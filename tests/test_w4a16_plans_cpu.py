"""The W4A16 plan mirror (w4a16_plans.py) and the GPU cases derived from it, on an H100 SXM (132 SMs) and an H100
PCIe (114 SMs): every plan class a served shape reaches has a GPU case, every case reaches the plan and edge it is
labelled with, and plan() agrees with values worked out by hand from the launchers.  The same for the MLP front half
(mlp_front_plan, mlp_front_cases): every fused split and ring depth has a case."""
import pytest

from w4a16_plans import (Rejected, SERVED, decode_plan, edge_cases, fused_reach, mlp_front_cases, mlp_front_plan, plan,
                         served_plans, served_shapes)

SMS = [pytest.param(132, id="h100_sxm"), pytest.param(114, id="h100_pcie")]


@pytest.mark.parametrize("sms", SMS)
def test_every_served_plan_class_has_a_gpu_case(sms):
    have = {plan(c.m, c.n, c.k, c.dtype, c.entry, sms).klass for c in edge_cases(sms)}
    missing = {k: v for k, v in served_plans(sms).items() if k not in have}
    assert not missing, f"plan classes a served shape reaches without a GPU case (class: first shape): {missing}"


@pytest.mark.parametrize("sms", SMS)
def test_edge_cases_reach_their_plan_and_edge(sms):
    cases = edge_cases(sms)
    assert len({c.id for c in cases}) == len(cases)
    for c in cases:
        p = plan(c.m, c.n, c.k, c.dtype, c.entry, sms)
        for attr, want in c.expect:
            assert getattr(p, attr) == want, (c.id, attr, getattr(p, attr), want)
    by = lambda route: [plan(c.m, c.n, c.k, c.dtype, c.entry, sms) for c in cases if c.label.startswith(route)]
    # decode: each split the SM count allows, with a unit of an odd quad-row count (a partial row block), and a
    # rank with an odd or uneven group count
    for S in (1, 2, 4):
        ps = [p for p in by("decode") if p.S == S]
        assert bool(ps) == (sms % S == 0), S
        if ps:
            assert any(p.per_unit[0] % 2 or p.per_unit[1] % 2 for p in ps)
    dk = {(c.k // 128, plan(c.m, c.n, c.k, c.dtype, c.entry, sms).S) for c in cases if c.label.startswith("decode")}
    assert any(g % s or (g // s) % 2 for g, s in dk)
    # ring: a unit without rows, one with an odd octet at its end; every token-column width, split and unsplit
    ring = by("ring_S")
    assert {(p.S, p.Mp) for p in ring} == {(s, mp) for s in (1, 2) for mp in (1, 2, 4)}
    assert any(p.per_unit[0] == 0 for p in ring) and any(p.per_unit[1] % 2 for p in ring)
    # stream: both octet widths, every split, CTA counts on both sides of 2 sms and 3 sms
    stream = by("stream")
    assert {(p.ro, p.S) for p in stream} >= {(ro, s) for ro in (1, 2) for s in (1, 2, 4, 8)}
    assert {p.grid <= 2 * sms for p in stream} == {True, False} and {p.grid <= 3 * sms for p in stream} == {True, False}
    # flat: every split 1..8
    assert {p.S for p in by("flat")} == set(range(1, 9))
    # tile: for each split > 1 under which a served shape's clusters walk several tiles, a case whose clusters walk
    # >= 3 tiles, some of them one tile fewer
    splits = {c[2] for c in served_plans(sms) if c[0] == "tile" and c[2] > 1 and c[3]}
    assert splits
    for S in splits:
        assert any(p.S == S and p.tiles_per_cluster >= 3 and p.short_clusters for p in by("tile")), S


def test_edge_cases_follow_the_sm_count():
    """The cases are derived from the SM count, not fixed: the ring's edge channel counts move with it."""
    n = lambda sms: sorted({c.n for c in edge_cases(sms) if c.label.startswith("ring_S1")})
    assert n(132) == [8 * o for o in (131, 132, 133, 2 * 132 + 1)]
    assert n(114) == [8 * o for o in (113, 114, 115, 2 * 114 + 1)]


# Worked by hand from the launchers (132 SMs unless stated).
PINNED = [
    # kMlpProjection (mlp_front's projections): no big-layer rule -- 12 tokens on 58.7 M weights take the flat launch
    # (32 groups; k per CTA 4096 / 2048 / 1024 with 112 x 4 = 448 >= 264 CTAs -> S = 4) where the GEMM takes tn 16 tiles
    ((12, 14336, 4096, "f16", "mlp", 132), dict(route="flat", kernel="w4a16_wgmma_kernel<16>", S=4, grid=448)),
    ((12, 14336, 4096, "f16", "gemm", 132), dict(route="tile", kernel="w4a16_wgmma_kernel<16>", S=1, grid=112)),
    # launch_flat: 12 groups, k per CTA 1536 / 768 (two CTAs per SM needs 264 CTAs, 12 x 2 < 264) / 512 -> S = 3
    ((6, 1536, 1536, "f16", "gemv", 132), dict(route="flat", kernel="w4a16_wgmma_kernel<16>", S=3, grid=36)),
    # 112 groups, no split <= 8 reaches 1024 k per CTA: the largest divisor, 8
    ((4, 1024, 14336, "f16", "gemv", 132), dict(route="flat", S=8, grid=64, fallbacks=("ring",))),
    # launch_umma at 129 tokens: tn 64 (96 tiles); S = 1 one wave of 224 x 400 + 640; S = 4: 33 clusters, 3 waves of
    # 56 x 400 + 6640 = 99120 < 102240 -> 96 tiles over 33 clusters, 3 per cluster (30 clusters take 3, 3 take 2)
    ((129, 4096, 14336, "f16", "gemm", 132), dict(route="tile", kernel="w4a16_wgmma_kernel<64>", S=4, tiles=96,
                                                  clusters=33, tiles_per_cluster=3, short_clusters=3, grid=132)),
    # 256 tokens: 128 tiles of 64 tokens fit one wave unsplit (102240) before any split (S = 2: 2 waves, 114880)
    ((256, 4096, 14336, "f16", "gemm", 132), dict(route="tile", S=1, tn=64, tiles=128, clusters=128, grid=128)),
    # 12 tokens on 58.7 M weights: the tile launch directly; tn 16, S = 4: 32 tiles on 33 clusters, one wave
    ((12, 4096, 14336, "f16", "gemm", 132), dict(route="tile", kernel="w4a16_wgmma_kernel<16>", S=4, clusters=32,
                                                 grid=128)),
    ((12, 4096, 4096, "f16", "gemm", 132), dict(route="flat", S=8, grid=256)),
    # launch_decode_impl: 112 groups > 64 digits -> S = 2, 66 units for 1024 quad rows (15 or 16), 4 row blocks;
    # 27392 B before the ring, 5 slots of 17536 B
    ((1, 4096, 14336, "f16", "gemv", 132), dict(route="decode", S=2, units=66, per_unit=(15, 16), ns=5, smem=115072,
                                                grid=132)),
    # 1032 quad rows over 132 CTAs: 7.8 per CTA (eff 0.98), 33 groups -> unsplit
    ((1, 4128, 4224, "f16", "gemv", 132), dict(route="decode", S=1, units=132, per_unit=(7, 8), grid=132)),
    # launch_ring: 32 groups -> S = 2; 512 octets over 66 units (<= 8: 4 row blocks); 27904 B before 5 slots
    ((4, 4096, 4096, "f16", "gemv", 132), dict(route="ring", S=2, units=66, Mp=4, ns=5, smem=27904 + 5 * 17536,
                                               grid=132)),
    ((1, 4096, 4096, "bf16", "gemv", 114), dict(route="ring", S=2, units=57, Mp=1, grid=114)),
    # launch_stream: 520 % 16 != 0 -> one octet per CTA, 65 CTAs <= 2 x 132: padded to 233472 / 3 - 512
    ((6, 520, 1024, "f16", "gemv", 132), dict(route="stream", ro=1, tt=1, S=1, grid=65, smem=77312)),
    ((7, 520, 8192, "bf16", "gemv", 132), dict(route="stream", ro=1, S=4, grid=260)),
]


@pytest.mark.parametrize("args,want", PINNED, ids=lambda v: "-".join(map(str, v)) if isinstance(v, tuple) else "")
def test_plan_matches_the_hand_worked_value(args, want):
    p = plan(*args)
    assert {a: getattr(p, a) for a in want} == want


def test_rejections_follow_the_entries():
    with pytest.raises(Rejected):
        plan(8, 4096, 4096, "f16", "gemv", 132)      # the GEMV envelope ends at 7 tokens
    with pytest.raises(Rejected):
        plan(5, 520, 1024, "f16", "gemm", 132)       # the GEMM needs n % 128 == 0
    with pytest.raises(Rejected):
        plan(8, 520, 1024, "f16", "linear", 132)     # ... and so does the linear from 8 tokens
    assert plan(5, 520, 1024, "f16", "linear", 132).route == "stream"


def test_two_token_tile_stream_plan_is_never_reached():
    """From 8 tokens every entry needs n % 128 == 0, and the flat launch takes such shapes up to 16 tokens: the stream
    kernel's 9..16-token instantiation is not part of any W4A16 entry's dispatch."""
    for _, n, k in served_shapes() + [("odd", 1152, 4224), ("odd", 2048, 11008)]:
        for m in range(9, 17):
            for entry in ("gemm", "linear"):
                assert plan(m, n, k, "f16", entry, 132).route in ("flat", "tile")


def test_served_lists_every_model():
    assert set(SERVED) == {"llama2_7b", "llama3_8b", "llama2_70b_tp8", "qwen2_0_5b", "qwen2_1_5b", "qwen2_7b"}
    shapes = {(n, k) for _, n, k in served_shapes()}
    assert {(6144, 4096), (14336, 4096), (4096, 14336), (2048, 1536), (8960, 1536), (1536, 8960), (3584, 18944),
            (1280, 8192), (8192, 1024), (3584, 8192), (8192, 3584), (1152, 896)} <= shapes


# ------------------------------------------------------------------------------------------------ MLP front half
@pytest.mark.parametrize("sms", SMS)
def test_mlp_front_cases_reach_their_plan(sms):
    cases = mlp_front_cases(sms)
    assert len({c.id for c in cases}) == len(cases)
    for c in cases:
        ps = mlp_front_plan(c.m, c.n, c.k, c.dtype, sms)
        for attr, want in c.expect:
            assert getattr(ps[0], attr) == want, (c.id, attr, getattr(ps[0], attr), want)
        if ps[0].route == "fused":
            assert len(ps) == 1 and c.m == 1 and c.dtype == "f16"
            # the composition the fused kernel must equal bit for bit runs the plain decode kernel with the same split
            # and the same partition of the quad rows
            pp = plan(1, c.n, c.k, "f16", "gemv", sms)
            assert pp.route == "decode" and (pp.S, pp.units, pp.per_unit) == (ps[0].S, ps[0].units, ps[0].per_unit)
        else:
            assert [p.route for p in ps[:2]] == [plan(c.m, c.n, c.k, c.dtype, "mlp", sms).route] * 2
            assert ps[2].kernel == "silu_mul_kernel"
    fused = [mlp_front_plan(c.m, c.n, c.k, c.dtype, sms)[0] for c in cases if c.label.startswith("fused_S")]
    # every split with a unit of an odd quad-row count (a partial row block) ...
    for S in {p.S for p in fused}:
        assert any(p.per_unit[0] % 2 or p.per_unit[1] % 2 for p in fused if p.S == S)
    # ... and a rank with an odd or uneven group count
    assert any((c.k // 128) % p.S or (c.k // 128 // p.S) % 2
               for c, p in zip([c for c in cases if c.label.startswith("fused_S")], fused) if p.S > 1)
    routes = {mlp_front_plan(c.m, c.n, c.k, c.dtype, sms)[0].route for c in cases}
    assert routes == {"fused", "decode", "ring", "flat", "stream", "tile"}
    # the token counts 9..16 on a layer of >= 48 M weights: flat here, where the GEMM would take the tile launch
    assert any(9 <= c.m <= 16 and c.n * c.k >= 48e6 and plan(c.m, c.n, c.k, c.dtype, "gemm", sms).route == "tile"
               for c in cases)
    # a wgmma tile launch whose last token tile is partial
    assert any((p := mlp_front_plan(c.m, c.n, c.k, c.dtype, sms)[0]).route == "tile" and c.m % p.tn for c in cases)


@pytest.mark.parametrize("sms", SMS)
def test_every_fused_split_and_ring_depth_has_a_case(sms):
    splits, depths, decline = fused_reach(sms)
    assert set(splits) == ({1, 2, 4} if sms % 4 == 0 else {1, 2})
    assert set(depths) == {3, 4, 5, 6}
    plans = [mlp_front_plan(c.m, c.n, c.k, c.dtype, sms)[0] for c in mlp_front_cases(sms)]
    assert {p.S for p in plans if p.route == "fused"} == set(splits)
    assert {p.ns for p in plans if p.route == "fused"} == set(depths)
    assert decline and any(p.route == "decode" for p in plans)


# Worked by hand from launch_decode_impl with two weight sets (32 floats per row block and warp in `red`, per row block
# in the exchange regions) and from b200awq_w4a16_mlp_front.
MLP_PINNED = [
    # Llama-3-8B gate / up: 3584 quad rows over 132 CTAs (27 or 28, eff 0.97), 32 groups -> unsplit, 7 row blocks;
    # 384 + 12288 + 512 + 7 x 16 x 32 x 4 + 7 x 32 x 4 = 28416 B before the ring: 4 slots of 17536 B
    ((1, 14336, 4096, "f16", 132), [dict(route="fused", kernel="w4a16_decode_kernel<true, false>", S=1, grid=132, ns=4,
                                         smem=98560)]),
    # 124672 x 6656: 237 quad rows per CTA (60 row blocks), 52 groups; 45696 B before the ring: 3 slots
    ((1, 124672, 6656, "f16", 132), [dict(route="fused", S=1, ns=3, smem=45696 + 3 * 17536)]),
    # 33272 x 16640: 130 groups -> S = 4, 33 units of 253 quad rows (64 row blocks); 63360 B before the ring: 2 slots,
    # declined.  The plain kernel (38784 B before its ring) keeps 4: two decode launches, then silu_mul over
    # 33272 / 8 = 4159 vectors, 17 CTAs
    ((1, 33272, 16640, "f16", 132), [dict(route="decode", S=4, units=33, ns=4, smem=38784 + 4 * 17536)] * 2
     + [dict(kernel="silu_mul_kernel", grid=17, smem=0)]),
    ((1, 4568, 31360, "f16", 114), [dict(route="decode")] * 2 + [dict(kernel="silu_mul_kernel")]),
    # 12 tokens: flat S = 4 on 448 CTAs per projection (the GEMM entry would take 112 tiles of 16 tokens);
    # 12 x 14336 / 8 / 256 -> 84 CTAs
    ((12, 14336, 4096, "f16", 132), [dict(route="flat", S=4, grid=448)] * 2 + [dict(kernel="silu_mul_kernel", grid=84)]),
    # 2048 tokens: 2048 x 14336 / 8 / 256 = 14336 CTAs, capped at 8 per SM
    ((2048, 14336, 4096, "bf16", 132), [dict(route="tile")] * 2 + [dict(kernel="silu_mul_kernel", grid=1056)]),
]


@pytest.mark.parametrize("args,want", MLP_PINNED, ids=lambda v: "-".join(map(str, v)) if isinstance(v, tuple) else "")
def test_mlp_front_plan_matches_the_hand_worked_value(args, want):
    ps = mlp_front_plan(*args)
    assert len(ps) == len(want)
    for p, w in zip(ps, want):
        assert {a: getattr(p, a) for a in w} == w


def test_decode_plan_weight_sets_change_only_the_ring():
    """Two weight sets double the red and exchange regions; the split and the partition are those of one."""
    for n, k in ((14336, 4096), (33272, 16640), (1048, 16896), (2104, 8448)):
        one, two = decode_plan(n, k, 132), decode_plan(n, k, 132, nt=2)
        assert one is not None
        if two is not None:
            assert (one.S, one.units, one.per_unit, one.grid) == (two.S, two.units, two.per_unit, two.grid)
            assert two.smem - two.ns * 17536 > one.smem - one.ns * 17536


def test_mlp_front_rejections_follow_the_entry():
    with pytest.raises(Rejected):
        mlp_front_plan(1, 4100, 4096, "f16", 132)      # n % 8
    with pytest.raises(Rejected):
        mlp_front_plan(8, 4104, 4096, "f16", 132)      # n % 128 from 8 tokens
    assert mlp_front_plan(7, 4104, 4096, "f16", 132)[0].route == "stream"
    assert mlp_front_plan(1, 4104, 4096, "f16", 132)[0].route == "fused"
    assert mlp_front_plan(1, 2048, 4096, "bf16", 132, y_aligned=False)[-1].grid == 8   # 2048 elements one at a time
