"""Every output element of the four attention entries within the bound of tests/attention_bounds.py, on inputs whose
scores are exact: the staircase, descending, needles, tiles and ties landscapes (one per batch row, or per packed
sequence), fp16 and bf16.  The largest err / B per entry and dtype is printed (-s) and is part of a failure message.

  * flash_attn_func, prefill route (Sq * G > 64) and split-key route (Sq * G <= 64);
  * flash_attn_varlen_qkvpacked_func, ragged sequences;
  * kv_cache_attention on the FT cache layout, the [B, L, Hkv, D] layout bit-identical to it;
  * single_query_attention without RoPE, one split and many, and the current step's key as the needle."""
import pytest
import torch

import llm_awq_b200 as P
import attention_bounds as AB
import attention_exact as AE
import prefill_attention_oracle as PO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
WORST = {}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _inputs(kinds, Sq, Sk, H, Hkv, D, causal, u, seed, edge=AB.TILE, n_keys=None, targets_at=None, shift=0.0):
    """q [B, Sq, H, D], K / V [B, n_keys (default Sk), Hkv, D] float64 on the GPU, batch row b with landscape
    kinds[b] (levels moved by `shift`); row i of head h has its needle among the keys it sees (`targets_at`: one key
    for every row)."""
    g = _gen(seed)
    n_keys = Sk if n_keys is None else n_keys
    G = H // Hkv
    qs, ks, vs = [], [], []
    for kind in kinds:
        K = torch.stack([AB.make_k(kind, n_keys, D, u, g, shift) for _ in range(Hkv)], 1)
        V = torch.stack([AB.make_v(n_keys, D, g) for _ in range(Hkv)], 1)
        hor = [min(Sk - 1, i + Sk - Sq) if causal else Sk - 1 for i in range(Sq)]
        tg = lambda i, h: (targets_at if targets_at is not None else
                           AB.needle_targets(0, hor[i], Sk, edge, i + 3 * h) if kind == "needles" else -1)
        q = torch.stack([AB.make_q(kind, [tg(i, h) for i in range(Sq)], n_keys, D, g) for h in range(H)], 1)
        AB.check_exact(q, K, V)
        qs.append(q), ks.append(K), vs.append(V)
    return tuple(torch.stack(x).to(DEV) for x in (qs, ks, vs))


def _check(entry, dtype, got, q, K, V, causal, scale, family, ctx, n_keys=None):
    """got [B, Sq, H, D] against the bound, for q [B, Sq, H, D], K / V [B, Sk, Hkv, D] (float64).  O comes from the
    float64 oracle of tests/prefill_attention_oracle.py on the K / V the caches were built from; one head at a time, so
    that the [B, Sq, Sk] float64 temporaries stay below 2 GB at the largest shapes."""
    B, Sq, H, D = q.shape
    Sk, Hkv = K.shape[1], K.shape[2]
    G = H // Hkv
    i = torch.arange(Sq, device=DEV).view(-1, 1)
    j = torch.arange(Sk, device=DEV).view(1, -1)
    vis = (j <= i + Sk - Sq) if causal else torch.ones(Sq, Sk, dtype=torch.bool, device=DEV)
    vis = vis.expand(B, Sq, Sk)
    for h in range(H):
        s = torch.einsum("bid,bjd->bij", q[:, :, h], K[:, :, h // G])
        O, Bnd = AB.bound(s, vis, V[:, :, h // G], scale, dtype, family, n_keys)
        del s
        want = PO.prefill_attention_torch(q, K, V, causal, scale, [h])[:, :, 0]
        assert torch.allclose(O, want, rtol=1e-12, atol=1e-12), f"{ctx}: the bound's attention is not the oracle's"
        r = AB.ratio(got[:, :, h], O, Bnd)
        worst = float(r.max())
        WORST[(entry, dtype)] = max(WORST.get((entry, dtype), 0.0), worst)
        if worst > 1.0:
            b, row, c = (int(x) for x in (r == r.max()).nonzero()[0])
            n = int((r > 1).sum())
            raise AssertionError(f"{ctx}: {n} elements of head {h} outside the bound, largest err / B {worst:.3g} at "
                                 f"batch row {b}, row {row}, channel {c}: got {float(got[b, row, h, c]):.6g}, O = "
                                 f"{float(O[b, row, c]):.6g}, B = {float(Bnd[b, row, c]):.3g}")


def _report(entry, dtype):
    print(f"\n{entry} {dtype}: largest err / B {WORST.get((entry, dtype), 0.0):.3f}")


# ------------------------------------------------------------------------------------------------ flash_attn_func
def _flash(entry, B_kinds, Sq, Sk, H, Hkv, D, causal, dtype, seed):
    eng = P.engine()
    scale = AB.wgmma_scale(D)
    ctx = f"flash_attn_func Sq={Sq} Sk={Sk} H={H} Hkv={Hkv} D={D} causal={causal} {dtype}"
    q, K, V = _inputs(B_kinds, Sq, Sk, H, Hkv, D, causal, AB.level_units(D, scale), seed)
    got = eng.flash_attn_func(q.to(dtype), K.to(dtype), V.to(dtype), 0.0, scale, causal)
    _check(entry, dtype, got, q, K, V, causal, scale, "wgmma", ctx)


def _prefill_cases():
    """Sq = Sk in {128, 129, 1000, 2048}, G in {1, 4, 7}, D in {64, 72, 128}, causal and not: Sq * G > 64."""
    for D in (64, 72, 128):
        for G in (1, 4, 7):
            for S in (128, 129, 1000, 2048):
                for causal in (False, True):
                    yield S, S, G, 1, D, causal


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attn_prefill(dtype):
    for i, (Sq, Sk, H, Hkv, D, causal) in enumerate(_prefill_cases()):
        _flash("flash_attn_func prefill", AB.KINDS, Sq, Sk, H, Hkv, D, causal, dtype, 100 + i)
    _report("flash_attn_func prefill", dtype)


def _splitkv_cases():
    """Sq in {1, 4, 8}, G in {1, 4, 8} (Sq * G <= 64, 64 included), Sk in {129, 4100, 16384}, D in {64, 128}."""
    n = 0
    for Sq in (1, 4, 8):
        for G in (1, 4, 8):
            for Sk in (129, 4100, 16384):
                for D in (64, 128):
                    yield AB.KINDS, Sq, Sk, G, 1, D, n % 2 == 0
                    n += 1
    for kind in ("staircase", "tiles", "needles"):  # one cell: as many splits as the SMs allow
        yield (kind,), 8, 16384, 8, 1, 128, True


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attn_splitkv(dtype):
    for i, (kinds, Sq, Sk, H, Hkv, D, causal) in enumerate(_splitkv_cases()):
        _flash("flash_attn_func split-key", kinds, Sq, Sk, H, Hkv, D, causal, dtype, 200 + i)
    _report("flash_attn_func split-key", dtype)


# ------------------------------------------------------------------------------------------------ varlen
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lengths,H,D,causal", [([129, 1000, 300, 2048, 128], 2, 64, True),
                                                ([2048, 128, 1000, 129, 300], 2, 72, False),
                                                ([300, 129, 128, 1000, 2048], 1, 128, True)])
def test_flash_attn_varlen(lengths, H, D, causal, dtype):
    """Sequence n carries landscape n."""
    eng = P.engine()
    entry = "flash_attn_varlen_qkvpacked_func"
    scale = AB.wgmma_scale(D)
    u = AB.level_units(D, scale)
    seqs = [_inputs((kind,), L, L, H, H, D, causal, u, 300 + n) for n, (kind, L) in enumerate(zip(AB.KINDS, lengths))]
    qkv = torch.cat([torch.stack([q[0], K[0], V[0]], 1) for q, K, V in seqs])
    cu = torch.tensor([0] + torch.tensor(lengths).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    got = eng.flash_attn_varlen_qkvpacked_func(qkv.to(dtype), cu, max(lengths), 0.0, scale, causal)
    for n, (q, K, V) in enumerate(seqs):
        ctx = f"{entry} lengths={lengths} sequence {n} H={H} D={D} causal={causal} {dtype}"
        _check(entry, dtype, got[int(cu[n]):int(cu[n + 1])].unsqueeze(0), q, K, V, causal, scale, "wgmma", ctx)
    _report(entry, dtype)


# ------------------------------------------------------------------------------------------------ kv_cache_attention
def _kv_cases():
    n = 0
    for G in (1, 4, 7):
        for Sq, Sk in ((1, 16384), (17, 4100), (128, 1000), (512, 2048)):
            yield Sq, Sk, G, (64, 128)[n % 2]
            n += 1


@pytest.mark.parametrize("dtype", DTYPES)
def test_kv_cache_attention(dtype):
    eng = P.engine()
    entry = "kv_cache_attention"
    for i, (Sq, Sk, G, D) in enumerate(_kv_cases()):
        scale = AB.wgmma_scale(D)
        L = Sk + 37  # cache slots past the keys in use
        ctx = f"{entry} Sq={Sq} Sk={Sk} L={L} G={G} D={D} causal=True {dtype}"
        q, K, V = _inputs(AB.KINDS, Sq, Sk, G, 1, D, True, AB.level_units(D, scale), 400 + i, n_keys=L)
        qt, Kt, Vt = q.to(dtype), K.to(dtype), V.to(dtype)
        ft = eng.kv_cache_attention(qt, AE.ft_k_cache(Kt), Vt.permute(0, 2, 1, 3).contiguous(), Sk, scale, True)
        bthd = eng.kv_cache_attention(qt, Kt, Vt, Sk, scale, True)
        assert torch.equal(ft, bthd), f"{ctx}: the FT and [B, L, Hkv, D] layouts differ"
        _check(entry, dtype, ft, q, K[:, :Sk], V[:, :Sk], True, scale, "wgmma", ctx)
    _report(entry, dtype)


# ------------------------------------------------------------------------------------------------ single_query_attention
def _sq_cases():
    """(G, Hkv, D, t, needle on the current step, shift): t = 100 runs one split, 3000 and 16383 many.  With shift =
    TOP the top scores lie above the range of exp (> 88 natural units): a combine weight exp(m_s) taken without
    subtracting the max overflows there, while elsewhere exp(M) cancels between numerator and denominator."""
    n = 0
    for G, Hkv in ((1, 2), (4, 2), (7, 1)):
        for D in (64, 128, 256):
            yield G, Hkv, D, (100, 3000)[n % 2], False, 0.0
            n += 1
    yield 71, 1, 64, 3000, False, 0.0    # Falcon-7B
    yield 71, 1, 64, 100, False, 0.0
    yield 8, 1, 128, 16383, False, 0.0
    yield 4, 2, 128, 3000, True, 0.0     # the split that holds the written slot wins the combine
    for G, Hkv, D, t, current in ((4, 2, 64, 100, False), (4, 2, 64, 3000, False), (7, 1, 128, 3000, False),
                                  (1, 2, 256, 16383, False), (71, 1, 64, 3000, False), (4, 2, 128, 3000, True)):
        yield G, Hkv, D, t, current, AB.TOP


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_query_attention(dtype):
    eng = P.engine()
    entry = "single_query_attention"
    for i, (G, Hkv, D, t, current, shift) in enumerate(_sq_cases()):
        H = G * Hkv
        L = t + 1 + 7
        scale = D ** -0.5
        ctx = f"{entry} H={H} Hkv={Hkv} D={D} t={t} L={L} needle on the current step={current} shift={shift} {dtype}"
        q, K, V = _inputs(AB.KINDS, 1, t + 1, H, Hkv, D, False, AB.level_units(D, scale), 600 + i, edge=32,
                          n_keys=L, targets_at=t if current else None, shift=shift)
        qt, Kt, Vt = q[:, 0].to(dtype).contiguous(), K.to(dtype), V.to(dtype)
        k, v = Kt[:, t].contiguous(), Vt[:, t].contiguous()
        kc = AE.ft_k_cache(Kt).contiguous()
        vc = Vt.permute(0, 2, 1, 3).contiguous()
        got = eng.single_query_attention(qt, k, v, kc, vc, None, None, t, 0, 10000.0, 1.0, True).unsqueeze(1)
        _check(entry, dtype, got, q, K[:, :t + 1], V[:, :t + 1], False, scale, "decode", ctx)
    _report(entry, dtype)
