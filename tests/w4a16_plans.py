"""The W4A16 dispatch and every launcher's plan, restated in Python from the shape and the SM count alone.

`plan(m, n, k, dtype, entry, sms)` mirrors api.cu's launch_w4a16 (envelopes, the 9..16-token big-layer rule, use_flat,
the fall-through from one kernel to the next on B200AWQ_ERR_SHAPE) and the planning lines of launch_decode_impl,
launch_ring, launch_flat, launch_stream and launch_umma.  It returns the kernel name and the grid the launch uses, as
the profiler reports them, and the quantities that decide where a kernel's partition edges fall.  This is the one copy
of the launchers' rules in the suite: a change to a launcher that is not made here fails the profiler test of
test_w4a16_plans_gpu.py, and the hand-worked values in test_w4a16_plans_cpu.py make such a change visible in review.

`edge_cases(sms)` derives the GPU cases from the SM count: shapes whose partition over the SMs is ragged, k splits
that leave odd group counts, every plan class the dispatch can reach, and the token counts at route boundaries.
`SERVED` lists the projections of the models the project serves.

`mlp_front_plan(m, n, k, dtype, sms)` mirrors b200awq_w4a16_mlp_front: the fused one-token kernel (launch_decode_impl
with two weight sets), else the two kMlpProjection products and silu_mul_kernel; `mlp_front_cases(sms)` derives its
GPU cases (test_mlp_front_plans_gpu.py)."""
import functools
from dataclasses import dataclass, field, replace

GROUP = 128
KB = 1024

# api.cu
RING_MAX_M, FLAT_MIN_M, FLAT_MIN_M_LONG_K, FLAT_MAX_M, STREAM_MAX_M = 4, 5, 3, 16, 16
BIG_MID_WEIGHTS = 48 * 1000 * 1000

# w4a16_decode.cu
DEC_PIECE, DEC_RED, DEC_MAX_SLOTS, DEC_MAX_RB, DEC_CONS = 32, 8, 8, 128, 16
DEC_SLOT_BYTES = -(-(2 * (DEC_PIECE * 256 + 16) + 2 * 2 * DEC_PIECE * 8) // 128) * 128
DEC_GROUP_BYTES = 6 * 4 * 16
DEC_BUDGET = 113 * KB

# w4a16_ring.cu
RING_CONS, RING_SLOT_GROUPS, RING_MAX_RB = 8, 16, 128
RING_SLOT_BYTES = -(-(4 * (RING_SLOT_GROUPS * 256 + 16) + 1024) // 128) * 128
RING_BUDGET = 113 * KB

# w4a16_stream.cu
STREAM_WARPS, STREAM_RPB, STREAM_SMEM_CAP = 8, 64, 200 * KB

# w4a16_wgmma.cu
BM, BK = 128, 64


def _align(v, a):
    return -(-v // a) * a


@dataclass(frozen=True)
class Plan:
    route: str           # decode, ring, flat, stream, tile; fused (the MLP front's decode kernel), silu_mul
    kernel: str          # as the profiler tests report it: w4a16_<route>_kernel, w4a16_wgmma_kernel<TN>,
                         # w4a16_decode_kernel<true, false> (fused), silu_mul_kernel
    grid: int            # CTAs of the launch
    smem: int            # dynamic shared memory of the launch, bytes
    S: int = 1           # k split: CTAs per cluster
    units: int = 0       # decode / ring: clusters the rows are dealt to
    per_unit: tuple = ()  # decode: (fewest, most) quad rows of a unit; ring: octets
    ns: int = 0          # decode / ring: ring slots
    Mp: int = 0          # ring: token columns of the exchange buffer
    ro: int = 0          # stream: octets per CTA
    tt: int = 0          # stream: 8-token MMA column tiles
    tn: int = 0          # flat / tile: token tile
    tiles: int = 0       # flat / tile: 128-channel x tn-token tiles
    clusters: int = 0    # flat / tile: clusters launched
    fallbacks: tuple = field(default=())  # kernels that returned B200AWQ_ERR_SHAPE before this one

    @property
    def tiles_per_cluster(self):
        return -(-self.tiles // self.clusters) if self.clusters else 0

    @property
    def short_clusters(self):
        """Clusters of a persistent tile launch that do one tile fewer than the others."""
        return (-self.tiles) % self.clusters if self.clusters else 0

    @property
    def klass(self):
        """The plan class: what decides which code of the kernel runs (instantiation, split, partition loop)."""
        if self.route in ("decode", "fused"):
            return (self.route, self.S)
        if self.route == "ring":
            return ("ring", self.S, self.Mp)
        if self.route == "stream":
            return ("stream", self.ro, self.tt, self.S)
        if self.route == "flat":
            return ("flat", self.S)
        return ("tile", self.tn, self.S, self.tiles_per_cluster > 1)


# ------------------------------------------------------------------------------------------------ launchers
def decode_plan(n, k, sms, nt=1):
    """launch_decode_impl (no override): None where it returns B200AWQ_ERR_SHAPE.  `nt` weight sets: 2 for the fused
    MLP front (w4a16_decode_kernel<true, false>), whose red and exchange regions hold 16 nt floats per row block; the
    split does not depend on it."""
    G, Q = k // GROUP, n // 4

    def eff(s):
        units = sms // s
        return Q / units / -(-Q // units)

    S, s = 1, 2
    while s <= 4 and eff(S) < 0.9:
        if sms % s == 0 and G // s >= 16 and eff(s) > eff(S) + 0.03:
            S = s
        s *= 2
    while G // S > 64 and S < 8 and sms % (2 * S) == 0:
        S *= 2
    if S > 1 and (sms % S or G < S):
        S = 1
    units = sms // S
    nrb_max = -(-(-(-Q // units)) // 4)
    if nrb_max > DEC_MAX_RB or Q * (units + 1) >= 2 ** 31:
        return None
    ngr = -(-G // S)
    off = _align(8 * (2 * DEC_MAX_SLOTS + 2 * DEC_RED + 1 + nrb_max), 128)
    off += ngr * DEC_GROUP_BYTES + ngr * 16 + min(DEC_RED, nrb_max) * DEC_CONS * 16 * nt * 4 + S * nrb_max * 16 * nt * 4
    off = _align(off, 128)
    ns = min((DEC_BUDGET - off) // DEC_SLOT_BYTES, DEC_MAX_SLOTS)
    if ns < 3:
        return None
    route, kernel = ("fused", "w4a16_decode_kernel<true, false>") if nt == 2 else ("decode", "w4a16_decode_kernel")
    return Plan(route, kernel, units * S, off + ns * DEC_SLOT_BYTES, S=S, units=units,
                per_unit=(Q // units, -(-Q // units)), ns=ns)


def ring_plan(m, n, k, sms):
    """launch_ring: None where it returns B200AWQ_ERR_SHAPE."""
    if sms < 2:
        return None
    G, O = k // GROUP, n // 8
    S = 2 if G >= 2 * RING_CONS and sms % 2 == 0 else 1
    units = sms // S
    Mp = 1 if m <= 1 else (2 if m <= 2 else 4)
    nrb_max = (-(-O // units) + 1) // 2
    if nrb_max > RING_MAX_RB:
        return None
    ngr = -(-G // S)
    off = _align(8 * (2 * 8 + 4 + RING_MAX_RB), 128)
    off += m * ngr * 256 + 8 * ngr * 8 + 2 * RING_CONS * 128 * 4 + nrb_max * 16 * Mp * 4
    off = _align(off, 128)
    ns = min((RING_BUDGET - off) // RING_SLOT_BYTES, 8)
    if ns < 3:
        return None
    return Plan("ring", "w4a16_ring_kernel", units * S, off + ns * RING_SLOT_BYTES, S=S, units=units,
                per_unit=(O // units, -(-O // units)), ns=ns, Mp=Mp)


def pick_splits(k, kc_target):
    groups, best = k // GROUP, 1
    for s in (1, 2, 4, 8):
        if groups % s:
            continue
        best = s
        if k // s <= kc_target:
            break
    return best


def stream_smem(ro, tt, bf16, m, kc, split):
    ng = kc // GROUP
    nbar = -(-(-(-ng // STREAM_WARPS)) // STREAM_RPB)
    off = 2 * ro * kc * 2 + 2 * ng * 8 * ro * 2
    off = _align(off, 16)
    off += m * (kc * 2 + 16) + STREAM_WARPS * tt * 128 * 4 + tt * 128 * 4
    off += 8 * tt * 128 * 4 if split else 0
    off += 0 if bf16 else 8 * tt * ng * 8
    return off + (nbar + 2) * 8


def stream_plan(m, n, k, bf16, sms):
    """launch_stream (no all-reduce): None where it returns B200AWQ_ERR_SHAPE."""
    ro = 2 if n % 16 == 0 else 1
    S = pick_splits(k, 4096 if m <= 4 else (2048 if m <= 8 else 1024))
    tt = 1 if m <= 8 else 2
    total = stream_smem(ro, tt, bf16, m, k // S, S > 1)
    if total > STREAM_SMEM_CAP:
        return None
    ctas = n // (8 * ro) * S
    dyn = total
    per_sm = 2 if ctas <= 2 * sms else (3 if ctas <= 3 * sms else 0)
    if per_sm and S == 1:
        dyn = max(dyn, 233472 // (per_sm + 1) - 512)
    if dyn > STREAM_SMEM_CAP:
        dyn = total
    return Plan("stream", "w4a16_stream_kernel", ctas, dyn, S=S, ro=ro, tt=tt)


def wgmma_smem(tn):
    stage = tn * 128 + BM * BK // 2
    stages = min(8, 160 * KB // stage)
    return stages * stage + max(tn * 272, tn * BM * 4) + 1024 + 256


def flat_plan(m, n, k, sms):
    """launch_flat: one 16-token tile, one cluster of S CTAs per 128 channels."""
    groups, S = k // GROUP, 1
    for s in range(1, 9):
        if groups % s:
            continue
        S = s
        if k // s <= 512 or (k // s <= 1024 and (n // BM) * s >= 2 * sms):
            break
    tiles = n // BM
    return Plan("flat", "w4a16_wgmma_kernel<16>", tiles * S, wgmma_smem(16), S=S, tn=16, tiles=tiles, clusters=tiles)


def umma_choice(m, n, k, sms):
    """launch_umma's cost model: (token tile, k split)."""
    best = None
    for c in (128, 64, 32, 16):
        if c > 16 and c // 2 >= m:
            continue
        tiles = -(-m // c) * (n // BM)
        for sp in (1, 2, 4, 8):
            if sp > 1 and (c > 64 or (k // GROUP) % sp or k // sp < 512):
                continue
            per_tile = (k // BK // sp) * max(4 * c + 100, 400) + 10 * c + (6000 if sp > 1 else 0)
            slots = sms // sp
            cost = 12000 + -(-tiles // slots) * per_tile
            if best is None or cost < best[0]:
                best = (cost, c, sp)
    return best[1], best[2]


def tile_plan(m, n, k, sms):
    """launch_umma: a persistent grid of min(tiles, sms / S) clusters walking the tiles."""
    tn, S = umma_choice(m, n, k, sms)
    tiles = -(-m // tn) * (n // BM)
    clusters = min(tiles, max(sms // S, 1))
    return Plan("tile", f"w4a16_wgmma_kernel<{tn}>", clusters * S, wgmma_smem(tn), S=S, tn=tn, tiles=tiles,
                clusters=clusters)


# ------------------------------------------------------------------------------------------------ dispatch
class Rejected(ValueError):
    """The entry returns an error for this shape."""


@functools.lru_cache(maxsize=None)
def plan(m, n, k, dtype, entry, sms):
    """The plan the entry `entry` ("gemv", "gemm" or "linear"; "mlp": one projection of b200awq_w4a16_mlp_front's
    composed path, the kMlpProjection envelope) launches for x [m, k], W [n, k] of `dtype` ("f16" or "bf16") on a device
    with `sms` SMs (api.cu launch_w4a16).  Raises Rejected where the entry returns an error."""
    assert dtype in ("f16", "bf16") and entry in ("gemv", "gemm", "linear", "mlp")
    if m < 1 or n < 8 or k < GROUP or n % 8 or k % GROUP:
        raise Rejected("shape")
    if entry == "gemv" and m > 7:
        raise Rejected("batch")
    if entry != "gemv" and n % BM and (entry == "gemm" or m >= 8):
        raise Rejected("shape")
    env = "gemv" if entry == "gemv" or (entry == "linear" and m < 8) else "gemm"
    # kMlpProjection is kGemm without the big-layer rule
    big_mid = env == "gemm" and entry != "mlp" and m > 8 and n * k >= BIG_MID_WEIGHTS
    failed = []
    if not big_mid:
        if m == 1 and dtype == "f16":
            p = decode_plan(n, k, sms)
            if p:
                return p
            failed.append("decode")
        if m <= RING_MAX_M:
            p = ring_plan(m, n, k, sms)
            if p:
                return _with(p, failed)
            failed.append("ring")
        if n % BM == 0 and (FLAT_MIN_M_LONG_K if k > 8192 else FLAT_MIN_M) <= m <= FLAT_MAX_M:
            return _with(flat_plan(m, n, k, sms), failed)
        if m <= STREAM_MAX_M:
            p = stream_plan(m, n, k, dtype == "bf16", sms)
            if p:
                return _with(p, failed)
            failed.append("stream")
    if env != "gemv" and n % BM == 0:
        return _with(tile_plan(m, n, k, sms), failed)
    raise Rejected("shape")


def _with(p, failed):
    return replace(p, fallbacks=tuple(failed)) if failed else p


# ------------------------------------------------------------------------------------------------ served shapes
def _decoder(hidden, inter, heads, kv_heads, head_dim):
    q, kv = heads * head_dim, kv_heads * head_dim
    return [("qkv", q + 2 * kv, hidden), ("q", q, hidden), ("kv", kv, hidden), ("o", hidden, q),
            ("gate_up", inter, hidden), ("down", hidden, inter)]


def _tp8(hidden, inter, heads, kv_heads, head_dim):
    """Column-parallel q/k/v and gate/up shards, row-parallel o and down shards (k is the sharded dimension)."""
    q, kv = heads * head_dim // 8, kv_heads * head_dim // 8
    return [("qkv", q + 2 * kv, hidden), ("q", q, hidden), ("kv", kv, hidden), ("o", hidden, q),
            ("gate_up", inter // 8, hidden), ("down", hidden, inter // 8)]


# model -> [(projection, n, k)]: a fused q/k/v projection and its q and k/v parts, gate and up (one shape), o, down.
# Qwen2-0.5B / 1.5B / 7B are the language models of InternVL3-1B / 2B and NVILA-Lite-2B / NVILA-8B.
SERVED = {
    "llama2_7b": _decoder(4096, 11008, 32, 32, 128),
    "llama3_8b": _decoder(4096, 14336, 32, 8, 128),
    "llama2_70b_tp8": _tp8(8192, 28672, 64, 8, 128),
    "qwen2_0_5b": _decoder(896, 4864, 14, 2, 64),
    "qwen2_1_5b": _decoder(1536, 8960, 12, 2, 128),
    "qwen2_7b": _decoder(3584, 18944, 28, 4, 128),
}


def served_shapes():
    """Distinct (n, k) over SERVED, with the first name that uses each."""
    seen = {}
    for model, projs in SERVED.items():
        for name, n, k in projs:
            seen.setdefault((n, k), f"{model}_{name}")
    return [(name, n, k) for (n, k), name in seen.items()]


@functools.lru_cache(maxsize=None)
def served_plans(sms, max_m=4096):
    """{plan class: (m, n, k, dtype, entry)} over every served shape, 1 <= m <= max_m, both dtypes, gemv and gemm."""
    found = {}
    for _, n, k in served_shapes():
        for dtype in ("f16", "bf16"):
            for m in range(1, max_m + 1):
                for entry in (("gemv", "gemm") if m <= 7 else ("gemm",)):
                    p = plan(m, n, k, dtype, entry, sms)
                    found.setdefault(p.klass, (m, n, k, dtype, entry))
    return found


# ------------------------------------------------------------------------------------------------ GPU cases
@dataclass(frozen=True)
class Case:
    label: str     # the plan and the edge the case targets
    m: int
    n: int
    k: int
    dtype: str
    entry: str
    expect: tuple  # (Plan attribute, value) pairs plan() must give

    @property
    def id(self):
        return f"{self.label}-m{self.m}-n{self.n}-k{self.k}-{self.dtype}"


def _case(label, m, n, k, dtype, entry, **expect):
    return Case(label, m, n, k, dtype, entry, tuple(sorted(expect.items())))


def _ks(lo=4 * GROUP, hi=32768):
    """Candidate k: from 4 groups (the probe tokens of the GPU tests fill groups 1..3 with special values)."""
    return range(lo, hi + 1, GROUP)


def _route(m, n, k, dtype, sms):
    try:
        return plan(m, n, k, dtype, "gemv", sms).route
    except Rejected:
        return None


def _decode_cases(sms):
    """Quad rows Q = 4 units j - 2, 4 units j, 4 units j + 2 (j = 1, 2; n = 4 Q stays a multiple of 8): two units get
    one quad row fewer or more than the rest, an odd count that leaves them a partial row block.  For each split S
    with sms % S == 0 the smallest k whose plan is that split, preferring an odd group count per rank."""
    out = []
    for S in (1, 2, 4):
        if sms % S:
            continue
        units = sms // S
        for j in (1, 2):
            for dq in (-2, 0, 2):
                Q = 4 * units * j + dq
                hits = [k for k in _ks() if (p := decode_plan(4 * Q, k, sms)) and p.S == S]
                # more than one 32-group piece per rank, and an odd or uneven group count per rank
                odd = [k for k in hits if k // GROUP // S > DEC_PIECE and ((k // GROUP) % S or (k // GROUP // S) % 2)]
                if not hits:
                    continue
                k = (odd or hits)[0]
                lo, hi = (4 * j - 1, 4 * j) if dq < 0 else ((4 * j, 4 * j) if dq == 0 else (4 * j, 4 * j + 1))
                out.append(_case(f"decode_S{S}_q{4 * j}{dq:+d}", 1, 4 * Q, k, "f16", "gemv", route="decode", S=S,
                                 units=units, per_unit=(lo, hi)))
    return out


def _ring_cases(sms):
    """Octets O = units - 1 (a unit without rows), units, units + 1, 2 units + 1 (an odd octet at the end of a unit),
    unsplit (15 groups) and split over two CTAs (17 groups: 8 | 9); every token-column width Mp; bf16 at one token."""
    out = []
    for S, k in ((1, 15 * GROUP), (2, 17 * GROUP)):
        if S == 2 and sms % 2:
            continue
        units = sms // S
        for tag, O, per_unit in (("u-1", units - 1, (0, 1)), ("u", units, (1, 1)), ("u+1", units + 1, (1, 2)),
                                 ("2u+1", 2 * units + 1, (2, 3))):
            for m, dtype in ((1, "bf16"), (2, "f16"), (3, "bf16"), (4, "f16")):
                Mp = 1 if m == 1 else (2 if m == 2 else 4)
                out.append(_case(f"ring_S{S}_O{tag}", m, 8 * O, k, dtype, "gemv", route="ring", S=S, units=units,
                                 per_unit=per_unit, Mp=Mp))
    # the activations of a long k leave fewer than 3 ring slots: the flat launch (n % 128 == 0, k > 8192) takes
    # 4 tokens, the stream kernel takes 2 tokens of a bf16 layer
    k4 = next(k for k in _ks() if ring_plan(4, 1024, k, sms) is None)
    out.append(_case("ring_ns_lt_3_to_flat", 4, 1024, k4, "f16", "gemv", route="flat", fallbacks=("ring",)))
    k2 = next(k for k in _ks(hi=65536) if ring_plan(2, 520, k, sms) is None and _route(2, 520, k, "bf16", sms) == "stream"
              and all(_route(m, 520, k, dt, sms) for m in (1, 2, 3, 4) for dt in ("f16", "bf16")))
    out.append(_case("ring_ns_lt_3_to_stream", 2, 520, k2, "bf16", "gemv", route="stream", fallbacks=("ring",)))
    return out


def _stream_cases(sms):
    """Only the GEMV envelope reaches the stream kernel with 5..7 tokens (n % 128 != 0; from 8 tokens the entries need
    n % 128 == 0 and the flat launch takes every such shape, so tt = 2 is never planned).  Octets per CTA ro = 1
    (n % 16 != 0) and 2, every split pick_splits returns for 5..7 tokens (k per CTA <= 2048), CTA counts just below and
    above 2 sms and 3 sms (the co-residency padding of the unsplit launch)."""
    out = []
    sides = (2 * sms - 1, 2 * sms + 1, 3 * sms - 1, 3 * sms + 1)
    i = 0
    for S, k in ((1, 1920), (2, 4096), (4, 8192), (8, 16384)):
        for ro in (1, 2):
            for side in (sides if S == 1 else sides[:1]):
                c = -(-side // S)  # row blocks: ctas = c S on the chosen side
                while c % (2 if ro == 1 else 8) == 0:  # n % 16 != 0 for ro = 1, n % 128 != 0 for ro = 2
                    c += 1
                n = 8 * ro * c
                m = (5, 7)[i % 2]
                dtype = ("f16", "bf16")[(i // 2) % 2]
                i += 1
                out.append(_case(f"stream_S{S}_ro{ro}_ctas{c * S - 2 * sms:+d}_2sms", m, n, k, dtype, "gemv",
                                 route="stream", S=S, ro=ro, tt=1, grid=c * S))
    # up to 4 tokens the stream kernel takes what the ring cannot (k per CTA <= 4096)
    k = next(k for k in _ks(hi=65536) if ring_plan(4, 1032, k, sms) is None and _route(4, 1032, k, "f16", sms) == "stream")
    out.append(_case("stream_after_ring_m4", 4, 1032, k, "f16", "gemv", route="stream", ro=1, tt=1,
                     S=pick_splits(k, 4096), fallbacks=("ring",)))
    return out


def _flat_cases(sms):
    """Every k split 1..8 that some k <= 32768 reaches with n % 128 == 0, for 5 tokens (a partial 16-token tile),
    13 and 16 tokens, and 3 tokens where k > 8192 and the ring does not take them."""
    out, seen, n = [], set(), 1024
    for k in _ks():
        p = flat_plan(5, n, k, sms)
        if p.S not in seen:
            seen.add(p.S)
            for m in (5, 13, 16):
                out.append(_case(f"flat_S{p.S}", m, n, k, ("f16", "bf16")[m % 2], "gemm", route="flat", S=p.S))
    k = next(k for k in _ks(8192 + GROUP) if _route(3, n, k, "f16", sms) == "flat")
    out.append(_case("flat_m3_long_k", 3, n, k, "f16", "gemv", route="flat", S=flat_plan(3, n, k, sms).S))
    return out


def _tile_cases(sms):
    """Every tile plan class the cost model picks for a served shape and m <= 4096, at m = j tn - 1, j tn, j tn + 1
    for the smallest j that keeps the class (one m where no such j exists); and for each split S > 1 a case with >= 3
    tiles per cluster where the tile count is not a multiple of the cluster count, so that some clusters do one tile
    fewer."""
    out, shapes, found = [], served_shapes(), served_plans(sms)
    for klass in sorted(c for c in found if c[0] == "tile"):
        _, tn, S, multi = klass
        hit = None
        for _, n, k in shapes:
            for j in range(1, 4096 // tn + 1):
                ms = (j * tn - 1, j * tn, j * tn + 1)
                if all(plan(mm, n, k, "f16", "gemm", sms).klass == klass for mm in ms):
                    hit = (ms, n, k)
                    break
            if hit:
                break
        if hit is None:
            m, n, k = found[klass][:3]
            hit = ((m,), n, k)
        ms, n, k = hit
        for mm, dtype in zip(ms, ("f16", "bf16", "f16")):
            out.append(_case(f"tile_tn{tn}_S{S}" + ("_multi" if multi else ""), mm, n, k, dtype, "gemm", route="tile",
                             tn=tn, S=S))
    splits = sorted({c[2] for c in found if c[0] == "tile" and c[2] > 1})
    for S in splits:
        best = None
        for _, n, k in shapes:
            for m in range(9, 4097):
                p = plan(m, n, k, "f16", "gemm", sms)
                if p.route == "tile" and p.S == S and p.tiles_per_cluster >= 3 and p.short_clusters:
                    if best is None or n * k * m < best[0]:
                        best = (n * k * m, m, n, k, p)
                    break
        if best:
            _, m, n, k, p = best
            out.append(_case(f"tile_S{S}_multi", m, n, k, "bf16", "gemm", route="tile", tn=p.tn, S=S,
                             tiles_per_cluster=p.tiles_per_cluster))
    return out


def _boundary_cases(sms):
    """m = 1, 4, 5, 7, 8, 9, 16, 17 on a served shape, both dtypes; and 9 / 16 tokens on n k just below and at the
    48 M weights from which the GEMM takes the tile launch directly."""
    out = []
    n, k = 4096, 4096
    for m in (1, 4, 5, 7, 8, 9, 16, 17):
        for dtype in ("f16", "bf16"):
            entry = "gemv" if m <= 7 else "gemm"
            out.append(_case(f"boundary_m{m}", m, n, k, dtype, entry, route=plan(m, n, k, dtype, entry, sms).route))
    pairs = [(a * BM, b * BM) for a in range(8, 257) for b in range(8, 257)]
    below = max((p for p in pairs if p[0] * p[1] < BIG_MID_WEIGHTS), key=lambda p: (p[0] * p[1], p[0]))
    at = min((p for p in pairs if p[0] * p[1] >= BIG_MID_WEIGHTS), key=lambda p: (p[0] * p[1], p[0]))
    for (n, k), route, tag in ((below, "flat", "below"), (at, "tile", "at")):
        for m, dtype in ((9, "f16"), (16, "bf16")):
            out.append(_case(f"big_mid_{tag}_48M", m, n, k, dtype, "gemm", route=route))
    return out


def edge_cases(sms):
    """The GPU cases for a device with `sms` SMs (see each generator's docstring)."""
    return (_decode_cases(sms) + _ring_cases(sms) + _stream_cases(sms) + _flat_cases(sms) + _tile_cases(sms)
            + _boundary_cases(sms))


# ------------------------------------------------------------------------------------------------ MLP front half
def silu_mul_plan(count, sms, vec=True):
    """launch_silu_mul over `count` elements of one flat row: 256 threads, 8 elements per thread when every pointer is
    16-byte aligned, grid-stride over at most 8 CTAs per SM."""
    return Plan("silu_mul", "silu_mul_kernel", max(1, min(-(-(count // 8 if vec else count) // 256), 8 * sms)), 0)


@functools.lru_cache(maxsize=None)
def mlp_front_plan(m, n, k, dtype, sms, y_aligned=True):
    """The launches of one b200awq_w4a16_mlp_front call, in stream order: the fused one-token kernel (one fp16 token,
    when its ring gets >= 3 slots), else gate and up through the kMlpProjection envelope into the workspace, then
    silu_mul_kernel over the m n products (vectorised when y is 16-byte aligned: the workspace always is).  Raises
    Rejected where the entry returns an error."""
    if m < 1 or n < 8 or k < GROUP or n % 8 or k % GROUP or (m >= 8 and n % BM):
        raise Rejected("shape")
    if m == 1 and dtype == "f16":
        p = decode_plan(n, k, sms, nt=2)
        if p:
            return (p,)
    proj = plan(m, n, k, dtype, "mlp", sms)
    return (proj, proj, silu_mul_plan(m * n, sms, y_aligned))


def _fused_candidates(sms):
    """(n, k) for k <= 32768 and, for every cluster count and row-block count r, the fewest even quad rows that give a
    CTA r row blocks and the most that do: the shapes at which the decode kernel's shared-memory layout changes."""
    qs = {2, 4}
    for S in (1, 2, 4, 8):
        if sms % S:
            continue
        u = sms // S
        for r in range(1, DEC_MAX_RB + 1):
            lo = 4 * u * (r - 1) + 1
            qs.update((lo + lo % 2, 4 * u * r))
    return [(4 * q, k) for k in _ks() for q in sorted(qs)]


@functools.lru_cache(maxsize=None)
def fused_reach(sms):
    """Over _fused_candidates: ({split: smallest (n, k)}, {ring slots: smallest-weight (n, k)}) of the fused kernel, and
    the smallest-weight (n, k) it declines while the plain decode kernel takes it."""
    splits, depths, decline = {}, {}, None
    for n, k in _fused_candidates(sms):
        p = decode_plan(n, k, sms, nt=2)
        if p is None:
            if decode_plan(n, k, sms) and (decline is None or n * k < decline[0] * decline[1]):
                decline = (n, k)
            continue
        for d, key in ((splits, p.S), (depths, p.ns)):
            if key not in d or n * k < d[key][0] * d[key][1]:
                d[key] = (n, k)
    return splits, depths, decline


def mlp_front_cases(sms):
    """The GPU cases of b200awq_w4a16_mlp_front on a device with `sms` SMs (entry "mlp_front"; `expect` holds attributes
    of the call's first launch):
      * fused: each split the fused kernel reaches, at Q = 4 units j -+ 2 quad rows (j = 1, 2: two units get one quad
        row fewer or more than the rest), the smallest k of that split, preferring an odd or uneven group count per rank;
      * fused: the smallest-weight shape of every ring depth it reaches;
      * the smallest shape the fused kernel declines (fewer than 3 ring slots) and the plain decode kernel takes: two
        plain decode launches and silu_mul;
      * the gate / up shapes of the Llama models in SERVED (make_fused_mlp replaces LlamaMLP only), one fp16 token;
      * composed on Llama-3-8B gate / up at m = 1 (bf16), 2 .. 17 tokens across every route boundary, among them 9..16
        tokens on this 58.7 M-weight layer, where kMlpProjection takes the flat launch and the GEMM the tile launch; a
        partial wgmma token tile; and 6 tokens with n % 128 != 0 (stream kernel)."""
    out = []
    splits, depths, decline = fused_reach(sms)
    for S in sorted(splits):
        units = sms // S
        for j in (1, 2):
            for dq in (-2, 2):
                Q = 4 * units * j + dq
                hits = [k for k in _ks() if (p := decode_plan(4 * Q, k, sms, nt=2)) and p.S == S]
                odd = [k for k in hits if k // GROUP // S > DEC_PIECE and ((k // GROUP) % S or (k // GROUP // S) % 2)]
                if not hits:
                    continue
                lo, hi = (4 * j - 1, 4 * j) if dq < 0 else (4 * j, 4 * j + 1)
                out.append(_case(f"fused_S{S}_q{4 * j}{dq:+d}", 1, 4 * Q, (odd or hits)[0], "f16", "mlp_front",
                                 route="fused", S=S, units=units, per_unit=(lo, hi)))
    for ns, (n, k) in sorted(depths.items()):
        out.append(_case(f"fused_ns{ns}", 1, n, k, "f16", "mlp_front", route="fused", ns=ns))
    if decline:
        n, k = decline
        out.append(_case("fused_declines", 1, n, k, "f16", "mlp_front", route="decode"))
    for model in ("llama2_7b", "llama3_8b", "llama2_70b_tp8"):
        n, k = next((n, k) for name, n, k in SERVED[model] if name == "gate_up")
        out.append(_case(f"{model}_gate_up", 1, n, k, "f16", "mlp_front", route="fused"))
    n, k = next((n, k) for name, n, k in SERVED["llama3_8b"] if name == "gate_up")
    for i, m in enumerate((1, 2, 4, 5, 7, 8, 9, 12, 16, 17)):
        dtype = "bf16" if m == 1 else ("f16", "bf16")[i % 2]
        out.append(_case(f"composed_m{m}", m, n, k, dtype, "mlp_front", route=plan(m, n, k, dtype, "mlp", sms).route))
    m = next(m for m in range(18, 4097) if (p := plan(m, n, k, "bf16", "mlp", sms)).route == "tile" and m % p.tn
             and m // p.tn >= 1)
    out.append(_case("composed_partial_tile", m, n, k, "bf16", "mlp_front", route="tile"))
    out.append(_case("composed_stream_n_not_128", 6, 2056, k, "f16", "mlp_front", route="stream"))
    return out


# ------------------------------------------------------------------------------------------------ sampled outputs
def edge_channels(p, n):
    """Output channels that carry the plan's edges: the first and last row block (decode) or octet (ring) of every
    unit, the first and last CTA row block (stream), the first and last channel of every 128-channel tile and the
    channels where a tile's warps and warpgroups meet (flat / tile); always the first and last channel."""
    ch = {0, n - 1}
    if p.route in ("decode", "fused", "ring"):
        size, block = (8, 8) if p.route == "ring" else (4, 16)
        rows = n // size
        for u in range(p.units):
            lo, hi = u * rows // p.units * size, (u + 1) * rows // p.units * size
            if hi > lo:
                ch.update(range(lo, min(hi, lo + block)))
                last = lo + (hi - lo - 1) // block * block
                ch.update(range(last, hi))
    elif p.route == "stream":
        r = 8 * p.ro
        ch.update(range(0, r))
        ch.update(range(n - r, n))
        ch.update(range(0, n, r))
        ch.update(range(r - 1, n, r))
    else:
        for t in range(0, n, BM):
            ch.update(t + o for o in (0, 7, 8, 63, 64, 127))
    return sorted(c for c in ch if c < n)


def edge_tokens(p, m):
    """Tokens that carry the plan's edges: every token up to 16; else the first and last token of every token tile
    and the last token (in the partial tile)."""
    if m <= 16:
        return list(range(m))
    t = {m - 1}
    for a in range(0, m, p.tn):
        t.update((a, min(a + p.tn, m) - 1))
    return sorted(t)
