"""Exact known-answer tests of the four attention entries (tests/attention_exact.py): which keys every output row sees,
and from which (batch row, KV head, slot) it reads them.

  * visibility probe over every block of the key range (and one block past it in a cache): exact zeros and w / n to
    one ulp of T, expected values from the float64 oracles (tests/prefill_attention_oracle.py,
    oracle/layer_oracle.single_query_attention);
  * pointer probe: every row returns its target key's value bit for bit.

Shapes come from the documented envelopes: single_query_attention (any G, D a multiple of 8 up to 256, ring caches,
per-sample lengths), flash_attn_func's split-key route (Sq * G <= 64, D in {64, 128}) and prefill route, the packed
varlen entry, and kv_cache_attention in both cache layouts (which must return the same bits)."""
import pytest
import torch

import llm_awq_b200 as P
import attention_exact as AE
import prefill_attention_oracle as PO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
NAME = {torch.float16: "f16", torch.bfloat16: "bf16"}
BETA = 16.0  # pointer probe with softmax_scale = 1: 32 per Hamming unit


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _visibility(run, oracle, w, n_keys, D, blocks, dtype, ctx, group=16):
    """Runs the visibility probe block by block and returns what the oracle reports as visible: [B, S, H, n_keys]
    (False in blocks not probed)."""
    vis = None
    for beta, want, exact in AE.visibility_expected(oracle, w, n_keys, D, blocks, dtype, group):
        got = run(AE.visibility_values(w, n_keys, D, beta).to(dtype))
        n, rep = AE.violations(got, want, dtype)
        assert n == 0, f"{ctx}: visibility block {beta} (keys from {beta * D}): {n} wrong, (b, i, h, c, got, want): {rep}"
        if vis is None:
            vis = torch.zeros(*exact.shape[:3], n_keys, dtype=torch.bool, device=exact.device)
        j1 = min(n_keys, (beta + 1) * D)
        if j1 > beta * D:
            vis[..., beta * D:j1] = exact[..., :j1 - beta * D] != 0
    return vis


def _pointer(run, oracle, vis, V, kv_heads, D, nbits, beta, dtype, ctx, seed):
    """The pointer probe over targets chosen from `vis`: the oracle gives V[target] exactly, and so must the kernel."""
    targets = AE.choose_targets(vis, seed)
    q = AE.pointer_queries(targets, kv_heads, D, nbits, beta)
    want = oracle(q).to(dtype)
    assert torch.equal(want, AE.gather_targets(V[:targets.shape[0]], targets, kv_heads).to(dtype)), ctx
    n, rep = AE.violations(run(q.to(dtype)), want, dtype, ulps=0)
    assert n == 0, f"{ctx}: pointer probe: {n} wrong, (b, i, h, c, got, want): {rep}"


# ------------------------------------------------------------------------------------------------ flash_attn_func
def _flash(B, Sq, Sk, H, Hkv, D, causal, dtype, seed):
    eng = P.engine()
    G = H // Hkv
    ctx = f"flash_attn_func B={B} Sq={Sq} Sk={Sk} H={H} Hkv={Hkv} D={D} causal={causal}"
    g = _gen(seed)
    w = AE.weights(B, Hkv, device=DEV)
    K = AE.random_keys(B, Sk, Hkv, D, g, DEV)
    q0 = torch.zeros(B, Sq, H, D, dtype=torch.float64, device=DEV)
    reps = [h * G for h in range(Hkv)]  # q = 0 in every head: one oracle head per KV head
    oracle = lambda V: PO.prefill_attention_torch(q0, K, V, causal, D ** -0.5, reps).repeat_interleave(G, 2)
    q0t, Kt = q0.to(dtype), K.to(dtype)
    vis = _visibility(lambda V: eng.flash_attn_func(q0t, Kt, V, 0.0, None, causal), oracle, w, Sk, D,
                      AE.all_blocks(Sk, D), dtype, ctx)
    nbits = AE.code_bits(Sk)
    Kp, Vp = AE.pointer_keys(B, Sk, Hkv, D, nbits, g, DEV), AE.pointer_values(B, Sk, Hkv, D, g, DEV)
    Kpt, Vpt = Kp.to(dtype), Vp.to(dtype)
    _pointer(lambda q: eng.flash_attn_func(q, Kpt, Vpt, 0.0, 1.0, causal),
             lambda q: PO.prefill_attention_torch(q, Kp, Vp, causal, 1.0), vis, Vp, Hkv, D, nbits, BETA, dtype, ctx, seed)


def _splitkv_cases():
    """Sq * G <= 64; odd G puts one query's heads across the 8-row halves of a thread's rows."""
    sks = (1, 127, 128, 129, 4097)
    for n, G in enumerate((1, 3, 5, 7, 8)):
        for m, Sq in enumerate((1, 2, 8)):
            for k, Sk in enumerate(sks):
                D = (64, 128)[(n + m + k) % 2]
                yield 2, Sq, Sk, 2 * G, 2, D, (n + m + k) % 3 != 2
    yield 1, 1, 16384, 8, 1, 128, True    # one cell, many splits
    yield 1, 8, 16384, 8, 1, 64, True
    yield 2, 8, 16384, 16, 2, 128, False
    yield 2, 8, 5, 8, 1, 64, True        # Sq > Sk: leading rows see no key
    yield 1, 64, 128, 1, 1, 128, True    # one split


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attn_splitkv(dtype):
    for i, case in enumerate(_splitkv_cases()):
        _flash(*case, dtype, seed=100 + i)


def _prefill_cases():
    """Sq * G > 64, so the prefill kernel runs."""
    for n, D in enumerate((64, 72, 128)):
        for m, G in enumerate((1, 4, 7)):
            for k, S in enumerate((127, 128, 129, 300)):
                yield 1 + (n + k) % 2, S, S, 2 * G, 2, D, (n + m + k) % 4 != 3
    yield 2, 17, 1000, 8, 2, 128, True    # bottom-right chunks
    yield 1, 200, 300, 14, 2, 64, True
    yield 1, 200, 300, 4, 4, 72, True
    yield 2, 300, 129, 8, 2, 128, True    # Sq > Sk
    yield 1, 129, 300, 2, 2, 64, False


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_attn_prefill(dtype):
    for i, case in enumerate(_prefill_cases()):
        _flash(*case, dtype, seed=300 + i)


# ------------------------------------------------------------------------------------------------ varlen
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lengths,H,D,causal", [([0, 1, 127, 128, 129, 300], 3, 64, True),
                                                ([300, 129, 0, 1, 128, 127], 3, 64, False),
                                                ([1, 129, 300, 0, 127], 2, 72, True),
                                                ([128, 1, 300, 127, 0], 4, 128, False)])
def test_flash_attn_varlen(lengths, H, D, causal, dtype):
    """Packed sequences: besides the masks, no row sees a key of another sequence (that key's channel stays 0)."""
    eng = P.engine()
    ctx = f"flash_attn_varlen_qkvpacked_func lengths={lengths} H={H} D={D} causal={causal}"
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    T = cu[-1]
    cu_t = torch.tensor(cu, dtype=torch.int32, device=DEV)
    g = _gen(T + H + D)

    def oracle_of(K):
        def oracle(q, V):  # the packed oracle returns D channels: one probe block per call
            a = lambda x: x[0].cpu().numpy()
            return torch.cat([torch.from_numpy(PO.prefill_attention(a(q), a(K), a(V[..., c:c + D]), causal, 1.0, cu))
                              for c in range(0, V.shape[-1], D)], -1).unsqueeze(0).to(DEV)
        return oracle

    def run(q, K, V):
        qkv = torch.stack([q[0], K[0], V[0]], 1)
        return eng.flash_attn_varlen_qkvpacked_func(qkv, cu_t, max(lengths), 0.0, 1.0, causal).unsqueeze(0)

    w = AE.weights(1, H, device=DEV)
    K = AE.random_keys(1, T, H, D, g, DEV)
    q0 = torch.zeros(1, T, H, D, dtype=torch.float64, device=DEV)
    orc = oracle_of(K)
    vis = _visibility(lambda V: run(q0.to(dtype), K.to(dtype), V), lambda V: orc(q0, V), w, T, D, AE.all_blocks(T, D),
                      dtype, ctx)
    nbits = AE.code_bits(T)
    Kp, Vp = AE.pointer_keys(1, T, H, D, nbits, g, DEV), AE.pointer_values(1, T, H, D, g, DEV)
    orc = oracle_of(Kp)
    _pointer(lambda q: run(q, Kp.to(dtype), Vp.to(dtype)), lambda q: orc(q, Vp), vis, Vp, H, D, nbits, BETA, dtype, ctx,
             T)


# ------------------------------------------------------------------------------------------------ kv_cache_attention
def _kv(B, Sq, Sk, G, D, causal, dtype, seed, Hkv=2, rows=None, sampled=None):
    """Batch B over caches of `rows` (default B + 1) rows and max_len past the last probe block; both layouts."""
    eng = P.engine()
    rows = B + 1 if rows is None else rows
    H = G * Hkv
    L = (-(-Sk // D) + 1) * D + 5
    ctx = f"kv_cache_attention B={B} rows={rows} Sq={Sq} Sk={Sk} L={L} H={H} Hkv={Hkv} D={D} causal={causal}"
    g = _gen(seed)

    def run(q, K, V):
        ft = eng.kv_cache_attention(q, AE.ft_k_cache(K), V.permute(0, 2, 1, 3).contiguous(), Sk, 1.0, causal)
        bthd = eng.kv_cache_attention(q, K, V, Sk, 1.0, causal)
        assert torch.equal(ft, bthd), f"{ctx}: the FT and [B, L, Hkv, D] layouts differ"
        return ft

    w = AE.weights(rows, Hkv, device=DEV)
    K = AE.random_keys(rows, L, Hkv, D, g, DEV)
    q0 = torch.zeros(B, Sq, H, D, dtype=torch.float64, device=DEV)
    reps = [h * G for h in range(Hkv)]
    oracle = lambda V: PO.prefill_attention_torch(q0, K[:B, :Sk], V[:B, :Sk], causal, 1.0, reps).repeat_interleave(G, 2)
    q0t, Kt = q0.to(dtype), K.to(dtype)
    blocks = AE.all_blocks(Sk, D, past=1) if sampled is None else sampled + [-(-Sk // D)]
    vis = _visibility(lambda V: run(q0t, Kt, V), oracle, w, L, D, blocks, dtype, ctx, group=16 if sampled is None else 4)
    nbits = AE.code_bits(L)
    Kp, Vp = AE.pointer_keys(rows, L, Hkv, D, nbits, g, DEV), AE.pointer_values(rows, L, Hkv, D, g, DEV)
    Kpt, Vpt = Kp.to(dtype), Vp.to(dtype)
    _pointer(lambda q: run(q, Kpt, Vpt), lambda q: PO.prefill_attention_torch(q, Kp[:B, :Sk], Vp[:B, :Sk], causal, 1.0),
             vis, Vp, Hkv, D, nbits, BETA, dtype, ctx, seed)


def _kv_cases():
    sks = (129, 1000, 4097, 300, 16384)
    n = 0
    for G in (1, 4, 7, 8):
        for Sq in (1, 17, 64, 65, 128, 129, 200, 512):
            Sk = max(sks[n % len(sks)], Sq) if Sq * G <= 1024 or sks[n % len(sks)] < 16384 else 4097
            yield 2, Sq, Sk, G, (128, 64)[n % 2], n % 4 != 3, n
            n += 1
    # a 128-row cell whose last row's horizon is the first key of a new 128-key tile
    yield 2, 128, 4097, 1, 128, True, n      # the only cell: rows 0 .. 127, last horizon 4096
    yield 2, 64, 1057, 4, 64, True, n + 1    # cell 0 of two: last row query 31, horizon 1024
    yield 2, 200, 100, 4, 128, True, n + 2   # Sq > Sk: leading rows see no key


@pytest.mark.parametrize("dtype", DTYPES)
def test_kv_cache_attention(dtype):
    for B, Sq, Sk, G, D, causal, i in _kv_cases():
        _kv(B, Sq, Sk, G, D, causal, dtype, seed=500 + i)


@pytest.mark.parametrize("dtype", DTYPES)
def test_kv_cache_attention_131072_sampled(dtype):
    """Block 0, every 64th block, the blocks of the causal horizons and the block past the keys."""
    Sk, Sq, D = 131072, 200, 128
    _kv(1, Sq, Sk, 4, D, True, dtype, seed=900, rows=1, sampled=AE.sampled_blocks(Sk, D, Sk - Sq, Sk, 64))


# ------------------------------------------------------------------------------------------------ single_query_attention
def _sq(B, G, Hkv, D, L, t, lps, dtype, seed):
    eng = P.engine()
    H = G * Hkv
    name = NAME[dtype]
    ctx = f"single_query_attention B={B} H={H} Hkv={Hkv} D={D} L={L} t={t} lps={lps}"
    ts = [t] * B if lps is None else list(lps)
    lps_t = None if lps is None else torch.tensor(lps, dtype=torch.int32, device=DEV)
    g = _gen(seed)

    def step(q, k, v, K, V, rot):
        kc = AE.ft_k_cache(K).to(dtype)
        vc = V.permute(0, 2, 1, 3).to(dtype).contiguous()
        return eng.single_query_attention(q.to(dtype).contiguous(), k.to(dtype).contiguous(), v.to(dtype).contiguous(), kc,
                                          vc, lps_t, None, t, rot, 10000.0, 1.0, True).unsqueeze(1)

    # visibility, RoPE over the whole head (q = 0 stays 0); the step's slot holds 0 in the cache, its value comes in v
    w = AE.weights(B, Hkv, device=DEV)
    K = AE.random_keys(B, L, Hkv, D, g, DEV)
    kin = AE.random_keys(B, 1, Hkv, D, g, DEV)[:, 0]
    q0 = torch.zeros(B, H, D, dtype=torch.float64, device=DEV)

    def run_vis(V):
        v = torch.stack([V[b, ts[b] % L] for b in range(B)])
        Vc = V.clone()
        for b in range(B):
            Vc[b, ts[b] % L] = 0
        return step(q0, kin, v, K, Vc, D)
    blocks = [b for b in AE.all_blocks(min(L, max(ts) + 1), D, past=1) if b * D < L]
    vis = _visibility(run_vis, AE.single_query_visibility_oracle(kin, K, t, D, H, name, lps), w, L, D, blocks, dtype, ctx)
    # pointer, no RoPE; the step's slot holds another key's code and another value
    nbits = AE.code_bits(L)
    Kt, Vt = AE.pointer_keys(B, L, Hkv, D, nbits, g, DEV), AE.pointer_values(B, L, Hkv, D, g, DEV)
    k, v, Kc, Vc = AE.single_query_step_inputs(Kt, Vt, t, lps)
    beta = float(round(16 * D ** 0.5))  # the scale is 1 / sqrt(D): about 32 per Hamming unit
    assert float(torch.tensor(beta).to(dtype)) == beta
    _pointer(lambda q: step(q[:, 0], k, v, Kc, Vc, 0),
             lambda q: AE.single_query_step(q[:, 0], k, v, Kc, Vc, t, 0, name, lps), vis, Vt, Hkv, D, nbits, beta, dtype,
             ctx, seed)


def _sq_cases():
    # (B, G, Hkv, D, L, t, lps): empty cache, short, on and beside 128-position edges, split over CTAs, wrapped ring
    contexts = [(1, 512, 0, None), (2, 512, 50, None), (1, 512, 127, None), (2, 512, 128, None), (1, 600, 256, None),
                (2, 4096, 3000, None), (2, 256, 700, None), (2, 300, 299, None), (3, 2304, 77, [5, 2100, 2400])]
    n = 0
    for G, Hkv in ((1, 2), (4, 2), (7, 2), (12, 2), (71, 1)):
        for D in (64, 128, 256, 80):
            B, L, t, lps = contexts[n % len(contexts)]
            yield B, G, Hkv, D, L, t, lps
            n += 1
    for B, L, t, lps in contexts:
        yield B, 7, 1, 224, L, t, lps


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_query_attention(dtype):
    for i, case in enumerate(_sq_cases()):
        _sq(*case, dtype, seed=700 + i)
