"""GPU tests of attention over a KV cache read in place: `awq_inference_engine.kv_cache_attention` and its C ABI
b200awq_kv_cache_attention (the split-key kernel of splitkv_attention.cu with two consumer warpgroups, in tinychat's
FasterTransformer cache layout or the [B, Lmax, Hkv, D] layout of long_forward).

The yardstick is the float64 definition in tests/prefill_attention_oracle.py over de-interleaved caches (`ft_keys` of
tests/test_kv_cache_attention_cpu.py indexes the FT cache as oracle/layer_oracle.py does), with the tolerances of the
other attention tests: 2e-3 (fp16) / 8e-3 (bf16) normwise per (batch row, head)."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P
import attention_gqa_cases as C
import prefill_attention_oracle as PO
from guard_bands import Op, guarded_call
from kernel_trace import trace
from test_kv_cache_attention_cpu import FT, BTHD, ft_keys, ft_values, _tinychat_chunk_kv, _tinychat_store

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
TOL = {torch.float16: 2e-3, torch.bfloat16: 8e-3}
COUNTER_BYTES = 4096 * 4
POISON = (float("nan"), float("inf"), -float("inf"), 65504.0, -65504.0)


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _poison_like(t):
    pat = torch.tensor(POISON, device=DEV).to(t.dtype)
    return pat[torch.arange(t.numel(), device=DEV) % len(POISON)].view(t.shape)


def _caches(layout, Bc, L, Hkv, D, Sk, dtype, seed, B=None, poison=False):
    """Caches of Bc rows and L slots in `layout`: slots < Sk of rows < B (default all) hold seeded data, the rest
    zeros, or NaN / +-inf / +-65504 when poisoned.  The data does not depend on the layout or on the fill."""
    B = Bc if B is None else B
    K, V = _rand((Bc, L, Hkv, D), dtype, seed), _rand((Bc, L, Hkv, D), dtype, seed + 1)
    for t in (K, V):
        rest = _poison_like(t) if poison else torch.zeros_like(t)
        keep = torch.zeros(Bc, L, 1, 1, dtype=torch.bool, device=DEV)
        keep[:B, :Sk] = True
        t.copy_(torch.where(keep, t, rest))
    if layout == BTHD:
        return K, V
    return K.view(Bc, L, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous(), V.permute(0, 2, 1, 3).contiguous()


def _logical(layout, kc, vc, B, Sk):
    """Keys / values 0 .. Sk - 1 of cache rows 0 .. B - 1 as [B, Sk, Hkv, D]."""
    if layout == FT:
        return ft_keys(kc[:B], Sk), ft_values(vc[:B], Sk)
    return kc[:B, :Sk], vc[:B, :Sk]


def _check(out, q, k, v, causal, scale, dtype, heads=None):
    """out [B, Sq, H, D] against the float64 oracle, normwise per (batch row, head); rows that see no key are zero."""
    H = q.shape[2]
    heads = (list(range(H)) if H <= 16 else sorted({0, H // 2, H - 1})) if heads is None else heads
    want = PO.prefill_attention_torch(q, k, v, causal, scale, heads)
    got = out[:, :, heads].double()
    assert torch.isfinite(got).all()
    for b in range(q.shape[0]):
        for n, h in enumerate(heads):
            w = want[b, :, n]
            wn = float(w.norm())
            if wn == 0.0:
                assert int(torch.count_nonzero(got[b, :, n])) == 0, (b, h)
                continue
            err = float((got[b, :, n] - w).norm() / wn)
            assert err <= TOL[dtype], (b, h, err)


def _near(a, b, tol):
    a, b = a.double(), b.double()
    for bb in range(a.shape[0]):
        for h in range(a.shape[2]):
            n = float(b[bb, :, h].norm())
            assert float((a[bb, :, h] - b[bb, :, h]).norm()) <= tol * max(n, 1e-30), (bb, h)


def _abi(q, kc, vc, out, layout, Sk, causal=True, ws=None, ws_bytes=None, scale=None):
    lib = P.lib()
    B, Sq, H, D = q.shape
    L = kc.shape[3] if layout == FT else kc.shape[1]
    Hkv = kc.shape[1] if layout == FT else kc.shape[2]
    if ws is None:
        ws_bytes = lib.b200awq_kv_cache_attention_workspace_bytes(layout, B, Sq, Sk, H, Hkv, D)
        ws = torch.zeros(max(ws_bytes, 16), dtype=torch.uint8, device=DEV)
    qs = (ctypes.c_longlong * 3)(q.stride(0), q.stride(1), q.stride(2))
    return lib.b200awq_kv_cache_attention(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), layout, B, Sq, Sk, L,
                                          H, Hkv, D, qs, ctypes.c_float(D ** -0.5 if scale is None else scale),
                                          1 if causal else 0, 0 if q.dtype == torch.float16 else 1, ws.data_ptr(),
                                          ws.numel() if ws_bytes is None else ws_bytes,
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


# ------------------------------------------------------------------------------------------------ oracle sweep
def _sweep_cases():
    for Sq in (1, 2, 16, 17, 33, 64, 65):
        for Sk in (Sq, 127, 128, 129, 1000, 4100, 16384):
            yield Sq, max(Sk, 1)
    for Sq in (128, 129, 512):
        for Sk in (Sq, Sq + 128, 1000, 4100):
            yield Sq, Sk


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [1, 4, 7, 8])
def test_oracle_sweep(G, D, dtype):
    """Both layouts on the same data return the same bits, and match the oracle: Sq from 1 to 512 (packed rows over
    one or more 128-row tiles), Sk at the 128-key tile edges and up to 16384, batch 2 of 3 cache rows (1 of 2 for long
    caches) with max_len > Sk; causal, and non-causal for the short chunks (Sq > Sk included)."""
    eng = P.engine()
    Hkv = 2
    H = G * Hkv
    for i, (Sq, Sk) in enumerate(_sweep_cases()):
        B = 2 if Sk <= 4100 else 1
        L = Sk + 37
        seed = 1000 * G + 10 * i + D
        q = _rand((B, Sq, H, D), dtype, seed)
        outs = {}
        for layout in (FT, BTHD):
            kc, vc = _caches(layout, B + 1, L, Hkv, D, Sk, dtype, seed + 1)
            for causal in (True, False) if Sq <= 65 and Sk <= 4100 else (True,):
                outs[layout, causal] = eng.kv_cache_attention(q, kc[:B], vc[:B], Sk, causal=causal)
                if layout == BTHD:
                    k, v = _logical(layout, kc, vc, B, Sk)
                    _check(outs[layout, causal], q, k, v, causal, D ** -0.5, dtype)
        for (layout, causal), o in outs.items():
            assert o.shape == q.shape and o.is_contiguous()
            assert torch.equal(o, outs[BTHD, causal]), (Sq, Sk, causal)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Sq", [1, 17, 200])
def test_131072_keys_sampled_heads(Sq, dtype):
    eng = P.engine()
    B, H, Hkv, D, Sk = 1, 32, 8, 128, 131072
    q = _rand((B, Sq, H, D), dtype, 77 + Sq)
    kc, vc = _caches(FT, B, Sk, Hkv, D, Sk, dtype, 78)
    out = eng.kv_cache_attention(q, kc, vc, Sk)
    k, v = _logical(FT, kc, vc, B, Sk)
    _check(out, q, k, v, True, D ** -0.5, dtype, heads=[0, 13, 31])


# ------------------------------------------------------------------------------------------------ in place, read only
@pytest.mark.parametrize("layout", [FT, BTHD])
@pytest.mark.parametrize("B,Sq,Sk,H,Hkv,D", [(2, 17, 4100, 32, 8, 128), (1, 300, 1300, 28, 4, 128), (2, 1, 9000, 14, 2, 64),
                                             (2, 65, 129, 8, 8, 64)])
def test_reads_only_its_slots_and_rows(layout, B, Sq, Sk, H, Hkv, D):
    """Cache slots >= Sk and cache rows >= B hold NaN / +-inf / +-65504: the output is bit-identical to that over clean
    caches, and both caches are unchanged afterwards."""
    eng = P.engine()
    dtype, L = torch.float16, Sk + 300
    q = _rand((B, Sq, H, D), dtype, Sq + Sk)
    kc, vc = _caches(layout, B + 1, L, Hkv, D, Sk, dtype, 5, B=B)
    clean = eng.kv_cache_attention(q, kc[:B], vc[:B], Sk)
    kp, vp = _caches(layout, B + 1, L, Hkv, D, Sk, dtype, 5, B=B, poison=True)
    k0, v0 = kp.clone(), vp.clone()
    got = eng.kv_cache_attention(q, kp[:B], vp[:B], Sk)
    torch.cuda.synchronize()
    assert torch.equal(got, clean)
    assert torch.equal(kp.view(torch.int16), k0.view(torch.int16)) and torch.equal(vp.view(torch.int16), v0.view(torch.int16))
    k, v = _logical(layout, kc, vc, B, Sk)
    _check(clean, q, k, v, True, D ** -0.5, dtype)


@pytest.mark.parametrize("case", ["ft_sq17_g4", "ft_r130_d64", "bthd_sq129_g1", "ft_single_split", "bthd_sq65_g7"])
def test_guard_bands(case):
    """Every operand, the workspace included, between 4 KiB guard bands: partial row tiles (R not a multiple of 8, of
    64 or of 128), Sk not a multiple of 128, several splits and one split (written directly, no workspace)."""
    layout, B, Sq, Sk, H, Hkv, D = {"ft_sq17_g4": (FT, 2, 17, 2000, 32, 8, 128), "ft_r130_d64": (FT, 1, 26, 1500, 10, 2, 64),
                                    "bthd_sq129_g1": (BTHD, 1, 129, 700, 4, 4, 128),
                                    "ft_single_split": (FT, 2, 40, 100, 8, 2, 64),
                                    "bthd_sq65_g7": (BTHD, 1, 65, 4100, 14, 2, 128)}[case]
    dtype = torch.float16
    L = Sk + 50
    q = _rand((B, Sq, H, D), dtype, Sk + H)
    kc, vc = _caches(layout, B, L, Hkv, D, Sk, dtype, 9)
    need = P.lib().b200awq_kv_cache_attention_workspace_bytes(layout, B, Sq, Sk, H, Hkv, D)
    assert (need == 0) == (case == "ft_single_split")
    ops = {"q": Op("in", q), "k": Op("in", kc), "v": Op("in", vc), "out": Op("out", shape=q.shape, dtype=dtype)}
    if need:
        ops["ws"] = Op("zeroed", shape=(need,), dtype=torch.uint8)

    def call(v):
        ws = v.get("ws", torch.empty(16, dtype=torch.uint8, device=DEV))
        rc = _abi(v["q"], v["k"], v["v"], v["out"], layout, Sk, ws=ws, ws_bytes=need)
        torch.cuda.synchronize()
        assert not need or int(torch.count_nonzero(ws[:COUNTER_BYTES])) == 0, "counters not left zero"
        return rc
    got = guarded_call(call, ops)["out"]
    k, v = _logical(layout, kc, vc, B, Sk)
    _check(got, q, k, v, True, D ** -0.5, dtype)


def traced_call(layout, Sq):
    """kernel_trace builder: one call over a cache of 9000 slots, q a strided view of the fused qkv output, read in
    place."""
    B, L, H, Hkv, D = 1, 9000, 32, 8, 128
    kc, vc = _caches(layout, B, L, Hkv, D, 8500, torch.float16, 1)
    q = torch.randn(B, Sq, H + 2 * Hkv, D, device=DEV).half()[:, :, :H]
    return lambda: P.engine().kv_cache_attention(q, kc, vc, 8500)


def test_one_kernel_per_call():
    """Each call over a cache, q a view of the fused qkv output, runs exactly one kernel (the split-key kernel; the
    combine is inside it) and no copy, fill or elementwise kernel."""
    cases = {"ft_sq17": (FT, 17), "ft_sq300": (FT, 300), "bthd_sq64": (BTHD, 64)}
    for name, rec in zip(cases, trace("test_kv_cache_attention_gpu:traced_call", cases.values(), per_process=8)):
        assert len(rec.names) == 1 and "splitkv_attention_kernel" in rec.names[0], (name, rec.names)


# ------------------------------------------------------------------------------------------------ agreement
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,Sq,Sk,H,Hkv,D,causal", [(1, 1, 16384, 32, 8, 128, True), (2, 16, 4100, 32, 8, 128, True),
                                                    (2, 8, 2048, 28, 4, 128, False), (1, 64, 1000, 8, 8, 64, True),
                                                    (3, 9, 20000, 14, 2, 64, True), (1, 4, 300, 64, 4, 64, True)])
def test_bthd_is_bit_identical_to_flash_attn_func_for_few_rows(B, Sq, Sk, H, Hkv, D, causal, dtype):
    """Sq * G <= 64 over a [B, Lmax, Hkv, D] cache: the same bits as flash_attn_func over the cache view (its split-key
    route), because both run the same kernel arithmetic with the same split plan."""
    eng = P.engine()
    L = Sk + 100
    q = _rand((B, Sq, H, D), dtype, Sq * 7 + Sk)
    kc, vc = _caches(BTHD, B + 1, L, Hkv, D, Sk, dtype, 13)
    want = eng.flash_attn_func(q, kc[:B, :Sk], vc[:B, :Sk], causal=causal)
    assert torch.equal(eng.kv_cache_attention(q, kc[:B], vc[:B], Sk, causal=causal), want)


@pytest.mark.parametrize("G,D", [(4, 64), (4, 128), (7, 128), (1, 128)])
def test_one_query_agrees_with_single_query_attention(G, D):
    """Sq = 1 over the FT caches that single_query_attention has just written its step into."""
    eng = P.engine()
    dtype, B, Hkv, L = torch.float16, 2, 2, 5000
    H, t = G * Hkv, 4321
    _, q, kn, vn = C.fused_qkv(B, H, Hkv, D, dtype, seed=G + D, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, t, seed=G * D, device=DEV)
    dec = eng.single_query_attention(q, kn, vn, kc, vc, None, None, t, 0, 10000.0, 1.0, True)
    got = eng.kv_cache_attention(q.reshape(B, 1, H, D), kc, vc, t + 1).reshape(B, 1, H, D)
    _near(got, dec.reshape(B, 1, H, D), 2e-3)


# ------------------------------------------------------------------------------------------------ tinychat's chunk branch
def _rope(eng, x, freqs):
    """x [B, S, h, D] -> rotated [B, S, h, D] through fused_rope_with_pos_forward_func(..., True), as tinychat calls it
    on its [s, b, h, d] view (the output is a transposed-memory view)."""
    return eng.fused_rope_with_pos_forward_func(x.transpose(0, 1), freqs, True).transpose(0, 1)


@pytest.mark.parametrize("H,Hkv,D", [pytest.param(32, 8, 128, id="llama3_8b"), pytest.param(28, 4, 128, id="qwen2_7b")])
def test_tinychat_multi_round(H, Hkv, D):
    """A prefill of 1000 tokens, then chunks of 17, 64 and 300.  For each chunk, q and k come from the fused qkv output
    through fused_rope_with_pos_forward_func(..., True), k / v are stored into the decode caches as the branch stores
    them, and kv_cache_attention over the caches matches the branch's copy + flash_attn_func route; the last chunk's
    rows match one attention over the whole sequence."""
    eng = P.engine()
    dtype, B, Lmax = torch.float16, 1, 2048
    cache_k = torch.zeros(B, Hkv, D // 8, Lmax, 8, dtype=dtype, device=DEV)
    cache_v = torch.zeros(B, Hkv, Lmax, D, dtype=dtype, device=DEV)
    qs, ks, vs = [], [], []
    start = 0
    for i, S in enumerate((1000, 17, 64, 300)):
        xqkv = _rand((B, S, H + 2 * Hkv, D), dtype, 40 + i)
        freqs = (torch.rand(B, S, D, generator=torch.Generator(device=DEV).manual_seed(50 + i), device=DEV) * 6.0)
        xq = _rope(eng, xqkv[:, :, :H], freqs)
        xk = _rope(eng, xqkv[:, :, H:H + Hkv], freqs)
        xv = xqkv[:, :, H + Hkv:]
        keys, values = _tinychat_chunk_kv(cache_k, cache_v, xk, xv, start)
        _tinychat_store(cache_k, cache_v, xk, xv, start)
        got = eng.kv_cache_attention(xq, cache_k[:B], cache_v[:B], start + S)
        want = eng.flash_attn_func(xq, keys, values, causal=True)
        _near(got, want, TOL[dtype])
        qs.append(xq), ks.append(xk), vs.append(xv)
        start += S
    whole = eng.flash_attn_func(torch.cat(qs, 1), torch.cat(ks, 1), torch.cat(vs, 1), causal=True)
    _near(got, whole[:, -300:], TOL[dtype])
    _check(got, xq, torch.cat(ks, 1), torch.cat(vs, 1), True, D ** -0.5, dtype)


# ------------------------------------------------------------------------------------------------ properties
def test_row_isolation():
    """The probe (batch row 1, query head 5, queries 60 .. 69, spanning the packed rows of two row tiles) is
    bit-identical whether every other query row holds data or NaN / inf."""
    eng = P.engine()
    dtype, B, Sq, Sk, H, Hkv, D = torch.float16, 2, 100, 3000, 16, 4, 128
    q = _rand((B, Sq, H, D), dtype, 123)
    kc, vc = _caches(FT, B, Sk, Hkv, D, Sk, dtype, 124)
    clean = eng.kv_cache_attention(q, kc, vc, Sk)
    qp = _poison_like(q)
    qp[1, 60:70, 5] = q[1, 60:70, 5]
    got = eng.kv_cache_attention(qp, kc, vc, Sk)
    assert torch.equal(got[1, 60:70, 5], clean[1, 60:70, 5])


def test_determinism_graph_and_side_stream():
    """More than one split: repeated calls, a call on a side stream (its own workspace) and the replays of a captured
    graph over new inputs all return the same bits as a direct call."""
    eng = P.engine()
    dtype, B, Sq, Sk, H, Hkv, D = torch.bfloat16, 1, 40, 20000, 32, 8, 128
    assert P.lib().b200awq_kv_cache_attention_workspace_bytes(FT, B, Sq, Sk, H, Hkv, D) > 0
    q = _rand((B, Sq, H, D), dtype, 41)
    kc, vc = _caches(FT, B, Sk + 10, Hkv, D, Sk, dtype, 42)
    first = eng.kv_cache_attention(q, kc, vc, Sk)
    for _ in range(3):
        assert torch.equal(eng.kv_cache_attention(q, kc, vc, Sk), first)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        on_side = eng.kv_cache_attention(q, kc, vc, Sk)
    side.synchronize()
    assert torch.equal(on_side, first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.kv_cache_attention(q, kc, vc, Sk)  # the capture stream's workspace exists before capture
    s.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        o = eng.kv_cache_attention(q, kc, vc, Sk)
    for seed in (44, 47):
        q.copy_(_rand((B, Sq, H, D), dtype, seed))
        k2, v2 = _caches(FT, B, Sk + 10, Hkv, D, Sk, dtype, seed + 1)
        kc.copy_(k2), vc.copy_(v2)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(o, eng.kv_cache_attention(q, kc, vc, Sk))


def test_interleaved_with_single_query_attention_on_one_workspace():
    """Decode steps (single_query_attention) and chunk calls alternate on one stream and one workspace, through the C
    ABI: results equal those of calls with workspaces of their own, and the counter block is zero after each sync."""
    lib = P.lib()
    dtype, B, H, Hkv, D, L, t = torch.float16, 2, 28, 4, 128, 6000, 5000
    _, q1, kn, vn = C.fused_qkv(B, H, Hkv, D, dtype, seed=5, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, t, seed=6, device=DEV)
    qc = _rand((B, 33, H, D), dtype, 7)
    need = max(lib.b200awq_single_query_attention_workspace_bytes(B, H, Hkv, D, L),
               lib.b200awq_kv_cache_attention_workspace_bytes(FT, B, 33, t + 1, H, Hkv, D))
    assert lib.b200awq_kv_cache_attention_workspace_bytes(FT, B, 33, t + 1, H, Hkv, D) > 0
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def decode(out, w):
        return lib.b200awq_single_query_attention(q1.data_ptr(), kn.data_ptr(), vn.data_ptr(), kc.data_ptr(), vc.data_ptr(),
                                                  out.data_ptr(), None, B, H, Hkv, D, L, t, q1.stride(0), kn.stride(0),
                                                  vn.stride(0), 0, ctypes.c_float(10000.0), ctypes.c_float(1.0), 1, 0,
                                                  w.data_ptr(), w.numel(), st)
    dec_own, chunk_own = torch.empty(B, H, D, dtype=dtype, device=DEV), torch.empty_like(qc)
    assert decode(dec_own, torch.zeros(need, dtype=torch.uint8, device=DEV)) == 0
    assert _abi(qc, kc, vc, chunk_own, FT, t + 1) == 0
    for _ in range(3):
        dec, chunk = torch.empty_like(dec_own), torch.empty_like(chunk_own)
        assert decode(dec, ws) == 0
        assert _abi(qc, kc, vc, chunk, FT, t + 1, ws=ws, ws_bytes=need) == 0
        torch.cuda.synchronize()
        assert int(torch.count_nonzero(ws[:COUNTER_BYTES])) == 0
        assert torch.equal(dec, dec_own) and torch.equal(chunk, chunk_own)


# ------------------------------------------------------------------------------------------------ rejected inputs
@pytest.mark.parametrize("what", ["seqlen_k", "negative_seqlen_k", "d96", "ratio", "fp32", "dtype_mix", "v_shape",
                                  "k_dims", "batch", "scale", "noncontiguous_cache"])
def test_rejected_inputs_raise(what):
    eng = P.engine()
    dtype, B, Sq, H, Hkv, D, L = torch.float16, 1, 5, 8, 2, 128, 300
    q = _rand((B, Sq, H, D), dtype, 3)
    kc, vc = _caches(FT, B, L, Hkv, D, L, dtype, 4)
    args, kw = [q, kc, vc, 200], {}
    if what == "seqlen_k":
        args[3] = L + 1
    elif what == "negative_seqlen_k":
        args[3] = -1
    elif what == "d96":
        args[0] = _rand((B, Sq, H, 96), dtype, 3)
        args[1], args[2] = _caches(FT, B, L, Hkv, 96, L, dtype, 4)
    elif what == "ratio":
        args[0] = _rand((B, Sq, 7, D), dtype, 3)
    elif what == "fp32":
        args[0], args[1], args[2] = q.float(), kc.float(), vc.float()
    elif what == "dtype_mix":
        args[0] = q.bfloat16()
    elif what == "v_shape":
        args[2] = vc[:, :, :L - 1].contiguous()
    elif what == "k_dims":
        args[1] = kc.view(B, Hkv, -1)
    elif what == "batch":
        args[0] = _rand((B + 1, Sq, H, D), dtype, 3)
    elif what == "scale":
        kw["softmax_scale"] = 0.0
    else:
        args[1] = kc.transpose(3, 4).contiguous().transpose(3, 4)
    with pytest.raises(RuntimeError):
        eng.kv_cache_attention(*args, **kw)
