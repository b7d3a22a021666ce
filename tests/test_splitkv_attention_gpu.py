"""GPU tests of attention of few queries over many keys: `flash_attn_func` calls with seqlen_q * (heads / kv_heads) <= 64
take the split-key kernel (splitkv_attention.cu, C ABI b200awq_splitkv_attention); everything else keeps the prefill
kernel.

The yardstick is the float64 definition in tests/prefill_attention_oracle.py, with the tolerances of the other attention
tests: 2e-3 (fp16) / 8e-3 (bf16) normwise per (batch row, head)."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P
import attention_gqa_cases as C
import prefill_attention_oracle as PO
from guard_bands import Op, guarded_call
from kernel_trace import trace
from test_prefill_attention_gpu import _siglip_qkv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
TOL = {torch.float16: 2e-3, torch.bfloat16: 8e-3}
SHAPE, ALIGN, WORKSPACE = -1, -3, -6
COUNTER_BYTES = 4096 * 4  # the workspace's counter block at offset 0 (kAttentionCounters u32)


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


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


def _inputs(B, Sq, Sk, H, Hkv, D, dtype, seed):
    return _rand((B, Sq, H, D), dtype, seed), _rand((B, Sk, Hkv, D), dtype, seed + 1), _rand((B, Sk, Hkv, D), dtype, seed + 2)


def _st(t):
    return (t.stride(0), t.stride(1), t.stride(2))


def _abi(q, k, v, out, causal, ws=None, ws_bytes=None, scale=None, strides=None, entry="splitkv", head_dim=None):
    """The C-ABI entry on torch tensors (or guard-banded views); returns its return code."""
    lib = P.lib()
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    D = head_dim or D
    arr = lambda s: (ctypes.c_longlong * 3)(*s)
    qs, ks, vs = strides or (_st(q), _st(k), _st(v))
    sc = ctypes.c_float(D ** -0.5 if scale is None else scale)
    dt = 0 if q.dtype == torch.float16 else 1
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if entry == "prefill":
        return lib.b200awq_prefill_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), None, None, B, Sq, Sk, H,
                                             Hkv, D, arr(qs), arr(ks), arr(vs), sc, 1 if causal else 0, dt, stream)
    if ws is None:
        need = lib.b200awq_splitkv_attention_workspace_bytes(B, Sq, Sk, H, Hkv, D)
        ws = torch.zeros(max(need, 16), dtype=torch.uint8, device=DEV)
        ws_bytes = need
    return lib.b200awq_splitkv_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, Sq, Sk, H, Hkv, D,
                                         arr(qs), arr(ks), arr(vs), sc, 1 if causal else 0, dt, ws.data_ptr(),
                                         ws.numel() if ws_bytes is None else ws_bytes, stream)


# ------------------------------------------------------------------------------------------------ oracle sweep
def _sweep_cases(G):
    sqs = sorted({s for s in (1, 2, 4, 8, 64 // G) if s * G <= 64}) if G <= 8 else [1]
    for Sq in sqs:
        for Sk in (1, 127, 128, 129, 1000, 4100, 16384):
            yield Sq, Sk


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [1, 4, 5, 7, 8, 16])
def test_oracle_sweep(G, D, dtype):
    """Sq in {1, 2, 4, 8} and Sq * G = 64 exactly; Sk at the 128-key tile edges and over many splits; batch 1 and 3;
    causal and not, including Sq > Sk (leading rows see no key)."""
    eng = P.engine()
    Hkv = 2
    H = G * Hkv
    for i, (Sq, Sk) in enumerate(_sweep_cases(G)):
        B = 3 if Sk <= 1000 else 1
        q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, 1000 * G + 10 * i + D)
        for causal in (False, True):
            out = eng.flash_attn_func(q, k, v, causal=causal)
            assert out.shape == q.shape and out.is_contiguous()
            _check(out, q, k, v, causal, D ** -0.5, dtype)
            if causal and Sq > Sk:
                assert int(torch.count_nonzero(out[:, :Sq - Sk])) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_131072_keys_sampled_heads(dtype):
    eng = P.engine()
    B, H, Hkv, D, Sk = 1, 32, 8, 128, 131072
    q, k, v = _inputs(B, 1, Sk, H, Hkv, D, dtype, 77)
    out = eng.flash_attn_func(q, k, v, causal=True)
    _check(out, q, k, v, True, D ** -0.5, dtype, heads=[0, 13, 31])


# ------------------------------------------------------------------------------------------------ tinychat's decode step
def _decode_step(eng, B, H, Hkv, D, Lmax, t, dtype, poison):
    """QuantLlamaAttentionFused.long_forward for one token: a fused qkv projection, q rotated by
    fused_rope_with_pos_forward_func(..., True) (transposed-memory output), k / v stored at slot t of [B, Lmax, Hkv, D]
    caches, attention over cache[:, :t + 1].  Slots past t hold `poison` (or zeros)."""
    qkv = _rand((B, 1, (H + 2 * Hkv) * D), dtype, 5)
    xq = qkv[..., :H * D].view(B, 1, H, D)
    xk = qkv[..., H * D:(H + Hkv) * D].view(B, 1, Hkv, D)
    xv = qkv[..., (H + Hkv) * D:].view(B, 1, Hkv, D)
    g = torch.Generator(device=DEV).manual_seed(6)
    freqs = (torch.rand(B, 1, D, generator=g, device=DEV) * 6.0).contiguous()
    q = eng.fused_rope_with_pos_forward_func(xq.transpose(0, 1), freqs, True).transpose(0, 1)  # [B, 1, H, D]
    kc = torch.zeros(B, Lmax, Hkv, D, dtype=dtype, device=DEV)
    vc = torch.zeros(B, Lmax, Hkv, D, dtype=dtype, device=DEV)
    kc[:, :t] = _rand((B, t, Hkv, D), dtype, 7)
    vc[:, :t] = _rand((B, t, Hkv, D), dtype, 8)
    kc[:, t:t + 1] = xk
    vc[:, t:t + 1] = xv
    if poison:
        tail = Lmax - t - 1
        pat = torch.tensor([float("nan"), float("inf"), -float("inf"), 65504.0, -65504.0], device=DEV).to(dtype)
        fill = pat[torch.arange(tail * Hkv * D, device=DEV) % 5].view(1, tail, Hkv, D)
        kc[:, t + 1:] = fill
        vc[:, t + 1:] = fill.flip(-1)
    return q, kc[:, :t + 1], vc[:, :t + 1]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Hkv,D,t", [(32, 8, 128, 9000), (28, 4, 128, 3000), (14, 2, 64, 129), (32, 8, 128, 0)])
def test_tinychat_decode_step(H, Hkv, D, t, dtype):
    eng = P.engine()
    B, Lmax = 2, t + 700
    q, k, v = _decode_step(eng, B, H, Hkv, D, Lmax, t, dtype, poison=False)
    assert k.stride(1) == Hkv * D and k.stride(0) == Lmax * Hkv * D  # views into the caches
    clean = eng.flash_attn_func(q, k, v, causal=True)
    _check(clean, q, k, v, True, D ** -0.5, dtype)
    q, k, v = _decode_step(eng, B, H, Hkv, D, Lmax, t, dtype, poison=True)
    assert torch.equal(eng.flash_attn_func(q, k, v, causal=True), clean)


# ------------------------------------------------------------------------------------------------ combine edge cases
@pytest.mark.parametrize("dtype", DTYPES)
def test_one_split_holds_the_max_by_a_wide_margin(dtype):
    """A few keys in one split score ~30 above every other key: the other splits' weights underflow towards 0."""
    eng = P.engine()
    B, Sq, H, Hkv, D, Sk = 1, 2, 32, 8, 128, 16384
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, 91)
    for j in (9000, 9001, 9100):
        k[:, j] = (q[:, 0].view(B, Hkv, H // Hkv, D).float().mean(2) * 6.0).to(dtype)
    out = eng.flash_attn_func(q, k, v, causal=False)
    _check(out, q, k, v, False, D ** -0.5, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,Sq,Sk,H,Hkv", [(1, 64, 160, 1, 1), (1, 16, 300, 4, 1), (2, 8, 40, 8, 1), (1, 64, 1000, 1, 1),
                                             (2, 64, 40, 1, 1), (1, 16, 140, 4, 1)])
def test_causal_splits_masked_for_some_rows(B, Sq, Sk, H, Hkv, dtype):
    """Bottom-right causal few-query tiles: the later splits are fully masked for the first rows and not for the last
    ones; with Sq > Sk the first rows see no key at all and are zero."""
    eng = P.engine()
    D = 64
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, Sq + Sk)
    out = eng.flash_attn_func(q, k, v, causal=True)
    _check(out, q, k, v, True, D ** -0.5, dtype)


# ------------------------------------------------------------------------------------------------ agreement with other routes
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,Sq,Sk,H,Hkv,D,causal", [(1, 1, 16384, 32, 8, 128, True), (3, 4, 4100, 28, 4, 128, True),
                                                    (2, 16, 2048, 8, 2, 64, False), (1, 8, 1000, 14, 2, 64, True)])
def test_agrees_with_the_prefill_kernel(B, Sq, Sk, H, Hkv, D, causal, dtype):
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, 3 * Sq + Sk)
    new, old = torch.empty_like(q), torch.empty_like(q)
    assert _abi(q, k, v, new, causal) == 0
    assert _abi(q, k, v, old, causal, entry="prefill") == 0
    torch.cuda.synchronize()
    a, b = new.double(), old.double()
    for bb in range(B):
        for h in range(H):
            assert float((a[bb, :, h] - b[bb, :, h]).norm() / b[bb, :, h].norm()) <= TOL[dtype], (bb, h)


@pytest.mark.parametrize("G,D", [(4, 64), (4, 128), (7, 64), (7, 128)])
def test_agrees_with_single_query_attention(G, D):
    eng = P.engine()
    dtype, B, Hkv, L = torch.float16, 2, 2, 5000
    H, t = G * Hkv, L - 1
    _, q, kn, vn = C.fused_qkv(B, H, Hkv, D, dtype, seed=G + D, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, t, seed=G * D, device=DEV)
    dec = eng.single_query_attention(q, kn, vn, kc, vc, None, None, t, 0, 10000.0, 1.0, True)
    keys = kc.permute(0, 3, 1, 2, 4).reshape(B, L, Hkv, D)  # the cache after the step stored kn, vn at slot t
    vals = vc.permute(0, 2, 1, 3)
    got = eng.flash_attn_func(q.reshape(B, 1, H, D), keys, vals, causal=True).reshape(B, H, D).double()
    d = dec.double()
    for b in range(B):
        for h in range(H):
            assert float((got[b, h] - d[b, h]).norm() / d[b, h].norm()) <= 2e-3, (b, h)


# ------------------------------------------------------------------------------------------------ isolation, determinism
def test_row_isolation():
    """The probe (batch row 1, query head 5, both queries) is bit-identical whether the other query heads, the other KV
    heads and the other batch rows hold data or NaN / inf / 65504."""
    eng = P.engine()
    dtype, B, Sq, Sk, H, Hkv, D = torch.float16, 3, 2, 5000, 16, 4, 128
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, 123)
    pb, ph = 1, 5
    clean = eng.flash_attn_func(q, k, v, causal=True)
    qp, kp, vp = q.clone(), k.clone(), v.clone()
    qp[:, :, [h for h in range(H) if h != ph]] = float("nan")
    qp[[b for b in range(B) if b != pb]] = float("inf")
    others = [h for h in range(Hkv) if h != ph // (H // Hkv)]
    kp[:, :, others] = float("nan")
    vp[:, :, others] = 65504.0
    kp[[b for b in range(B) if b != pb]] = -float("inf")
    vp[[b for b in range(B) if b != pb]] = float("nan")
    got = eng.flash_attn_func(qp, kp, vp, causal=True)
    assert torch.equal(got[pb, :, ph], clean[pb, :, ph])


def test_determinism_graph_and_side_stream():
    eng = P.engine()
    dtype, B, Sq, Sk, H, Hkv, D = torch.bfloat16, 2, 1, 20000, 32, 8, 128
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, 41)
    first = eng.flash_attn_func(q, k, v, causal=True)
    for _ in range(3):
        assert torch.equal(eng.flash_attn_func(q, k, v, causal=True), first)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # a stream of its own: its own workspace
        on_side = eng.flash_attn_func(q, k, v, causal=True)
    side.synchronize()
    assert torch.equal(on_side, first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.flash_attn_func(q, k, v, causal=True)  # the capture stream's workspace exists before capture
    s.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        o = eng.flash_attn_func(q, k, v, causal=True)
    for seed in (44, 47):
        q2, k2, v2 = _inputs(B, Sq, Sk, H, Hkv, D, dtype, seed)
        q.copy_(q2), k.copy_(k2), v.copy_(v2)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(o, eng.flash_attn_func(q, k, v, causal=True))


# ------------------------------------------------------------------------------------------------ guard bands
@pytest.mark.parametrize("case", ["sk1000_r4", "sk4100_r5_d64", "r21_causal", "single_split", "r64"])
def test_guard_bands(case):
    """Every operand between guard bands, the workspace included (zeroed before the call, beyond
    b200awq_splitkv_attention_workspace_bytes): Sk not a multiple of 128, the last split's partial tile, R = Sq * G not
    a multiple of 8, and one split (written directly).  After every call the workspace's counter block is zero again, as
    the header promises (single_query_attention shares the buffer)."""
    dtype = torch.float16
    B, Sq, Sk, H, Hkv, D, causal = {"sk1000_r4": (2, 1, 1000, 8, 2, 128, True), "sk4100_r5_d64": (1, 1, 4100, 10, 2, 64, True),
                                    "r21_causal": (2, 3, 2000, 14, 2, 128, True), "single_split": (3, 2, 100, 8, 2, 64, False),
                                    "r64": (1, 16, 700, 8, 2, 128, True)}[case]
    q, k, v = _inputs(B, Sq, Sk, H, Hkv, D, dtype, Sk + H)
    need = P.lib().b200awq_splitkv_attention_workspace_bytes(B, Sq, Sk, H, Hkv, D)
    assert (need == 0) == (case == "single_split")
    ops = {"q": Op("in", q), "k": Op("in", k), "v": Op("in", v), "out": Op("out", shape=(B, Sq, H, D), dtype=dtype)}
    if need:
        ops["ws"] = Op("zeroed", shape=(need,), dtype=torch.uint8)

    def call(vw):
        ws = vw.get("ws")
        if ws is None:
            ws = torch.empty(0, dtype=torch.uint8, device=DEV)
        rc = _abi(vw["q"], vw["k"], vw["v"], vw["out"], causal, ws=ws, ws_bytes=need)
        if rc == 0 and need:
            torch.cuda.synchronize()
            assert int(torch.count_nonzero(ws[:COUNTER_BYTES])) == 0, "counters not left zero"
        return rc
    plain = guarded_call(call, ops)
    _check(plain["out"], q, k, v, causal, D ** -0.5, dtype)


def test_shared_workspace_grows_without_freeing_a_captured_buffer():
    """flash_attn_func's split-key calls and single_query_attention share one workspace per stream.  A graph captured
    while it was small keeps replaying correctly after larger calls of both entries have grown it."""
    eng = P.engine()
    dtype = torch.float16
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        q, k, v = _inputs(1, 1, 300, 8, 2, 64, dtype, 501)   # a small workspace
        eng.flash_attn_func(q, k, v, causal=True)
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            o = eng.flash_attn_func(q, k, v, causal=True)
        big = _inputs(2, 4, 40000, 32, 8, 128, dtype, 502)  # grows the workspace
        want_big = eng.flash_attn_func(*big, causal=True)
        _, q1, k1, v1 = C.fused_qkv(4, 28, 4, 128, dtype, seed=503, device=DEV)
        kc, vc = C.caches(4, 4, 128, 6000, dtype, 5000, seed=504, device=DEV)
        dec = eng.single_query_attention(q1, k1, v1, kc, vc, None, None, 5000, 0, 10000.0, 1.0, True)
        for seed in (505, 506):
            q2, k2, v2 = _inputs(1, 1, 300, 8, 2, 64, dtype, seed)
            q.copy_(q2), k.copy_(k2), v.copy_(v2)
            gr.replay()
            assert torch.equal(o, eng.flash_attn_func(q, k, v, causal=True))
        assert torch.equal(eng.flash_attn_func(*big, causal=True), want_big)
        assert torch.equal(eng.single_query_attention(q1, k1, v1, kc, vc, None, None, 5000, 0, 10000.0, 1.0, True), dec)
    s.synchronize()
    _check(want_big, *big, True, 128 ** -0.5, dtype)


# ------------------------------------------------------------------------------------------------ routes
def traced_call(name):
    """kernel_trace builder: the calls of test_routes and test_decode_over_a_cache_view_is_not_copied, their inputs
    made before the call."""
    eng = P.engine()
    rnd = lambda *s: torch.randn(*s, device=DEV).half()  # noqa: E731
    if name == "siglip":
        qkv = _siglip_qkv(2, 729, 16, 72, torch.float16, 5)
        return lambda: eng.flash_attn_func(*qkv)
    if name == "internvit":
        qkv, cu = rnd(2 * 1025, 3, 16, 64), torch.tensor([0, 1025, 2050], dtype=torch.int32, device=DEV)
        return lambda: eng.flash_attn_varlen_qkvpacked_func(qkv, cu, 1025)
    B, Sq, Sk = {"decode_view": (1, 1, 8200), "sq17_g4": (1, 17, 4000), "chunk512": (1, 512, 2048),
                 "decode_b2": (2, 1, 8200)}[name]
    kc, vc, q = rnd(B, 9000, 8, 128), rnd(B, 9000, 8, 128), rnd(B, Sq, 32, 128)
    return lambda: eng.flash_attn_func(q, kc[:, :Sk], vc[:, :Sk], causal=True)


def test_routes():
    """A single query over a cache view runs the split-key kernel; Sq * G > 64, a 512-token chunk, SigLIP and InternViT
    run the prefill kernel."""
    cases = ["decode_view", "sq17_g4", "chunk512", "siglip", "internvit"]
    res = {c: r.names for c, r in zip(cases, trace("test_splitkv_attention_gpu:traced_call", [[c] for c in cases],
                                                   per_process=8))}
    assert any("splitkv_attention_kernel" in n for n in res["decode_view"]), res["decode_view"]
    assert not any("prefill_attention_kernel" in n for n in res["decode_view"]), res["decode_view"]
    for name in ("sq17_g4", "chunk512", "siglip", "internvit"):
        assert any("prefill_attention_kernel" in n for n in res[name]), (name, res[name])
        assert not any("splitkv_attention_kernel" in n for n in res[name]), (name, res[name])


def test_decode_over_a_cache_view_is_not_copied():
    (rec,) = trace("test_splitkv_attention_gpu:traced_call", [["decode_b2"]], per_process=8)
    names = rec.names
    assert any("splitkv_attention_kernel" in n for n in names), names
    assert not any(("copy" in n.lower() or "elementwise" in n.lower() or "fill" in n.lower()) for n in names), names


# ------------------------------------------------------------------------------------------------ rejected inputs
@pytest.mark.parametrize("what", ["d72", "d96", "sqg65", "scale", "workspace", "stride", "pointer"])
def test_rejected_inputs(what):
    dtype = torch.float16
    D = {"d72": 72, "d96": 96}.get(what, 128)
    Sq, H, Hkv, Sk = (17, 32, 8, 2000) if what == "sqg65" else (1, 32, 8, 2000)
    q, k, v = _inputs(1, Sq, Sk, H, Hkv, D, dtype, 3)
    out = torch.empty_like(q)
    if what in ("d72", "d96", "sqg65"):
        assert _abi(q, k, v, out, True) == SHAPE
        # flash_attn_func falls through to the prefill kernel (D = 72, Sq * G > 64) or raises (D = 96)
        if what == "d96":
            with pytest.raises(RuntimeError):
                P.engine().flash_attn_func(q, k, v, causal=True)
        else:
            _check(P.engine().flash_attn_func(q, k, v, causal=True), q, k, v, True, D ** -0.5, dtype)
    elif what == "scale":
        for s in (0.0, -0.125, float("inf"), float("nan")):
            assert _abi(q, k, v, out, True, scale=s) == SHAPE
    elif what == "workspace":
        need = P.lib().b200awq_splitkv_attention_workspace_bytes(1, Sq, Sk, H, Hkv, D)
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        assert _abi(q, k, v, out, True, ws=ws, ws_bytes=need - 16) == WORKSPACE
    elif what == "stride":
        bad = (_st(q), (k.stride(0), k.stride(1) + 4, k.stride(2)), _st(v))
        assert _abi(q, k, v, out, True, strides=bad) == ALIGN
    else:
        buf = torch.empty(q.numel() + 8, dtype=dtype, device=DEV)
        qm = buf[1:1 + q.numel()].view(q.shape)
        assert _abi(qm, k, v, out, True) == ALIGN
