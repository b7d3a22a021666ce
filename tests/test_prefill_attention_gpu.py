"""GPU parity of attention over many queries (`flash_attn_func`, `flash_attn_varlen_qkvpacked_func`, sm_90a TMA + wgmma
kernel) against the float64 definition in tests/prefill_attention_oracle.py and the stored outputs of flash-attn 2.8.3
(tests/golden/reference_kernels_prefill_attention.npz).

Tolerances are those of the decode-attention tests: 2e-3 (fp16) / 8e-3 (bf16) normwise per (sequence, head).  Full-size
cases check every row of sampled heads, the first and the last among them."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import attention_gqa_cases as C
import prefill_attention_oracle as PO
from awq_testutil import np64
from guard_bands import Op, guarded_call
from kernel_trace import trace

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
TOL = {torch.float16: 2e-3, torch.bfloat16: 8e-3}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kernels_prefill_attention.npz")


def _rand(shape, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV).to(dtype)


def _sample_heads(H):
    return sorted({0, H // 2, H - 1})


def _check(out, q, k, v, causal, scale, dtype, heads=None):
    """out [B, Sq, H, D] against the float64 oracle, normwise per (batch row, sampled head)."""
    H = q.shape[2]
    heads = _sample_heads(H) if heads is None else heads
    want = PO.prefill_attention_torch(q, k, v, causal, scale, heads)
    got = out[:, :, heads].double()
    for b in range(q.shape[0]):
        for n, h in enumerate(heads):
            w = want[b, :, n]
            err = float((got[b, :, n] - w).norm() / max(float(w.norm()), 1e-30))
            assert err <= TOL[dtype], (b, h, err)


def _zero_rows(Sq, Sk):
    return max(0, Sq - Sk)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G", [1, 4, 7])
@pytest.mark.parametrize("B", [1, 3])
def test_causal_square(B, G, D, dtype):
    eng = P.engine()
    Hkv = 2
    H = G * Hkv
    for S in (1, 2, 63, 64, 65, 127, 128, 129, 1000, 2048):
        seed = S * 7 + G * 3 + D + B
        q, k, v = _rand((B, S, H, D), dtype, seed), _rand((B, S, Hkv, D), dtype, seed + 1), _rand((B, S, Hkv, D), dtype, seed + 2)
        out = eng.flash_attn_func(q, k, v, causal=True)
        assert out.shape == q.shape and out.is_contiguous()
        _check(out, q, k, v, True, D ** -0.5, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Sq,Sk", [(1, 4100), (16, 2048), (129, 700), (512, 4096), (300, 200)])
def test_causal_bottom_right(Sq, Sk, dtype):
    eng = P.engine()
    B, H, Hkv, D = 2, 8, 2, 128
    q, k, v = _rand((B, Sq, H, D), dtype, Sq), _rand((B, Sk, Hkv, D), dtype, Sk), _rand((B, Sk, Hkv, D), dtype, Sk + 1)
    out = eng.flash_attn_func(q, k, v, 0.0, None, True)
    _check(out, q, k, v, True, D ** -0.5, dtype)
    z = _zero_rows(Sq, Sk)
    if z:  # rows that see no key
        assert int(torch.count_nonzero(out[:, :z])) == 0
        assert torch.isfinite(out).all()


def _siglip_qkv(bsz, seqlen, heads, head_dim, dtype, seed):
    """q, k, v exactly as tinychat's QuantSiglipFlashAttention2 builds them (fused_siglipdecoder.py:162-167)."""
    embed = heads * head_dim
    buf = _rand((bsz * seqlen, 3 * embed), dtype, seed)
    q, k, v = buf.split([embed, embed, embed], dim=-1)
    return (q.reshape(bsz, seqlen, heads, head_dim), k.reshape(bsz, seqlen, heads, head_dim),
            v.reshape(bsz, seqlen, heads, head_dim))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("S", [729, 1024])
def test_siglip_views(S, B, dtype):
    eng = P.engine()
    q, k, v = _siglip_qkv(B, S, 16, 72, dtype, S + B)
    assert not q.is_contiguous()
    out = eng.flash_attn_func(q, k, v, softmax_scale=None, causal=False)
    _check(out, q, k, v, False, 72 ** -0.5, dtype, heads=list(range(16)) if B == 1 else None)


def traced_call():
    """kernel_trace builder: flash_attn_func on SigLIP's views of a fused qkv buffer."""
    q, k, v = _siglip_qkv(2, 729, 16, 72, torch.float16, 5)
    return lambda: P.engine().flash_attn_func(q, k, v)


def test_siglip_views_are_not_copied():
    """The profiler sees the attention kernel and no copy kernel."""
    (rec,) = trace("test_prefill_attention_gpu:traced_call", [[]], per_process=8)
    names = rec.names
    assert any("prefill_attention_kernel" in n for n in names), names
    assert not any(("copy" in n.lower() or "elementwise" in n.lower()) for n in names), names


def _packed(lengths, H, D, dtype, seed):
    total = sum(lengths)
    qkv = _rand((total, 3, H, D), dtype, seed)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lengths)]), dtype=torch.int32, device=DEV)
    return qkv, cu


def _check_packed(out, qkv, cu, lengths, causal, scale, dtype, heads=None):
    c = cu.tolist()
    for b, L in enumerate(lengths):
        if L == 0:
            continue
        s = slice(c[b], c[b + 1])
        _check(out[None, s], qkv[None, s, 0], qkv[None, s, 1], qkv[None, s, 2], causal, scale, dtype, heads)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,D,B", [(16, 64, 1), (16, 64, 3), (25, 128, 1), (25, 128, 2)])
def test_internvit_uniform(H, D, B, dtype):
    """cu_seqlens as internvit.py:64 builds them."""
    eng = P.engine()
    S = 1025
    qkv = _rand((B * S, 3, H, D), dtype, H + D + B)
    cu = torch.arange(0, (B + 1) * S, step=S, dtype=torch.int32, device=DEV)
    out = eng.flash_attn_varlen_qkvpacked_func(qkv, cu, S, 0.0, softmax_scale=None, causal=False)
    assert out.shape == (B * S, H, D)
    _check_packed(out, qkv, cu, [S] * B, False, D ** -0.5, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_ragged(causal, dtype):
    eng = P.engine()
    lengths = [1, 17, 0, 300, 1025]
    H, D = 4, 64
    qkv, cu = _packed(lengths, H, D, dtype, 9)
    out = eng.flash_attn_varlen_qkvpacked_func(qkv, cu, max(lengths), causal=causal, softmax_scale=0.1)
    _check_packed(out, qkv, cu, lengths, causal, 0.1, dtype, heads=list(range(H)))


def _poison_k(k, rows):
    k[:, rows] = float("nan")
    k[:, rows[::2], :, 0] = float("inf")
    k[:, rows[1::2], :, 1] = -float("inf")


def test_row_isolation_causal():
    eng = P.engine()
    dtype, B, S, H, Hkv, D = torch.float16, 1, 700, 4, 2, 128
    q, k, v = _rand((B, S, H, D), dtype, 1), _rand((B, S, Hkv, D), dtype, 2), _rand((B, S, Hkv, D), dtype, 3)
    clean = eng.flash_attn_func(q, k, v, causal=True)
    for p in (0, S - 1, 300):  # first, last and a mid-tile row
        qp, kp, vp = q.clone(), k.clone(), v.clone()
        others = [r for r in range(S) if r != p]
        qp[:, others] = float("nan")
        if p + 1 < S:
            _poison_k(kp, list(range(p + 1, S)))
            vp[:, p + 1::2] = 65504.0
            vp[:, p + 2::2] = -65504.0
        got = eng.flash_attn_func(qp, kp, vp, causal=True)
        assert torch.equal(got[:, p], clean[:, p]), p


def test_row_isolation_varlen():
    """The middle sequence is shorter than a tile: its Q and K / V tiles are shifted back and read rows of the first
    sequence, which must stay masked."""
    eng = P.engine()
    dtype, H, D = torch.bfloat16, 4, 64
    lengths = [200, 90, 260]
    qkv, cu = _packed(lengths, H, D, dtype, 4)
    clean = eng.flash_attn_varlen_qkvpacked_func(qkv, cu, max(lengths))
    neighbours = list(range(0, 200)) + list(range(290, 550))
    for p in (200, 200 + 45, 289):  # first, middle and last row of the middle sequence
        bad = qkv.clone()
        others = [r for r in range(sum(lengths)) if r != p]
        bad[others, 0] = float("nan")
        bad[neighbours, 1] = float("nan")
        bad[neighbours[::2], 1, :, 0] = float("inf")
        bad[neighbours[::2], 2] = 65504.0
        bad[neighbours[1::2], 2] = -65504.0
        got = eng.flash_attn_varlen_qkvpacked_func(bad, cu, max(lengths))
        assert torch.equal(got[p], clean[p]), p


def test_operands_the_tma_cannot_take_are_copied():
    """A contiguous view 2 bytes past an aligned address, and a size-1 batch dimension whose stride is not a multiple
    of 8 elements: both are copied (torch calls them contiguous) and give the same bits as aligned inputs."""
    eng = P.engine()
    dtype, S, H, D = torch.float16, 300, 4, 64
    q, k, v = _rand((1, S, H, D), dtype, 61), _rand((1, S, H, D), dtype, 62), _rand((1, S, H, D), dtype, 63)
    want = eng.flash_attn_func(q, k, v, causal=True)
    buf = torch.empty(q.numel() + 1, dtype=dtype, device=DEV)
    qm = buf[1:].view(1, S, H, D)
    qm.copy_(q)
    assert qm.is_contiguous() and qm.data_ptr() % 16 == 2
    assert torch.equal(eng.flash_attn_func(qm, k, v, causal=True), want)
    ks = k.as_strided(k.shape, (3,) + k.stride()[1:])
    assert ks.is_contiguous() and ks.stride(0) % 8
    assert torch.equal(eng.flash_attn_func(q, ks, v, causal=True), want)


def test_chunked_prefill_is_bit_identical():
    """A 2048-token causal prefill and four 512-token chunks over the growing prefix (bottom-right)."""
    eng = P.engine()
    dtype, S, H, Hkv, D = torch.float16, 2048, 8, 2, 128
    q, k, v = _rand((1, S, H, D), dtype, 21), _rand((1, S, Hkv, D), dtype, 22), _rand((1, S, Hkv, D), dtype, 23)
    full = eng.flash_attn_func(q, k, v, causal=True)
    for c in range(4):
        lo, hi = 512 * c, 512 * (c + 1)
        part = eng.flash_attn_func(q[:, lo:hi], k[:, :hi], v[:, :hi], causal=True)
        assert torch.equal(part, full[:, lo:hi]), c


def test_single_query_matches_decode_kernel():
    """long_forward's decode: Sq = 1 over a context through flash_attn_func, and single_query_attention without
    rotary on the same cache content."""
    eng = P.engine()
    dtype, B, H, Hkv, D, L = torch.float16, 2, 32, 8, 128, 3000
    t = L - 1
    _, q, kn, vn = C.fused_qkv(B, H, Hkv, D, dtype, seed=31, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, t, seed=32, device=DEV)
    dec = eng.single_query_attention(q, kn, vn, kc, vc, None, None, t, 0, 10000.0, 1.0, True)
    keys = kc.permute(0, 3, 1, 2, 4).reshape(B, L, Hkv, D)  # the cache after the step stored kn, vn at slot t
    vals = vc.permute(0, 2, 1, 3)
    pre = eng.flash_attn_func(q.reshape(B, 1, H, D), keys, vals, causal=True)
    d, p = dec.double(), pre.reshape(B, H, D).double()
    assert float((d - p).norm() / d.norm()) <= 2e-3


def test_determinism_graph_and_side_stream():
    eng = P.engine()
    dtype, B, S, H, Hkv, D = torch.bfloat16, 2, 777, 8, 2, 64
    q, k, v = _rand((B, S, H, D), dtype, 41), _rand((B, S, Hkv, D), dtype, 42), _rand((B, S, Hkv, D), dtype, 43)
    first = eng.flash_attn_func(q, k, v, causal=True)
    for _ in range(3):
        assert torch.equal(eng.flash_attn_func(q, k, v, causal=True), first)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        on_side = eng.flash_attn_func(q, k, v, causal=True)
    side.synchronize()
    assert torch.equal(on_side, first)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        o = eng.flash_attn_func(q, k, v, causal=True)
    q2, k2, v2 = _rand(q.shape, dtype, 44), _rand(k.shape, dtype, 45), _rand(v.shape, dtype, 46)
    q.copy_(q2), k.copy_(k2), v.copy_(v2)
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(o, eng.flash_attn_func(q, k, v, causal=True))


def _abi(views, cu, B, Sq, Sk, H, Hkv, D, causal, dtype, q_st, k_st, v_st):
    lib = P.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    arr = lambda s: (ctypes.c_longlong * 3)(*s)
    cup = p(views["cu"]) if cu else None
    return lib.b200awq_prefill_attention(p(views["q"]), p(views["k"]), p(views["v"]), p(views["out"]), cup, cup, B, Sq, Sk,
                                         H, Hkv, D, arr(q_st), arr(k_st), arr(v_st), ctypes.c_float(D ** -0.5),
                                         1 if causal else 0, 0 if dtype == torch.float16 else 1,
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("case", ["s129_d128_causal", "d72", "varlen_tails", "strided_qkv"])
def test_guard_bands(case):
    dtype = torch.float16
    if case == "varlen_tails":
        lengths, H, D = [5, 129, 1, 200], 4, 64
        qkv, cu = _packed(lengths, H, D, dtype, 51)
        total = sum(lengths)
        ops = {"qkv": Op("in", qkv), "cu": Op("in", cu), "out": Op("out", shape=(total, H, D), dtype=dtype)}
        st = (0, 3 * H * D, D)

        def call(vw):
            base = vw["qkv"]
            views = {"q": base[:, 0], "k": base[:, 1], "v": base[:, 2], "out": vw["out"], "cu": vw["cu"]}
            return _abi(views, True, len(lengths), max(lengths), max(lengths), H, H, D, True, dtype, st, st, st)
        plain = guarded_call(call, ops)
        _check_packed(plain["out"], plain["qkv"], plain["cu"], lengths, True, D ** -0.5, dtype, heads=list(range(H)))
        return
    if case == "strided_qkv" or case == "d72":
        B, S, H, D = 2, 129, 4, (72 if case == "d72" else 64)
        qkv = _rand((B, S, 3 * H * D), dtype, 52)
        ops = {"qkv": Op("in", qkv), "out": Op("out", shape=(B, S, H, D), dtype=dtype)}
        st = (S * 3 * H * D, 3 * H * D, D)

        def call(vw):
            base = vw["qkv"].view(B, S, 3, H, D)
            views = {"q": base[:, :, 0], "k": base[:, :, 1], "v": base[:, :, 2], "out": vw["out"]}
            return _abi(views, False, B, S, S, H, H, D, False, dtype, st, st, st)
        plain = guarded_call(call, ops)
        base = plain["qkv"].view(B, S, 3, H, D)
        _check(plain["out"], base[:, :, 0], base[:, :, 1], base[:, :, 2], False, D ** -0.5, dtype, list(range(H)))
        return
    B, S, H, Hkv, D = 1, 129, 4, 2, 128
    q, k, v = _rand((B, S, H, D), dtype, 53), _rand((B, S, Hkv, D), dtype, 54), _rand((B, S, Hkv, D), dtype, 55)
    ops = {"q": Op("in", q), "k": Op("in", k), "v": Op("in", v), "out": Op("out", shape=(B, S, H, D), dtype=dtype)}
    plain = guarded_call(lambda vw: _abi(vw, False, B, S, S, H, Hkv, D, True, dtype, (S * H * D, H * D, D),
                                         (S * Hkv * D, Hkv * D, D), (S * Hkv * D, Hkv * D, D)), ops)
    _check(plain["out"], q, k, v, True, D ** -0.5, dtype, list(range(H)))


def _golden_module():
    spec = importlib.util.spec_from_file_location("_prefill_golden", os.path.join(os.path.dirname(GOLDEN),
                                                                                   "make_prefill_attention_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("dtype", DTYPES)
def test_vs_stored_flash_attn_outputs(dtype):
    """flash-attn 2.8.3 on the same seeded inputs (sampled heads and rows)."""
    eng = P.engine()
    M = _golden_module()
    g = np.load(GOLDEN)
    tag = "f16" if dtype == torch.float16 else "bf16"
    for name, (kind, B, Sq, Sk, H, Hkv, D, causal) in M.CASES.items():
        heads, rows = (torch.from_numpy(a).to(DEV) for a in M.sampled(name))
        want = torch.from_numpy(g[f"{name}__{tag}"]).view(dtype).to(DEV).double()
        x = M.inputs(name, dtype, DEV)
        if kind == "fixed":
            got = eng.flash_attn_func(*x, 0.0, softmax_scale=D ** -0.5, causal=causal)[:, rows][:, :, heads]
        else:
            got = eng.flash_attn_varlen_qkvpacked_func(*x, 0.0, softmax_scale=D ** -0.5, causal=causal)[rows][:, heads]
        got = got.double()
        assert want.shape == got.shape, name
        # normwise per head (and batch row)
        if kind == "fixed":
            w, o = want.permute(0, 2, 1, 3).reshape(B * len(heads), -1), got.permute(0, 2, 1, 3).reshape(B * len(heads), -1)
        else:
            w, o = want.permute(1, 0, 2).reshape(len(heads), -1), got.permute(1, 0, 2).reshape(len(heads), -1)
        err = ((o - w).norm(dim=1) / w.norm(dim=1)).max().item()
        assert err <= TOL[dtype], (name, err)


@pytest.mark.parametrize("what", ["d96", "d256", "dropout", "fp32", "heads", "keyword", "scale"])
def test_rejected_inputs_raise(what):
    eng = P.engine()
    D = {"d96": 96, "d256": 256}.get(what, 64)
    dtype = torch.float32 if what == "fp32" else torch.float16
    Hkv = 3 if what == "heads" else 2
    q, k, v = _rand((1, 16, 4, D), dtype, 0), _rand((1, 16, Hkv, D), dtype, 1), _rand((1, 16, Hkv, D), dtype, 2)
    if what == "keyword":
        with pytest.raises(TypeError):
            eng.flash_attn_func(q, k, v, window_size=(-1, -1))
        return
    with pytest.raises(RuntimeError):
        eng.flash_attn_func(q, k, v, dropout_p=0.1 if what == "dropout" else 0.0,
                            softmax_scale=-0.125 if what == "scale" else None)
