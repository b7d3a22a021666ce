"""Every kernel-launching entry of the C ABI (include/b200awq.h) reads and writes only its own operands: each runs
on guard-banded buffers with two fills and on plain tensors (`guarded_call` of tests/guard_bands.py).

The cases sit at the tails of the kernels: partial token tiles of the W4A16 and W8A8 GEMMs, the decode kernel's last row
blocks, the ring kernel's odd last octet, the stream kernel's channel tails, the masked spare heads of attention's last
head group, and the row ops on pointers that are not 16-byte aligned (their one-element paths).

The checker itself is tested on the CPU: fake kernels written in torch that write one element too many, skip one, or
read one past their input must each be flagged."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import attention_gqa_cases as C
import w8a8_cases as W
from awq_testutil import gen_layer, gen_x
from guard_bands import DEV, Op, _code, _p, _st, guarded_call
from oracle import w8a8_oracle as O8

DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]


# ------------------------------------------------------------------------------------------------ checker self-tests
def _fake_double(fault):
    """y = 2 x over n elements, written in torch, with one injected fault."""
    def call(v):
        x, y = v["x"], v["y"]
        n = x.numel()
        if fault == "write_past":
            y.as_strided((n + 1,), (1,), y.storage_offset()).copy_(torch.cat([2 * x, 2 * x[:1]]))
        elif fault == "skip":
            y[:-1] = 2 * x[:-1]
        elif fault == "read_past":
            xr = x.as_strided((n + 1,), (1,), x.storage_offset())
            y.copy_(2 * x + 0 * xr[1:])        # reads x[n], one past the end: 0 * NaN is NaN
        else:
            y.copy_(2 * x)
        return 0
    return call


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("fault,message", [("write_past", "guard after"), ("skip", "differs between fills"),
                                           ("read_past", "differs between fills")])
def test_checker_flags_faulty_fake_kernels(fault, message, dtype):
    x = torch.randn(37).to(dtype)
    ops = {"x": Op("in", x), "y": Op("out", shape=(37,), dtype=dtype)}
    with pytest.raises(AssertionError, match=message):
        guarded_call(_fake_double(fault), ops, device="cpu")


@pytest.mark.parametrize("offset", [0, 2, 8])
def test_checker_passes_a_correct_fake_kernel(offset):
    x = torch.randn(37).half()
    ops = {"x": Op("in", x, offset=offset), "y": Op("out", shape=(37,), dtype=torch.float16, offset=offset)}
    y = guarded_call(_fake_double(None), ops, device="cpu")["y"]
    assert torch.equal(y, 2 * x)


def test_checker_flags_a_write_into_an_input():
    def call(v):
        v["y"].copy_(v["x"])
        v["x"][3] = 0
        return 0
    ops = {"x": Op("in", torch.ones(8).half()), "y": Op("out", shape=(8,), dtype=torch.float16)}
    with pytest.raises(AssertionError, match="read-only operand written"):
        guarded_call(call, ops, device="cpu")


# ------------------------------------------------------------------------------------------------ W4A16 linears
def _w4_ops(M, N, K, dtype, seed):
    qw, s, z = gen_layer(N, K, dtype, seed=seed)
    x = gen_x(M, K, dtype, seed=seed + 1)
    return {"x": Op("in", x), "qw": Op("in", qw), "s": Op("in", s), "z": Op("in", z),
            "y": Op("out", shape=(M, N), dtype=dtype)}


def _gemv(M, N, K, dtype):
    def call(v):
        return P.lib().b200awq_w4a16_gemv(_p(v["x"]), _p(v["qw"]), _p(v["s"]), _p(v["z"]), _p(v["y"]), M, N, K, 128,
                                          _code(dtype), _st())
    return call


def _gemm(M, N, K, dtype):
    def call(v):
        return P.lib().b200awq_w4a16_gemm(_p(v["x"]), _p(v["qw"]), _p(v["s"]), _p(v["z"]), _p(v["y"]), M, N, K, 128,
                                          _code(dtype), None, 0, _st())
    return call


# (M, N, K, dtype): decode (one fp16 token), ring (2-4 tokens, one bf16 token; odd last octets), skinny wgmma (5-7
# tokens, n % 128 == 0), stream (5-7 tokens, n % 128 != 0)
GEMV_CASES = [
    (1, 8, 128, torch.float16), (1, 1192, 2176, torch.float16), (1, 4104, 11008, torch.float16),
    (1, 4096, 14336, torch.float16), (1, 1192, 2176, torch.bfloat16), (1, 8, 128, torch.bfloat16),
    (2, 1192, 2176, torch.float16), (3, 40, 1920, torch.bfloat16), (4, 4104, 11008, torch.float16),
    (3, 8, 14336, torch.float16), (4, 1192, 2176, torch.bfloat16),
    (5, 384, 2176, torch.float16), (7, 128, 128, torch.bfloat16), (6, 4096, 14336, torch.float16),
    (5, 8, 128, torch.float16), (7, 24, 2176, torch.bfloat16), (6, 1192, 11008, torch.float16),
    (7, 1192, 2176, torch.float16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,dtype", GEMV_CASES, ids=lambda v: str(v).replace("torch.", ""))
def test_gemv_guarded(M, N, K, dtype):
    guarded_call(_gemv(M, N, K, dtype), _w4_ops(M, N, K, dtype, seed=M + N + K))


# every token tile (16 / 32 / 64 / 128) ending in a partial tile, the 9-16-token tile launch on a large layer
# (n k >= 48 M), split-k clusters with a partial last tile
GEMM_CASES = [
    (8, 384, 512, torch.float16), (9, 4096, 14336, torch.float16), (16, 4096, 14336, torch.bfloat16),
    (17, 384, 4096, torch.float16), (31, 128, 512, torch.bfloat16), (33, 4096, 4096, torch.float16),
    (63, 384, 4096, torch.float16), (65, 128, 14336, torch.bfloat16), (127, 4096, 512, torch.float16),
    (129, 384, 4096, torch.bfloat16), (300, 4096, 4096, torch.float16), (777, 384, 512, torch.float16),
    (777, 128, 14336, torch.bfloat16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,dtype", GEMM_CASES, ids=lambda v: str(v).replace("torch.", ""))
def test_gemm_guarded(M, N, K, dtype):
    guarded_call(_gemm(M, N, K, dtype), _w4_ops(M, N, K, dtype, seed=M + N + K))


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,dtype", [(1, 2376, 4224, torch.float16), (4, 2376, 4224, torch.float16),
                                         (4, 600, 2048, torch.bfloat16), (40, 384, 1024, torch.float16)],
                         ids=["fused", "composed_4", "composed_4_bf16", "composed_40"])
def test_mlp_front_guarded(M, N, K, dtype):
    """One fp16 token: the fused decode kernel; otherwise the two products into the workspace, then silu * mul.  The
    workspace is guarded beyond b200awq_w4a16_mlp_front_workspace_bytes and pattern-filled: the elementwise tail must
    read only what the products wrote."""
    gq, gs, gz = gen_layer(N, K, dtype, seed=1)
    uq, us, uz = gen_layer(N, K, dtype, seed=2)
    ops = {"x": Op("in", gen_x(M, K, dtype, seed=3)), "gq": Op("in", gq), "gs": Op("in", gs), "gz": Op("in", gz),
           "uq": Op("in", uq), "us": Op("in", us), "uz": Op("in", uz), "y": Op("out", shape=(M, N), dtype=dtype)}
    nbytes = P.lib().b200awq_w4a16_mlp_front_workspace_bytes(M, N, K)
    ops["ws"] = Op("scratch", shape=(nbytes,), dtype=torch.uint8)

    def call(v):
        return P.lib().b200awq_w4a16_mlp_front(_p(v["x"]), _p(v["gq"]), _p(v["gs"]), _p(v["gz"]), _p(v["uq"]), _p(v["us"]),
                                               _p(v["uz"]), _p(v["y"]), M, N, K, 128, _code(dtype), _p(v["ws"]), nbytes,
                                               _st())
    guarded_call(call, ops)


@pytest.mark.gpu
def test_gemv_allreduce_loopback_guarded():
    """The fused decode GEMV + all-reduce at world 2 on one GPU (tests/test_tp_loopback_gpu.py), both ranks' y guarded;
    the two ranks' outputs are bit-identical."""
    from test_tp_loopback_gpu import LoopbackExchange, _allreduce_call, _shards
    dtype, world, N, Kr, M = torch.float16, 2, 264, 256, 3
    qw, s, z = gen_layer(N, Kr * world, dtype, seed=5, device=DEV)
    shards = _shards(qw, s, z, world)
    ex = LoopbackExchange(world, 8, 512)
    x = gen_x(M, Kr * world, dtype, seed=6)
    ops = {f"x{r}": Op("in", x[:, r * Kr:(r + 1) * Kr].contiguous()) for r in range(world)}
    ops.update({f"y{r}": Op("out", shape=(M, N), dtype=dtype) for r in range(world)})

    def call(v):
        _allreduce_call(ex, shards, [v["x0"], v["x1"]], [v["y0"], v["y1"]], M, N, Kr)
        return 0
    y = guarded_call(call, ops)
    assert torch.equal(y["y0"], y["y1"])


# ------------------------------------------------------------------------------------------------ attention and RoPE
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ctx", [(2, 2304, 2100), (2, 256, 700)], ids=["split", "wrap"])
@pytest.mark.parametrize("D", [80, 128])
@pytest.mark.parametrize("G,Hkv", [(7, 2), (71, 1)])
def test_single_query_attention_guarded(G, Hkv, D, ctx, dtype):
    """Guards around the fused QKV buffer (q, k, v are views into it), the caches, `out` and the workspace beyond
    b200awq_single_query_attention_workspace_bytes; G = 71 masks the spare heads of its last head group."""
    B, L, t = ctx
    H = G * Hkv
    qkv, _, _, _ = C.fused_qkv(B, H, Hkv, D, dtype, seed=H + D + t, device="cpu")
    kc, vc = C.caches(B, Hkv, D, L, dtype, min(t, L), seed=t + D, device="cpu")
    nbytes = P.lib().b200awq_single_query_attention_workspace_bytes(B, H, Hkv, D, L)
    ops = {"qkv": Op("in", qkv), "kc": Op("io", kc), "vc": Op("io", vc), "out": Op("out", shape=(B, H, D), dtype=dtype),
           "ws": Op("zeroed", shape=(nbytes,), dtype=torch.uint8)}
    stride = (H + 2 * Hkv) * D

    def call(v):
        base, e = _p(v["qkv"]), v["qkv"].element_size()
        return P.lib().b200awq_single_query_attention(base, base + H * D * e, base + (H + Hkv) * D * e, _p(v["kc"]), _p(v["vc"]),
                                                      _p(v["out"]), None, B, H, Hkv, D, L, t, stride, stride, stride, D,
                                                      C.ROPE_BASE, 1.0, 1, _code(dtype), _p(v["ws"]), nbytes, _st())
    guarded_call(call, ops)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("transpose", [False, True], ids=["same_layout", "transposed"])
@pytest.mark.parametrize("S,Bt,H,D,d2", [(7, 3, 5, 128, 128), (5, 2, 3, 80, 32)])
def test_rope_with_pos_guarded(S, Bt, H, D, d2, transpose, dtype):
    g = torch.Generator().manual_seed(S * D + d2)
    x = torch.randn(S, Bt, H, D, generator=g).to(dtype)
    freqs = torch.rand(Bt * S * d2, generator=g) * 50
    ops = {"x": Op("in", x), "f": Op("in", freqs),
           "y": Op("out", shape=(Bt, S, H, D) if transpose else (S, Bt, H, D), dtype=dtype)}
    ins = (ctypes.c_longlong * 4)(Bt * H * D, H * D, D, 1)
    outs = (ctypes.c_longlong * 4)(*((H * D, S * H * D, D, 1) if transpose else (Bt * H * D, H * D, D, 1)))

    def call(v):
        return P.lib().b200awq_rope_with_pos(_p(v["x"]), _p(v["f"]), _p(v["y"]), S, Bt, H, D, d2, ins, outs, _code(dtype),
                                             _st())
    guarded_call(call, ops)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("tokens,qh,kh,vh,hs,rot", [(9, 8, 2, 2, 128, 128), (5, 7, 1, 1, 80, 32), (3, 4, 3, 0, 64, 64)])
def test_rotary_embedding_neox_guarded(tokens, qh, kh, vh, hs, rot, dtype):
    """In place on query and key views of one fused buffer with different head counts; the value heads that follow
    them in each token row must stay untouched (the buffer is compared as a whole)."""
    g = torch.Generator().manual_seed(tokens * hs + rot)
    row = (qh + kh + vh) * hs
    buf = torch.randn(tokens, row, generator=g).to(dtype)
    pos = torch.randint(0, 300, (tokens,), generator=g, dtype=torch.int64)
    ang = torch.arange(300).double()[:, None] / (10000.0 ** (torch.arange(rot // 2).double() / (rot // 2)))[None]
    cache = torch.cat([ang.cos(), ang.sin()], dim=1).to(dtype)
    ops = {"buf": Op("io", buf), "pos": Op("in", pos), "cache": Op("in", cache)}

    def call(v):
        q = _p(v["buf"])
        return P.lib().b200awq_rotary_embedding_neox(_p(v["pos"]), q, q + qh * hs * 2, _p(v["cache"]), tokens, qh, kh, hs, rot,
                                                     row, row, _code(dtype), _st())
    guarded_call(call, ops)


# ------------------------------------------------------------------------------------------------ row ops
# (m, n, byte offset of every operand): the 16-byte kernels, their generic / one-element paths through n % 8 and
# through pointers that are 2 or 8 bytes past a 16-byte boundary
ROW_CASES = [(3, 4096, 0), (3, 4096, 2), (3, 4096, 8), (5, 100, 0), (2, 40000, 0), (4, 4104, 8), (1, 8, 2), (7, 1152, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,n,off", ROW_CASES)
def test_rmsnorm_guarded(m, n, off, dtype):
    g = torch.Generator().manual_seed(m + n)
    x = (torch.randn(m, n, generator=g) * 1.7).to(dtype)
    gamma = (1.0 + 0.2 * torch.randn(n, generator=g)).to(dtype)
    ops = {"x": Op("in", x, offset=off), "g": Op("in", gamma, offset=off), "y": Op("out", shape=(m, n), dtype=dtype, offset=off)}

    def call(v):
        return P.lib().b200awq_rmsnorm(_p(v["x"]), _p(v["g"]), _p(v["y"]), m, n, 1e-5, _code(dtype), _st())
    guarded_call(call, ops)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,d,off", [(3, 1024, 0), (3, 1024, 2), (3, 1024, 8), (5, 1001, 0), (1, 1001, 0), (1, 13, 2),
                                     (2, 4304, 8)])
def test_silu_and_mul_guarded(m, d, off, dtype):
    """A single row with d % 8 != 0 runs the 16-byte part and the one-element tail in one launch."""
    g = torch.Generator().manual_seed(m + d)
    x = (torch.randn(m, 2 * d, generator=g) * 2).to(dtype)
    ops = {"x": Op("in", x, offset=off), "y": Op("out", shape=(m, d), dtype=dtype, offset=off)}

    def call(v):
        return P.lib().b200awq_silu_and_mul(_p(v["x"]), _p(v["y"]), m, d, _code(dtype), _st())
    r = guarded_call(call, ops)
    lo, hi = O8.silu_and_mul_bounds(x.float().numpy(), "f16" if dtype == torch.float16 else "bf16")
    O8.assert_between(r["y"].float().cpu().numpy(), lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("M,N,K", [(130, 4304, 1152), (5, 24, 48), (129, 136, 144), (300, 256, 16), (65, 1160, 4304)])
def test_w8a8_gemm_guarded(M, N, K, bias):
    """M / N tails (masked 16-byte stores), k % 64 != 0 (zero-filled TMA tails)."""
    x, w, ws, a, b = W.gemm_inputs(M, N, K)
    ops = {"x": Op("in", x), "w": Op("in", w), "ws": Op("in", ws), "a": Op("in", a), "y": Op("out", shape=(M, N), dtype=torch.float16)}
    if bias:
        ops["b"] = Op("in", b)

    def call(v):
        return P.lib().b200awq_w8a8_gemm(_p(v["x"]), _p(v["w"]), _p(v["ws"]), _p(v["a"]), _p(v["b"]) if bias else None,
                                         _p(v["y"]), M, N, K, _st())
    guarded_call(call, ops)


W8_ROW_CASES = [(n, off) for n in (1152, 4304) for off in (0, 2, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,off", W8_ROW_CASES)
def test_quant_per_token_guarded(n, off, dtype):
    """Offsets 2 and 8 run the one-element kernel on n % 8 == 0 rows; its codes and scales lie inside the oracle's
    admissible sets as the 16-byte kernel's do (tests/test_w8a8_gpu.py)."""
    m = 5
    x = W.act_rows(m, n, dtype, seed=n + off)
    ops = {"x": Op("in", x, offset=off), "q": Op("out", shape=(m, n), dtype=torch.int8, offset=off),
           "s": Op("out", shape=(m,), dtype=torch.float16, offset=off)}

    def call(v):
        return P.lib().b200awq_quant_per_token(_p(v["x"]), _p(v["q"]), _p(v["s"]), m, n, _code(dtype), _st())
    r = guarded_call(call, ops)
    O8.assert_admissible(r["q"].cpu().numpy(), r["s"].cpu().numpy(), O8.quant_per_token_bounds(x.float().numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("per_token", [1, 0], ids=["per_token", "per_tensor"])
@pytest.mark.parametrize("n,off", W8_ROW_CASES)
def test_layernorm_quant_guarded(n, off, per_token, dtype):
    m = 5
    x = W.act_rows(m, n, dtype, seed=n + off)
    gamma, beta = W.ln_params(n, dtype, seed=n)
    ops = {"x": Op("in", x, offset=off), "g": Op("in", gamma, offset=off), "b": Op("in", beta, offset=off),
           "q": Op("out", shape=(m, n), dtype=torch.int8, offset=off)}
    if per_token:
        ops["s"] = Op("out", shape=(m,), dtype=torch.float16, offset=off)
    else:
        ops["s"] = Op("in", torch.full((1,), 30.0, dtype=torch.float16), offset=off)

    def call(v):
        return P.lib().b200awq_layernorm_quant(_p(v["x"]), _p(v["g"]), _p(v["b"]), _p(v["q"]), _p(v["s"]), m, n, W.LN_EPS,
                                               per_token, _code(dtype), _st())
    r = guarded_call(call, ops)
    xf, gf, bf = (t.float().numpy() for t in (x, gamma, beta))
    tag = "f16" if dtype == torch.float16 else "bf16"
    vec = O8.row_vec(n, off == 0)
    if per_token:
        b = O8.layernorm_quant_bounds(xf, gf, bf, W.LN_EPS, tag, vec=vec)
        O8.assert_admissible(r["q"].cpu().numpy(), r["s"].cpu().numpy(), b)
    else:
        b = O8.layernorm_quant_bounds(xf, gf, None, W.LN_EPS, tag, per_token=False, scale=np.array([30.0], np.float16),
                                      vec=vec)
        O8.assert_admissible(r["q"].cpu().numpy(), None, b)


@pytest.mark.gpu
@pytest.mark.parametrize("n,off", W8_ROW_CASES)
def test_gelu_quant_guarded(n, off):
    m = 5
    x = W.gelu_rows(m, n, seed=n + off)
    ops = {"x": Op("in", x, offset=off), "q": Op("out", shape=(m, n), dtype=torch.int8, offset=off),
           "s": Op("out", shape=(m,), dtype=torch.float16, offset=off),
           "tmp": Op("out", shape=(m, n), dtype=torch.float16, offset=off)}

    def call(v):
        return P.lib().b200awq_gelu_quant(_p(v["x"]), _p(v["q"]), _p(v["s"]), _p(v["tmp"]), m, n, _st())
    r = guarded_call(call, ops)
    b = O8.gelu_quant_bounds(x.numpy())
    O8.assert_between(r["tmp"].cpu().numpy(), b["g_lo"], b["g_hi"])
    O8.assert_admissible(r["q"].cpu().numpy(), r["s"].cpu().numpy(), b)


@pytest.mark.gpu
def test_row_ops_refuse_long_misaligned_rows():
    """Above 8192 elements only the 16-byte kernels hold a row: the same n is taken on 16-byte aligned pointers and
    refused with B200AWQ_ERR_SHAPE on pointers 2 bytes off, before anything is launched."""
    L, m, n = P.lib(), 2, 8200
    buf = torch.zeros(4 * m * n + 64, dtype=torch.float16, device=DEV)   # bytes: x [0, 2mn), scales, tmp [4mn + 128, 6mn + 128)
    q = torch.zeros(m * n + 64, dtype=torch.int8, device=DEV)
    base, qb = _p(buf), _p(q)
    s = base + 4 * m * n + 32
    for off, want in ((0, 0), (2, -1)):
        x, qq = base + off, qb + off
        assert L.b200awq_quant_per_token(x, qq, s, m, n, 0, _st()) == want
        assert L.b200awq_layernorm_quant(x, x, None, qq, s, m, n, 1e-6, 1, 0, _st()) == want
        assert L.b200awq_gelu_quant(x, qq, s, base + 4 * m * n + 128 + off, m, n, _st()) == want
    torch.cuda.synchronize()
