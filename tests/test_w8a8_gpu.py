"""W8A8 vision-tower ops on the GPU: the C ABI and the `awq_inference_engine` entries against the reference kernels'
stored outputs (tests/golden/reference_kernels_w8a8.npz) and against the numpy oracle (oracle/w8a8_oracle.py): the GEMM
bit-exact, every row-op code, scale and GELU value inside its admissible set."""
import ctypes
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import w8a8_cases as W
from oracle import w8a8_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kernels_w8a8.npz")
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}
SIGLIP = [(3456, 1152), (1152, 1152), (4304, 1152), (1152, 4304)]      # (N, K): qkv, out, fc1, fc2
INTERNVIT = [(3072, 1024), (1024, 1024), (4096, 1024), (1024, 4096)]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ordered(bits16):
    """fp16 / bf16 raw bits -> integers whose differences count ulps across the sign."""
    b = np.asarray(bits16).view(np.uint16).astype(np.int32)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def ulps(a, b):
    return np.abs(ordered(np.asarray(a).view(np.uint16)) - ordered(np.asarray(b).view(np.uint16)))


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def abi_gemm(x, w, ws, a, b):
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=torch.float16, device=x.device)
    rc = P.lib().b200awq_w8a8_gemm(ptr(x), ptr(w), ptr(ws), ptr(a), ptr(b), ptr(y), M, N, K, stream())
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


def check_gemm_oracle(x, w, ws, a, b, y):
    rows = W.sample_rows(x.shape[0])
    o = O.gemm(x.cpu().numpy()[rows], w.cpu().numpy(), ws.cpu().numpy(), a.cpu().numpy()[rows],
               None if b is None else b.cpu().numpy())
    np.testing.assert_array_equal(bits(y)[rows], o.view(np.uint16))


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M", [1, 7, 64, 729, 1024, 1025, 8192])
@pytest.mark.parametrize("NK", SIGLIP + INTERNVIT)
def test_gemm_abi_vs_oracle(M, NK):
    N, K = NK
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    for bias in (None, b):
        y = abi_gemm(x, w, ws, a, bias)
        torch.cuda.synchronize()
        check_gemm_oracle(x, w, ws, a, bias, y)


@pytest.mark.parametrize("MNK", [(130, 4304, 1152), (257, 1152, 4304), (300, 256, 16), (5, 24, 48), (129, 136, 144)])
def test_gemm_tails_vs_oracle(MNK):
    M, N, K = MNK
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    for bias in (None, b):
        check_gemm_oracle(x, w, ws, a, bias, abi_gemm(x, w, ws, a, bias))


def test_gemm_extreme_codes_and_zero_rows():
    M, N, K = 200, 264, 4304
    x = torch.full((M, K), 127, dtype=torch.int8)
    x[1::3] = -128
    x[2::7] = 0
    w = torch.full((N, K), -127, dtype=torch.int8)
    w[::2] = 127
    w[5] = -128
    x, w = x.to(DEV), w.to(DEV)
    ws, a, b = W.gen_scales(N, 1, 1e-5, 2e-5).to(DEV), W.gen_scales(M, 2, 1e-5, 2e-5).to(DEV), W.gen_bias(N, 3).to(DEV)
    for bias in (None, b):
        check_gemm_oracle(x, w, ws, a, bias, abi_gemm(x, w, ws, a, bias))


def test_gemm_plugin_vs_reference(gold):
    e = P.engine()
    for (M, N, K) in W.REF_GEMM:
        x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
        rows, cols = W.sample_rows(M), np.arange(0, N, W.GEMM_COLS)
        for tag in ("nobias", "bias"):
            key = f"{tag}_{M}x{N}x{K}"
            y = torch.empty(M, N, dtype=torch.float16, device=DEV)
            if tag == "bias":
                e.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, y, b)
            else:
                e.w8a8_gemm_forward_cuda(x, w, ws, a, y)
            torch.cuda.synchronize()
            check_gemm_oracle(x, w, ws, a, b if tag == "bias" else None, y)
            if bool(gold[f"gemm_ok_{key}"]):
                np.testing.assert_array_equal(bits(y)[rows][:, cols], gold[f"gemm_{key}"], err_msg=key)


def test_gemm_abi_rejects_bad_shapes():
    L = P.lib()
    x = torch.zeros(64, 64, dtype=torch.int8, device=DEV)
    s = torch.ones(64, dtype=torch.float16, device=DEV)
    y = torch.empty(64, 64, dtype=torch.float16, device=DEV)
    assert L.b200awq_w8a8_gemm(ptr(x), ptr(x), ptr(s), ptr(s), None, ptr(y), 64, 64, 24, stream()) == -1
    assert L.b200awq_w8a8_gemm(ptr(x), ptr(x), ptr(s), ptr(s), None, ptr(y), 64, 60, 64, stream()) == -1
    assert L.b200awq_w8a8_gemm(ctypes.c_void_p(x.data_ptr() + 8), ptr(x), ptr(s), ptr(s), None, ptr(y), 8, 8, 32,
                               stream()) == -3


# ------------------------------------------------------------------------------------------------ row ops
def row_inputs(tag, M, N):
    dtype = DTYPES[tag]
    x = W.act_rows(M, N, dtype, seed=M + N, device=DEV)
    gamma, beta = W.ln_params(N, dtype, seed=N, device=DEV)
    return x, gamma, beta


def code_diff(a, b):
    d = np.abs(np.asarray(a, np.int32) - np.asarray(b, np.int32))
    return d.max(), float(np.mean(d != 0))


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_quant_per_token(gold, tag, MN):
    M, N = MN
    key = f"{tag}_{M}x{N}"
    x, _, _ = row_inputs(tag, M, N)
    q = torch.empty(M, N, dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=torch.float16, device=DEV)
    P.engine().invoke_quant(q, x, s)
    q2 = torch.empty_like(q)
    s2 = torch.empty_like(s)
    assert P.lib().b200awq_quant_per_token(ptr(x), ptr(q2), ptr(s2), M, N, 0 if tag == "f16" else 1, stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(q, q2) and torch.equal(s, s2)
    np.testing.assert_array_equal(q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], gold[f"quant_q_{key}"])
    np.testing.assert_array_equal(bits(s), gold[f"quant_s_{key}"])
    assert int(q[1].abs().max()) == 0 and float(s[1]) == 0.0  # zero row
    O.assert_admissible(q.cpu().numpy(), s.cpu().numpy(), O.quant_per_token_bounds(x.float().cpu().numpy()), key)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_layernorm_quant(gold, tag, MN):
    M, N = MN
    key = f"{tag}_{M}x{N}"
    x, gamma, beta = row_inputs(tag, M, N)
    e = P.engine()
    q = torch.empty(M, N, dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=torch.float16, device=DEV)
    e.rms_norm_general(q, x, gamma, beta, s, W.LN_EPS)  # default: per token
    qt = torch.empty(M, N, dtype=torch.int8, device=DEV)
    st = torch.full((1,), 30.0, dtype=torch.float16, device=DEV)
    e.rms_norm_general(out=qt, input=x, weight=gamma, bias=beta, scaling=st, epsilon=W.LN_EPS, use_per_token_quant=False)
    torch.cuda.synchronize()
    # against the reference's kernel: codes +-1 (summation order), scales <= 1 ulp
    mx, share = code_diff(q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], gold[f"ln_q_{key}"])
    assert mx <= 1 and share < 0.01, (mx, share)
    assert ulps(bits(s), gold[f"ln_s_{key}"]).max() <= 1
    mx, share = code_diff(qt.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], gold[f"lnt_q_{key}"])
    assert mx <= 1 and share < 0.01, (mx, share)
    # against the oracle's admissible sets
    xf, gf, bf = (t.float().cpu().numpy() for t in (x, gamma, beta))
    O.assert_admissible(q.cpu().numpy(), s.cpu().numpy(), O.layernorm_quant_bounds(xf, gf, bf, W.LN_EPS, tag), key)
    bt = O.layernorm_quant_bounds(xf, gf, None, W.LN_EPS, tag, per_token=False, scale=np.array([30.0], np.float16))
    O.assert_admissible(qt.cpu().numpy(), None, bt, key)


@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_gelu_quant(gold, MN):
    M, N = MN
    key = f"f16_{M}x{N}"
    x = W.gelu_rows(M, N, seed=7 * M + N, device=DEV)
    q = torch.empty(M, N, dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=torch.float16, device=DEV)
    tmp = torch.empty(M, N, dtype=torch.float16, device=DEV)
    P.engine().gelu_and_quant(q, x, s, tmp)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(bits(tmp.reshape(-1)[::W.ROW_SAMPLE]), gold[f"gelu_t_{key}"])
    np.testing.assert_array_equal(q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], gold[f"gelu_q_{key}"])
    np.testing.assert_array_equal(bits(s), gold[f"gelu_s_{key}"])
    b = O.gelu_quant_bounds(x.cpu().numpy())
    O.assert_between(tmp.cpu().numpy(), b["g_lo"], b["g_hi"], key)
    O.assert_admissible(q.cpu().numpy(), s.cpu().numpy(), b, key)
    # the tiny row: 127 / amax overflows fp16, so every non-zero code saturates
    assert float(s[2]) < 2e-5 and set(np.unique(q[2].cpu().numpy())) <= {-127, 0, 127}


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_silu_and_mul(gold, tag, MN):
    M, N = MN
    x, _, _ = row_inputs(tag, M, N)
    xx = torch.cat([x, x.flip(0)], dim=1).contiguous()
    y = P.engine().silu_and_mul(xx)
    y2 = torch.empty_like(y)
    assert P.lib().b200awq_silu_and_mul(ptr(xx), ptr(y2), M, N, 0 if tag == "f16" else 1, stream()) == 0
    torch.cuda.synchronize()
    assert y.shape == (M, N) and torch.equal(y, y2)
    assert ulps(bits(y.reshape(-1)[::W.ROW_SAMPLE]), gold[f"silu_{tag}_{M}x{N}"]).max() <= 1
    lo, hi = O.silu_and_mul_bounds(xx.float().cpu().numpy(), tag)
    O.assert_between(y.float().cpu().numpy(), lo, hi, f"{tag}_{M}x{N}")


def test_row_ops_odd_width_and_fp32_rejected():
    M, N = 33, 1001  # n % 8 != 0: one element per access
    x = W.act_rows(M, N, torch.float16, seed=5, device=DEV)
    q = torch.empty(M, N, dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=torch.float16, device=DEV)
    P.engine().invoke_quant(q, x, s)
    torch.cuda.synchronize()
    O.assert_admissible(q.cpu().numpy(), None, O.quant_per_token_bounds(x.float().cpu().numpy()))
    with pytest.raises(RuntimeError):
        P.engine().invoke_quant(q, x.float(), s)
    assert P.lib().b200awq_quant_per_token(ptr(x), ptr(q), ptr(s), M, N, 2, stream()) == -4


# ------------------------------------------------------------------------------------------------ composition
def oracle_linear(xq, xs, w, ws, b):
    return O.gemm(xq, w, ws, xs, b)


def test_siglip_layer_chain():
    """LN-quant -> qkv -> quant(stand-in attention output) -> out -> residual -> LN-quant -> fc1 -> gelu-quant -> fc2,
    each step fed with the GPU's own previous output and compared with the oracle."""
    e = P.engine()
    M, H, I = 729, 1152, 4304
    g = torch.Generator().manual_seed(11)
    h = (torch.randn(M, H, generator=g)).half().to(DEV)
    ln1, ln2 = W.ln_params(H, torch.float16, 1, DEV), W.ln_params(H, torch.float16, 2, DEV)
    lin = {}
    for name, (n, k) in {"qkv": (3 * H, H), "out": (H, H), "fc1": (I, H), "fc2": (H, I)}.items():
        wf = torch.randn(n, k, generator=g) * 0.02
        lin[name] = P.W8A8OF16LinearDynamicInputScale.from_linear(_linear(wf, g), device=DEV)

    def run_ln(x, p):
        q = torch.empty(M, H, dtype=torch.int8, device=DEV)
        s = torch.empty(M, dtype=torch.float16, device=DEV)
        e.rms_norm_general(q, x, p[0], p[1], s, 1e-6)
        return q, s

    def run_lin(name, q, s):
        y = torch.empty(M, lin[name].out_features, dtype=torch.float16, device=DEV)
        lin[name](q, s, y)
        return y

    def check_lin(name, q, s, y):
        L = lin[name]
        o = O.gemm(q.cpu().numpy(), L.weight.cpu().numpy(), L.dequant_scale.cpu().numpy(), s.cpu().numpy(),
                   L.bias.cpu().numpy())
        np.testing.assert_array_equal(bits(y), o.view(np.uint16), err_msg=name)

    q, s = run_ln(h, ln1)
    O.assert_admissible(q.cpu().numpy(), s.cpu().numpy(),
                        O.layernorm_quant_bounds(h.float().cpu().numpy(), *(t.float().cpu().numpy() for t in ln1), 1e-6,
                                                 "f16"), "ln1")
    qkv = run_lin("qkv", q, s)
    check_lin("qkv", q, s, qkv)
    attn = qkv[:, :H].contiguous()  # fixed stand-in for the attention output
    aq = torch.empty(M, H, dtype=torch.int8, device=DEV)
    as_ = torch.empty(M, dtype=torch.float16, device=DEV)
    e.invoke_quant(aq, attn, as_)
    o = run_lin("out", aq, as_)
    check_lin("out", aq, as_, o)
    h2 = h + o
    q2, s2 = run_ln(h2, ln2)
    f1 = run_lin("fc1", q2, s2)
    check_lin("fc1", q2, s2, f1)
    gq = torch.empty(M, I, dtype=torch.int8, device=DEV)
    gs = torch.empty(M, dtype=torch.float16, device=DEV)
    tmp = torch.empty(M, I, dtype=torch.float16, device=DEV)
    e.gelu_and_quant(gq, f1, gs, tmp)
    O.assert_admissible(gq.cpu().numpy(), gs.cpu().numpy(), O.gelu_quant_bounds(f1.cpu().numpy()), "gelu")
    f2 = run_lin("fc2", gq, gs)
    check_lin("fc2", gq, gs, f2)
    torch.cuda.synchronize()
    assert torch.isfinite(f2).all()


def _linear(wf, g):
    n, k = wf.shape
    lin = torch.nn.Linear(k, n).half().requires_grad_(False)
    lin.weight.copy_(wf.half())
    lin.bias.copy_((torch.randn(n, generator=g) * 0.1).half())
    return lin


def test_graph_capture_and_side_stream():
    M, N, K = 1024, 1152, 4304
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    xa = W.act_rows(M, K, torch.float16, seed=3, device=DEV)
    e = P.engine()
    ref_y = torch.empty(M, N, dtype=torch.float16, device=DEV)
    e.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, ref_y, b)
    q0 = torch.empty(M, K, dtype=torch.int8, device=DEV)
    s0 = torch.empty(M, dtype=torch.float16, device=DEV)
    e.invoke_quant(q0, xa, s0)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    y = torch.zeros_like(ref_y)
    q = torch.empty_like(q0)
    s = torch.empty_like(s0)
    with torch.cuda.stream(side):
        e.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, y, b)
        e.invoke_quant(q, xa, s)
    side.synchronize()
    assert torch.equal(y, ref_y) and torch.equal(q, q0) and torch.equal(s, s0)
    y.zero_()
    q.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            e.invoke_quant(q, xa, s)
            e.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, y, b)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, ref_y) and torch.equal(q, q0)


def test_mirror_forward_with_and_without_bias():
    g = torch.Generator().manual_seed(4)
    for has_bias in (True, False):
        lin = torch.nn.Linear(1152, 4304, bias=has_bias).half().requires_grad_(False)
        lin.weight.copy_((torch.randn(4304, 1152, generator=g) * 0.02).half())
        m = P.W8A8OF16LinearDynamicInputScale.from_linear(lin, device=DEV)
        assert (m.bias is not None) == has_bias
        x, _, _, a, _ = W.gemm_inputs(64, 4304, 1152, DEV)
        y = torch.empty(64, 4304, dtype=torch.float16, device=DEV)
        m(x, a, y)
        torch.cuda.synchronize()
        o = O.gemm(x.cpu().numpy(), m.weight.cpu().numpy(), m.dequant_scale.cpu().numpy(), a.cpu().numpy(),
                   m.bias.cpu().numpy() if has_bias else None)
        np.testing.assert_array_equal(bits(y), o.view(np.uint16))
