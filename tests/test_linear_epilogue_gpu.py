"""The W4A16 linear with its bias and residual adds in the kernel's epilogue (b200awq_w4a16_linear,
awq_inference_engine.w4a16_linear_forward_cuda, WQLinear.forward(x, residual)).

The contract is bit-identity with what callers do today: the existing engine call (gemv_forward_cuda_new below 8
tokens, gemm_forward_cuda_new from 8, the reference's dispatch rule) followed by PyTorch's `out + bias` and then
`residual + out`.  Every comparison here is torch.equal.  The route each case takes is pinned by kernel name with the
profiler (tests/kernel_trace.py), so that every kernel's epilogue (decode single-CTA and k-split cluster, ring, stream,
the wgmma kernel's skinny launch and its tile launch with and without the split-k reduction) is covered by name."""
import ctypes
import os

import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer, gen_x
from guard_bands import Op, guarded_call
from kernel_trace import short_names, trace
from w4a16_plans import plan

DEV = "cuda:0"
F16, BF16 = torch.float16, torch.bfloat16
DTYPES = [pytest.param(F16, id="f16"), pytest.param(BF16, id="bf16")]
OPS = ("neither", "bias", "residual", "both")
MS = (1, 2, 3, 4, 5, 7, 8, 16, 17, 64, 193, 2048)

# (name, n, k): the projections that carry a bias (Qwen2's q / k / v) or a residual (o_proj, down_proj) in tinychat
SHAPES = [
    ("qwen2_7b_q", 3584, 3584), ("qwen2_7b_kv", 512, 3584), ("qwen2_7b_o", 3584, 3584), ("qwen2_7b_down", 3584, 18944),
    ("llama3_8b_o", 4096, 4096), ("llama3_8b_down", 4096, 14336), ("qwen2_0_5b_kv", 128, 896),
]
STREAM_SHAPE = ("stream_n520", 520, 1024)  # n % 128 != 0: only the GEMV envelope (m < 8), 5..7 tokens take the stream kernel

_layers = {}


def layer(n, k, dtype):
    key = (n, k, dtype)
    if key not in _layers:
        _layers.clear()  # one layer at a time on the device
        _layers[key] = gen_layer(n, k, dtype, seed=n * 7 + k, device=DEV)
    return _layers[key]


def operands(m, n, dtype, op, seed):
    g = torch.Generator().manual_seed(seed)
    bias = torch.randn(n, generator=g).to(dtype).to(DEV) if op in ("bias", "both") else None
    res = (4 * torch.randn(m, n, generator=g)).to(dtype).to(DEV) if op in ("residual", "both") else None
    return bias, res


def unfused(x, qw, s, z, bias=None, residual=None):
    """Today's calls: the engine call the reference's WQLinear makes, then the callers' PyTorch adds in their order."""
    eng = P.engine()
    m, k = x.numel() // x.shape[-1], x.shape[-1]
    if m < 8:
        out = eng.gemv_forward_cuda_new(x, qw, s, z, m, s.shape[1], k, 128)
    else:
        out = eng.gemm_forward_cuda_new(x, qw, s, z)
    if bias is not None:
        out = out + bias
    if residual is not None:
        out = residual + out
    return out


def fused(x, qw, s, z, bias=None, residual=None):
    return P.engine().w4a16_linear_forward_cuda(x, qw, s, z, 128, bias=bias, residual=residual)


def traced_call(m, n, k, dt, entry, op):
    """kernel_trace builder: entry "linear" is w4a16_linear_forward_cuda with the given operands ("none", "bias",
    "residual", "both"), "engine" the gemv / gemm call of today."""
    dtype = getattr(torch, dt)
    eng = P.engine()
    qw, s, z = gen_layer(n, k, dtype, seed=n + k, device="cuda")
    x = gen_x(m, k, dtype, seed=m).cuda()
    bias = torch.randn(n, device="cuda").to(dtype) if op in ("bias", "both") else None
    res = torch.randn(m, n, device="cuda").to(dtype) if op in ("residual", "both") else None
    if entry == "linear":
        return lambda: eng.w4a16_linear_forward_cuda(x, qw, s, z, 128, bias=bias, residual=res)
    if m < 8:
        return lambda: eng.gemv_forward_cuda_new(x, qw, s, z, m, n, k, 128)
    return lambda: eng.gemm_forward_cuda_new(x, qw, s, z)


def profiled_kernels(cases, env=None):
    """The names of the GPU work of one call per case (see traced_call), eight cases per profiling process."""
    cases = [[m, n, k, "float16" if dt == F16 else "bfloat16", entry, op] for m, n, k, dt, entry, op in cases]
    return [r.names for r in trace("test_linear_epilogue_gpu:traced_call", cases, per_process=8, env=env)]


def check_equal(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    if not torch.equal(got.view(torch.int16), want.view(torch.int16)):
        bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} elements differ; first at {i}: {got[i].item()!r} vs {want[i].item()!r}")


# ------------------------------------------------------------------------------------------------ bit-identity
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", SHAPES + [STREAM_SHAPE], ids=lambda s: s[0])
def test_bit_identical_to_engine_call_then_torch_adds(shape, dtype):
    name, n, k = shape
    qw, s, z = layer(n, k, dtype)
    ms = (5, 6, 7, 1, 3) if n % 128 else MS
    for m in ms:
        x = gen_x(m, k, dtype, seed=m + n).to(DEV)
        for op in OPS:
            bias, res = operands(m, n, dtype, op, seed=m * 3 + n)
            check_equal(fused(x, qw, s, z, bias, res), unfused(x, qw, s, z, bias, res), f"{name} m={m} {op}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_leading_dimensions_and_3d_inputs(dtype):
    """in_feats [b, s, k] and a residual of the output's shape [b, s, n], as the decoder blocks hold them."""
    n, k = 4096, 4096
    qw, s, z = layer(n, k, dtype)
    for b, t in ((1, 1), (1, 5), (2, 4), (1, 300)):
        x = gen_x(b * t, k, dtype, seed=t).to(DEV).view(b, t, k)
        bias, res = operands(b * t, n, dtype, "both", seed=b + t)
        res = res.view(b, t, n)
        check_equal(fused(x, qw, s, z, bias, res), unfused(x, qw, s, z, bias, res), f"[{b}, {t}, k]")


# ------------------------------------------------------------------------------------------------ routes
# (route, m, n, k, dtype, kernel name as short_names reports it; None = the tile launch, name from its plan)
ROUTES = [
    ("decode", 1, 4096, 4096, F16, "w4a16_decode_kernel"),
    ("decode_ksplit", 1, 4096, 14336, F16, "w4a16_decode_kernel"),   # k = 14336: the plan splits k over a cluster
    ("ring", 3, 4096, 4096, F16, "w4a16_ring_kernel"),
    ("ring_bf16_m1", 1, 3584, 3584, BF16, "w4a16_ring_kernel"),
    ("stream", 6, 520, 1024, F16, "w4a16_stream_kernel"),
    ("stream_bf16", 7, 520, 1024, BF16, "w4a16_stream_kernel"),
    ("flat", 6, 4096, 4096, F16, "w4a16_wgmma_kernel<16>"),
    ("flat_bf16", 5, 3584, 3584, BF16, "w4a16_wgmma_kernel<16>"),
    ("tile_split", 12, 4096, 14336, F16, None),                      # 9..16 tokens on a >= 48 M weight layer
    ("tile_split_bf16", 16, 3584, 18944, BF16, None),
    ("tile", 2048, 4096, 4096, F16, None),
    ("tile_bf16", 193, 3584, 3584, BF16, None),
]


@pytest.mark.gpu
def test_every_route_pinned_by_kernel_name():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    names = profiled_kernels([(m, n, k, dtype, "linear", "both") for _, m, n, k, dtype, _ in ROUTES])
    wrong, rows = [], []
    for (route, m, n, k, dtype, want), got in zip(ROUTES, names):
        if want is None:
            p = plan(m, n, k, "f16" if dtype == F16 else "bf16", "linear", sms)
            assert p.route == "tile" and (p.S > 1) == route.startswith("tile_split"), (route, p)
            want = p.kernel
        got = short_names(got)
        rows.append(f"| {route} | {m} | {n} | {k} | {dtype} | {', '.join(sorted(got))} |")
        if got != {want}:
            wrong.append((route, sorted(got), want))
        qw, s, z = layer(n, k, dtype)
        x = gen_x(m, k, dtype, seed=m).to(DEV)
        bias, res = operands(m, n, dtype, "both", seed=m + 1)
        check_equal(fused(x, qw, s, z, bias, res), unfused(x, qw, s, z, bias, res), route)
    print("\n| route | m | n | k | dtype | kernel |\n|---|---|---|---|---|---|\n" + "\n".join(rows))
    assert not wrong, wrong


@pytest.mark.gpu
@pytest.mark.parametrize("split", [2, 4])
def test_decode_split_forced_through_the_test_override(split):
    """The k-split cluster plan of the one-token kernel on a shape that would not pick it (B200AWQ_DECODE_SPLIT)."""
    lib = P.lib()
    n, k = 4096, 4096
    names = profiled_kernels([(1, n, k, F16, "linear", op) for op in OPS], env={"B200AWQ_DECODE_SPLIT": str(split)})
    for op, got in zip(OPS, names):
        assert short_names(got) == {"w4a16_decode_kernel"}, (op, got)
    qw, s, z = layer(n, k, F16)
    x = gen_x(1, k, F16, seed=11).to(DEV)
    old = os.environ.get("B200AWQ_DECODE_SPLIT")
    os.environ["B200AWQ_DECODE_SPLIT"] = str(split)
    lib.b200awq_reload_config()
    try:
        for op in OPS:
            bias, res = operands(1, n, F16, op, seed=split)
            check_equal(fused(x, qw, s, z, bias, res), unfused(x, qw, s, z, bias, res), f"split {split} {op}")
    finally:
        if old is None:
            del os.environ["B200AWQ_DECODE_SPLIT"]
        else:
            os.environ["B200AWQ_DECODE_SPLIT"] = old
        lib.b200awq_reload_config()


NEITHER = [(m, n, k, dtype) for dtype in (F16, BF16)
           for m, n, k in ((1, 4096, 4096), (3, 4096, 4096), (6, 520, 1024), (6, 4096, 4096), (12, 4096, 14336),
                           (64, 4096, 4096), (2048, 3584, 3584))]


@pytest.mark.gpu
def test_neither_operand_is_the_existing_launch():
    """Without bias and residual the entry launches what gemv / gemm launch: one kernel, the same kernel (full name,
    template arguments included), the same bits."""
    eng = P.engine()
    names = profiled_kernels([(m, n, k, dt, entry, "none") for m, n, k, dt in NEITHER for entry in ("linear", "engine")])
    for i, (m, n, k, dtype) in enumerate(NEITHER):
        got, want = names[2 * i], names[2 * i + 1]
        assert got == want and len(got) == 1, (m, n, k, dtype, got, want)
        qw, s, z = layer(n, k, dtype)
        x = gen_x(m, k, dtype, seed=m).to(DEV)
        fused(x, qw, s, z)
        c0 = eng.launch_count()
        y = fused(x, qw, s, z)
        assert eng.launch_count() == c0 + 1
        check_equal(y, unfused(x, qw, s, z), f"no operands, m={m} n={n} k={k} {dtype}")


# ------------------------------------------------------------------------------------------------ PDL ordering
def decoder_chain(xs, layers, gamma, linear):
    """A chain of launches whose residuals come from the launches just before: per pair of layers
    a = rmsnorm(h); h = linear(a, residual=h)        residual written two launches earlier (by the linear)
    a = rmsnorm(h); r = h * 0.5; h = linear(a, residual=r)   residual written by a PyTorch op right before
    h = linear(h, residual=h)                         input and residual written by the launch right before
    a = rmsnorm(h); h = linear(a, residual=a)         residual written by layernorm_forward_cuda right before"""
    eng = P.engine()
    h = xs
    for i, (qw, s, z, bias) in enumerate(layers):
        a = torch.empty_like(h)
        kind = i % 4
        if kind != 2:
            eng.layernorm_forward_cuda(h, gamma, a, 1e-6)
        if kind == 0:
            h = linear(a, qw, s, z, bias, h)
        elif kind == 1:
            h = linear(a, qw, s, z, bias, h * 0.5)
        elif kind == 2:
            h = linear(h, qw, s, z, bias, h)
        else:
            h = linear(a, qw, s, z, bias, a)
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m", [1, 3, 6, 16, 64])
def test_graph_captured_chain_reads_residuals_in_stream_order(m, dtype):
    n = k = 4096
    layers = []
    for i in range(8):
        qw, s, z = gen_layer(n, k, dtype, seed=100 + i, device=DEV)
        bias = operands(1, n, dtype, "bias", seed=i)[0] if i % 2 else None
        layers.append((qw, s, z, bias))
    gamma = (1 + 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(5))).to(dtype).to(DEV)
    x = gen_x(m, k, dtype, seed=m).to(DEV)
    want = decoder_chain(x, layers, gamma, unfused)
    results = {}
    lib = P.lib()
    for pdl in (True, False):
        prev = lib.b200awq_set_pdl(1 if pdl else 0)
        try:
            eager = decoder_chain(x, layers, gamma, fused)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                decoder_chain(x, layers, gamma, fused)  # warm-up of the capture stream
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = decoder_chain(x, layers, gamma, fused)
            g.replay()
            torch.cuda.synchronize()
            results[pdl] = (eager, out.clone())
        finally:
            lib.b200awq_set_pdl(prev)
    for pdl, (eager, graphed) in results.items():
        check_equal(eager, want, f"eager chain, pdl={pdl}")
        check_equal(graphed, want, f"graph replay, pdl={pdl}")


# ------------------------------------------------------------------------------------------------ guard bands
def _linear_abi(v, m, n, k, dtype, with_bias, with_res):
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    return P.lib().b200awq_w4a16_linear(p(v["x"]), p(v["qw"]), p(v["s"]), p(v["z"]), p(v["b"]) if with_bias else None,
                                        p(v["r"]) if with_res else None, p(v["y"]), m, n, k, 128,
                                        0 if dtype == F16 else 1, st)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,n,k", [(1, 4104, 4096), (1, 4096, 14336), (3, 4104, 4096), (6, 520, 1024), (7, 3584, 3584),
                                   (12, 4096, 14336), (193, 3584, 3584)])
def test_guard_bands_around_bias_residual_and_output(m, n, k, dtype):
    """bias and residual inside NaN-filled bands: a read past them poisons the result; y's bands stay unchanged."""
    qw, s, z = gen_layer(n, k, dtype, seed=n + k, device="cpu")
    x = gen_x(m, k, dtype, seed=m)
    bias, res = operands(m, n, dtype, "both", seed=m)
    ops = {"x": Op("in", x), "qw": Op("in", qw), "s": Op("in", s), "z": Op("in", z), "b": Op("in", bias.cpu()),
           "r": Op("in", res.cpu()), "y": Op("out", shape=(m, n), dtype=dtype)}
    out = guarded_call(lambda v: _linear_abi(v, m, n, k, dtype, True, True), ops)
    want = unfused(x.to(DEV), qw.to(DEV), s.to(DEV), z.to(DEV), bias, res)
    check_equal(out["y"], want, "guarded call")


# ------------------------------------------------------------------------------------------------ rejections
@pytest.mark.gpu
def test_bad_operands_raise():
    eng = P.engine()
    n, k, m = 4096, 4096, 4
    qw, s, z = layer(n, k, F16)
    x = gen_x(m, k, F16, seed=1).to(DEV)
    buf = torch.zeros(m * n + 8, dtype=F16, device=DEV)
    good_res = torch.zeros(m, n, dtype=F16, device=DEV)
    bad = [
        dict(residual=buf[1:1 + m * n].view(m, n)),                     # misaligned view
        dict(bias=buf[4:4 + n]),                                         # misaligned bias
        dict(residual=torch.zeros(m, n + 8, dtype=F16, device=DEV)),     # wrong shape
        dict(residual=torch.zeros(m * n, dtype=F16, device=DEV)),        # wrong rank
        dict(residual=torch.zeros(m, n, dtype=BF16, device=DEV)),        # wrong dtype
        dict(bias=torch.zeros(n, dtype=torch.float32, device=DEV)),
        dict(bias=torch.zeros(n + 8, dtype=F16, device=DEV)),
        dict(residual=torch.zeros(m, n, dtype=F16)),                     # CPU tensor
        dict(bias=torch.zeros(n, dtype=F16)),
        dict(residual=torch.zeros(n, m, dtype=F16, device=DEV).t()),     # not contiguous
    ]
    for kw in bad:
        with pytest.raises(RuntimeError):
            eng.w4a16_linear_forward_cuda(x, qw, s, z, 128, **kw)
    with pytest.raises(RuntimeError):  # n % 128 != 0 from 8 tokens (the GEMM envelope)
        q2, s2, z2 = gen_layer(520, 1024, F16, seed=1, device=DEV)
        eng.w4a16_linear_forward_cuda(gen_x(8, 1024, F16).to(DEV), q2, s2, z2, 128, residual=torch.zeros(8, 520, dtype=F16, device=DEV))
    eng.w4a16_linear_forward_cuda(x, qw, s, z, 128, residual=good_res)


# ------------------------------------------------------------------------------------------------ module, streams
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_wqlinear_with_bias_matches_its_old_forward(dtype):
    """The mirror's WQLinear with a bias: the same bits as the engine call + `out + self.bias` it made before, on the
    current stream, on a side stream, and replayed from a CUDA graph; residual= adds the decoder block's add."""
    n, k = 3584, 3584
    lin = P.WQLinear(4, 128, k, n, True, DEV, dtype=dtype)
    lin.qweight, lin.scales, lin.scaled_zeros = gen_layer(n, k, dtype, seed=9, device=DEV)
    lin.bias = operands(1, n, dtype, "bias", seed=9)[0]
    for t in (1, 5, 8, 40):
        x = gen_x(t, k, dtype, seed=t).to(DEV).view(1, t, k)
        _, res = operands(t, n, dtype, "residual", seed=t)
        res = res.view(1, t, n)
        check_equal(lin(x), unfused(x, lin.qweight, lin.scales, lin.scaled_zeros, lin.bias), f"bias, {t} tokens")
        check_equal(lin(x, residual=res), unfused(x, lin.qweight, lin.scales, lin.scaled_zeros, lin.bias, res),
                    f"bias + residual, {t} tokens")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            y_side = lin(x, residual=res)
        torch.cuda.current_stream().wait_stream(side)
        check_equal(y_side, lin(x, residual=res), f"side stream, {t} tokens")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side):
            lin(x, residual=res)
        torch.cuda.current_stream().wait_stream(side)
        with torch.cuda.graph(g):
            y_graph = lin(x, residual=res)
        g.replay()
        torch.cuda.synchronize()
        check_equal(y_graph, lin(x, residual=res), f"graph replay, {t} tokens")
    plain = P.WQLinear(4, 128, k, n, False, DEV, dtype=dtype)
    plain.qweight, plain.scales, plain.scaled_zeros = lin.qweight, lin.scales, lin.scaled_zeros
    x = gen_x(3, k, dtype, seed=3).to(DEV)
    check_equal(plain(x), unfused(x, plain.qweight, plain.scales, plain.scaled_zeros), "no bias, no residual")
