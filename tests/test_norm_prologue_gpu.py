"""RMSNorm prologues of the W4A16 launches (b200awq_w4a16_norm_linear, b200awq_w4a16_norm_mlp_front; DESIGN §3.5c).

The contract is bit-identity with the composition: layernorm_forward_cuda (x^ = RMSNorm(x)) followed by
w4a16_linear_forward_cuda / mlp_front_forward_cuda on x^.  Every comparison below is on the int16 views of the outputs
(which also holds NaN payloads to the bit), and every output buffer starts as NaN.
* Bit-identity over dtypes, bias, token counts from 1 to 2048 and the served shapes, on rows that are random, all
  zero (r = rsqrt(eps)), hit the fp16 clamp of x^, carry a single huge element, or hold inf / NaN.
* The same at every decode plan the test-only overrides B200AWQ_DECODE_SPLIT / B200AWQ_DECODE_SLOTS reach.
* The profiler: one W4A16 kernel and no RMSNorm launch where the plain launch is the decode or ring kernel, with the
  plain launch's grid and shared memory (tests/w4a16_plans.py); RMSNorm and then the plain launches elsewhere.
* Stream order: graph-captured chains in which the launch right before writes x, with PDL on and off, on a side stream
  and over graph replays.
* Guard bands around every operand (tests/guard_bands.py), and the Python mirrors."""
import ctypes
import functools
import os
import re

import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from guard_bands import Op, guarded_call
from kernel_trace import short_names, trace
from oracle import w4a16_oracle as O
from w4a16_plans import mlp_front_plan, plan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16, BF16 = torch.float16, torch.bfloat16
DTYPE = {"f16": F16, "bf16": BF16}
EPS = 1e-6
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132

# (label, n, k): Llama-3-8B q/k/v and gate/up, Qwen2-7B q/k/v (biased), Qwen2-0.5B q/k/v and gate/up, Llama-2-70B q/k/v,
# and the shortest k
SHAPES = [("l3_qkv", 6144, 4096), ("l3_gate_up", 14336, 4096), ("q7_qkv", 4608, 3584), ("q05_qkv", 1152, 896),
          ("q05_gate_up", 4864, 896), ("l2_70_qkv", 10240, 8192), ("k128", 512, 128)]
TOKENS = [1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 64, 2048]
OPS = ["linear", "linear_bias", "front"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st(stream=None):
    return ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def _code(T):
    return 0 if T == F16 else 1


@functools.lru_cache(maxsize=None)
def layer(n, k, T, seed=0):
    return gen_layer(n, k, T, seed=seed + n + 3 * k, device=DEV)


@functools.lru_cache(maxsize=None)
def bias_of(n, T):
    g = torch.Generator().manual_seed(n)
    return (0.5 * torch.randn(n, generator=g)).to(T).to(DEV)


def gammas(k, T):
    """(plain, clamping): RMSNorm weights around 1, and the same with +-65000 on every 61st element, which sends x^ of
    a constant row (and many elements of the others) into the fp16 clamp at +-(65504 - 1000)."""
    g = torch.Generator().manual_seed(k)
    plain = 1.0 + 0.3 * torch.randn(k, generator=g)
    big = plain.clone()
    big[::61] = 65000.0 * torch.sign(torch.randn(big[::61].shape, generator=g))
    return plain.to(T).to(DEV), big.to(T).to(DEV)


LANDSCAPES = ("random", "zeros", "huge_one", "inf_nan", "tiny", "constant")


def rows(m, k, T, shift, seed):
    """m rows whose landscapes cycle through LANDSCAPES from `shift`."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m, k, generator=g)
    for i in range(m):
        kind = LANDSCAPES[(i + shift) % len(LANDSCAPES)]
        if kind == "zeros":
            x[i] = 0.0
        elif kind == "huge_one":
            x[i] *= 1e-2
            x[i, (i * 37) % k] = 30000.0
        elif kind == "inf_nan":
            x[i, (i * 11) % k] = float("inf")
            x[i, (i * 13 + 5) % k] = float("nan")
        elif kind == "tiny":
            x[i] *= 2.0 ** -20
        elif kind == "constant":
            x[i] = -3.0
    return x.to(T).to(DEV)


# ------------------------------------------------------------------------------------------------ entries
def norm_linear(x, gamma, W, bias=None, eps=EPS, y=None, ws=None, stream=None):
    m, k = x.shape
    n = W[1].shape[1]
    y = torch.full((m, n), float("nan"), dtype=x.dtype, device=DEV) if y is None else y
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k)
    ws = torch.full((nb,), 0x7F, dtype=torch.uint8, device=DEV) if ws is None else ws
    rc = P.lib().b200awq_w4a16_norm_linear(_p(x), _p(gamma), eps, *map(_p, W), _p(bias), _p(y), m, n, k, 128,
                                           _code(x.dtype), _p(ws), ws.numel(), _st(stream))
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


def norm_front(x, gamma, G, U, eps=EPS, y=None, ws=None, stream=None):
    m, k = x.shape
    n = G[1].shape[1]
    y = torch.full((m, n), float("nan"), dtype=x.dtype, device=DEV) if y is None else y
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k)
    ws = torch.full((nb,), 0x7F, dtype=torch.uint8, device=DEV) if ws is None else ws
    rc = P.lib().b200awq_w4a16_norm_mlp_front(_p(x), _p(gamma), eps, *map(_p, G), *map(_p, U), _p(y), m, n, k, 128,
                                              _code(x.dtype), _p(ws), ws.numel(), _st(stream))
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


def rmsnorm(x, gamma, eps=EPS):
    out = torch.full_like(x, float("nan"))
    P.engine().layernorm_forward_cuda(x, gamma, out, eps)
    return out


def composed_linear(x, gamma, W, bias=None, eps=EPS):
    return P.engine().w4a16_linear_forward_cuda(rmsnorm(x, gamma, eps), *W, 128, bias=bias)


def composed_front(x, gamma, G, U, eps=EPS):
    return P.engine().mlp_front_forward_cuda(rmsnorm(x, gamma, eps), *G, *U)


def assert_bits(got, want, what):
    a, b = got.reshape(want.shape).view(torch.int16), want.view(torch.int16)
    if not torch.equal(a, b):
        bad = (a != b).nonzero()
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {len(bad)} of {a.numel()} elements differ; first at {i}: {got.reshape(want.shape)[i].item()!r} "
                    f"against {want[i].item()!r}")


def run_op(op, x, gamma, n, k, T, eps=EPS, count=False):
    """(fused, composed) outputs of op on x; with count, also the launches of the fused call (launch_count())."""
    c0 = P.engine().launch_count()
    if op == "front":
        G, U = layer(n, k, T, 1), layer(n, k, T, 2)
        fused = norm_front(x, gamma, G, U, eps)
        launches = P.engine().launch_count() - c0
        out = fused, composed_front(x, gamma, G, U, eps)
    else:
        W = layer(n, k, T)
        b = bias_of(n, T) if op == "linear_bias" else None
        fused = norm_linear(x, gamma, W, b, eps)
        launches = P.engine().launch_count() - c0
        out = fused, composed_linear(x, gamma, W, b, eps)
    return out + (launches,) if count else out


# ------------------------------------------------------------------------------------------------ 1. bit-identity
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("m", TOKENS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: s[0])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_bit_identical_to_the_composition(dtype, shape, m, op):
    _, n, k = shape
    T = DTYPE[dtype]
    plain, big = gammas(k, T)
    # every landscape on every token count: few tokens take one call per starting landscape
    shifts = range(len(LANDSCAPES)) if m < len(LANDSCAPES) else [0]
    for shift in shifts:
        x = rows(m, k, T, shift, seed=m * 31 + k + shift)
        for gname, gamma in (("plain", plain), ("clamping", big)):
            got, want = run_op(op, x, gamma, n, k, T)
            assert_bits(got, want, f"{dtype} {shape[0]} m={m} {op}, landscapes from {LANDSCAPES[shift]}, {gname} gamma")


def test_clamp_and_zero_rows_are_exercised():
    """The landscapes do what their names say on x^ itself: the clamp is reached, zero rows give zeros."""
    k = 4096
    plain, big = gammas(k, F16)
    x = rows(len(LANDSCAPES), k, F16, 0, seed=1)
    xh = rmsnorm(x, big)
    const = LANDSCAPES.index("constant")
    assert (xh[const].float().abs() == 64512.0).any()   # rn_fp16(65504 - 1000)
    assert (rmsnorm(x, plain)[LANDSCAPES.index("zeros")] == 0).all()


# ------------------------------------------------------------------------------------------------ 2. every plan
PLAN_SHAPES = [("q05_qkv", 1152, 896), ("q05_gate_up", 4864, 896), ("l3_qkv", 6144, 4096), ("k128", 512, 128),
               ("l2_70_qkv", 10240, 8192)]


@pytest.mark.parametrize("slots", [3, 4, 5, 6])
@pytest.mark.parametrize("split", list(range(1, 9)))
def test_every_decode_plan(split, slots):
    os.environ["B200AWQ_DECODE_SPLIT"] = str(split)
    os.environ["B200AWQ_DECODE_SLOTS"] = str(slots)
    P.lib().b200awq_reload_config()
    try:
        for label, n, k in PLAN_SHAPES:
            plain, big = gammas(k, F16)
            for shift in (0, 3):
                x = rows(1, k, F16, shift, seed=k + shift)
                for op in OPS:
                    got, want, launches = run_op(op, x, plain, n, k, F16, count=True)
                    # the prologue ran inside the W4A16 launch: one kernel, no RMSNorm launch
                    assert launches == 1, (label, op, launches)
                    assert_bits(got, want, f"split {split} slots {slots} {label} {op} shift {shift}")
            x = rows(1, k, F16, LANDSCAPES.index("constant"), seed=k)
            got, want = run_op("linear", x, big, n, k, F16)
            assert_bits(got, want, f"split {split} slots {slots} {label} clamping gamma")
    finally:
        os.environ.pop("B200AWQ_DECODE_SPLIT"), os.environ.pop("B200AWQ_DECODE_SLOTS")
        P.lib().b200awq_reload_config()


def override_call(entry, op, n, k):
    """kernel_trace builder: the norm entry ("norm") or the plain entry on x^ ("plain") of one m = 1 fp16 case."""
    T = F16
    x, y = torch.zeros(1, k, dtype=T, device=DEV), torch.empty(1, n, dtype=T, device=DEV)
    gamma = torch.ones(k, dtype=T, device=DEV)
    W = [(torch.zeros(n // 4, k, dtype=torch.int16, device=DEV),
          *(torch.zeros(O.scale_rows(k), n, dtype=T, device=DEV) for _ in range(2))) for _ in range(2)]
    bias = torch.zeros(n, dtype=T, device=DEV) if op == "linear_bias" else None
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(1, n, k)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st, L = _st(), P.lib()
    if entry == "plain" and op == "front":
        return lambda: L.b200awq_w4a16_mlp_front(_p(x), *map(_p, W[0]), *map(_p, W[1]), _p(y), 1, n, k, 128, 0, _p(ws), nb, st)
    if entry == "plain":
        return lambda: L.b200awq_w4a16_linear(_p(x), *map(_p, W[0]), _p(bias), None, _p(y), 1, n, k, 128, 0, st)
    return traced_call(op, 1, n, k, "f16")


@pytest.mark.parametrize("split", list(range(1, 9)))
def test_overridden_plans_run_the_prologue_kernel(split):
    """Under each B200AWQ_DECODE_SPLIT (and the shallowest ring, B200AWQ_DECODE_SLOTS=3), every case of
    test_every_decode_plan launches the normed decode kernel, with the grid and shared memory of the plain launch
    under the same override."""
    cases = [[e, op, n, k] for (_, n, k) in PLAN_SHAPES for op in OPS for e in ("norm", "plain")]
    recs = trace("test_norm_prologue_gpu:override_call", cases, per_process=len(cases),
                 env={"B200AWQ_DECODE_SPLIT": str(split), "B200AWQ_DECODE_SLOTS": "3"})
    wrong = []
    for i in range(0, len(cases), 2):
        norm, plain = recs[i], recs[i + 1]
        have = [(kernel_name(e.name), e.grid, e.smem) for e in norm.events]
        want = [("norm:" + kernel_name(e.name), e.grid, e.smem) for e in plain.events]
        if len(want) != 1 or not want[0][0].startswith("norm:w4a16_decode_kernel") or have != want or norm.launches != 1:
            wrong.append((cases[i][1:], have, want, norm.launches))
    assert not wrong, wrong


def test_rmsnorm_reproduces_the_stored_order_bits():
    """b200awq_rmsnorm (both of its kernels) still gives the stored outputs of tests/golden/rmsnorm_order.npz, which
    tests/test_norm_prologue_cpu.py reproduces from the numpy restatement of rmsnorm_stat.cuh's order: the order the
    prologues share with rmsnorm.cu cannot change unnoticed."""
    import numpy as np
    import norm_order as N
    data = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rmsnorm_order.npz"))
    for dt in ("f16", "bf16"):
        for n in N.WIDTHS:
            x, g = N.inputs(n, dt)
            xd, gd = torch.from_numpy(x).to(DTYPE[dt]).to(DEV), torch.from_numpy(g).to(DTYPE[dt]).to(DEV)
            got = rmsnorm(xd, gd, N.EPS).view(torch.int16).cpu().numpy().view(np.uint16)
            assert np.array_equal(got, data[f"{dt}_{n}"]), (dt, n)
            if n % 8 == 0 and n >= 128:   # the same rows through the prologue: x^ W~^T equals the plain entry on x^
                W = layer(256, n, DTYPE[dt])
                assert_bits(norm_linear(xd[:1], gd, W, eps=N.EPS), composed_linear(xd[:1], gd, W, eps=N.EPS), (dt, n))


# ------------------------------------------------------------------------------------------------ 3. routes pinned
TRACE_CASES = [[op, m, n, k, dt] for op in OPS for (_, n, k) in SHAPES for m in (1, 2, 3, 4, 5, 9, 17)
               for dt in ("f16", "bf16")]


def traced_call(op, m, n, k, dt):
    """kernel_trace builder: the norm entry of one case on zero weights."""
    T = DTYPE[dt]
    x, y = torch.zeros(m, k, dtype=T, device=DEV), torch.empty(m, n, dtype=T, device=DEV)
    gamma = torch.ones(k, dtype=T, device=DEV)
    W = [(torch.zeros(n // 4, k, dtype=torch.int16, device=DEV),
          *(torch.zeros(O.scale_rows(k), n, dtype=T, device=DEV) for _ in range(2))) for _ in range(2)]
    bias = torch.zeros(n, dtype=T, device=DEV) if op == "linear_bias" else None
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st = _st()
    if op == "front":
        return lambda: P.lib().b200awq_w4a16_norm_mlp_front(_p(x), _p(gamma), EPS, *map(_p, W[0]), *map(_p, W[1]), _p(y),
                                                            m, n, k, 128, _code(T), _p(ws), nb, st)
    return lambda: P.lib().b200awq_w4a16_norm_linear(_p(x), _p(gamma), EPS, *map(_p, W[0]), _p(bias), _p(y), m, n, k,
                                                     128, _code(T), _p(ws), nb, st)


def kernel_name(name):
    """The kernel's name as w4a16_plans.py writes it, prefixed "norm:" for the instantiations with the prologue
    (w4a16_decode_norm_kernel<FUSED, EPI>, w4a16_ring_norm_kernel<T, M1, EPI>)."""
    if "rmsnorm" in name:
        return "rmsnorm"
    if "silu_mul_kernel" in name:
        return "silu_mul_kernel"
    mt = re.search(r"w4a16_decode(_norm)?_kernel<\s*(true|false)", name)
    if mt:
        return ("norm:" if mt.group(1) else "") + ("w4a16_decode_kernel<true, false>" if mt.group(2) == "true"
                                                   else "w4a16_decode_kernel")
    mt = re.search(r"w4a16_ring(_norm)?_kernel<", name)
    if mt:
        return ("norm:" if mt.group(1) else "") + "w4a16_ring_kernel"
    found = short_names([name])
    return found.pop() if found else name


def expected(op, m, n, k, dt):
    """[(kernel, grid, smem)] the norm entry launches: the plain plan's kernels, behind one RMSNorm launch unless the
    plain plan's single kernel is the decode or ring kernel (grid and shared memory then those of the plain launch)."""
    if op == "front":
        ps = mlp_front_plan(m, n, k, dt, SMS)
        fused = len(ps) == 1
    else:
        ps = (plan(m, n, k, dt, "linear", SMS),)
        fused = ps[0].route in ("decode", "ring")
    want = [(p.kernel, [p.grid, 1, 1], p.smem + (128 if p.route == "stream" else 0)) for p in ps]
    if fused:
        return [("norm:" + w[0],) + w[1:] for w in want]
    return [("rmsnorm", [m, 1, 1], None)] + want


def test_routes_pinned_by_profiler():
    records = trace("test_norm_prologue_gpu:traced_call", TRACE_CASES, per_process=64)
    wrong = []
    for c, rec in zip(TRACE_CASES, records):
        want = expected(*c)
        have = [(kernel_name(e.name), e.grid, e.smem) for e in rec.events]
        have_cmp = [(h[0], h[1], None if w[2] is None else h[2]) for h, w in zip(have, want)] if len(have) == len(want) else have
        if have_cmp != want or rec.launches != len(want):
            wrong.append((c, have, want, rec.launches))
    assert not wrong, wrong[:10]
    fused = sum(1 for c in TRACE_CASES if len(expected(*c)) == 1)
    assert fused >= 40, fused   # fp16 m = 1 (plain, bias, front), ring m = 2..4 and bf16 m = 1 are among the cases


# ------------------------------------------------------------------------------------------------ 4. stream order
def _chain(fused, n_o, k_o, n, k, T, pdl, stream=None):
    """h = o(a) + residual (the o projection's epilogue writes the norm's input), then the normed q/k/v and the normed
    MLP front on h; returns a closure over fixed buffers and the outputs."""
    a = rows(1, k_o, T, 0, seed=5)
    res = rows(1, n_o, T, 0, seed=6)
    Wo, Wq = layer(n_o, k_o, T, 7), layer(n, k, T)
    G, U = layer(n, k, T, 1), layer(n, k, T, 2)
    gamma, _ = gammas(k, T)
    bias = bias_of(n, T)
    h = torch.empty(1, n_o, dtype=T, device=DEV)
    xh = torch.empty(1, k, dtype=T, device=DEV)
    q = torch.empty(1, n, dtype=T, device=DEV)
    f = torch.empty(1, n, dtype=T, device=DEV)
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(1, n, k)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    wsf = torch.empty(P.lib().b200awq_w4a16_mlp_front_workspace_bytes(1, n, k), dtype=torch.uint8, device=DEV)
    L = P.lib()
    c = _code(T)

    def step():
        st = _st(stream)
        assert L.b200awq_w4a16_linear(_p(a), *map(_p, Wo), None, _p(res), _p(h), 1, n_o, k_o, 128, c, st) == 0
        if fused:
            assert L.b200awq_w4a16_norm_linear(_p(h), _p(gamma), EPS, *map(_p, Wq), _p(bias), _p(q), 1, n, k, 128, c,
                                               _p(ws), nb, st) == 0
            assert L.b200awq_w4a16_norm_mlp_front(_p(h), _p(gamma), EPS, *map(_p, G), *map(_p, U), _p(f), 1, n, k, 128, c,
                                                  _p(ws), nb, st) == 0
        else:
            assert L.b200awq_rmsnorm(_p(h), _p(gamma), _p(xh), 1, k, EPS, c, st) == 0
            assert L.b200awq_w4a16_linear(_p(xh), *map(_p, Wq), _p(bias), None, _p(q), 1, n, k, 128, c, st) == 0
            assert L.b200awq_w4a16_mlp_front(_p(xh), *map(_p, G), *map(_p, U), _p(f), 1, n, k, 128, c, _p(wsf),
                                             wsf.numel(), st) == 0
    return step, (h, q, f), a


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("pdl", [True, False])
def test_graph_chain_with_the_writer_right_before(pdl, dtype):
    T = DTYPE[dtype]
    n_o = k = 4096
    old = P.engine().set_pdl(pdl)
    try:
        outs = {}
        for fused in (False, True):
            step, bufs, a = _chain(fused, n_o, 4096, 6144, k, T, pdl)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()   # warm-up outside capture
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
            results = []
            for r in range(3):   # replays on fresh activations: every replay reads what the writer just stored
                a.copy_(rows(1, 4096, T, r, seed=100 + r))
                g.replay()
                torch.cuda.synchronize()
                results.append([b.clone() for b in bufs])
            outs[fused] = results
        for r in range(3):
            for name, got, want in zip(("h", "qkv", "front"), outs[True][r], outs[False][r]):
                assert_bits(got, want, f"replay {r} {name}, pdl {pdl}")
    finally:
        P.engine().set_pdl(old)


@pytest.mark.parametrize("pdl", [True, False])
def test_side_stream_after_attention(pdl):
    """single_query_attention writes the o projection's input on a side stream; o (+ residual) writes the norm's input."""
    T = F16
    heads, hd, max_len = 32, 128, 64
    old = P.engine().set_pdl(pdl)
    try:
        s = torch.cuda.Stream()
        g = torch.Generator().manual_seed(3)
        qkv = [torch.randn(1, heads, hd, generator=g).to(T).to(DEV) for _ in range(3)]
        outs = {}
        for fused in (False, True):
            step, bufs, a = _chain(fused, 4096, heads * hd, 6144, 4096, T, pdl, stream=s)
            kc = torch.zeros(1, heads, hd // 8, max_len, 8, dtype=T, device=DEV)
            vc = torch.zeros(1, heads, max_len, hd, dtype=T, device=DEV)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for t in range(4):
                    att = P.engine().single_query_attention(*qkv, kc, vc, None, None, t, hd, 10000.0, 1.0, True)
                    a.copy_(att.reshape(1, heads * hd))
                    step()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            outs[fused] = [b.clone() for b in bufs]
        for name, got, want in zip(("h", "qkv", "front"), outs[True], outs[False]):
            assert_bits(got, want, f"{name} after attention, pdl {pdl}")
    finally:
        P.engine().set_pdl(old)


# ------------------------------------------------------------------------------------------------ 5. guard bands
GUARD_CASES = [("linear", 1, "f16"), ("linear_bias", 1, "f16"), ("front", 1, "f16"), ("linear_bias", 3, "f16"),
               ("linear", 1, "bf16"), ("linear_bias", 9, "f16"), ("front", 2, "bf16"), ("linear", 64, "bf16")]


@pytest.mark.parametrize("offset", [0, 16])
@pytest.mark.parametrize("case", GUARD_CASES, ids=lambda c: f"{c[0]}-m{c[1]}-{c[2]}")
def test_guard_bands(case, offset):
    op, m, dt = case
    T = DTYPE[dt]
    n, k = 1152, 896
    x = rows(m, k, T, 0, seed=m)
    gamma, _ = gammas(k, T)
    nb = P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k)
    ops = {"x": Op("in", x, offset=offset), "gamma": Op("in", gamma, offset=offset),
           "y": Op("out", shape=(m, n), dtype=T, offset=offset), "ws": Op("scratch", shape=(nb,), dtype=torch.uint8, offset=offset)}
    if op == "front":
        G, U = layer(n, k, T, 1), layer(n, k, T, 2)
        for name, t in zip(("gq", "gs", "gz", "uq", "us", "uz"), (*G, *U)):
            ops[name] = Op("in", t)

        def call(v):
            return P.lib().b200awq_w4a16_norm_mlp_front(_p(v["x"]), _p(v["gamma"]), EPS, *(_p(v[s]) for s in ("gq", "gs", "gz")),
                                                        *(_p(v[s]) for s in ("uq", "us", "uz")), _p(v["y"]), m, n, k, 128,
                                                        _code(T), _p(v["ws"]), nb, _st())
        want = composed_front(x, gamma, G, U)
    else:
        W = layer(n, k, T)
        for name, t in zip(("q", "s", "z"), W):
            ops[name] = Op("in", t)
        b = bias_of(n, T) if op == "linear_bias" else None
        if b is not None:
            ops["bias"] = Op("in", b, offset=offset)

        def call(v):
            return P.lib().b200awq_w4a16_norm_linear(_p(v["x"]), _p(v["gamma"]), EPS, *(_p(v[s]) for s in ("q", "s", "z")),
                                                     _p(v.get("bias")), _p(v["y"]), m, n, k, 128, _code(T), _p(v["ws"]), nb,
                                                     _st())
        want = composed_linear(x, gamma, W, b)
    plain = guarded_call(call, ops)
    assert_bits(plain["y"], want, f"{case} offset {offset}")


# ------------------------------------------------------------------------------------------------ 6. Python mirrors
@pytest.mark.parametrize("tokens", [1, 3, 8, 40])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_python_mirrors(dtype, tokens):
    from llm_awq_b200.fused_mlp import QuantLlamaMLP
    T = DTYPE[dtype]
    H, I = 896, 4864

    def wq(K, N, seed, bias=False):
        m = P.WQLinear(4, 128, K, N, bias, DEV, dtype=T)
        m.qweight, m.scales, m.scaled_zeros = layer(N, K, T, seed)
        if bias:
            m.bias = bias_of(N, T)
        return m
    qkv, plain_proj = wq(H, 1152, 11, bias=True), wq(H, 1152, 12)
    mlp = QuantLlamaMLP(wq(H, I, 13), wq(I, H, 14), wq(H, I, 15))
    legacy = QuantLlamaMLP(wq(H, I, 13), wq(I, H, 14), wq(H, I, 15), legacy_gemm_zero_offset=True)
    gamma, _ = gammas(H, T)
    x = rows(tokens, H, T, 0, seed=tokens).view(1, tokens, H)
    xh = rmsnorm(x, gamma)
    for lin in (qkv, plain_proj):
        assert_bits(lin.norm_forward(x, (gamma, EPS)), lin(xh), f"WQLinear bias={lin.bias is not None}")
        assert_bits(lin.norm_forward(x, None), lin(x), "WQLinear norm=None")
    for mod in (mlp, legacy):
        assert_bits(mod(x, norm=(gamma, EPS)), mod(xh), f"QuantLlamaMLP legacy={mod.legacy_gemm_zero_offset}")
        assert_bits(mod(x, norm=None), mod.down_proj(mod.our_llama_mlp(x)), "QuantLlamaMLP norm=None")
        assert_bits(mod.our_llama_mlp(x, (gamma, EPS)), mod.our_llama_mlp(xh), "our_llama_mlp")
