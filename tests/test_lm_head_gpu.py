"""GPU checks of the LM head (b200awq_lm_head, lm_head_forward_cuda).

Oracle: every logit meets the elementwise bound of tests/lm_head_oracle.py.  Restated:
    |y - Y| <= ulp_T(|Y| + e) + e,   e = gamma_n A + n 2^-149 + k 2^-53 A,   n = 8 ceil(k / 256) + 5,
where Y and A = sum |x^ W| are float64.  n counts the fp32 roundings a product passes through in the kernel's order:
lane l owns chunks l, l + 32, ... of 8 elements, and each element is one fmaf, so a lane makes at most 8 ceil(k / 256)
roundings.  The xor butterfly over 32 lanes adds 5 more.  gamma_n A bounds the recursive sum (Higham §3.1).  n 2^-149
covers fp32 subnormal results.  k 2^-53 A is float64's own error in Y.  The last term, ulp_T, is twice the half ulp of
the final rounding to T.  Y, A and the check are computed on the GPU in float64 (torch), from the bits the kernel read:
x^ is b200awq_rmsnorm's output when the norm is on.

Beyond the bound: the prologue is bit-identical to b200awq_rmsnorm followed by the plain head.  A logit's bits do not
depend on its row's index, vocab, m or its neighbours.  The envelope covers vocab sizes, partition edges from the SM
count, strided x and guard bands.  The argmax and sample_next_token agree with F.linear wherever torch's margin is safe.
Each call is one launch of a named kernel.  Graphs and side streams give the same bits, with PDL on and off."""
import ctypes
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import llm_awq_b200 as P
import lm_head_oracle as O
from awq_testutil import gen_layer
from guard_bands import Op, guarded_call
from kernel_trace import trace

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16, BF16 = torch.float16, torch.bfloat16
DTYPE = {"f16": F16, "bf16": BF16}
EPS = 1e-6
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132

# (label, vocab, k): the heads of Llama-3-8B, Qwen2-7B, Qwen2.5-1.5B, Qwen2-0.5B and Falcon-7B, and the narrowest and
# widest k
HEADS = [("llama3_8b", 128256, 4096), ("qwen2_7b", 152064, 3584), ("qwen25_15b", 151936, 1536),
         ("qwen2_05b", 151936, 896), ("falcon_7b", 65024, 4544), ("k8", 5000, 8), ("k16", 5000, 16),
         ("k8192", 20000, 8192)]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st(stream=None):
    return ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def _code(T):
    return 0 if T == F16 else 1


def partition(vocab):
    """(rows per CTA, grid) of the kernel's plan: ceil(vocab / SMs) rows per CTA, as many CTAs as that needs."""
    rpc = -(-vocab // SMS)
    return rpc, -(-vocab // rpc)


@functools.lru_cache(maxsize=4)
def weight(vocab, k, T, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed + vocab + 7 * k)
    return (0.02 * torch.randn(vocab, k, generator=g, device=DEV)).to(T)


def hidden(m, k, T, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed + 31 * k + m)
    return (torch.randn(m, k, generator=g, device=DEV) * 2.0).to(T)


def gamma_of(k, T):
    g = torch.Generator(device=DEV).manual_seed(k)
    return (1.0 + 0.3 * torch.randn(k, generator=g, device=DEV)).to(T)


def head(x, W, gamma=None, eps=EPS, logits=None, stride=None, stream=None):
    """b200awq_lm_head on x [m, k] (row stride `stride`, default x.stride(0)) into logits (fresh NaN-filled if None)."""
    m, k = x.shape
    vocab = W.shape[0]
    logits = torch.full((m, vocab), float("nan"), device=DEV) if logits is None else logits
    s = x.stride(0) if stride is None else stride
    rc = P.lib().b200awq_lm_head(_p(x), s, _p(gamma), eps, _p(W), _p(logits), m, vocab, k, _code(x.dtype), _st(stream))
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return logits


def rmsnorm(x, gamma, eps=EPS):
    out = torch.full_like(x, float("nan"))
    P.engine().layernorm_forward_cuda(x.contiguous(), gamma, out, eps)
    return out


def check_oracle(got, xhat, W):
    """Asserts the bound of the module docstring for every logit."""
    x64, w64 = xhat.double(), W.double()
    Y = (x64 @ w64.T).cpu().numpy()
    A = (x64.abs() @ w64.abs().T).cpu().numpy()
    bad = O.violations_of(got.cpu().numpy(), Y, A, W.shape[1], xhat.dtype == BF16)
    if bad.any():
        i, v = np.argwhere(bad)[0]
        pytest.fail(f"{bad.sum()} of {bad.size} logits out of bound; first [{i}, {v}]: {got[i, v].item()!r} against "
                    f"{Y[i, v]!r} (A = {A[i, v]!r})")


def assert_bits(got, want, what):
    a, b = got.view(torch.int32), want.view(torch.int32)
    if not torch.equal(a, b):
        bad = (a != b).nonzero()
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {len(bad)} of {a.numel()} logits differ; first at {i}: {got[i].item()!r} against {want[i].item()!r}")


# ------------------------------------------------------------------------------------------------ 1. oracle
@pytest.mark.parametrize("norm", [False, True], ids=["plain", "norm"])
@pytest.mark.parametrize("m", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("shape", HEADS, ids=lambda s: s[0])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_oracle(dtype, shape, m, norm):
    _, vocab, k = shape
    T = DTYPE[dtype]
    W, x = weight(vocab, k, T), hidden(m, k, T)
    gamma = gamma_of(k, T) if norm else None
    got = head(x, W, gamma)
    check_oracle(got, rmsnorm(x, gamma) if norm else x, W)


# ------------------------------------------------------------------------------------------------ 2. prologue bits
LANDSCAPES = ("random", "zeros", "huge_one", "inf_nan", "tiny", "constant")


def rows(m, k, T, shift=0):
    g = torch.Generator().manual_seed(m + k)
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


@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("m", [6, 8])
@pytest.mark.parametrize("shape", [HEADS[0], HEADS[3], HEADS[5], HEADS[7]], ids=lambda s: s[0])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_prologue_bit_identical_to_rmsnorm_then_head(dtype, shape, m, shift):
    _, vocab, k = shape
    T = DTYPE[dtype]
    W, x = weight(vocab, k, T), rows(m, k, T, shift)
    gamma = gamma_of(k, T)
    if T == F16:  # elements at 65000 x gamma send x^ of the constant and huge rows into the fp16 clamp
        gamma = gamma.clone()
        gamma[::61] = 65000.0
    assert_bits(head(x, W, gamma), head(rmsnorm(x, gamma), W), "norm prologue")


# ------------------------------------------------------------------------------------------------ 3. order invariance
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_row_index_vocab_and_m_do_not_change_bits(dtype):
    T = DTYPE[dtype]
    vocab, k = 65024, 4544
    W, x = weight(vocab, k, T), hidden(8, k, T, seed=5)
    full = head(x, W)
    rpc, _ = partition(vocab)
    # views whose first row moves every row across CTA-block edges of the view's own partition
    for r0 in (1, rpc - 1, rpc, rpc + 1, 3 * rpc + 5, vocab // 2):
        for r1 in (vocab, vocab - 1, r0 + 1, r0 + 2 * rpc + 3):
            r1 = min(r1, vocab)
            assert_bits(head(x, W[r0:r1]), full[:, r0:r1], f"weight[{r0}:{r1}]")
    for m in (1, 2, 5, 7):
        for first in (0, 8 - m):
            assert_bits(head(x[first:first + m], W), full[first:first + m], f"m = {m} from row {first}")


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_neighbours_do_not_change_bits(dtype):
    T = DTYPE[dtype]
    vocab, k = 4099, 896
    W, x = weight(vocab, k, T).clone(), hidden(3, k, T, seed=9)
    want = head(x, W)
    probe = list(range(1, vocab, 97))
    for fill in (65504.0, -65504.0, float("inf"), -float("inf"), float("nan"), None):
        V = W.clone()
        for v in probe:
            for nb in (v - 1, v + 1):
                if nb < vocab and nb not in probe:
                    if fill is None:
                        V[nb] = torch.randn(k, device=DEV).to(T) * 100
                    else:
                        V[nb] = fill
        got = head(x, V)
        assert_bits(got[:, probe], want[:, probe], f"neighbours {fill}")


# ------------------------------------------------------------------------------------------------ 4. envelope
def edge_vocabs():
    """One row short of, at and one row past the vocab sizes where the plan's rows per CTA changes, for a few
    multiples of the SM count, and vocab sizes below the SM count."""
    out = set()
    for j in (1, 2, 3, 8, 64):
        for d in (-1, 0, 1):
            out.add(j * SMS + d)
    return sorted(out | {SMS // 2, SMS - 3})


VOCABS = [1, 2, 7, 8, 9, 31, 32000, 65024, 128256, 151936, 152064, 262144]


@pytest.mark.parametrize("vocab", VOCABS + edge_vocabs())
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_vocab_sizes(dtype, vocab):
    T = DTYPE[dtype]
    k = 1536 if vocab > 100000 else 896
    W, x = weight(vocab, k, T), hidden(2, k, T)
    gamma = gamma_of(k, T)
    got = head(x, W, gamma)
    assert not torch.isnan(got).any()
    check_oracle(got, rmsnorm(x, gamma), W)


@pytest.mark.parametrize("norm", [False, True], ids=["plain", "norm"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_strided_rows(dtype, norm):
    T = DTYPE[dtype]
    vocab, k = 32000, 4096
    W = weight(vocab, k, T)
    gamma = gamma_of(k, T) if norm else None
    h = hidden(10, k, T).view(2, 5, k)
    want = head(h[:, -1, :].contiguous(), W, gamma)
    assert_bits(P.engine().lm_head_forward_cuda(h[:, -1, :], W, gamma, EPS), want, "h[:, -1, :]")
    for pad in (8, 64, 4096):
        xp = torch.full((3, k + pad), float("nan"), dtype=T, device=DEV)
        xp[:, :k] = hidden(3, k, T)
        assert_bits(head(xp[:, :k], W, gamma), head(xp[:, :k].contiguous(), W, gamma), f"pad {pad}")


@pytest.mark.parametrize("case", [(1, 7, 8, "f16", False), (3, 1000, 896, "bf16", True), (8, 3 * 132 + 1, 4096, "f16", True),
                                  (2, 65024, 4544, "bf16", False)], ids=str)
def test_guard_bands(case):
    m, vocab, k, dt, norm = case
    T = DTYPE[dt]
    ops = {"x": Op("in", hidden(m, k, T)), "w": Op("in", weight(vocab, k, T)), "y": Op("out", shape=(m, vocab), dtype=torch.float32)}
    if norm:
        ops["g"] = Op("in", gamma_of(k, T))

    def call(v):
        return P.lib().b200awq_lm_head(_p(v["x"]), k, _p(v.get("g")), EPS, _p(v["w"]), _p(v["y"]), m, vocab, k,
                                       _code(T), _st())
    plain = guarded_call(call, ops)
    assert not torch.isnan(plain["y"]).any()


def test_overflow_and_nan_rows():
    k, vocab = 1024, 300
    W = torch.full((vocab, k), 1.0, dtype=F16, device=DEV)
    W[1] = -1.0
    W[2, :] = 0.0
    x = torch.full((3, k), 100.0, dtype=F16, device=DEV)   # 102400 > fp16's max
    x[2, 5] = float("nan")
    got = head(x, W)
    assert got[0, 0].item() == float("inf") and got[0, 1].item() == -float("inf") and got[0, 2].item() == 0.0
    assert torch.isnan(got[2]).all()


# ------------------------------------------------------------------------------------------------ 5. the current tail
@pytest.mark.parametrize("shape", [HEADS[0], HEADS[1], HEADS[3]], ids=lambda s: s[0])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_argmax_and_token_match_the_torch_tail(dtype, shape):
    _, vocab, k = shape
    T = DTYPE[dtype]
    W, x, gamma = weight(vocab, k, T), hidden(8, k, T, seed=2), gamma_of(k, T)
    xhat = rmsnorm(x, gamma)
    ref = F.linear(xhat, W).float()
    got = P.engine().lm_head_forward_cuda(x, W, gamma, EPS)
    top2 = ref.topk(2, dim=1).values
    Y, A = (xhat.double() @ W.double().T).cpu().numpy(), (xhat.double().abs() @ W.double().abs().T).cpu().numpy()
    b = torch.from_numpy(O.bound(Y, A, k, T == BF16).max(axis=1)).to(DEV)
    safe = (top2[:, 0] - top2[:, 1]).double() > 2 * b
    assert safe.sum() >= 2, safe
    assert torch.equal(got.argmax(1)[safe], ref.argmax(1)[safe])
    tok = P.engine().sample_next_token(got, None, 1.0, 1.0, 1.0, 0, True)
    assert torch.equal(tok[safe], ref.argmax(1)[safe])


# ------------------------------------------------------------------------------------------------ 6. launches
def traced_call(m, vocab, k, dt, norm):
    """kernel_trace builder: one head call."""
    T = DTYPE[dt]
    x, W = torch.zeros(m, k, dtype=T, device=DEV), torch.zeros(vocab, k, dtype=T, device=DEV)
    g = torch.ones(k, dtype=T, device=DEV) if norm else None
    y = torch.empty(m, vocab, device=DEV)
    st = _st()
    return lambda: P.lib().b200awq_lm_head(_p(x), k, _p(g), EPS, _p(W), _p(y), m, vocab, k, _code(T), st)


TRACE_CASES = [(m, vocab, k, dt, norm) for (m, vocab, k) in [(1, 128256, 4096), (8, 151936, 896), (3, 7, 8)]
               for dt in ("f16", "bf16") for norm in (False, True)]


def test_one_named_launch_per_call():
    records = trace("test_lm_head_gpu:traced_call", TRACE_CASES, per_process=len(TRACE_CASES))
    for (m, vocab, k, dt, norm), rec in zip(TRACE_CASES, records):
        assert rec.launches == 1, rec
        kernels = [e for e in rec.events if e.cat == "kernel"]
        assert len(kernels) == 1, rec.names
        name = kernels[0].name
        want = "lm_head_norm_kernel" if norm else "lm_head_kernel"
        tname = "__half" if dt == "f16" else "__nv_bfloat16"
        assert f"{want}<{tname}, {m}>" in name, name
        assert kernels[0].grid is None or kernels[0].grid[0] == partition(vocab)[1], kernels[0]
    x, W = hidden(2, 64, F16), weight(100, 64, F16)
    c0 = P.engine().launch_count()
    P.engine().lm_head_forward_cuda(x, W, gamma_of(64, F16), EPS)
    P.engine().lm_head_forward_cuda(x, W)
    assert P.engine().launch_count() - c0 == 2
    assert P.engine().lm_head_forward_cuda(x[:0], W).shape == (0, 100)
    assert P.engine().launch_count() - c0 == 2


# ------------------------------------------------------------------------------------------------ 7. graphs and streams
def _chain(T, pdl_tag):
    """The decoder's last down projection + residual, then the normed head, then greedy sampling, as three entries."""
    k_in, k, vocab, m = 14336, 4096, 128256, 2
    qw, sc, sz = gen_layer(k, k_in, T, seed=11, device=DEV)
    act = hidden(m, k_in, T, seed=3) * 0.05
    resid = hidden(m, k, T, seed=4)
    W, gamma = weight(vocab, k, T), gamma_of(k, T)
    h = torch.empty(m, k, dtype=T, device=DEV)
    logits = torch.empty(m, vocab, device=DEV)
    tokens = torch.empty(m, dtype=torch.int64, device=DEV)

    def step():
        rc = P.lib().b200awq_w4a16_linear(_p(act), _p(qw), _p(sc), _p(sz), None, _p(resid), _p(h), m, k, k_in, 128,
                                          _code(T), _st())
        assert rc == 0
        head(h, W, gamma, logits=logits)
        rc = P.lib().b200awq_sample_next_token(_p(logits), vocab, m, vocab, None, 0, 0, 1.0, 1.0, 1.0, 0, 1, None,
                                               _p(tokens), _st())
        assert rc == 0
    return step, h, logits, tokens


@pytest.mark.parametrize("pdl", [True, False], ids=["pdl", "nopdl"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_graph_chain_bit_identical(dtype, pdl):
    T = DTYPE[dtype]
    old = P.engine().set_pdl(pdl)
    try:
        step, h, logits, tokens = _chain(T, pdl)
        step()
        torch.cuda.synchronize()
        want_h, want_l, want_t = h.clone(), logits.clone(), tokens.clone()
        check_oracle(logits, rmsnorm(h, gamma_of(h.shape[1], T)), weight(logits.shape[1], h.shape[1], T))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
            g = torch.cuda.CUDAGraph()
            for t in (h, logits, tokens):
                t.fill_(0)
            with torch.cuda.graph(g, stream=s):
                step()
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(3):
            for t in (h, logits, tokens):
                t.fill_(-1)
            g.replay()
            torch.cuda.synchronize()
            assert_bits(logits, want_l, "graph replay")
            assert torch.equal(h, want_h) and torch.equal(tokens, want_t)
    finally:
        P.engine().set_pdl(old)


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_side_stream(dtype):
    T = DTYPE[dtype]
    vocab, k = 151936, 1536
    W, x, gamma = weight(vocab, k, T), hidden(4, k, T), gamma_of(k, T)
    want = head(x, W, gamma)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x2 = x * 1  # written on the side stream right before the head reads it
        got = P.engine().lm_head_forward_cuda(x2, W, gamma, EPS)
    s.synchronize()
    assert_bits(got, want, "side stream")
