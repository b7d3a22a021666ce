"""The W8A8 vision-tower ops across their whole envelope, every output against its admissible set
(oracle/w8a8_oracle.py *_bounds): every width where the row kernels' thread count or chunks per thread change, on the
16-byte and the one-element path, up to 32768; more than 65535 rows; rows whose maximum sits on the edges of each
thread's last chunk; zero, single-element, constant, cancelling, inf / NaN and overflowing rows; every LayerNorm mode;
exact known answers for the code rounding; silu_and_mul through its tail and grid-stride paths; and the GEMM at every
tile residue, bit-exact with and without bias.  Every call goes through the C ABI into poisoned outputs.

Run with -s to see the share of elements that had two admissible codes (lines starting TWO-CODE)."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import w8a8_cases as W
from oracle import w8a8_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TT = {"f16": torch.float16, "bf16": torch.bfloat16}
CODE = {"f16": 0, "bf16": 1}
POISON_Q = 77
ONE_ELEMENT = list(range(1, 32))
# (n, byte offset of every pointer): the 16-byte path's thread-count and chunk changes, then the one-element path's
WIDTHS = [(8, 0), (16, 0), (24, 0), (256, 0), (264, 0), (3200, 0), (8192, 0), (8200, 0), (12800, 0), (16384, 0),
          (16392, 0), (24576, 0), (24584, 0), (32760, 0), (32768, 0),
          (1023, 0), (2049, 0), (4097, 0), (8191, 0), (8192, 2)]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _report(op, tag, b):
    print(f"TWO-CODE {op} {tag}: {O.two_code_share(b):.3e} of {b['lo'].size} elements")


def dev_buf(shape, dtype, off, fill):
    """A device tensor of `shape` whose data starts `off` bytes past a 256-byte boundary, filled with `fill`."""
    n = int(np.prod(shape))
    es = torch.empty((), dtype=dtype).element_size()
    base = torch.full((n + 256 // es,), fill, dtype=dtype, device=DEV)
    return base[off // es:off // es + n].view(shape)


def to_dev(x, dtype, off=0):
    t = dev_buf(x.shape, dtype, off, 0)
    t.copy_(torch.as_tensor(x).to(dtype))
    return t


def thread_edges(n, vec):
    """Columns of the first and last element of every thread's last chunk."""
    nc = n // vec
    thr = O.row_threads(nc)
    last = [max(ci for ci in range(t, nc, thr)) for t in range(min(thr, nc))]
    return np.unique(np.array([c * vec for c in last] + [c * vec + vec - 1 for c in last]))


def rows_for(n, vec, tag, seed, gelu=False):
    """T values as float32 [M, n]: a spread row, zeros, one non-zero element, the maximum on the last / first of the
    thread-edge columns, a large mean with a tiny spread, a constant row, and inf / NaN elements."""
    rng = np.random.default_rng(seed)
    sd = 2.0 if gelu else 1.0
    rows = [rng.standard_normal(n) * sd * np.exp(rng.standard_normal()), np.zeros(n)]
    one = np.zeros(n)
    one[rng.integers(n)] = -3.0
    rows.append(one)
    e = thread_edges(n, vec)
    for order in (1, -1):
        r = rng.standard_normal(n) * 0.5
        r[e] = 4.0 + 0.25 * np.arange(len(e))[::order] / max(len(e), 1)
        rows.append(r)
    if not gelu:
        rows += [100.0 + 0.1 * rng.standard_normal(n), np.full(n, 100.0)]
    special = rng.standard_normal(n)
    special[rng.integers(n)] = np.nan
    if not gelu:
        special[rng.integers(n)] = np.inf
        special[rng.integers(n)] = -np.inf
    rows.append(special)
    if gelu:  # gelu amax below ~0.0019 (127 / amax overflows fp16), and values in (0, 1e-4]
        rows += [rng.random(n) * 3e-3, rng.random(n) * 2e-4]
    elif tag == "bf16":  # amax above 2^126 (127 / amax is 0), and an fp16 scale that overflows
        big = rng.standard_normal(n) * 1e37
        big[rng.integers(n)] = 2.0 ** 127
        rows += [big, rng.standard_normal(n) * 3e6]
    return O.round_t(np.stack(rows).astype(np.float32), tag)


# ------------------------------------------------------------------------------------------------ quant_per_token
def run_quant(x, tag, off=0):
    M, n = x.shape
    xd = to_dev(x, TT[tag], off)
    q = dev_buf((M, n), torch.int8, off, POISON_Q)
    s = dev_buf((M,), torch.float16, off, float("nan"))
    assert P.lib().b200awq_quant_per_token(_p(xd), _p(q), _p(s), M, n, CODE[tag], _st()) == 0
    torch.cuda.synchronize()
    return q.cpu().numpy(), s.cpu().numpy()


def check_quant(x, tag, off=0):
    q, s = run_quant(x, tag, off)
    b = O.quant_per_token_bounds(x)
    O.assert_admissible(q, s, b, f"quant {tag} n={x.shape[1]} off={off}")
    return b


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("n,off", WIDTHS)
def test_quant_per_token_widths(tag, n, off):
    vec = O.row_vec(n, off == 0)
    _report(f"quant n={n}", tag, check_quant(rows_for(n, vec, tag, seed=n), tag, off))


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_quant_per_token_narrow_rows(tag):
    for n in ONE_ELEMENT:
        check_quant(rows_for(n, 1, tag, seed=n), tag)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("n", [8, 5])
def test_quant_per_token_70000_rows(tag, n):
    rng = np.random.default_rng(n)
    x = O.round_t((rng.standard_normal((70000, n)) * np.exp(rng.standard_normal((70000, 1)))).astype(np.float32), tag)
    _report(f"quant 70000x{n}", tag, check_quant(x, tag))


# ------------------------------------------------------------------------------------------------ layernorm_quant
LN_MODES = [("beta", 1e-6, None), ("nobeta", 1e-5, None), ("tensor", 1e-6, 30.0), ("tensor", 1e-5, 0.5),
            ("tensor", 1e-6, 1024.0)]


def run_ln(x, gamma, beta, tag, mode, eps, scale, off=0):
    M, n = x.shape
    xd, gd = to_dev(x, TT[tag], off), to_dev(gamma, TT[tag], off)
    bd = to_dev(beta, TT[tag], off) if mode == "beta" else None
    q = dev_buf((M, n), torch.int8, off, POISON_Q)
    if mode == "tensor":
        s = dev_buf((1,), torch.float16, off, scale)
    else:
        s = dev_buf((M,), torch.float16, off, float("nan"))
    rc = P.lib().b200awq_layernorm_quant(_p(xd), _p(gd), _p(bd), _p(q), _p(s), M, n, ctypes.c_float(eps),
                                         int(mode != "tensor"), CODE[tag], _st())
    assert rc == 0
    torch.cuda.synchronize()
    return q.cpu().numpy(), (None if mode == "tensor" else s.cpu().numpy())


def check_ln(x, tag, mode, eps, scale, off=0, seed=0):
    n = x.shape[1]
    rng = np.random.default_rng(seed)
    gamma = O.round_t((1 + 0.2 * rng.standard_normal(n)).astype(np.float32), tag)
    beta = O.round_t((0.1 * rng.standard_normal(n)).astype(np.float32), tag)
    q, s = run_ln(x, gamma, beta, tag, mode, eps, scale, off)
    b = O.layernorm_quant_bounds(x, gamma, beta if mode == "beta" else None, eps, tag, per_token=mode != "tensor",
                                 scale=None if scale is None else np.array([scale], np.float16),
                                 vec=O.row_vec(n, off == 0))
    O.assert_admissible(q, s, b, f"layernorm {mode} {tag} n={n} off={off}")
    return b


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("mode,eps,scale", LN_MODES, ids=[f"{m}-{e}-{s}" for m, e, s in LN_MODES])
@pytest.mark.parametrize("n,off", WIDTHS)
def test_layernorm_quant_widths(tag, mode, eps, scale, n, off):
    b = check_ln(rows_for(n, O.row_vec(n, off == 0), tag, seed=n + 1), tag, mode, eps, scale, off, seed=n)
    _report(f"layernorm-{mode} n={n}", tag, b)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("mode,eps,scale", LN_MODES[:3], ids=["beta", "nobeta", "tensor"])
def test_layernorm_quant_narrow_rows(tag, mode, eps, scale):
    for n in ONE_ELEMENT:
        check_ln(rows_for(n, 1, tag, seed=n + 1), tag, mode, eps, scale, seed=n)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("n", [8, 5])
def test_layernorm_quant_70000_rows(tag, n):
    rng = np.random.default_rng(n)
    x = O.round_t((rng.standard_normal((70000, n)) * 3 + rng.standard_normal((70000, 1))).astype(np.float32), tag)
    _report(f"layernorm-beta 70000x{n}", tag, check_ln(x, tag, "beta", 1e-6, None, seed=n))


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("n,off", [(64, 0), (1152, 0), (9, 0), (1152, 2)])
def test_layernorm_quant_known_rounding(tag, n, off):
    """x alternates +1 / -1, so every partial sum is an exact integer, mean = 0 and rn_T(y) = x * gamma whatever
    rstd's error; with scale[0] = 0.5 the code is cvt(x gamma / 2), an exact product on k + 0.5 or past the int8 range:
    round-half-even and saturation pinned exactly."""
    n -= n % 2
    x = np.where(np.arange(n) % 2 == 0, 1.0, -1.0).astype(np.float32)[None, :].repeat(2, axis=0)
    targets = [127.5, -127.5, 126.5, -126.5, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 200.0, -200.0, 129.0, -129.0, 127.0, -128.0]
    want_codes = [127, -128, 126, -126, 0, 0, 2, -2, 2, -2, 127, -128, 127, -128, 127, -128]
    if tag == "f16":
        targets += [128.5, -128.5, 3.5, -3.5]
        want_codes += [127, -128, 4, -4]
    k = np.arange(n) % len(targets)
    gamma = (2 * np.array(targets, np.float32)[k] * x[0]).astype(np.float32)
    assert (O.round_t(gamma, tag) == gamma).all()
    xd, gd = to_dev(x, TT[tag], off), to_dev(gamma, TT[tag], off)
    q = dev_buf((2, n), torch.int8, off, POISON_Q)
    s = dev_buf((1,), torch.float16, off, 0.5)
    assert P.lib().b200awq_layernorm_quant(_p(xd), _p(gd), None, _p(q), _p(s), 2, n, ctypes.c_float(1e-6), 0,
                                           CODE[tag], _st()) == 0
    torch.cuda.synchronize()
    np.testing.assert_array_equal(q.cpu().numpy(), np.array(want_codes, np.int8)[k][None, :].repeat(2, axis=0))
    b = O.layernorm_quant_bounds(x, gamma, None, 1e-6, tag, per_token=False, scale=np.array([0.5], np.float16),
                                 vec=O.row_vec(n, off == 0))
    assert (b["lo"] == b["hi"]).all() and (b["lo"] == q.cpu().numpy()).all()


# ------------------------------------------------------------------------------------------------ gelu_quant
def check_gelu(x, off=0):
    M, n = x.shape
    xd = to_dev(x, torch.float16, off)
    q = dev_buf((M, n), torch.int8, off, POISON_Q)
    s = dev_buf((M,), torch.float16, off, float("nan"))
    tmp = dev_buf((M, n), torch.float16, off, float("nan"))
    assert P.lib().b200awq_gelu_quant(_p(xd), _p(q), _p(s), _p(tmp), M, n, _st()) == 0
    torch.cuda.synchronize()
    b = O.gelu_quant_bounds(x.astype(np.float16))
    O.assert_between(tmp.cpu().numpy(), b["g_lo"], b["g_hi"], f"gelu n={n} off={off}")
    O.assert_admissible(q.cpu().numpy(), s.cpu().numpy(), b, f"gelu_quant n={n} off={off}")
    return b


@pytest.mark.parametrize("n,off", WIDTHS)
def test_gelu_quant_widths(n, off):
    b = check_gelu(rows_for(n, O.row_vec(n, off == 0), "f16", seed=n + 2, gelu=True), off)
    _report(f"gelu n={n}", "f16", b)


def test_gelu_quant_narrow_rows():
    for n in ONE_ELEMENT:
        check_gelu(rows_for(n, 1, "f16", seed=n + 2, gelu=True))


@pytest.mark.parametrize("n", [8, 5])
def test_gelu_quant_70000_rows(n):
    rng = np.random.default_rng(n)
    _report(f"gelu 70000x{n}", "f16", check_gelu(O.round_t((rng.standard_normal((70000, n)) * 2).astype(np.float32), "f16")))


def test_row_ops_refuse_rows_past_their_kernel():
    """n = 32769 on any pointers and n = 8193 on the one-element kernel are refused before anything is launched."""
    L = P.lib()
    buf = torch.zeros(4 * 32776 + 256, dtype=torch.float16, device=DEV)
    q = torch.zeros(2 * 32776 + 256, dtype=torch.int8, device=DEV)
    base, qb = buf.data_ptr(), q.data_ptr()
    for n, off in ((32769, 0), (32776, 0), (8193, 0), (8200, 2)):
        x, qq, s = ctypes.c_void_p(base + off), ctypes.c_void_p(qb + off), ctypes.c_void_p(base + 2 * 32776 * 2)
        assert L.b200awq_quant_per_token(x, qq, s, 1, n, 0, _st()) == -1
        assert L.b200awq_layernorm_quant(x, x, None, qq, s, 1, n, ctypes.c_float(1e-6), 1, 0, _st()) == -1
        assert L.b200awq_gelu_quant(x, qq, s, x, 1, n, _st()) == -1
    torch.cuda.synchronize()
    assert int(q.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------ silu_and_mul
def silu_rows(m, d, tag, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((m, 2 * d)) * 3
    x[:, rng.integers(d, size=4)] = [-100.0, 100.0, -20.0, 1e-30]   # exp overflow, saturation, a flushed-looking gate
    return O.round_t(x.astype(np.float32), tag)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,d,off", [(1, 4104, 0), (1, 4100, 0), (1, 4096, 2), (1, 13, 0), (7, 1001, 0), (5, 1024, 0),
                                     (300, 8192, 0), (3, 100001, 0)])
def test_silu_and_mul(tag, m, d, off):
    """One row on the 16-byte path, with its up half misaligned, and at a 2-byte offset; rows with cols % 8 != 0; more
    vectors (300 x 8192 / 8) and more elements (3 x 100001) than one pass of the grid covers on an H100."""
    x = silu_rows(m, d, tag, seed=m * d)
    xd = to_dev(x, TT[tag], off)
    y = dev_buf((m, d), TT[tag], off, float("nan"))
    assert P.lib().b200awq_silu_and_mul(_p(xd), _p(y), m, d, CODE[tag], _st()) == 0
    torch.cuda.synchronize()
    lo, hi = O.silu_and_mul_bounds(x, tag)
    O.assert_between(y.float().cpu().numpy(), lo, hi, f"silu_and_mul {tag} {m}x{d} off={off}")
    print(f"TWO-VALUE silu_and_mul {tag} {m}x{d}: {float(np.mean(lo != hi)):.3e}")


# ------------------------------------------------------------------------------------------------ GEMM
def check_gemm(M, N, K, rows=None):
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    rows = np.arange(M) if rows is None else rows
    ridx = torch.from_numpy(rows).to(DEV)
    acc = (x.index_select(0, ridx).double() @ w.double().T).cpu().numpy()   # exact: |acc| < 2^53
    for bias in (None, b):
        y = torch.full((M, N), float("nan"), dtype=torch.float16, device=DEV)
        assert P.lib().b200awq_w8a8_gemm(_p(x), _p(w), _p(ws), _p(a), _p(bias), _p(y), M, N, K, _st()) == 0
        torch.cuda.synchronize()
        want = O.gemm_exact(acc, ws.cpu().numpy(), a.cpu().numpy()[rows], None if bias is None else bias.cpu().numpy())
        got = y.index_select(0, ridx).cpu().numpy()
        bad = np.flatnonzero((got.view(np.uint16) != want.view(np.uint16)).any(axis=1))
        assert bad.size == 0, (M, N, K, bias is not None, rows[bad[:4]].tolist())


@pytest.mark.parametrize("N", list(range(8, 129, 8)) + [136, 264, 392, 1160])
def test_gemm_n_residues(N):
    check_gemm(129, N, 144)


@pytest.mark.parametrize("K", list(range(16, 385, 16)) + [752, 768, 784])
def test_gemm_k_residues(K):
    check_gemm(65, 136, K)


@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 257])
def test_gemm_m_residues(M):
    check_gemm(M, 264, 784)


@pytest.mark.parametrize("M,N,K", [(64 * 729, 1152, 4304), (64 * 1025, 1024, 4096)], ids=["siglip", "internvit"])
def test_gemm_tinychat_batch(M, N, K):
    """tinychat's default batch of 64 images through the out-projection / fc2 shapes, on sampled rows."""
    check_gemm(M, N, K, rows=W.sample_rows(M))
