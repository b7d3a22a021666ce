"""W4A16 routes under AWQ-like activations: every output element depends on its own token only, and is within an
elementwise bound of the float64 oracle.

Probe tokens look like the activations AWQ is built for: N(0, 1) with about 1 % fixed outlier channels scaled by 100
to 3000, one 128-k group of values near +40 (a non-zero mean: the fp16 ring and stream kernels subtract the staged
per-group sums C = 1024 X_lo + 64 X_hi from a 1024-biased accumulator, and this is where that cancellation is
largest), one all-zero group, one group of fp16 subnormals, a -0.0 and one element at +-60000.  Neighbour tokens are
extreme: +-65504, zero, subnormal, +-inf and NaN, group by group.

Isolation: at a fixed token count a probe token's output is bit-identical whether its neighbours are extreme or
ordinary randn tokens.  Every route computes an output element from its own token only: tokens are independent MMA
columns, and split-k partials are reduced in a fixed order.

Accuracy, element by element (`bound_violations`): |y - Y| <= ulp_T(Y) + gamma A + delta, where Y = x . w~^T is the
oracle in float64 with w~ = rn_T(q s + z), A = |x| . |w~|^T, and
  * ulp_T(Y) covers the one rounding of the result to T (half an ulp, doubled for the fp32 sum's last bits);
  * gamma = 2^-11 on the routes that apply scale and zero unrounded (fp16 decode, ring and stream kernels): their
    weight is q s + z in fp32 instead of rn_f16(q s + z), off by at most half an fp16 ulp, 2^-11 |w~|, per product;
  * gamma = 2^-14 on the operand-exact routes (wgmma, and bf16 everywhere): the products are exact and only the fp32
    accumulation rounds.  Its error is n u A in the worst case, but it grows like sqrt(K) u for the random signs
    here: sqrt(14336) 2^-24 ~ 2^-17, so 2^-14 keeps a margin of 8;
  * delta = 2^-21 sum_g max_g |x| sum_{k in g} |w~| on the fp16 decode kernel only: it splits each 128-k group of the
    activations into three 7-bit digits of a block-fixed-point number exact to 2^-21 of the group's largest magnitude
    (DESIGN.md 3.1).  Zero on every other route.
Where the oracle's value rounded to T overflows, the output must be an infinity of the same sign.

The profiler test (tests/kernel_trace.py) pins the kernel each case runs, so a change of the dispatch cannot quietly
move a case to another route.  The bound itself is tested on the CPU: the oracle rounded to T passes, and an output
missing one group's contribution in a single element, or using the neighbouring channel's scale in a single element,
fails."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from kernel_trace import short_names, trace
from oracle import w4a16_oracle as O
from w4a16_plans import plan

DEV = "cuda:0"
F16, BF16 = torch.float16, torch.bfloat16
TAG = {F16: "f16", BF16: "bf16"}

# (route, M, N, K, dtype, entry): every W4A16 route of api.cu, fp16 and bf16 where the route exists
CASES = [
    ("decode", 1, 1032, 4224, F16, "gemv"),
    ("decode", 1, 2056, 14336, F16, "gemv"),         # k split over a 2-CTA cluster
    ("ring", 1, 1032, 4224, BF16, "gemv"),           # bf16 single token
    ("ring", 2, 1032, 4224, F16, "gemv"),
    ("ring", 3, 1032, 4224, BF16, "gemv"),
    ("ring", 4, 264, 11008, F16, "gemv"),
    ("ring", 4, 264, 11008, BF16, "gemv"),
    ("skinny", 5, 384, 3584, F16, "gemv"),           # k split 7
    ("skinny", 7, 384, 3584, BF16, "gemv"),
    ("skinny", 12, 1024, 2048, F16, "gemm"),
    ("skinny", 16, 256, 3584, BF16, "gemm"),
    ("stream", 6, 1032, 2048, F16, "gemv"),
    ("stream", 6, 1032, 2048, BF16, "gemv"),
    ("stream", 7, 24, 4224, F16, "gemv"),
    ("tile_9_16", 13, 4096, 14336, F16, "gemm"),     # n k >= 48 M: the tile launch, not the skinny one
    ("tile_9_16", 13, 4096, 14336, BF16, "gemm"),
    ("wgmma", 17, 384, 4096, F16, "gemm"),
    ("wgmma", 40, 1024, 2048, BF16, "gemm"),
    ("wgmma", 100, 512, 4096, F16, "gemm"),
    ("wgmma", 300, 1024, 1024, BF16, "gemm"),
]


def case_id(c):
    return f"{c[0]}-M{c[1]}-N{c[2]}-K{c[3]}-{TAG[c[4]]}"


def gamma(route, dtype):
    return 2.0 ** -11 if dtype == F16 and route in ("decode", "ring", "stream") else 2.0 ** -14


# ------------------------------------------------------------------------------------------------ inputs
def probe_tokens(n, K, seed):
    """n AWQ-like activation rows (float32; see the module docstring)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, K, generator=g)
    outl = torch.randperm(K, generator=g)[: max(1, K // 100)]
    x[:, outl] *= 100 + 2900 * torch.rand(len(outl), generator=g)
    x[:, 128:256] = 40 + 0.5 * torch.randn(n, 128, generator=g)                         # non-zero mean
    x[:, 256:384] = 0.0                                                                  # all zero
    x[:, 384:512] = torch.randint(-1023, 1024, (n, 128), generator=g).float() * 2.0 ** -24   # fp16 subnormals
    x[:, 5] = -0.0
    x[:, K - 1] = 60000.0 * (1 - 2 * (torch.arange(n) % 2))
    return x


EXTREMES = [65504.0, -65504.0, 0.0, 3 * 2.0 ** -24, float("inf"), float("-inf"), float("nan")]


def extreme_tokens(n, K):
    """Group by group one of EXTREMES, cycling, shifted per row."""
    grp = torch.arange(K) // 128
    rows = [torch.tensor(EXTREMES)[(grp + r) % len(EXTREMES)] for r in range(n)]
    return torch.stack(rows)


def probe_rows(M):
    return sorted({i for i in range(M) if i % 3 == 0} | ({M - 1} if M >= 4 else set()))


def batches(M, K, dtype, seed):
    """(x with extreme neighbours, x with randn neighbours, probe row indices)."""
    pr = probe_rows(M)
    nb = [i for i in range(M) if i not in pr]
    probes = probe_tokens(len(pr), K, seed)
    g = torch.Generator().manual_seed(seed + 1)
    x_ord = torch.randn(M, K, generator=g)
    x_ord[pr] = probes
    x_ext = x_ord.clone()
    if nb:
        x_ext[nb] = extreme_tokens(len(nb), K)
    return x_ext.to(dtype), x_ord.to(dtype), pr


# ------------------------------------------------------------------------------------------------ oracle and bound
def oracle_terms(x, qw, s, z, dtype, cols=None, chunk=512):
    """(Y, A, D) in float64 over the output channels `cols` (all by default): Y = x w~^T, A = |x| |w~|^T,
    D = sum_g max_g |x| sum_{k in g} |w~|.  w~ is dequantised for the packed rows (4 channels each) that hold `cols`,
    `chunk` channels at a time."""
    x = x.detach().cpu().double().numpy()
    qw, s, z = qw.cpu().numpy(), s.cpu().double().numpy(), z.cpu().double().numpy()
    M, K = x.shape
    cols = np.arange(s.shape[1]) if cols is None else np.asarray(cols)
    ax = np.abs(x)
    mx = ax.reshape(M, K // 128, 128).max(axis=2)
    Y, A, D = (np.zeros((M, len(cols))) for _ in range(3))
    for c0 in range(0, len(cols), chunk):
        cc = cols[c0:c0 + chunk]
        quads = np.unique(cc // 4)
        ch = (4 * quads[:, None] + np.arange(4)).ravel()
        w = O.dequant_weight(qw[quads], s[:, ch], z[:, ch], dtype=TAG[dtype])[np.searchsorted(ch, cc)]
        aw = np.abs(w)
        Y[:, c0:c0 + len(cc)] = x @ w.T
        A[:, c0:c0 + len(cc)] = ax @ aw.T
        D[:, c0:c0 + len(cc)] = mx @ aw.reshape(len(cc), K // 128, 128).sum(axis=2).T
    return Y, A, D


def ulp(v, dtype):
    """Spacing of T at |v| (normal or subnormal)."""
    lo, mant = (-14, 10) if dtype == F16 else (-126, 7)
    e = np.floor(np.log2(np.maximum(np.abs(v), 2.0 ** lo)))
    return 2.0 ** (np.maximum(e, lo) - mant)


def bound_violations(y, Y, A, D, dtype, gam, digits):
    """Boolean mask of the elements of y outside |y - Y| <= ulp_T(Y) + gam A + (2^-21 D if digits)."""
    y = np.asarray(y, dtype=np.float64)
    rn = O.rounder(TAG[dtype])
    slack = gam * A + (2.0 ** -21 * D if digits else 0.0)
    with np.errstate(invalid="ignore", over="ignore"):
        bound = ulp(Y, dtype) + slack        # the spacing at the unrounded Y: finite even where rn(Y) overflows
        ok = np.abs(y - Y) <= bound
        # an infinity is right where every value within the slack of Y rounds to it
        may_overflow = np.isinf(rn(Y + np.sign(Y) * slack))
        ok_inf = np.isinf(y) & (np.sign(y) == np.sign(Y)) & may_overflow
        must_overflow = np.isinf(rn(Y - np.sign(Y) * slack)) & np.isinf(rn(Y))
    return ~((ok & ~must_overflow) | ok_inf)


# ------------------------------------------------------------------------------------------------ calls
def run(entry, x, qw, s, z):
    """y of b200awq_w4a16_gemv / _gemm, into a NaN-filled buffer."""
    M, K = x.shape
    N = s.shape[1]
    y = torch.full((M, N), float("nan"), dtype=x.dtype, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    code = 0 if x.dtype == F16 else 1
    L = P.lib()
    if entry == "gemv":
        rc = L.b200awq_w4a16_gemv(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), M, N, K, 128, code, st)
    else:
        rc = L.b200awq_w4a16_gemm(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), M, N, K, 128, code,
                                  None, 0, st)
    assert rc == 0, L.b200awq_strerror(rc)
    return y


def layer(N, K, dtype):
    return gen_layer(N, K, dtype, seed=N + K, device=DEV)


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_probe_tokens_isolated_and_within_elementwise_bound(case):
    route, M, N, K, dtype, entry = case
    qw, s, z = layer(N, K, dtype)
    x_ext, x_ord, pr = batches(M, K, dtype, seed=M * 7 + K)
    y_ext = run(entry, x_ext.to(DEV), qw, s, z)
    y_ord = run(entry, x_ord.to(DEV), qw, s, z)
    torch.cuda.synchronize()
    for i in pr:
        assert torch.equal(y_ext[i].view(torch.int16), y_ord[i].view(torch.int16)), f"probe token {i} depends on its neighbours"
    Y, A, D = oracle_terms(x_ord[pr], qw, s, z, dtype)
    y = y_ord[pr].double().cpu().numpy()
    bad = bound_violations(y, Y, A, D, dtype, gamma(route, dtype), digits=route == "decode")
    if bad.any():
        t, n = np.argwhere(bad)[0]
        pytest.fail(f"{int(bad.sum())} of {bad.size} elements outside the bound; first: token {pr[t]}, channel {n}: "
                    f"y = {y[t, n]!r}, oracle = {Y[t, n]!r}, A = {A[t, n]!r}")


def expected_kernel(route, M, N, K, dtype, entry, sms):
    p = plan(M, N, K, TAG[dtype], entry, sms)
    assert {"skinny": "flat", "tile_9_16": "tile", "wgmma": "tile"}.get(route, route) == p.route, (route, p)
    return p.kernel


def traced_call(i):
    """kernel_trace builder: CASES[i]'s entry on a randn batch."""
    route, M, N, K, dtype, entry = CASES[i]
    qw, s, z = layer(N, K, dtype)
    x = torch.randn(M, K).to(dtype).to(DEV)
    return lambda: run(entry, x, qw, s, z)


@pytest.mark.gpu
def test_routes_pinned_by_profiler():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    records = trace("test_token_isolation_gpu:traced_call", [[i] for i in range(len(CASES))], per_process=64)
    rows, wrong = [], []
    for case, rec in zip(CASES, records):
        route, M, N, K, dtype, entry = case
        got = short_names(rec.names)
        want = expected_kernel(route, M, N, K, dtype, entry, sms)
        rows.append(f"| {route} | {M} | {N} | {K} | {TAG[dtype]} | {entry} | {', '.join(sorted(got))} |")
        if got != {want}:
            wrong.append((case_id(case), sorted(got), want))
    print("\n| route | M | N | K | dtype | entry | kernel |\n|---|---|---|---|---|---|---|\n" + "\n".join(rows))
    assert not wrong, wrong


# ------------------------------------------------------------------------------------------------ CPU self-tests
def _small_case(dtype):
    N, K, M = 256, 1024, 2
    qw, s, z = gen_layer(N, K, dtype, seed=3)
    x = probe_tokens(M, K, seed=4).to(dtype)
    return x, qw, s, z


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_bound_accepts_the_rounded_oracle(dtype):
    x, qw, s, z = _small_case(dtype)
    Y, A, D = oracle_terms(x, qw, s, z, dtype)
    y = O.rounder(TAG[dtype])(Y)
    for gam in (2.0 ** -11, 2.0 ** -14):
        assert not bound_violations(y, Y, A, D, dtype, gam, digits=False).any()


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_bound_flags_one_missing_group_contribution(dtype):
    x, qw, s, z = _small_case(dtype)
    Y, A, D = oracle_terms(x, qw, s, z, dtype)
    t, n, grp = 1, 77, 6
    s0, z0 = s.clone(), z.clone()
    s0[grp, n] = 0
    z0[grp, n] = 0
    Yc, _, _ = oracle_terms(x, qw, s0, z0, dtype)
    y = O.rounder(TAG[dtype])(Y)
    y[t, n] = O.rounder(TAG[dtype])(Yc[t, n])
    bad = bound_violations(y, Y, A, D, dtype, 2.0 ** -11, digits=True)   # the loosest bound of any route
    assert bad[t, n] and bad.sum() == 1


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["f16", "bf16"])
def test_bound_flags_the_neighbouring_channels_scale(dtype):
    x, qw, s, z = _small_case(dtype)
    Y, A, D = oracle_terms(x, qw, s, z, dtype)
    t, n = 1, 77
    s1 = s.clone()
    s1[:, n] = s[:, n + 1]
    Yc, _, _ = oracle_terms(x, qw, s1, z, dtype)
    y = O.rounder(TAG[dtype])(Y)
    y[t, n] = O.rounder(TAG[dtype])(Yc[t, n])
    bad = bound_violations(y, Y, A, D, dtype, 2.0 ** -11, digits=True)
    assert bad[t, n] and bad.sum() == 1


def test_probe_and_neighbour_tokens_have_the_promised_content():
    x_ext, x_ord, pr = batches(5, 1024, F16, seed=0)
    assert pr == [0, 3, 4]
    assert torch.equal(x_ext[pr], x_ord[pr])
    p = x_ord[0].float()
    assert (p[128:256] > 35).all() and (p[256:384] == 0).all() and (p[384:512].abs() < 2.0 ** -14).all()
    assert p.abs().max() >= 1000 and torch.signbit(p[5]) and p[1023] == 60000
    nb = x_ext[[1, 2]].float()
    assert torch.isnan(nb).any() and torch.isinf(nb).any() and (nb.abs() == 65504).any()
