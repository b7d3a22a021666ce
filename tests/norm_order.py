"""The RMSNorm row statistic's summation order (llm_awq_b200/csrc/rmsnorm_stat.cuh), restated in numpy, and the inputs
of tests/golden/rmsnorm_order.npz (outputs of b200awq_rmsnorm on an H100, made by tests/golden/make_rmsnorm_order_golden.py).

The order: 256 threads; thread t owns the 8-element chunks t, t + 256, ... and accumulates x_i^2 with fmaf in element
order from 0.f; an xor butterfly 16, 8, 4, 2, 1 inside each warp of 32 threads; the 8 warp totals added in warp order
from 0.f; r = rsqrtf(total / n + eps); y_i = rn_T((x_i * r) * gamma_i), fp16 clamped to +-(65504 - 1000).

Everything but rsqrtf is restated exactly: x_i^2 of an fp16 / bf16 value is exact in fp32 (at most 22 significant
bits, inside the range of the inputs below), so fmaf(x, x, s) is the fp32 sum s + x_i^2 rounded once, and every other
step is one IEEE fp32 operation.  rsqrtf is the hardware's approximate reciprocal square root (a few ulp), so the
restatement gives the correctly rounded value and the candidates within RSQRT_ULPS ulp of it; the stored row must equal
the output of one of them, bit for bit.

The ROWS are built so that the order shows in the output: a large element whose square absorbs the small squares added
after it in a sequential sum, placed at the start, at the end and every few chunks, moves the total by far more than the
rsqrtf tolerance when the order changes."""
import numpy as np

THREADS, WARP = 256, 32
RSQRT_ULPS = 4
EPS = 1e-6
WIDTHS = (100, 128, 896, 4096, 4100, 8192)   # 100 and 4100: the generic kernel (n % 8 != 0); the rest: the register kernel
ROWS = ("normal", "heavy_tailed", "absorb_first", "absorb_last", "absorb_strided")


def inputs(n, dtype):
    """(x [len(ROWS), n], gamma [n]) as float32 arrays holding values of `dtype` ("f16" or "bf16")."""
    rng = np.random.default_rng(1000 * n + (dtype == "bf16"))
    x = np.empty((len(ROWS), n), dtype=np.float64)
    sign = np.where(rng.random((len(ROWS), n)) < 0.5, -1.0, 1.0)
    x[0] = 2.0 * rng.standard_normal(n)
    x[1] = sign[1] * np.exp2(rng.uniform(-10.0, 8.0, n))
    x[2:] = sign[2:] * (1.0 + rng.integers(0, 4, (3, n)) / 8.0)   # squares of 1 .. 1.375: absorbed next to 2^24
    x[2, 0] = 4096.0
    x[3, n - 1] = -4096.0
    x[4, ::24] = 4096.0
    gamma = 1.0 + 0.25 * rng.standard_normal(n)
    return round_to(x, dtype), round_to(gamma, dtype)


def round_to(v, dtype):
    """float32 array of the values of v rounded to fp16 / bf16 (round to nearest even)."""
    v = np.asarray(v, dtype=np.float32)
    if dtype == "f16":
        return v.astype(np.float16).astype(np.float32)
    b = v.view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32)


def thread_sums(sq):
    """The 256 threads' accumulators over one row of squares (rmsnorm_stat.cuh's chunk ownership)."""
    n = sq.shape[0]
    nchunk = -(-n // 8)
    rounds = -(-nchunk // THREADS)
    pad = np.zeros(rounds * THREADS * 8, dtype=np.float32)
    pad[:n] = sq
    chunks = pad.reshape(rounds, THREADS, 8)          # [round j][thread t] = chunk t + 256 j
    s = np.zeros(THREADS, dtype=np.float32)
    for j in range(rounds):
        for e in range(8):
            s = s + chunks[j, :, e]                    # + 0 for the chunks past the row: exact
    return s


def butterfly(s):
    """Each warp's xor butterfly 16 .. 1; returns the 8 warp totals (lane 0's value)."""
    v = s.reshape(THREADS // WARP, WARP).copy()
    lanes = np.arange(WARP)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lanes ^ o]
    return v[:, 0]


def ordered_total(w):
    t = np.float32(0.0)
    for x in w:
        t = np.float32(t + x)
    return t


def total_in_order(x):
    """The row statistic's sum of squares in rmsnorm_stat.cuh's order."""
    return ordered_total(butterfly(thread_sums(x * x)))


def total_sequential(x):
    """Another order, for the tests' discrimination check: one accumulator over the row."""
    return ordered_total(x * x)


def total_blocked(x):
    """Another order: thread t owns one contiguous block of the row instead of every 256th chunk."""
    n = x.shape[0]
    per = -(-n // THREADS)
    pad = np.zeros(per * THREADS, dtype=np.float32)
    pad[:n] = x * x
    s = np.zeros(THREADS, dtype=np.float32)
    for e in range(per):
        s = s + pad.reshape(THREADS, per)[:, e]
    return ordered_total(butterfly(s))


def norm_round(v, dtype):
    if dtype == "f16":
        lim = np.float32(65504.0 - 1000.0)
        v = np.where(v > 0, np.minimum(v, lim), np.maximum(v, -lim)).astype(np.float32)
    return round_to(v, dtype)


def rsqrt_candidates(total, n, eps=EPS):
    q = np.float32(np.float32(total / np.float32(n)) + np.float32(eps))
    r0 = np.float32(1.0 / np.sqrt(np.float64(q)))
    i0 = int(np.array([r0], dtype=np.float32).view(np.int32)[0])
    return [np.array([i0 + d], dtype=np.int32).view(np.float32)[0] for d in range(-RSQRT_ULPS, RSQRT_ULPS + 1)]


def outputs(x, gamma, total, dtype, eps=EPS):
    """[candidate][n] float32 values of rn_T((x r) gamma) for each rsqrtf candidate r of `total`."""
    return [norm_round(np.float32(x * r) * gamma, dtype) for r in rsqrt_candidates(total, x.shape[0], eps)]


def bits(v, dtype):
    """uint16 bit patterns of float32 values that are fp16 / bf16 values."""
    if dtype == "f16":
        return v.astype(np.float16).view(np.uint16)
    return (v.view(np.uint32) >> 16).astype(np.uint16)


def matches(x, gamma, stored_bits, total, dtype, eps=EPS):
    """Whether some rsqrtf candidate of `total` reproduces the stored row bit for bit."""
    return any(np.array_equal(bits(y, dtype), stored_bits) for y in outputs(x, gamma, total, dtype, eps))
