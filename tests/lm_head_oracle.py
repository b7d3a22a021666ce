"""The float64 oracle of the LM head (b200awq_lm_head) and the elementwise bound its logits must meet.

Contract: logits[i, v] = (float) rn_T(s), where s is the fp32 sum of the products x^[i, j] W[v, j] over j < k.  The kernel
forms s as follows: lane l of a warp owns the 8-element chunks l, l + 32, ... and accumulates each product with one fmaf,
then the 32 lane sums meet in an xor butterfly of 5 adds.  So each product passes through at most
    n = 8 ceil(k / 256) + 5
fp32 roundings.  Products of two fp16 or two bf16 values are exact in float64, and so is Y = sum_j x^_ij W_vj up to
float64's own summation error, which is at most k 2^-53 A and is counted below.  Let A = sum_j |x^_ij W_vj|.  The textbook
bound for a recursive sum with one rounding per operation (Higham, Accuracy and Stability, §3.1) gives
    |s - Y| <= gamma_n A + n 2^-149,    gamma_n = n u / (1 - n u),  u = 2^-24.
The second term covers operations whose result lies in fp32's subnormal range: there the absolute error of one rounding
is at most 2^-150, so the relative model does not hold.  The last rounding to T adds at most half an ulp of T at |s|, and
|s| <= |Y| + gamma_n A + n 2^-149.  So every finite logit y must satisfy
    |y - Y| <= ulp_T(|Y| + e) + e,    e = gamma_n A + n 2^-149 + k 2^-53 A,
with ulp_T the spacing of T at that magnitude, or its smallest subnormal below T's normal range.  A full ulp here is
twice what the last rounding needs.  y must also be a value of T: the fp32 logit is T's value widened exactly.
Non-finite cases: if Y is NaN, y is NaN.  If Y is +-inf, y is the same inf.  If Y is finite, y may be +-inf only when
[Y - b, Y + b] reaches T's rounding threshold for overflow (65520 for fp16; bf16 overflows in fp32 first, above
2^128 (1 - 2^-25))."""
import numpy as np

U32 = 2.0 ** -24
FP16_OVERFLOW = 65520.0
BF16_OVERFLOW = 2.0 ** 128 * (1 - 2.0 ** -25)


def roundings(k):
    return 8 * -(-k // 256) + 5


def t_spacing(a, bf16):
    """ulp of T at |a| (float64 array): 2^(e - p) for 2^e <= |a| < 2^(e+1), T's subnormal spacing below its normal
    range."""
    p, emin = (7, -126) if bf16 else (10, -14)
    a = np.abs(a)
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.maximum(np.where(a > 0, e, emin), emin)
    return np.exp2(e - p)


def oracle(xhat, w):
    """(Y, A): float64 [m, vocab] of the exact sums and the sums of the absolute products, from float64 copies of the
    T-valued xhat [m, k] and w [vocab, k]."""
    x = np.asarray(xhat, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return x @ w.T, np.abs(x) @ np.abs(w).T


def bound(Y, A, k, bf16):
    n = roundings(k)
    e = (n * U32 / (1 - n * U32) + k * 2.0 ** -53) * A + n * 2.0 ** -149
    with np.errstate(over="ignore"):
        return t_spacing(np.abs(Y) + e, bf16) + e


def is_t_value(y, bf16):
    """whether each fp32 y is a value of T (fp16: exactly representable; bf16: low 16 bits zero)."""
    y = np.asarray(y, dtype=np.float32)
    if bf16:
        return (y.view(np.uint32) & 0xFFFF) == 0
    with np.errstate(over="ignore"):
        return np.isnan(y) | (y.astype(np.float16).astype(np.float32) == y)


def violations(got, xhat, w, bf16):
    """Boolean [m, vocab]: the logits that break the contract (see the module docstring)."""
    Y, A = oracle(xhat, w)
    return violations_of(got, Y, A, np.asarray(w).shape[1], bf16)


def violations_of(got, Y, A, k, bf16):
    """violations() from the oracle's (Y, A) of a k-wide product."""
    got = np.asarray(got, dtype=np.float32)
    b = bound(np.nan_to_num(Y), np.nan_to_num(A), k, bf16)
    g = got.astype(np.float64)
    thr = BF16_OVERFLOW if bf16 else FP16_OVERFLOW
    with np.errstate(invalid="ignore"):
        finite_ok = np.isfinite(g) & (np.abs(g - Y) <= b)
        inf_ok = (g == np.inf) & (Y + b >= thr) | (g == -np.inf) & (Y - b <= -thr)
        ok_finite_y = np.isfinite(Y) & (finite_ok | inf_ok)
        ok_inf_y = np.isinf(Y) & (g == Y)
        ok_nan_y = np.isnan(Y) & np.isnan(g)
    return ~((ok_finite_y | ok_inf_y | ok_nan_y) & is_t_value(got, bf16))


def emulate(xhat, w, bf16):
    """The kernel's summation order on the host (module docstring), with each fmaf formed in float64 and rounded to
    fp32 (exact for these products; the rare double rounding stays inside the bound).  Returns fp32 [m, vocab]."""
    x = np.asarray(xhat, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    m, k = x.shape
    nchunk = k // 8
    lanes = np.zeros((32, m, w.shape[0]), dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for lane in range(32):
            for c in range(lane, nchunk, 32):
                for j in range(8 * c, 8 * c + 8):
                    prod = x[:, j][:, None] * w[:, j][None, :]
                    lanes[lane] = (lanes[lane].astype(np.float64) + prod).astype(np.float32)
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[np.arange(32) ^ o]
        s = lanes[0]
        if bf16:
            t = s.view(np.uint32).astype(np.uint64)
            t = ((t + 0x7FFF + ((t >> 16) & 1)) >> 16 << 16).astype(np.uint32)
            t = np.where(np.isnan(s), np.uint32(0x7FC00000), t)
            return t.view(np.float32)
        return s.astype(np.float16).astype(np.float32)
