"""numpy restatement of the reference's W8A8 vision-tower ops, step by step at the reference's rounding points.

Reference: awq/kernels/csrc/w8a8/{w8a8_gemm_cuda,quantization,layernorm,act}.cu, built with --use_fast_math.
The restatements use exact divisions, np.tanh and float64 sums where the GPU uses div.approx, tanh.approx and its own
summation order; the *_bounds functions further down model those exactly or by their documented error bounds and give
every element's admissible outputs.  The GEMM is exact: its int32 accumulator (int64 here) and every epilogue step
rounded once, as the GPU rounds it.
"""
import numpy as np

F16, F32 = np.float16, np.float32


def round_bf16(x):
    """float32 -> nearest-even bfloat16, returned as float32."""
    b = np.asarray(x, dtype=F32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16 << 16
    return b.astype(np.uint32).view(F32)


def round_t(x, dtype):
    """Round float32 values to the activation type ("f16" / "bf16"), result as float32."""
    x = np.asarray(x, dtype=F32)
    return x.astype(F16).astype(F32) if dtype == "f16" else round_bf16(x)


def cvt_s8(x):
    """cvt.rni.sat.s8.f32: round half to even, saturate to [-128, 127], NaN -> 0."""
    x = np.asarray(x, dtype=F32)
    r = np.rint(np.nan_to_num(x, nan=0.0, posinf=127.0, neginf=-128.0))
    return np.clip(r, -128, 127).astype(np.int8)


def gemm(x, w, wscales, ascales, bias=None):
    """x int8 [M, K], w int8 [N, K], wscales fp16 [N], ascales fp16 [M], bias fp16 [N] or None -> fp16 [M, N].
    no bias: rn_f16(f32(acc) * (ws * as));  bias: rn_f16(f32(f32(acc) * ws) * as + bias) (w8a8_gemm_cuda.cu:573-577,
    :893-899)."""
    return gemm_exact(x.astype(np.int64) @ w.astype(np.int64).T, wscales, ascales, bias)


def quant_per_token(x):
    """invoke_quant (quantization.cu:54-112): x [M, N] (fp16 / bf16 values as float32) -> (int8 codes, fp16 scales)."""
    x = np.asarray(x, dtype=F32)
    amax = np.abs(x).max(axis=1).astype(F32)
    scale = (amax / F32(127)).astype(F16)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (F32(127) / amax).astype(F32)
        q = cvt_s8(x * inv[:, None])
    return q, scale


def layernorm_quant(x, gamma, beta, eps, dtype, per_token=True, scale=None):
    """rms_norm_general (layernorm.cu:55-231).  Per token: (codes, fp16 scales); per tensor: codes, with beta ignored
    and the T-rounded value multiplied by scale[0]."""
    x = np.asarray(x, dtype=F32)
    n = x.shape[1]
    mean = (x.astype(np.float64).sum(axis=1) / n).astype(F32)
    ex2 = ((x.astype(np.float64) ** 2).sum(axis=1) / n).astype(F32)
    var = (ex2 - mean * mean).astype(F32)
    rstd = (F32(1) / np.sqrt(var + F32(eps))).astype(F32)
    d = ((x - mean[:, None]) * rstd[:, None]).astype(F32)
    g = np.asarray(gamma, dtype=F32)[None, :]
    if per_token:
        y = (d * g + np.asarray(beta, dtype=F32)[None, :]) if beta is not None else d * g
        y = y.astype(F32)
        yt = round_t(y, dtype)
        amax = np.maximum(np.abs(yt).max(axis=1), round_t(np.array([1e-6], F32), dtype)[0]).astype(F32)
        q = cvt_s8(y * (F32(127) / amax)[:, None])
        return q, (amax / F32(127)).astype(F16)
    yt = round_t((d * g).astype(F32), dtype)
    return cvt_s8(yt * F32(np.asarray(scale, dtype=F16).reshape(-1)[0]))


def gelu_fast_f16(x):
    """The reference's gelu_fast on fp16 values (act.cu:22-28) with np.tanh for tanh.approx.  `1 + (c2 x) x` is one
    fused multiply-add in the reference's SASS (HFMA2) and is formed exactly here before its single rounding."""
    x = np.asarray(x, dtype=F16)
    c1, c2 = F16(0.79788456), F16(0.044715)
    a = (x * c1).astype(F16)
    b = (c2 * x).astype(F16)
    d = (b.astype(np.float64) * x.astype(np.float64) + 1.0).astype(F16)
    inner = (a * d).astype(F16)
    t = np.tanh(inner.astype(F32)).astype(F16)
    return ((F16(0.5) * x).astype(F16) * (F16(1) + t).astype(F16)).astype(F16)


def gelu_quant(x):
    """gelu_and_quant (act.cu:34-77): x fp16 [M, N] -> (int8 codes, fp16 scales, fp16 gelu)."""
    g = gelu_fast_f16(x)
    a = np.where(g > F16(0.0001), g, -g).astype(F32)
    amax = np.maximum(a.max(axis=1), F32(0))
    scale = (amax / F32(127)).astype(F16)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        hs = (F32(127) / amax).astype(F16)
        q = cvt_s8((hs[:, None] * g).astype(F16).astype(F32))
    return q, scale, g


def silu_and_mul(x, dtype):
    """silu_and_mul (act.cu:101-140): x [M, 2d] -> rn_T(rn_T(silu(x[:, :d])) * x[:, d:])."""
    x = np.asarray(x, dtype=F32)
    d = x.shape[1] // 2
    g, u = x[:, :d], x[:, d:]
    s = round_t((g.astype(np.float64) / (1.0 + np.exp(-g.astype(np.float64)))).astype(F32), dtype)
    return round_t(s * u, dtype)


def quantize_weight(w, dtype):
    """W8A8OF16LinearDynamicInputScale's quantiser (w8a8_linear.py:156-166) on float32 values of a layer of `dtype`
    ("f16" / "bf16" / "f32"): s = max|w| per row, clamped at 1e-5, / 127, then round(w / s), every step rounded to
    the layer's dtype.  Returns (int8 codes, fp16 scales)."""
    w = np.asarray(w, dtype=F32)
    rt = (lambda v: np.asarray(v, F32)) if dtype == "f32" else (lambda v: round_t(v, dtype))
    s = rt(np.maximum(np.abs(w).max(axis=1, keepdims=True), rt(np.array(1e-5, F32))) / F32(127))
    q = np.rint(rt(w / s)).astype(np.int8)
    return q, s.reshape(-1).astype(F16)


# ================================================================================================================
# Admissible outputs.  The functions above restate the reference's formulas; the ones below say, element by element,
# which outputs the GPU kernels may produce given the instructions they issue (llm_awq_b200/csrc/w8a8_math.cuh):
#   * add / sub / mul / fma .rn.ftz, cvt.rni.sat, the fp16 / bf16 roundings: emulated exactly (one rounding of the
#     exact value; subnormal inputs and results flushed to signed zero);
#   * the LayerNorm's summation order: emulated exactly (ln_sums);
#   * the approximate instructions, by their documented bounds (PTX ISA; CUDA C Programming Guide for expf):
#       div.approx.ftz  2 ulp for |b| in [2^-126, 2^126]; outside, d = a * (1 / b): 0 for |b| > 2^126 (b = inf too),
#                       inf for b = 0, NaN for inf / inf and 0 / 0
#       rsqrt.approx    relative error 2^-22.9
#       tanh.approx     relative error 2^-10.987
#       expf            2 ulp (silu_mul.cu is built without fast math: its `+` and `/` are IEEE, nothing flushes).
# Every output is a monotone function of each approximate quantity once the sign of the element is fixed: codes are
# cvt(v * inv) with cvt and every .rn step monotone; y = ((x - mean) * rstd) * gamma (+ beta) is monotone in mean for a
# fixed rstd and in rstd for a fixed mean; gelu = rn(rn(0.5 x) * rn(1 + t)) in t; silu = g / (1 + e) in e.  A
# function monotone in each variable separately (whatever the direction) takes its extremes over a box at the box's
# corners, so evaluating the extreme candidates of every approximate quantity and taking the per-element min / max
# gives sets that contain every output the bounds allow.  Treating the LayerNorm's mean and rstd (and a row's amax)
# as independent boxes, though rstd and amax depend on the mean, only enlarges the sets.
# The LayerNorm's var = fma(-mean, mean, sq / n) can fall below -eps (a large mean, a tiny spread); then rstd is NaN,
# every code 0 and amax its floor rn_T(1e-6), the reference's formula.  Such rows carry `deg` and may instead hold that
# outcome as a whole.
# ================================================================================================================
F64 = np.float64
TINY32 = 2.0 ** -126
DIV_ULPS = 2
RSQRT_REL = 2.0 ** -22.9
TANH_REL = 2.0 ** -10.987
EXPF_ULPS = 2
_CHUNKS = {8: 4, 1: 8}      # chunks_per_thread<VEC>() of w8a8_rowops.cu
_MAX_THREADS = 1024


def _f32(x):
    return np.asarray(x, dtype=F32)


def ftz(x):
    """float32 values with subnormals flushed to zero of the same sign."""
    x = _f32(x)
    return np.where(np.abs(x) < F32(TINY32), np.copysign(F32(0), x), x).astype(F32)


def _round32(s, e):
    """float32 nearest-even to the exact s + e (float64 s, and e its exact remainder with |e| <= ulp(s) / 2): s rounds
    correctly unless it sits exactly halfway between two floats, where the sign of e picks the side."""
    with np.errstate(all="ignore"):
        r = s.astype(F32)
        r64 = r.astype(F64)
        other = np.nextafter(r, np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32))
        tie = (s != r64) & (s == (r64 + other.astype(F64)) * 0.5) & (e != 0)
        return np.where(tie & ((e > 0) == (other > r)), other, r).astype(F32)


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def add_ftz(a, b):
    """add.rn.ftz.f32"""
    with np.errstate(all="ignore"):
        s, e = _two_sum(ftz(a).astype(F64), ftz(b).astype(F64))
    return ftz(_round32(s, e))


def sub_ftz(a, b):
    """sub.rn.ftz.f32"""
    return add_ftz(a, -_f32(b))


def mul_ftz(a, b):
    """mul.rn.ftz.f32 (the float64 product of two floats is exact)"""
    with np.errstate(all="ignore"):
        return ftz((ftz(a).astype(F64) * ftz(b).astype(F64)).astype(F32))


def fma_ftz(a, b, c):
    """fma.rn.ftz.f32: a * b is exact in float64; the sum is rounded once through TwoSum."""
    with np.errstate(all="ignore"):
        s, e = _two_sum(ftz(a).astype(F64) * ftz(b).astype(F64), ftz(c).astype(F64))
    return ftz(_round32(s, e))


def rn16(x):
    """float32 / float64 -> nearest-even fp16 (numpy rounds a float64 once, from all its bits)."""
    with np.errstate(all="ignore"):
        return np.asarray(x).astype(F16)


def steps32(x, k):
    """x moved k float32 steps (k < 0: down); infinities, NaN and zeros stay."""
    x = _f32(x)
    out = x.copy()
    fin = np.isfinite(x) & (x != 0)
    for _ in range(abs(k)):
        out = np.where(fin, np.nextafter(out, F32(np.inf if k > 0 else -np.inf)), out).astype(F32)
    return out


def _floor32(v):
    r = _f32(v)
    return np.where(r.astype(F64) > v, np.nextafter(r, F32(-np.inf)), r).astype(F32)


def _ceil32(v):
    r = _f32(v)
    return np.where(r.astype(F64) < v, np.nextafter(r, F32(np.inf)), r).astype(F32)


def div_approx(a, b):
    """div.approx.ftz.f32: (lowest, highest) admissible result, elementwise."""
    a, b = ftz(a), ftz(b)
    with np.errstate(all="ignore"):
        q = (a.astype(F64) / b.astype(F64)).astype(F32)          # one rounding: innocuous after float64
        rule = (a.astype(F64) * (F64(1) / b.astype(F64))).astype(F32)
        rule = np.where(np.abs(b) > F32(2.0 ** 126), (a.astype(F64) * 0.0).astype(F32), rule)
    inr = (np.abs(b) >= F32(TINY32)) & (np.abs(b) <= F32(2.0 ** 126)) & np.isfinite(a)
    lo = np.where(inr, steps32(q, -DIV_ULPS), rule)
    hi = np.where(inr, steps32(q, DIV_ULPS), rule)
    return ftz(lo), ftz(hi)


def rsqrt_approx(x):
    """rsqrt.approx.ftz.f32: (lowest, highest) admissible result; +-0 -> +-inf, negative -> NaN, inf -> 0."""
    x = ftz(x)
    with np.errstate(all="ignore"):
        r = 1.0 / np.sqrt(x.astype(F64))
        lo, hi = _ceil32(r * (1 - RSQRT_REL)), _floor32(r * (1 + RSQRT_REL))
    special = (x <= 0) | ~np.isfinite(x)
    with np.errstate(all="ignore"):
        sp = (1.0 / np.sqrt(x.astype(F64))).astype(F32)
    return np.where(special, sp, lo).astype(F32), np.where(special, sp, hi).astype(F32)


def expf_range(x):
    """expf (2 ulp): (lowest, highest) admissible float32 result."""
    with np.errstate(all="ignore"):
        e = np.exp(_f32(x).astype(F64)).astype(F32)
    return steps32(e, -EXPF_ULPS), steps32(e, EXPF_ULPS)


def tanh_range(x):
    """tanh.approx.f32 rounded to fp16: (lowest, highest) admissible fp16 result (rn16 is monotone, so rounding the
    real bounds bounds the rounding of every float32 between them)."""
    t = np.tanh(_f32(x).astype(F64))
    a, b = t * (1 - TANH_REL), t * (1 + TANH_REL)
    return rn16(np.minimum(a, b)), rn16(np.maximum(a, b))


def round_t64(x, dtype):
    """float32 -> activation type, kept as float32 (round_t without its float32 cast of the input)."""
    return round_t(_f32(x), dtype)


# ---------------------------------------------------------------------------------------------- kernel geometry
def row_threads(chunks):
    """Threads of a row kernel for `chunks` accesses (w8a8_rowops.cu row_threads)."""
    per = -(-chunks // _MAX_THREADS)
    t = -(-chunks // per)
    return -(-t // 32) * 32


def row_vec(n, aligned=True):
    """Elements per access: 8 (16-byte kernel) when n % 8 == 0 and every pointer is 16-byte aligned, else 1."""
    return 8 if n % 8 == 0 and aligned else 1


def row_fits(n, vec):
    """Whether a row of n elements fits the kernel of width `vec` (else B200AWQ_ERR_SHAPE)."""
    return n // vec <= _CHUNKS[vec] * _MAX_THREADS


def warp_butterfly(a):
    """The xor butterfly (16 ... 1) of add.rn.ftz over the last axis (32 lanes); every lane ends with the same sum."""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        a = add_ftz(a, a[..., lane ^ o])
    return a


def block_sum(part):
    """block_sum2 of w8a8_rowops.cu on per-thread partials [..., threads]: each warp's butterfly, then the butterfly
    over the warps' results (lanes >= the warp count contribute 0)."""
    thr = part.shape[-1]
    nw = thr // 32
    w = warp_butterfly(part.reshape(part.shape[:-1] + (nw, 32)))[..., 0]
    red = np.zeros(part.shape[:-1] + (32,), F32)
    red[..., :nw] = w
    return warp_butterfly(red)[..., 0]


def ln_sums(x, vec):
    """(sum, sq) of each row of x [M, n] as layernorm_quant_kernel forms them: thread t takes chunks t + j * threads
    in ascending j and element order, sum = add(sum, v), sq = fma(v, v, sq), then block_sum."""
    x = _f32(x)
    M, n = x.shape
    nc = n // vec
    thr = row_threads(nc)
    s = np.zeros((M, thr), F32)
    q = np.zeros((M, thr), F32)
    for j in range(_CHUNKS[vec]):
        ci = np.arange(thr) + j * thr
        ok = ci < nc
        if not ok.any():
            break
        for e in range(vec):
            v = x[:, np.minimum(ci, nc - 1) * vec + e]
            s = np.where(ok, add_ftz(s, v), s)
            q = np.where(ok, fma_ftz(v, v, q), q)
    return block_sum(s), block_sum(q)


# ---------------------------------------------------------------------------------------------- admissible sets
def cvt_range(vals):
    """Codes of a stack of candidate values [k, ...] -> (lowest, highest) code per element."""
    c = cvt_s8(vals)
    return c.min(axis=0), c.max(axis=0)


def _abs_range(lo, hi):
    """(min, max) of |v| for v in [lo, hi], NaN-free bounds; NaN where both bounds are NaN."""
    mn = np.where((lo <= 0) & (hi >= 0), 0, np.minimum(np.abs(lo), np.abs(hi)))
    return mn, np.maximum(np.abs(lo), np.abs(hi))


def _scale_range(amax_lo, amax_hi):
    return rn16(div_approx(amax_lo, F32(127))[0]), rn16(div_approx(amax_hi, F32(127))[1])


def quant_per_token_bounds(x):
    """invoke_quant: x [M, N] (T values as float32) -> dict of code bounds lo / hi [M, N] and scale bounds s_lo / s_hi
    [M] (fp16)."""
    x = _f32(x)
    with np.errstate(all="ignore"):
        amax = np.fmax.reduce(np.abs(x), axis=1, initial=F32(0)).astype(F32)   # fmaxf: NaN never wins
    ilo, ihi = div_approx(F32(127), amax)
    lo, hi = cvt_range(np.stack([mul_ftz(x, ilo[:, None]), mul_ftz(x, ihi[:, None])]))
    s_lo, s_hi = _scale_range(amax, amax)
    return dict(lo=lo, hi=hi, s_lo=s_lo, s_hi=s_hi)


def layernorm_quant_bounds(x, gamma, beta, eps, dtype, per_token=True, scale=None, vec=None):
    """rms_norm_general as layernorm_quant_kernel computes it, on x [M, n], gamma / beta [n] (T values as float32;
    beta None, and ignored per tensor), vec the access width (default: row_vec(n)).  Returns the dict of
    quant_per_token_bounds (per tensor: no scale bounds) plus `deg` [M]: rows that may instead be all codes 0 with
    scale rn_f16(floor / 127), d_lo / d_hi."""
    x = _f32(x)
    M, n = x.shape
    vec = row_vec(n) if vec is None else vec
    s, q = ln_sums(x, vec)
    k = np.arange(-DIV_ULPS, DIV_ULPS + 1)
    mq = div_approx(s, F32(n))[0]
    qq = div_approx(q, F32(n))[0]
    means = np.stack([steps32(mq, DIV_ULPS + i) for i in k])          # every div.approx candidate [5, M]
    sqns = np.stack([steps32(qq, DIV_ULPS + i) for i in k])
    var = fma_ftz(-means[:, None], means[:, None], sqns[None, :])        # [5, 5, M]
    ve = add_ftz(var, F32(eps))
    rlo, rhi = rsqrt_approx(ve)
    ok = ~np.isnan(rlo)                                                  # var + eps >= 0
    with np.errstate(all="ignore"):
        r_lo = np.where(ok, rlo, np.inf).min(axis=(0, 1)).astype(F32)
        r_hi = np.where(ok, rhi, -np.inf).max(axis=(0, 1)).astype(F32)
    deg = ~ok.all(axis=(0, 1))
    regular = ok.any(axis=(0, 1))
    r_lo, r_hi = np.where(regular, r_lo, 0), np.where(regular, r_hi, 0)
    g = _f32(gamma)[None, :]
    ys = []
    for mc in (means.min(axis=0), means.max(axis=0)):
        dm = sub_ftz(x, mc[:, None])
        for rc in (r_lo, r_hi):
            d = mul_ftz(dm, rc[:, None])
            if per_token and beta is not None:
                ys.append(fma_ftz(d, g, _f32(beta)[None, :]))
            else:
                ys.append(mul_ftz(d, g))
    ys = np.stack(ys)
    yt = round_t64(ys, dtype)
    floor = round_t64(np.array([1e-6], F32), dtype)[0]
    if not per_token:
        lo, hi = cvt_range(mul_ftz(yt, F32(np.asarray(scale, dtype=F16).reshape(-1)[0])))
        return dict(lo=lo, hi=hi, deg=deg)
    with np.errstate(all="ignore"):
        amn, amx = _abs_range(np.fmin.reduce(yt, axis=0), np.fmax.reduce(yt, axis=0))
        a_lo = np.fmax(np.fmax.reduce(np.where(np.isnan(amn), 0, amn), axis=1), floor).astype(F32)
        a_hi = np.fmax(np.fmax.reduce(np.where(np.isnan(amx), 0, amx), axis=1), floor).astype(F32)
    ilo, ihi = div_approx(F32(127), a_hi)[0], div_approx(F32(127), a_lo)[1]
    lo, hi = cvt_range(np.concatenate([mul_ftz(ys, ilo[None, :, None]), mul_ftz(ys, ihi[None, :, None])]))
    s_lo, s_hi = _scale_range(a_lo, a_hi)
    d_lo, d_hi = _scale_range(np.full(M, floor, F32), np.full(M, floor, F32))
    return dict(lo=lo, hi=hi, s_lo=s_lo, s_hi=s_hi, deg=deg, d_lo=d_lo, d_hi=d_hi)


GELU_SMALL = F16(0.0001)


def gelu_front_f16(x):
    """The fp16 chain of gelu_fast up to tanh's argument and the half factor: (inner, rn(0.5 x)).  Every fp16 step is
    one rounding of the float64 value, which is exact for a product or sum of two fp16 values and for
    `1 + (c2 x) x` (HFMA2)."""
    x = np.asarray(x, dtype=F16).astype(F64)
    c1, c2 = F64(F16(0.79788456)), F64(F16(0.044715))
    with np.errstate(all="ignore"):
        a = rn16(x * c1).astype(F64)
        b = rn16(c2 * x).astype(F64)
        d = rn16(b * x + 1.0).astype(F64)
        return rn16(a * d), rn16(0.5 * x)


def gelu_tail_f16(h, t):
    """rn(h * rn(1 + t)) on fp16 h, t."""
    with np.errstate(all="ignore"):
        return rn16(h.astype(F64) * rn16(1.0 + np.asarray(t, F16).astype(F64)).astype(F64))


def gelu_quant_bounds(x):
    """gelu_and_quant on fp16 x [M, N]: the dict of quant_per_token_bounds plus g_lo / g_hi, the admissible GELU
    values (fp16)."""
    inner, h = gelu_front_f16(x)
    t_lo, t_hi = tanh_range(inner.astype(F32))
    ga, gb = gelu_tail_f16(h, t_lo), gelu_tail_f16(h, t_hi)
    g_lo, g_hi = np.minimum(ga, gb), np.maximum(ga, gb)
    nxt = np.nextafter(GELU_SMALL, F16(np.inf))

    def a_of(g):
        return np.where(g > GELU_SMALL, g, -g).astype(F32)
    cand = [a_of(g_lo), a_of(g_hi)]
    span = (g_lo <= GELU_SMALL) & (g_hi > GELU_SMALL)
    cand += [np.where(span, a_of(GELU_SMALL), np.nan), np.where(span, a_of(nxt), np.nan)]
    with np.errstate(all="ignore"):
        cand = np.stack(cand)
        a_min, a_max = np.fmin.reduce(cand, axis=0), np.fmax.reduce(cand, axis=0)
        # max.f32 orders -0 below +0, so a row of +0 and negated values keeps amax = +0 (127 / amax = +inf)
        amax_lo = np.fmax.reduce(np.where(np.isnan(a_min), 0, a_min), axis=1, initial=F32(0)).astype(F32) + F32(0)
        amax_hi = np.fmax.reduce(np.where(np.isnan(a_max), 0, a_max), axis=1, initial=F32(0)).astype(F32) + F32(0)
    hs_lo = rn16(div_approx(F32(127), amax_hi)[0])
    hs_hi = rn16(div_approx(F32(127), amax_lo)[1])
    with np.errstate(all="ignore"):
        prods = [rn16(hs[:, None].astype(F64) * g.astype(F64)).astype(F32) for hs in (hs_lo, hs_hi) for g in (g_lo, g_hi)]
    lo, hi = cvt_range(np.stack(prods))
    s_lo, s_hi = _scale_range(amax_lo, amax_hi)
    return dict(lo=lo, hi=hi, s_lo=s_lo, s_hi=s_hi, g_lo=g_lo, g_hi=g_hi)


def silu_and_mul_bounds(x, dtype):
    """silu_and_mul on x [M, 2d] (T values as float32): (lowest, highest) admissible output, T values as float32.
    IEEE fp32 arithmetic with subnormals, expf within 2 ulp."""
    x = _f32(x)
    d = x.shape[1] // 2
    g, u = x[:, :d].astype(F64), x[:, d:].astype(F64)
    outs = []
    for e in expf_range(-x[:, :d]):
        with np.errstate(all="ignore"):
            den = (1.0 + e.astype(F64)).astype(F32).astype(F64)
            s = round_t((g / den).astype(F32), dtype).astype(F64)
            outs.append(round_t((s * u).astype(F32), dtype))
    return np.minimum(*outs), np.maximum(*outs)


def gemm_exact(acc, wscales, ascales, bias=None):
    """The GEMM epilogue, every step one rounding: acc [M, N] exact integers (any dtype that holds them) -> fp16.
    no bias: rn_f16(mul(f32(acc), mul(ws, as)));  bias: rn_f16(fma(mul(f32(acc), ws), as, bias))."""
    accf = np.asarray(acc, dtype=F64).astype(F32)
    ws = np.asarray(wscales, dtype=F16).astype(F32)[None, :]
    a = np.asarray(ascales, dtype=F16).astype(F32)[:, None]
    if bias is None:
        return rn16(mul_ftz(accf, mul_ftz(ws, a)))
    return rn16(fma_ftz(mul_ftz(accf, ws), a, np.asarray(bias, dtype=F16).astype(F32)[None, :]))


# ---------------------------------------------------------------------------------------------- checks
def admissible_rows(q, s, b):
    """Per row: every code within [lo, hi] and the scale within [s_lo, s_hi] (when the op has one), or -- rows marked
    `deg` -- every code 0 and the scale within [d_lo, d_hi]."""
    q = np.asarray(q, np.int32)
    ok = ((q >= b["lo"]) & (q <= b["hi"])).all(axis=1)
    if s is not None and "s_lo" in b:
        sf = np.asarray(s, F16).astype(F32)
        ok &= (sf >= b["s_lo"].astype(F32)) & (sf <= b["s_hi"].astype(F32))
    if "deg" in b:
        alt = b["deg"] & (q == 0).all(axis=1)
        if s is not None and "d_lo" in b:
            alt &= (sf >= b["d_lo"].astype(F32)) & (sf <= b["d_hi"].astype(F32))
        ok |= alt
    return ok


def two_code_share(b):
    """Share of the elements with more than one admissible code."""
    return float(np.mean(b["hi"] != b["lo"]))


def assert_admissible(q, s, b, what=""):
    ok = admissible_rows(q, s, b)
    if not ok.all():
        r = int(np.flatnonzero(~ok)[0])
        qr = np.asarray(q, np.int32)[r]
        bad = np.flatnonzero((qr < b["lo"][r]) | (qr > b["hi"][r]))[:8]
        msg = f"{what}: {int((~ok).sum())} rows outside their admissible sets; row {r}, columns {bad.tolist()}: codes " \
              f"{qr[bad].tolist()}, admissible [{b['lo'][r][bad].tolist()}, {b['hi'][r][bad].tolist()}]"
        if s is not None and "s_lo" in b:
            msg += f"; scale {float(np.asarray(s, F16)[r])} in [{float(b['s_lo'][r])}, {float(b['s_hi'][r])}]"
        raise AssertionError(msg)


def assert_between(v, lo, hi, what=""):
    """Values (fp16 / bf16 as float32 or fp16) within [lo, hi] elementwise; NaN where both bounds are NaN."""
    v, lo, hi = (np.asarray(t).astype(F32) for t in (v, lo, hi))
    ok = ((v >= lo) & (v <= hi)) | (np.isnan(v) & np.isnan(lo) & np.isnan(hi))
    if not ok.all():
        i = np.argwhere(~ok)[:8]
        raise AssertionError(f"{what}: {int((~ok).sum())} values outside [lo, hi]; first at {i.tolist()}: "
                             f"{v[~ok][:8].tolist()} vs [{lo[~ok][:8].tolist()}, {hi[~ok][:8].tolist()}]")
