"""numpy restatement of the reference's W8A8 vision-tower ops, step by step at the reference's rounding points.

Reference: awq/kernels/csrc/w8a8/{w8a8_gemm_cuda,quantization,layernorm,act}.cu, built with --use_fast_math.
What numpy cannot reproduce, and so what the tests allow for:
  * divisions are exact here, div.approx.ftz on the GPU (scales <= 1 fp16 ulp, codes +-1);
  * tanh is np.tanh, tanh.approx on the GPU (gelu <= 2 fp16 ulp, codes +-1);
  * the fused-bias GEMM epilogue is one fused multiply-add on the GPU; here the product is formed exactly in float64
    and rounded to float32 after the add (<= 1 fp16 ulp);
  * LayerNorm statistics are summed in another order (codes +-1, scale <= 1 ulp).
The GEMM accumulator is exact (int64), as the GPU's int32 accumulator is.
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
    acc = x.astype(np.int64) @ w.astype(np.int64).T
    accf = acc.astype(F32)
    ws = np.asarray(wscales, dtype=F16).astype(F32)[None, :]
    a = np.asarray(ascales, dtype=F16).astype(F32)[:, None]
    if bias is None:
        return (accf * (ws * a)).astype(F16)
    p = (accf * ws).astype(F32).astype(np.float64)
    y = (p * a.astype(np.float64) + np.asarray(bias, dtype=F16).astype(np.float64)[None, :]).astype(F32)
    return y.astype(F16)


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
