"""CPU oracle for the W4A16 (AWQ v2 / "gemv_new") quantized-linear path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``llm_awq_b200/`` may import this file; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs use it, and there only as the checker / the timed CPU arm.

Parity status: the reference ships no tests or golden vectors for this path
(SURVEY.md §4), so it is *pinned by us*: every function below is checked against the
reference's own Python (``awq/quantize/qmodule.py``, ``awq/quantize/quantizer.py``)
imported on CPU; the resulting vectors are committed under
``tests/golden/`` together with ``tests/golden/make_golden.py``.  The CUDA kernels of
the reference's kernels need a GPU; on the GPU the parity
tests additionally compare against stored outputs of the reference kernels built for sm_90a
(``oracle/_ref``, built by ``oracle/build_ref.py``).

Each function cites the reference file:line it restates (paths relative to the
reference checkout).
"""
from __future__ import annotations

import numpy as np

INTERLEAVE = 4   # awq/quantize/qmodule.py:90
KSTRIDE = 64     # awq/quantize/qmodule.py:187  (pack_intweight(..., interleave=4, kstride=64))
PACK_NUM = 8     # awq/quantize/qmodule.py:94   (32 // w_bit)


# --------------------------------------------------------------------------------------
# shapes
# --------------------------------------------------------------------------------------
def calculate_zeros_width(in_features: int, group_size: int = 128, pack_num: int = 8) -> int:
    """Number of 8-row blocks of the scales / scaled_zeros buffers.

    Restates awq/quantize/qmodule.py:11-23.
    """
    if group_size >= 128:
        mult = 1
    elif group_size == 64:
        mult = 2
    elif group_size == 32:
        mult = 4
    else:
        raise NotImplementedError(group_size)
    width = -(-(in_features // group_size) // pack_num)
    width = -(-width // mult) * mult
    return width


def scale_rows(in_features: int, group_size: int = 128) -> int:
    """Row count of ``scales`` / ``scaled_zeros`` (awq/quantize/qmodule.py:109-130)."""
    return calculate_zeros_width(in_features, group_size) * PACK_NUM


# --------------------------------------------------------------------------------------
# packed layout (closed form of awq/quantize/qmodule.py:26-65)
# --------------------------------------------------------------------------------------
def packed_index(n, k):
    """Where weight (n, k) lives in ``qweight`` viewed as uint16 ``P[r, c]``.

    Returns (r, c, j): nibble ``j`` (bits 4j..4j+3) of ``P[r, c]``.

    Derivation from pack_intweight (qmodule.py:32-55): inside every 32-k block the
    order is first permuted to [0,1,8,9,16,17,24,25, 2,3,...] (:32-34), then every
    run of 8 is re-ordered [0,2,4,6,1,3,5,7] (:38-40), then 4 rows x 64 k are
    interleaved row-major into one 128-byte segment (:43-48) and 4 consecutive
    elements are packed into one int16, lowest nibble first (:50-55).
    Equivalent statement: in the 16-byte chunk of (row n, 32-k block), viewed as four
    little-endian uint32 ``u``, nibble ``i`` of word ``u`` holds
    ``k_local = 8*(i % 4) + 2*u + i // 4``.
    """
    n = np.asarray(n)
    k = np.asarray(k)
    r = n // 4
    row = n % 4
    tile = k // 64
    blk = (k % 64) // 32
    o = k % 32
    u = (o >> 1) & 3
    i = (o >> 3) + 4 * (o & 1)
    c = tile * 64 + row * 16 + blk * 8 + u * 2 + i // 4
    j = i % 4
    return r, c, j


def pack_intweight(q: np.ndarray) -> np.ndarray:
    """q[N, K] integers  ->  int16 [N//4, K]  (qmodule.py:26-65).

    The reference ORs the four shifted values of one int16 WITHOUT masking (:50-55) and
    then wraps to int16 (:59): integers outside 0..15 corrupt the neighbouring nibbles.
    Restated as is (values in 0..15 are the only ones the quantiser is meant to produce)."""
    q = np.asarray(q).astype(np.int64)
    N, K = q.shape
    assert N % INTERLEAVE == 0 and K % KSTRIDE == 0
    nn, kk = np.meshgrid(np.arange(N), np.arange(K), indexing="ij")
    r, c, j = packed_index(nn, kk)
    out = np.zeros((N // 4, K), dtype=np.int64)
    np.bitwise_or.at(out, (r, c), q << (4 * j))
    return out.astype(np.int16)


def unpack_intweight(qweight: np.ndarray) -> np.ndarray:
    """int16 [N//4, K] -> q[N, K] uint8 in 0..15 (inverse of pack_intweight).

    Structured form of packed_index(): P[r, 64*tile + 16*row + 8*blk + 2*u + hi] nibble j
    is q[4r + row, 64*tile + 32*blk + 8*j + 2*u + hi]."""
    P = np.ascontiguousarray(qweight).view(np.uint16)
    R, K = P.shape
    a = P.reshape(R, K // 64, 4, 2, 4, 2)                           # r, tile, row, blk, u, hi
    nib = (a[..., None] >> (4 * np.arange(4, dtype=np.uint16))) & 0xF   # ..., j
    q = nib.transpose(0, 2, 1, 3, 6, 4, 5)                           # r, row, tile, blk, j, u, hi
    return np.ascontiguousarray(q).reshape(R * 4, K).astype(np.uint8)


def unpack_intweight_indexed(qweight: np.ndarray) -> np.ndarray:
    """Same as unpack_intweight, through packed_index() (slow; cross-check only)."""
    P = np.ascontiguousarray(qweight).view(np.uint16)
    R, K = P.shape
    nn, kk = np.meshgrid(np.arange(R * 4), np.arange(K), indexing="ij")
    r, c, j = packed_index(nn, kk)
    return ((P[r, c] >> (4 * j).astype(np.uint16)) & 0xF).astype(np.uint8)


# --------------------------------------------------------------------------------------
# rounding helpers (exact single rounding from float64)
# --------------------------------------------------------------------------------------
def rn_f16(x: np.ndarray) -> np.ndarray:
    """float64 -> nearest fp16 (RNE), returned as float64."""
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def rn_bf16(x: np.ndarray) -> np.ndarray:
    """float64 -> nearest bfloat16 (RNE, incl. subnormals), returned as float64.

    Done directly from float64 so there is no double rounding through float32.
    """
    x = np.asarray(x, dtype=np.float64)
    m, e = np.frexp(x)                       # x = m * 2**e, 0.5 <= |m| < 1
    e = np.maximum(e, -125)                  # bf16 min normal exponent (2**-126) -> frexp e = -125
    quantum = np.ldexp(1.0, e - 8)           # 8 significant bits
    y = np.round(x / quantum) * quantum      # np.round is round-half-even; division is exact
    big = np.float64(3.3895313892515355e38)  # max bf16
    y = np.where(np.abs(y) > big, np.copysign(np.inf, y), y)
    return np.where(np.isfinite(x), y, x)


def rounder(dtype: str):
    """Round-to-nearest-even into ``dtype``; "f64" = no rounding (the unrounded restatement, used where a fixture
    was produced by the reference's fp32 / fp64 Python)."""
    return {"f16": rn_f16, "fp16": rn_f16, "half": rn_f16,
            "bf16": rn_bf16, "bfloat16": rn_bf16,
            "f64": lambda v: np.asarray(v, dtype=np.float64)}[dtype]


# --------------------------------------------------------------------------------------
# dequantised weight and forward
# --------------------------------------------------------------------------------------
def dequant_weight(qweight, scales, szeros, group_size: int = 128, dtype: str = "f16", rows=None) -> np.ndarray:
    """w~[n,k] = rn_T( q[n,k] * S[k//G, n] + Z[k//G, n] ) as float64 [N, K] (or [len(rows), K]).

    q is the *unsigned* nibble 0..15 (quantization_new/dequantize.cuh:63,69 subtract
    1024 / 64 only, no -8); scale and zero are applied with ONE fused multiply-add in
    the activation dtype (gemv_cuda.cu:161,165; gemm_cuda.cu:306-308,916).
    ``scales``/``szeros`` are the [>=K/G, N] buffers of WQLinear (qmodule.py:109-130);
    padding rows are ignored.  ``rows`` selects output channels (full-size spot checks).
    """
    q = unpack_intweight(qweight)                                # [N, K] uint8
    N, K = q.shape
    G = group_size
    S = np.asarray(scales, dtype=np.float64)[: K // G].T         # [N, K/G]
    Z = np.asarray(szeros, dtype=np.float64)[: K // G].T
    if rows is not None:
        q, S, Z = q[rows], S[rows], Z[rows]
    q = q.astype(np.float64)
    S = np.repeat(S, G, axis=1)
    Z = np.repeat(Z, G, axis=1)
    return rounder(dtype)(q * S + Z)


def wq_linear_forward(x, qweight, scales, szeros, bias=None, group_size: int = 128,
                      dtype: str = "f16", rows=None) -> np.ndarray:
    """Y = X . w~^T (+ bias) in float64 (WQLinear.forward, qmodule.py:201-224).

    The reference accumulates in fp16 (GEMV chains gemv_cuda.cu:195-198, fp16 mma
    gemm_cuda.cu:124-131); accumulation order is not part of the contract, so the
    oracle accumulates exactly (float64) and the tests bound ||Y - Y64|| / ||Y64||.
    """
    w = dequant_weight(qweight, scales, szeros, group_size, dtype, rows)
    x = np.asarray(x, dtype=np.float64)
    y = x.reshape(-1, x.shape[-1]) @ w.T
    if bias is not None:
        b = np.asarray(bias, dtype=np.float64)
        y = y + (b if rows is None else b[rows])
    return y.reshape(*x.shape[:-1], w.shape[0])


def dispatch_is_gemv(x_shape) -> bool:
    """M = numel / last dim; M < 8 -> GEMV, else GEMM (qmodule.py:206)."""
    m = int(np.prod(x_shape)) // int(x_shape[-1])
    return m < 8


# --------------------------------------------------------------------------------------
# quantiser side (produces the tensors the kernels consume)
# --------------------------------------------------------------------------------------
def pseudo_quantize_scales_zeros(w: np.ndarray, group_size: int = 128, n_bit: int = 4):
    """scales, integer zeros per (row, group): awq/quantize/quantizer.py:61-79."""
    w = np.asarray(w, dtype=np.float32)
    N, K = w.shape
    g = w.reshape(-1, group_size)
    mx = g.max(axis=1, keepdims=True)
    mn = g.min(axis=1, keepdims=True)
    max_int = 2 ** n_bit - 1
    scales = np.maximum(mx - mn, np.float32(1e-5)) / np.float32(max_int)
    zeros = np.clip(-np.round(mn / scales), 0, max_int)
    return scales.reshape(N, -1), zeros.reshape(N, -1)


def from_linear(weight, scales, zeros, group_size: int = 128, dtype: str = "f16"):
    """Restates WQLinear.from_linear (qmodule.py:139-199).

    weight [N, K]; scales, zeros [N, K/G] as produced by pseudo_quantize_tensor
    (zeros integer-valued).  ``dtype`` is the dtype of ``linear.weight`` ("f32", "f16",
    "bf16"): torch evaluates every element-wise op in float32 and rounds the result to
    that dtype, which is what ``_r`` mimics.
    Returns (qweight int16 [N/4, K], scales_buf [rows, N], szeros_buf [rows, N]); the
    two buffers are float32 arrays whose values are exactly representable in ``dtype``.
    """
    if dtype == "f32":
        _r = lambda a: np.asarray(a, dtype=np.float32)
    else:
        rn = rounder(dtype)
        _r = lambda a: rn(np.asarray(a, dtype=np.float32).astype(np.float64)).astype(np.float32)
    w = _r(weight)
    s = _r(scales)
    z = _r(zeros)
    N, K = w.shape
    ng = K // group_size
    rows = scale_rows(K, group_size)
    scale_zeros = _r(z * s)                                        # :155
    s_rep = np.repeat(s, group_size, axis=1)
    sz_rep = np.repeat(scale_zeros, group_size, axis=1)
    q = np.round(_r(_r(w + sz_rep) / s_rep)).astype(np.int32)      # :177-184
    qweight = pack_intweight(q)                                    # :186-188 (`|` of nibbles)
    sbuf = np.zeros((rows, N), dtype=np.float32)
    zbuf = np.zeros((rows, N), dtype=np.float32)
    sbuf[:ng] = s.T                                                # :162-172
    zi = np.trunc(z).astype(np.float32)                            # zeros.to(int32) :190
    zbuf[:ng] = (-_r(s * zi)).T                                    # :193-196 (f32 product, cast, negate)
    return qweight, sbuf, zbuf
