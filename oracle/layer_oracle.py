"""CPU oracle for the ops adjacent to the W4A16 linears inside a decoder layer (SURVEY.md §8f).

TEST INFRASTRUCTURE ONLY -- same rules as ``oracle/w4a16_oracle.py``: nothing under ``llm_awq_b200/`` may import
this file.

Parity status: the reference has no tests or golden vectors for these ops and its kernels are CUDA-only.  The
restatements below are pinned twice:
  * on CPU (``tests/test_layer_oracle_golden.py``) against fixtures produced by the reference's own PYTHON definitions
    of the same ops, imported on the CPU by ``tests/golden/make_golden.py::layer_ops_golden`` ->
    ``tests/golden/reference_layer_ops.npz``: ``RMSNorm._norm`` (tinychat/models/llama.py:24-31),
    ``precompute_freqs_cis`` + ``apply_rotary_emb`` (:39-47, :68-84), ``precompute_freqs`` (:50-57: the table
    ``fused_rope_with_pos`` consumes), and the KV-cache store + softmax attention of the prefill branch
    (tinychat/modules/fused_attn.py:256-305) whose last row a decode step must reproduce; ``mlp_front`` against the
    reference's unmodified ``QuantLlamaMLP.our_llama_mlp`` EXECUTED on CPU over oracle-backed engine calls
    (``make_golden.py::mlp_callsite_golden`` -> ``tests/golden/reference_mlp_callsite.npz``);
  * on the GPU against the reference's own kernels' outputs stored under ``tests/golden/`` (``oracle/_ref``:
    ``layernorm_forward_cuda``) and, for the fused MLP front half, against the composition the reference executes
    (two engine calls + ``F.silu`` + multiply, ``tinychat/modules/fused_mlp.py:36-83``) evaluated with torch.
The reference's attention KERNEL (FasterTransformer template) is not rebuilt (DESIGN.md §4).

Each function cites the reference file:line it restates.
"""
from __future__ import annotations

import numpy as np

from . import w4a16_oracle as O

HALF_CLAMP = 65504.0 - 1000.0   # awq/kernels/csrc/layernorm/reduction.cuh:81 (HALF_FLT_MAX - 1000)


def rmsnorm(x: np.ndarray, gamma: np.ndarray, eps: float, dtype: str = "f16", rounded: bool = True) -> np.ndarray:
    """``generalT5LayerNorm`` (awq/kernels/csrc/layernorm/layernorm.cu:38-64): per row,
    ``var = sum x^2`` (:50-53), ``r = rsqrt(var / n + eps)`` (:57), ``y = clamp_T((x * r) * gamma)`` (:62; the clamp is
    fp16-only, reduction.cuh:72-82).  float64 statistics; one rounding to ``dtype`` when ``rounded``."""
    x = np.asarray(x, dtype=np.float64)
    g = np.asarray(gamma, dtype=np.float64)
    n = x.shape[-1]
    r = 1.0 / np.sqrt((x * x).sum(axis=-1, keepdims=True) / n + eps)
    y = (x * r) * g
    if not rounded:
        return y
    if dtype == "f16":
        y = np.clip(y, -HALF_CLAMP, HALF_CLAMP)
    return O.rounder(dtype)(y)


def silu(x: np.ndarray) -> np.ndarray:
    """``F.silu`` (tinychat/modules/fused_mlp.py:50,78): x * sigmoid(x), float64."""
    x = np.asarray(x, dtype=np.float64)
    return x / (1.0 + np.exp(-x))


def mlp_front(x, gate, up, dtype: str = "f16", rows=None) -> np.ndarray:
    """``QuantLlamaMLP.our_llama_mlp`` (tinychat/modules/fused_mlp.py:36-83) with the zeros tensors AS GIVEN
    (the caller applies the ``- 8 * scales`` of the GEMM branch, :69,76, when it wants that branch):
        gate_out = rn_T(x @ w~_gate^T)   (:40-49 / :65-71)      up_out = rn_T(x @ w~_up^T)   (:51-60 / :72-77)
        c = rn_T( rn_T(silu(gate_out)) * up_out )               (:50,78,80)
    ``gate`` / ``up`` are (qweight, scales, szeros) triples.  Every intermediate is rounded to ``dtype`` exactly
    where the reference materialises a tensor."""
    rn = O.rounder(dtype)
    g = rn(O.wq_linear_forward(x, *gate, dtype=dtype, rows=rows))
    u = rn(O.wq_linear_forward(x, *up, dtype=dtype, rows=rows))
    return rn(rn(silu(g)) * u)


# ------------------------------------------------------------------------------------------------- attention + RoPE
def rope_pair_angles(n_pairs: int, rot_dim: int, t: float, base: float, scale: float) -> np.ndarray:
    """``rotary_embedding_coefficient`` (awq/kernels/csrc/attention/decoder_masked_multihead_attention_utils.h:
    1282-1287): angle of pair ``i`` at step ``t`` = ``(t * scale) / base ** (2 i / rot_dim)``."""
    i = np.arange(n_pairs, dtype=np.float64)
    return (t * scale) / np.power(float(base), 2.0 * i / rot_dim)


def rope_rotate(x: np.ndarray, t: float, rot_dim: int, base: float, scale: float, neox: bool, dtype: str) -> np.ndarray:
    """Rotate the last dimension of ``x`` ([..., D]) at position ``t`` and round to ``dtype``
    (decoder_masked_multihead_attention_template.hpp:1080-1135 with utils.h:1290-1296: x' = c x - s y, y' = c y + s x;
    neox style pairs (i, i + rot_dim / 2), :1088-1135, else (2 i, 2 i + 1), :1080-1087; the vectors are of T)."""
    x = np.array(x, dtype=np.float64)
    out = x.copy()
    half = rot_dim // 2
    ang = rope_pair_angles(half, rot_dim, t, base, scale)
    c, s = np.cos(ang), np.sin(ang)
    if neox:
        a, b = x[..., :half], x[..., half:rot_dim]
        out[..., :half], out[..., half:rot_dim] = c * a - s * b, c * b + s * a
    else:
        a, b = x[..., 0:rot_dim:2], x[..., 1:rot_dim:2]
        out[..., 0:rot_dim:2], out[..., 1:rot_dim:2] = c * a - s * b, c * b + s * a
    return O.rounder(dtype)(out)


def single_query_attention(q, k, v, k_cache, v_cache, timestep, rot_dim, base=10000.0, scale=1.0, neox=True, dtype="f16",
                           length_per_sample=None):
    """``single_query_attention`` (awq/kernels/csrc/attention/ft_attention.cpp:112-184 ->
    decoder_masked_multihead_attention_template.hpp).  q [B, H, D], k / v [B, Hkv, D]; k_cache [B, Hkv, D / 8, L, 8] and
    v_cache [B, Hkv, L, D] are UPDATED IN PLACE (float64 arrays holding T values) at slot t % L (:1148-1175, :1424-1440);
    returns out [B, H, D] rounded to T.  tlength per sample = length_per_sample[b] or timestep (:975-978); positions
    attended to: max(0, t + 1 - L) .. t (:979); logits = q . k / sqrt(D) (:1200, :1323), softmax and the sum over
    positions in float64 (the reference: fp32, logits rounded to T before the product with V -- accumulation-level
    differences, covered by the tests' tolerance)."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    B, H, D = q.shape
    Hkv, L = v_cache.shape[1], v_cache.shape[2]
    G = H // Hkv
    rn = O.rounder(dtype)
    out = np.zeros((B, H, D))
    for b in range(B):
        t = int(length_per_sample[b]) if length_per_sample is not None else int(timestep)
        qr = rope_rotate(q[b], t, rot_dim, base, scale, neox, dtype) if rot_dim > 0 else q[b]
        kr = rope_rotate(k[b], t, rot_dim, base, scale, neox, dtype) if rot_dim > 0 else k[b]
        slot = t % L
        k_cache[b, :, :, slot, :] = kr.reshape(Hkv, D // 8, 8)
        v_cache[b, :, slot, :] = v[b]
        first = max(0, t + 1 - L)
        slots = [p % L for p in range(first, t + 1)]
        for h in range(H):
            kv = h // G
            K = k_cache[b, kv][:, slots, :].transpose(1, 0, 2).reshape(len(slots), D)
            V = v_cache[b, kv][slots]
            s = (K @ qr[h]) / np.sqrt(D)
            p = np.exp(s - s.max())
            out[b, h] = (p / p.sum()) @ V
    return rn(out)


def rope_with_pos(x: np.ndarray, freqs: np.ndarray, dtype: str = "f16") -> np.ndarray:
    """``fused_rope_with_pos_forward_func`` (awq/kernels/csrc/rope_new/fused_rope_with_pos.cu:33-75): x [s, b, h, d],
    angle of (s_id, b_id, i) = freqs.flat[(b_id * S + s_id) * d2 + i] (:46); y = x cos + rot(x) sin for i < d2 with
    rot(x)[i] = -x[i + d2/2] (i < d2/2) else x[i - d2/2] (:51-56); the rest copied (:60-72); fp32 math, one rounding."""
    x = np.asarray(x, dtype=np.float64)
    S, B, Hh, D = x.shape
    d2 = freqs.shape[-1]
    f = np.asarray(freqs, dtype=np.float64).reshape(-1)[: B * S * d2].reshape(B, S, d2).transpose(1, 0, 2)[:, :, None, :]
    y = x.copy()
    xr = x[..., :d2]
    rot = np.concatenate([-xr[..., d2 // 2:], xr[..., : d2 // 2]], axis=-1)
    y[..., :d2] = xr * np.cos(f) + rot * np.sin(f)
    return O.rounder(dtype)(y)


def neox_cos_sin_cache(dim: int, max_position: int, base: float = 10000.0, dtype: str = "f16") -> np.ndarray:
    """``QuantLlamaRotaryEmbedding._set_cos_sin_cache`` (tinychat/modules/fused_attn.py:26-59): row p =
    [cos(p f_0) .. cos(p f_{dim/2-1}), sin(p f_0) .. sin(p f_{dim/2-1})] with f_i = base ** (-2 i / dim), computed in
    fp32 by the reference and stored as fp16 (:59); here float64, rounded to ``dtype``."""
    inv = 1.0 / np.power(float(base), np.arange(0, dim, 2, dtype=np.float64) / dim)
    ang = np.outer(np.arange(max_position, dtype=np.float64), inv)
    return O.rounder(dtype)(np.concatenate([np.cos(ang), np.sin(ang)], axis=-1))


def rotary_embedding_neox(positions, query, key, head_size: int, cos_sin_cache, dtype: str = "f16"):
    """``rotary_embedding_neox`` (awq/kernels/csrc/position_embedding/pos_encoding_kernels.cu:13-88): query / key
    [tokens, heads, head_size] (any leading shape with tokens * heads * head_size elements), positions [tokens],
    cos_sin_cache [max_position, rot_dim].  Per token and head, pair r < rot_dim / 2 (:33-36):
    x' = x cos_r - y sin_r, y' = y cos_r + x sin_r with x = head[r], y = head[rot_dim / 2 + r] (:44-52); the rest of the
    head is untouched.  Returns NEW arrays (the kernel works in place); float64 products, one rounding to ``dtype``
    (the reference rounds after every operation of T: <= 2 ulp of T away)."""
    pos = np.asarray(positions).reshape(-1)
    cache = np.asarray(cos_sin_cache, dtype=np.float64)
    rot = cache.shape[1]
    e = rot // 2
    rn = O.rounder(dtype)
    outs = []
    for t in (query, key):
        a = np.array(t, dtype=np.float64)
        v = a.reshape(len(pos), -1, head_size)
        c, s = cache[pos][:, None, :e], cache[pos][:, None, e:rot]
        x, y = v[..., :e].copy(), v[..., e:rot].copy()
        v[..., :e], v[..., e:rot] = rn(x * c - y * s), rn(y * c + x * s)
        outs.append(v.reshape(a.shape))
    return outs[0], outs[1]
