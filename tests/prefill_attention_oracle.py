"""Float64 definition of attention over many queries (flash-attn's flash_attn_func / flash_attn_varlen_*_func for the
parameters tinychat passes), the yardstick of ``awq_inference_engine.flash_attn_func`` and
``flash_attn_varlen_qkvpacked_func``.  Test infrastructure only: nothing under ``llm_awq_b200/`` imports it.

  out[b, i, h] = sum_j softmax_j(scale * q[b, i, h] . k[b, j, h // G]) v[b, j, h // G],   G = H / Hkv
over the keys j that query i sees: all of them, or with ``causal`` the keys j <= i + Sk - Sq (bottom-right alignment,
flash-attn >= 2.1).  A row that sees no key is zero.  Packed sequences (``cu_seqlens``) are the concatenation of the
per-sequence results.

``prefill_attention`` is numpy on the CPU; ``prefill_attention_torch`` is the same computation in float64 torch, for the
large GPU cases (pinned to the numpy one in tests/test_prefill_attention_cpu.py)."""
import numpy as np


def _fixed(q, k, v, causal, scale):
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    G = H // Hkv
    kk = np.repeat(k, G, axis=2)
    vv = np.repeat(v, G, axis=2)
    s = np.einsum("bihd,bjhd->bhij", q, kk) * scale
    if causal:
        i = np.arange(Sq)[:, None]
        j = np.arange(Sk)[None, :]
        s = np.where(j <= i + Sk - Sq, s, -np.inf)
    m = s.max(axis=-1, keepdims=True) if Sk else np.zeros(s.shape[:-1] + (1,))
    m = np.where(np.isfinite(m), m, 0.0)
    p = np.exp(s - m)
    l = p.sum(axis=-1, keepdims=True)
    o = np.einsum("bhij,bjhd->bhid", p, vv) / np.where(l > 0, l, 1.0)
    return o.transpose(0, 2, 1, 3)


def prefill_attention(q, k, v, causal, scale, cu_seqlens=None, cu_seqlens_k=None):
    """q [B, Sq, H, D], k / v [B, Sk, Hkv, D] -> [B, Sq, H, D]; with ``cu_seqlens`` ([batch + 1] offsets; for the keys
    ``cu_seqlens_k`` when given, else the same) q [total_q, H, D], k / v [total_k, Hkv, D] -> [total_q, H, D]."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    if cu_seqlens is None:
        return _fixed(q, k, v, causal, scale)
    cq = [int(c) for c in cu_seqlens]
    ck = cq if cu_seqlens_k is None else [int(c) for c in cu_seqlens_k]
    out = np.zeros(q.shape)
    for b in range(len(cq) - 1):
        if cq[b + 1] > cq[b]:
            out[cq[b]:cq[b + 1]] = _fixed(q[None, cq[b]:cq[b + 1]], k[None, ck[b]:ck[b + 1]], v[None, ck[b]:ck[b + 1]],
                                          causal, scale)[0]
    return out


def prefill_attention_torch(q, k, v, causal, scale, heads=None):
    """Fixed-length ``prefill_attention`` in float64 torch on q's device for the query heads ``heads`` (default all):
    returns [B, Sq, len(heads), D]."""
    import torch
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    G = H // Hkv
    heads = list(range(H)) if heads is None else list(heads)
    kv = [h // G for h in heads]
    qd = q[:, :, heads].double().permute(0, 2, 1, 3)
    kd = k[:, :, kv].double().permute(0, 2, 1, 3)
    vd = v[:, :, kv].double().permute(0, 2, 1, 3)
    s = torch.matmul(qd, kd.transpose(-1, -2)) * scale
    if causal:
        i = torch.arange(Sq, device=q.device)[:, None]
        j = torch.arange(Sk, device=q.device)[None, :]
        s = s.masked_fill(j > i + Sk - Sq, float("-inf"))
    m = s.amax(dim=-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp(s - m)
    l = p.sum(dim=-1, keepdim=True)
    o = torch.matmul(p, vd) / torch.where(l > 0, l, torch.ones_like(l))
    return o.permute(0, 2, 1, 3)
