"""Seeded inputs of the grouped-query decode-attention cases shared by tests/test_attention_gqa_gpu.py and
tests/golden/make_attention_ref_kernel_golden.py (the stored outputs of the reference's own kernel are regenerated from
the same seeds, bit for bit).

q, k and v are views of one fused QKV buffer [B, H + 2 Hkv, D], as tinychat slices its QKV projection: their batch
stride is (H + 2 Hkv) D, and the reference applies q's batch stride to all three
(awq/kernels/csrc/attention/decoder_masked_multihead_attention_template.hpp:967-969)."""
import torch

# (B, H, Hkv, D, L, t): the model shapes of the grouped-query ratios and the head sizes the reference dispatches
# (decoder_masked_multihead_attention.cu:68-99) beyond 64 / 128 / 256, at single-CTA, split and wrapped contexts.
REF_CASES = [
    (1, 28, 4, 128, 4096, 2500),   # Qwen2-7B, G = 7, split over CTAs
    (2, 12, 2, 128, 512, 300),     # Qwen2-1.5B, G = 6, batch 2
    (1, 14, 2, 64, 256, 300),      # Qwen2.5-0.5B, G = 7, circular wrap
    (1, 40, 8, 128, 1024, 37),     # Qwen2.5-14B, G = 5
    (1, 24, 8, 128, 512, 0),       # Llama-3.2-3B, G = 3, empty cache
    (2, 71, 1, 64, 2304, 2100),    # Falcon-7B, G = 71 (nine head groups), split, batch 2
    (1, 24, 2, 64, 300, 100),      # G = 12 (two head groups of six)
] + [(1, 14, 2, d, 512, 200) for d in (48, 80, 96, 112, 160, 192, 224)] \
  + [(1, 4, 4, d, 300, 299) for d in (48, 80, 96, 112, 160, 192, 224)]
ROPE_BASE = 1000000.0  # Qwen2's rope_theta; neox style over the whole head


def case_id(case):
    return "B{}_H{}_Hkv{}_D{}_L{}_t{}".format(*case)


def fused_qkv(B, H, Hkv, D, dtype, seed, device):
    """Returns (qkv, q, k, v): q [B, H, D], k / v [B, Hkv, D] as views of qkv [B, H + 2 Hkv, D]."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, H + 2 * Hkv, D, generator=g).to(dtype).to(device)
    return qkv, qkv[:, :H], qkv[:, H:H + Hkv], qkv[:, H + Hkv:]


def caches(B, Hkv, D, L, dtype, fill_to, seed, device):
    """k_cache [B, Hkv, D / 8, L, 8] and v_cache [B, Hkv, L, D] with slots 0 .. fill_to - 1 random, the rest zero."""
    g = torch.Generator().manual_seed(seed)
    kc = torch.zeros(B, Hkv, D // 8, L, 8)
    vc = torch.zeros(B, Hkv, L, D)
    kc[:, :, :, :fill_to] = torch.randn(B, Hkv, D // 8, fill_to, 8, generator=g)
    vc[:, :, :fill_to] = torch.randn(B, Hkv, fill_to, D, generator=g)
    return kc.to(dtype).to(device), vc.to(dtype).to(device)


def ref_case_inputs(case, dtype, device):
    """(q, k, v, k_cache, v_cache) of a REF_CASES entry."""
    B, H, Hkv, D, L, t = case
    _, q, k, v = fused_qkv(B, H, Hkv, D, dtype, seed=1000 * B + H + D + t, device=device)
    kc, vc = caches(B, Hkv, D, L, dtype, min(t, L), seed=t + D + 7, device=device)
    return q, k, v, kc, vc
