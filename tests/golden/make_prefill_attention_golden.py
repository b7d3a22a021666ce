#!/usr/bin/env python
"""Stored outputs of flash-attn 2.8.3 (the installed package, not the reference checkout) on an H100, for the callers'
attention shapes at reduced sizes, in fp16 and bf16 -> tests/golden/reference_kernels_prefill_attention.npz.

    python tests/golden/make_prefill_attention_golden.py [OUT.npz]

Cases (seeded inputs): Llama-3 / Qwen2 causal prefill with grouped-query heads (D = 128, 64), a bottom-right chunk
(512 queries over 1536 keys), SigLIP (D = 72, non-causal, views of a fused qkv buffer), InternViT through
flash_attn_varlen_qkvpacked_func with uniform and ragged cu_seqlens.  Only sampled heads and rows of the outputs are
stored, as raw 16-bit patterns; the inputs are rebuilt from their seeds by `inputs` (shared with the test)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
DEV = "cuda:0"

# name: (kind, B, Sq, Sk, H, Hkv, D, causal); kind "fixed" or the varlen sequence lengths
CASES = {
    "llama3_prefill": ("fixed", 1, 384, 384, 8, 2, 128, True),
    "qwen2_small_prefill": ("fixed", 2, 200, 200, 14, 2, 64, True),
    "chunk_bottom_right": ("fixed", 1, 512, 1536, 4, 1, 128, True),
    "siglip": ("fixed", 2, 729, 729, 4, 4, 72, False),
    "internvit_uniform": ([257, 257], 0, 0, 0, 4, 4, 64, False),
    "varlen_ragged": ([1, 17, 0, 300, 129], 0, 0, 0, 4, 4, 128, True),
}


def bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy()


def inputs(name, dtype, device):
    """Seeded inputs of a case (CPU generator, so the test rebuilds them bit for bit): (q, k, v) for the fixed-length
    cases, (qkv, cu_seqlens, max_seqlen) for the packed ones."""
    kind, B, Sq, Sk, H, Hkv, D, _ = CASES[name]
    g = torch.Generator().manual_seed(100 + list(CASES).index(name))
    if kind != "fixed":
        qkv = torch.randn(sum(kind), 3, H, D, generator=g).to(dtype).to(device)
        cu = torch.tensor(np.concatenate([[0], np.cumsum(kind)]), dtype=torch.int32, device=device)
        return qkv, cu, max(kind)
    if name == "siglip":  # views of a fused qkv buffer, as fused_siglipdecoder.py:162-167 builds them
        buf = torch.randn(B * Sq, 3 * H * D, generator=g).to(dtype).to(device)
        return tuple(t.reshape(B, Sq, H, D) for t in buf.split([H * D] * 3, dim=-1))
    return (torch.randn(B, Sq, H, D, generator=g).to(dtype).to(device), torch.randn(B, Sk, Hkv, D, generator=g).to(dtype).to(device),
            torch.randn(B, Sk, Hkv, D, generator=g).to(dtype).to(device))


def sampled(name):
    """(heads, rows) stored of a case's output: first, middle and last head; 64 (packed: 96) rows spread evenly."""
    kind, B, Sq, Sk, H, Hkv, D, _ = CASES[name]
    n = Sq if kind == "fixed" else sum(kind)
    return (np.array(sorted({0, H // 2, H - 1}), dtype=np.int64),
            np.unique(np.linspace(0, n - 1, 64 if kind == "fixed" else 96).astype(np.int64)))


def main(path):
    from flash_attn import flash_attn_func, flash_attn_varlen_qkvpacked_func
    import flash_attn
    assert flash_attn.__version__ == "2.8.3", flash_attn.__version__
    out = {}
    for name, (kind, B, Sq, Sk, H, Hkv, D, causal) in CASES.items():
        heads, rows = sampled(name)
        h, r = torch.from_numpy(heads).to(DEV), torch.from_numpy(rows).to(DEV)
        for dtype, tag in ((torch.float16, "f16"), (torch.bfloat16, "bf16")):
            x = inputs(name, dtype, DEV)
            if kind == "fixed":
                o = flash_attn_func(*x, 0.0, softmax_scale=D ** -0.5, causal=causal)[:, r][:, :, h]
            else:
                o = flash_attn_varlen_qkvpacked_func(*x, 0.0, softmax_scale=D ** -0.5, causal=causal)[r][:, h]
            out[f"{name}__{tag}"] = bits(o)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "reference_kernels_prefill_attention.npz"))
