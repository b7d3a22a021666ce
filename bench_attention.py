#!/usr/bin/env python
"""Benchmark of the decode-step attention (`b200awq_single_query_attention`) at the grouped-query shapes of the
language models tinychat decodes, on 1 x H100.

    python bench_attention.py [--steps K] [--warmup W]

Prints one JSON line.  For each model shape, context (512, 2048, 8192 positions) and batch (1, 8), a step is one
decode-attention call per layer, every layer with its own KV cache (so the caches are read from HBM, not from L2), timed
as a CUDA graph of C-ABI launches (include/b200awq.h), K steps after W warm-up steps, CUDA events.  Per case the line
gives the time of one call, the algorithmic bytes of one call (the KV cache read once: 2 n_pos D sizeof(T) per KV head
and batch row, plus q, k, v and the output) and their share of 3.35 TB/s (H100 SXM data sheet).  The G = 8 control has
Qwen2-7B's KV heads, head size and contexts with 32 query heads: it reads the same KV bytes as Qwen2-7B's G = 7.
Falcon-7B's G = 71 runs as nine head groups per KV head; the groups re-read the KV head's bytes, counted once here.
Synthetic, seeded fp16 data.  Writes nothing in the tree.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import timed_steps  # noqa: E402  (the timing helper of the main benchmark)
from bench_siglip import card_info  # noqa: E402

# name: (query heads, KV heads, head size, layers), from the models' config.json
MODELS = {
    "Llama-3-8B": (32, 8, 128, 32),
    "Qwen2-7B": (28, 4, 128, 28),
    "G8-control (Qwen2-7B KV, 32 query heads)": (32, 4, 128, 28),
    "Qwen2-1.5B": (12, 2, 128, 28),
    "Falcon-7B": (71, 1, 64, 32),
}
CONTEXTS = (512, 2048, 8192)
BATCHES = (1, 8)
HBM_TBPS = 3.35


def run(args):
    import torch
    import llm_awq_b200 as P
    device = torch.device("cuda", 0)
    lib = P.lib()
    dtype = torch.float16
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    ws_bytes = max(lib.b200awq_single_query_attention_workspace_bytes(b, h, hk, d, c)
                   for (h, hk, d, _) in MODELS.values() for b in BATCHES for c in CONTEXTS)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=device)
    g = torch.Generator(device=device).manual_seed(0)
    results = []
    for name, (H, Hkv, D, layers) in MODELS.items():
        for B in BATCHES:
            for ctx in CONTEXTS:
                t = ctx - 1  # the cache is full: ctx positions attended to
                qkv = (torch.randn(B, H + 2 * Hkv, D, generator=g, device=device)).to(dtype)
                q, k, v = qkv[:, :H], qkv[:, H:H + Hkv], qkv[:, H + Hkv:]
                kcs = [torch.randn(B, Hkv, D // 8, ctx, 8, generator=g, device=device).to(dtype) for _ in range(layers)]
                vcs = [torch.randn(B, Hkv, ctx, D, generator=g, device=device).to(dtype) for _ in range(layers)]
                out = torch.empty(B, H, D, dtype=dtype, device=device)

                def step():
                    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
                    for kc, vc in zip(kcs, vcs):
                        rc = lib.b200awq_single_query_attention(p(q), p(k), p(v), p(kc), p(vc), p(out), None, B, H, Hkv, D, ctx,
                                                                t, q.stride(0), k.stride(0), v.stride(0), D, 1e6, 1.0, 1, 0,
                                                                p(ws), ws_bytes, st)
                        if rc != 0:
                            raise RuntimeError(lib.b200awq_strerror(rc).decode())

                sg = torch.cuda.Stream()
                with torch.cuda.stream(sg):
                    step()
                sg.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    step()
                ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
                us = ms * 1e3 / (args.steps * layers)
                kv_bytes = 2 * B * Hkv * ctx * D * 2
                byt = kv_bytes + 2 * B * (2 * H + 2 * Hkv) * D
                results.append({"model": name, "H": H, "Hkv": Hkv, "G": H // Hkv, "head_dim": D, "batch": B, "context": ctx,
                                "us_per_call": us, "kv_bytes": kv_bytes, "bytes": byt, "GBps": byt / us / 1e3,
                                "frac_hbm": byt / (us * 1e-6) / (HBM_TBPS * 1e12)})
                del kcs, vcs, gr
                torch.cuda.empty_cache()
    line = {"metric": "decode attention, one call per layer in a CUDA graph, 1xH100", "unit": "us per call",
            "steps": args.steps, "warmup": args.warmup, "dtype": "fp16", "data": "synthetic",
            "peaks": {"hbm_tbps": HBM_TBPS, "source": "H100 SXM data sheet (700 W)"},
            "card": card_info(0), "cases": results}
    print(json.dumps(line))
    for r in results:
        print(f"{r['model']:<42} G={r['G']:<3} D={r['head_dim']:<4} B={r['batch']} ctx={r['context']:<5} "
              f"{r['us_per_call']:8.2f} us  {r['kv_bytes'] / 1e6:8.2f} MB KV  {100 * r['frac_hbm']:5.1f} % of 3.35 TB/s",
              file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_attention.py runs on one GPU")
    run(args)


if __name__ == "__main__":
    main()
