#!/usr/bin/env python
"""Benchmark of attention over many queries (`flash_attn_func` / `flash_attn_varlen_qkvpacked_func` of this build:
the sm_90a TMA + wgmma kernel) at the callers' shapes, on 1 x H100, against flash-attn 2.8.3 (when it can be imported)
and torch's scaled_dot_product_attention with the flash backend, timed on the same inputs in the same process,
alternating.

    python bench_prefill_attention.py [--steps K] [--warmup W]

Prints one JSON line.  A step is one call per layer, every layer with its own q, k, v and output (8 layers), captured
in a CUDA graph and timed with CUDA events, K steps after W warm-up steps.  Per case and implementation: us per call,
algorithmic TFLOP/s = 4 D H (visible query-key pairs) / time, and its share of 989 TFLOP/s (H100 SXM data sheet, dense
fp16, 700 W).  A causal pair count is sum_i clamp(i + Sk - Sq + 1, 0, Sk) (bottom-right alignment).  The Sq = 1 case
(tinychat's long_forward decode) is also timed through single_query_attention on the same context.  Synthetic, seeded
fp16 data.  Writes nothing in the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import timed_steps  # noqa: E402  (the timing helper of the main benchmark)
from bench_siglip import card_info  # noqa: E402

PEAK_TFLOPS = 989.0
LAYERS = 8

# name: (H, Hkv, D, batch, Sq, Sk, causal, packed)
CASES = {
    "Llama-3-8B prefill S=2048": (32, 8, 128, 1, 2048, 2048, True, False),
    "Llama-3-8B prefill S=8192": (32, 8, 128, 1, 8192, 8192, True, False),
    "Llama-3-8B chunk 512 over 4096 prefix": (32, 8, 128, 1, 512, 4608, True, False),
    "Qwen2-7B prefill S=2048": (28, 4, 128, 1, 2048, 2048, True, False),
    "SigLIP-so400m 1 image": (16, 16, 72, 1, 1024, 1024, False, False),
    "SigLIP-so400m 8 images": (16, 16, 72, 8, 1024, 1024, False, False),
    "InternViT-300M 1 image (varlen)": (16, 16, 64, 1, 1025, 1025, False, True),
    "InternViT-300M 8 images (varlen)": (16, 16, 64, 8, 1025, 1025, False, True),
    "Llama-3-8B Sq=1 over 16384 keys": (32, 8, 128, 1, 1, 16384, True, False),
}


def visible_pairs(Sq, Sk, causal):
    if not causal:
        return Sq * Sk
    return sum(min(max(i + Sk - Sq + 1, 0), Sk) for i in range(Sq))


def run(args):
    import torch
    import torch.nn.functional as F
    import llm_awq_b200 as P
    eng = P.engine()
    device = torch.device("cuda", 0)
    dtype = torch.float16
    try:
        import flash_attn
        from flash_attn import flash_attn_func as fa_func, flash_attn_varlen_qkvpacked_func as fa_varlen
        fa_version = flash_attn.__version__
    except Exception:  # noqa: BLE001
        fa_func = fa_varlen = fa_version = None
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from torch.nn.attention.bias import causal_lower_right
    g = torch.Generator(device=device).manual_seed(0)
    results = []
    for name, (H, Hkv, D, B, Sq, Sk, causal, packed) in CASES.items():
        layers = []
        for _ in range(LAYERS):
            if packed:
                qkv = torch.randn(B * Sq, 3, H, D, generator=g, device=device).to(dtype)
                layers.append((qkv,))
            elif "SigLIP" in name:  # views of the fused qkv output, as the tower passes them
                buf = torch.randn(B * Sq, 3 * H * D, generator=g, device=device).to(dtype)
                layers.append(tuple(t.reshape(B, Sq, H, D) for t in buf.split([H * D] * 3, dim=-1)))
            else:
                layers.append((torch.randn(B, Sq, H, D, generator=g, device=device).to(dtype),
                               torch.randn(B, Sk, Hkv, D, generator=g, device=device).to(dtype),
                               torch.randn(B, Sk, Hkv, D, generator=g, device=device).to(dtype)))
        cu = torch.arange(0, (B + 1) * Sq, step=Sq, dtype=torch.int32, device=device)

        def ours(x):
            if packed:
                return eng.flash_attn_varlen_qkvpacked_func(x[0], cu, Sq, 0.0, None, causal)
            return eng.flash_attn_func(*x, 0.0, None, causal)

        def fa(x):
            if packed:
                return fa_varlen(x[0], cu, Sq, 0.0, None, causal)
            return fa_func(*x, 0.0, None, causal)

        bias = causal_lower_right(Sq, Sk) if causal and Sq != Sk else None

        def sdpa(x):
            if packed:
                q, k, v = (x[0].view(B, Sq, 3, H, D)[:, :, i].transpose(1, 2) for i in range(3))
            else:
                q, k, v = (t.transpose(1, 2) for t in x)
            with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
                if bias is not None:
                    return F.scaled_dot_product_attention(q, k, v, attn_mask=bias, enable_gqa=H != Hkv)
                return F.scaled_dot_product_attention(q, k, v, is_causal=causal, enable_gqa=H != Hkv)

        impls = {"this": ours, "sdpa_flash": sdpa}
        if fa_func is not None:
            impls["flash_attn"] = fa
        graphs, errors = {}, {}
        for key, fn in impls.items():
            try:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for x in layers:
                        fn(x)
                side.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    for x in layers:
                        fn(x)
                graphs[key] = gr
            except Exception as e:  # noqa: BLE001  (a backend that cannot take the shape is reported, not timed)
                errors[key] = f"{type(e).__name__}: {str(e).splitlines()[0][:160]}"
        times = {k: [] for k in graphs}
        for _ in range(3):  # alternate the implementations
            for key, gr in graphs.items():
                ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
                times[key].append(ms * 1e3 / (args.steps * LAYERS))
        flops = 4.0 * D * H * B * visible_pairs(Sq, Sk, causal)
        row = {"case": name, "H": H, "Hkv": Hkv, "head_dim": D, "batch": B, "Sq": Sq, "Sk": Sk, "causal": causal,
               "varlen": packed, "flop": flops, "impls": {}}
        for key, ts in times.items():
            us = min(ts)
            row["impls"][key] = {"us_per_call": us, "us_runs": ts, "tflops": flops / us / 1e6,
                                 "frac_peak": flops / us / 1e6 / PEAK_TFLOPS}
        for key, err in errors.items():
            row["impls"][key] = {"error": err}
        if Sq == 1:  # the decode kernel on the same context
            kc = [torch.randn(B, Hkv, D // 8, Sk, 8, generator=g, device=device).to(dtype) for _ in range(LAYERS)]
            vc = [torch.randn(B, Hkv, Sk, D, generator=g, device=device).to(dtype) for _ in range(LAYERS)]
            qd = torch.randn(B, H + 2 * Hkv, D, generator=g, device=device).to(dtype)
            q1, k1, v1 = qd[:, :H], qd[:, H:H + Hkv], qd[:, H + Hkv:]

            def dec():
                for a, b in zip(kc, vc):
                    eng.single_query_attention(q1, k1, v1, a, b, None, None, Sk - 1, 0, 10000.0, 1.0, True)
            dec()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                dec()
            ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
            us = ms * 1e3 / (args.steps * LAYERS)
            row["impls"]["single_query_attention"] = {"us_per_call": us, "tflops": flops / us / 1e6,
                                                      "frac_peak": flops / us / 1e6 / PEAK_TFLOPS}
            del kc, vc
        results.append(row)
        del layers, graphs
        torch.cuda.empty_cache()
    line = {"metric": "attention over many queries, one call per layer in a CUDA graph, 1xH100", "unit": "us per call",
            "steps": args.steps, "warmup": args.warmup, "layers": LAYERS, "dtype": "fp16", "data": "synthetic",
            "flash_attn_version": fa_version, "torch_version": torch.__version__,
            "peaks": {"fp16_dense_tflops": PEAK_TFLOPS, "source": "H100 SXM data sheet (700 W)"},
            "card": card_info(0), "cases": results}
    print(json.dumps(line))
    for r in results:
        parts = []
        for k, v in r["impls"].items():
            parts.append(f"{k} {v['us_per_call']:9.1f} us {v['tflops']:6.1f} TF/s" if "us_per_call" in v else f"{k} n/a")
        print(f"{r['case']:<40} " + " | ".join(parts), file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_prefill_attention.py runs on one GPU")
    run(args)


if __name__ == "__main__":
    main()
