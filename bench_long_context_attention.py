#!/usr/bin/env python
"""Benchmark of attention of few queries over many keys (tinychat's long_forward decode: `flash_attn_func(q, k, v,
causal=True)` with q [B, Sq, H, D] and k / v views cache[:, :Sk] of [B, Lmax, Hkv, D] caches) on 1 x H100.

    python bench_long_context_attention.py [--steps K] [--warmup W]

Callers, timed on the same inputs in the same process, alternating, three rounds each:
  this            this build's flash_attn_func (the split-key kernel when Sq * H / Hkv <= 64, else the prefill kernel)
  prefill_kernel  b200awq_prefill_attention called directly (the route every such call took before the split-key kernel)
  single_query    single_query_attention over the same context in tinychat's decode-cache layout (Sq = 1 only)
  flash_attn      flash-attn 2.8.3's flash_attn_func, when it can be imported
  sdpa_flash      torch's scaled_dot_product_attention with the flash backend
A step is one call per layer, every layer with its own caches, query and output (8 layers), captured in a CUDA graph and
timed with CUDA events, K steps after W warm-up steps.  Per case and caller: us per call (the best round; all rounds
listed), achieved GB/s = (K + V + q + out bytes of the call) / time, and its share of 3.35 TB/s (H100 SXM data sheet
HBM3 bandwidth).  Prints one JSON line with the card's name and power limit.  Synthetic, seeded fp16 data.  Writes
nothing in the tree.
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

PEAK_GBPS = 3350.0
LAYERS = 8

# name: (H, Hkv, D, batch, Sq, Sk)
CASES = {
    "Llama-3-8B Sq=1 Sk=8192": (32, 8, 128, 1, 1, 8192),
    "Llama-3-8B Sq=1 Sk=16384": (32, 8, 128, 1, 1, 16384),
    "Llama-3-8B Sq=1 Sk=32768": (32, 8, 128, 1, 1, 32768),
    "Llama-3-8B Sq=1 Sk=131072": (32, 8, 128, 1, 1, 131072),
    "Llama-3-8B B=8 Sq=1 Sk=8192": (32, 8, 128, 8, 1, 8192),
    "Llama-3-8B B=8 Sq=1 Sk=32768": (32, 8, 128, 8, 1, 32768),
    "Qwen2-7B Sq=1 Sk=16384": (28, 4, 128, 1, 1, 16384),
    "Qwen2-7B Sq=1 Sk=32768": (28, 4, 128, 1, 1, 32768),
    "Qwen2-0.5B Sq=1 Sk=16384": (14, 2, 64, 1, 1, 16384),
    "Qwen2-0.5B Sq=1 Sk=32768": (14, 2, 64, 1, 1, 32768),
    "Llama-3-8B Sq=4 Sk=16384": (32, 8, 128, 1, 4, 16384),
    "Llama-3-8B Sq=8 Sk=16384": (32, 8, 128, 1, 8, 16384),
    "Llama-3-8B Sq=16 Sk=16384 (Sq*G=64: split-key)": (32, 8, 128, 1, 16, 16384),
    "Llama-3-8B Sq=17 Sk=16384 (Sq*G=68: prefill)": (32, 8, 128, 1, 17, 16384),
}


def run(args):
    import torch
    import torch.nn.functional as F
    import llm_awq_b200 as P
    eng = P.engine()
    lib = P.lib()
    device = torch.device("cuda", 0)
    dtype = torch.float16
    try:
        import flash_attn
        from flash_attn import flash_attn_func as fa_func
        fa_version = flash_attn.__version__
    except Exception:  # noqa: BLE001
        fa_func = fa_version = None
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from torch.nn.attention.bias import causal_lower_right
    g = torch.Generator(device=device).manual_seed(0)
    results = []
    for name, (H, Hkv, D, B, Sq, Sk) in CASES.items():
        Lmax = Sk + 256  # the caches are longer than the context: k / v are views, as in long_forward
        layers = []
        for _ in range(LAYERS):
            kc = torch.randn(B, Lmax, Hkv, D, generator=g, device=device).to(dtype)
            vc = torch.randn(B, Lmax, Hkv, D, generator=g, device=device).to(dtype)
            q = torch.randn(B, Sq, H, D, generator=g, device=device).to(dtype)
            layers.append((q, kc[:, :Sk], vc[:, :Sk], torch.empty_like(q)))
        st = lambda t: (ctypes.c_longlong * 3)(t.stride(0), t.stride(1), t.stride(2))
        stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def this(x):
            return eng.flash_attn_func(x[0], x[1], x[2], 0.0, None, True)

        def prefill_kernel(x):
            q, k, v, out = x
            rc = lib.b200awq_prefill_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), None, None, B, Sq,
                                               Sk, H, Hkv, D, st(q), st(k), st(v), ctypes.c_float(D ** -0.5), 1, 0, stream())
            assert rc == 0, rc

        def fa(x):
            return fa_func(x[0], x[1], x[2], 0.0, None, True)

        bias = causal_lower_right(Sq, Sk) if Sq > 1 else None

        def sdpa(x):
            q, k, v = (t.transpose(1, 2) for t in x[:3])
            with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
                if bias is not None:
                    return F.scaled_dot_product_attention(q, k, v, attn_mask=bias, enable_gqa=H != Hkv)
                return F.scaled_dot_product_attention(q, k, v, enable_gqa=H != Hkv)  # one query sees every key

        impls = {"this": lambda: [this(x) for x in layers], "prefill_kernel": lambda: [prefill_kernel(x) for x in layers],
                 "sdpa_flash": lambda: [sdpa(x) for x in layers]}
        if fa_func is not None:
            impls["flash_attn"] = lambda: [fa(x) for x in layers]
        dec_state = None
        if Sq == 1:  # the decode kernel on the same context, tinychat's FT cache layout
            kcs = [torch.randn(B, Hkv, D // 8, Sk, 8, generator=g, device=device).to(dtype) for _ in range(LAYERS)]
            vcs = [torch.randn(B, Hkv, Sk, D, generator=g, device=device).to(dtype) for _ in range(LAYERS)]
            qd = torch.randn(B, H + 2 * Hkv, D, generator=g, device=device).to(dtype)
            dec_state = (kcs, vcs)
            q1, k1, v1 = qd[:, :H], qd[:, H:H + Hkv], qd[:, H + Hkv:]
            impls["single_query"] = lambda: [eng.single_query_attention(q1, k1, v1, a, b, None, None, Sk - 1, 0, 10000.0, 1.0,
                                                                        True) for a, b in zip(kcs, vcs)]
        graphs, errors = {}, {}
        for key, fn in impls.items():
            try:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    fn()
                side.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=side):
                    fn()
                graphs[key] = gr
            except Exception as e:  # noqa: BLE001  (a backend that cannot take the shape is reported, not timed)
                errors[key] = f"{type(e).__name__}: {str(e).splitlines()[0][:160]}"
        times = {k: [] for k in graphs}
        for _ in range(3):  # alternate the callers
            for key, gr in graphs.items():
                ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
                times[key].append(ms * 1e3 / (args.steps * LAYERS))
        nbytes = 2 * (2 * B * Sk * Hkv * D + 2 * B * Sq * H * D)
        row = {"case": name, "H": H, "Hkv": Hkv, "head_dim": D, "batch": B, "Sq": Sq, "Sk": Sk, "causal": True,
               "bytes": nbytes, "route": "split-key" if Sq * (H // Hkv) <= 64 else "prefill", "impls": {}}
        for key, ts in times.items():
            us = min(ts)
            row["impls"][key] = {"us_per_call": us, "us_runs": ts, "gbps": nbytes / us / 1e3,
                                 "frac_hbm": nbytes / us / 1e3 / PEAK_GBPS}
        for key, err in errors.items():
            row["impls"][key] = {"error": err}
        results.append(row)
        del layers, graphs, dec_state, impls
        torch.cuda.empty_cache()
    line = {"metric": "attention of few queries over a long context, one call per layer in a CUDA graph, 1xH100",
            "unit": "us per call", "steps": args.steps, "warmup": args.warmup, "layers": LAYERS, "dtype": "fp16",
            "data": "synthetic", "flash_attn_version": fa_version, "torch_version": torch.__version__,
            "peaks": {"hbm_gbps": PEAK_GBPS, "source": "H100 SXM data sheet"}, "card": card_info(0), "cases": results}
    print(json.dumps(line))
    for r in results:
        parts = []
        for k, v in r["impls"].items():
            parts.append(f"{k} {v['us_per_call']:8.1f} us {v['frac_hbm']:5.2f}" if "us_per_call" in v else f"{k} n/a")
        print(f"{r['case']:<48} " + " | ".join(parts), file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_long_context_attention.py runs on one GPU")
    run(args)


if __name__ == "__main__":
    main()
