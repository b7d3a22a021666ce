#!/usr/bin/env python
"""Benchmark of attention of a prefill chunk over a KV cache (tinychat's multi-round chat and --chunk_prefilling: a chunk
of Sq new tokens after a history, every layer, every chunk) on 1 x H100.

    python bench_kv_cache_attention.py [--steps K] [--warmup W]

Callers, timed on the same inputs in the same process, alternating, three rounds each:
  this            kv_cache_attention(q, cache_k, cache_v, Sk): the caches read in place
  copy+fa         the route it replaces.  FT layout (short_forward's chunk branch): the history copied out of the decode
                  caches with permute / transpose + reshape + contiguous, the chunk's k / v appended, then this build's
                  flash_attn_func; BTHD layout (long_forward): flash_attn_func over the cache views, no copy
  fa_only         the same flash_attn_func call over copies made beforehand (attention alone; FT only)
  flash_attn      flash-attn 2.8.3's flash_attn_func over the same copies (FT) or views (BTHD), when it can be imported
Sk = history + Sq, causal.  A step is one call per layer, every layer with its own caches, chunk and output (8 layers,
more than the 50 MB L2), captured in a CUDA graph and timed with CUDA events, K steps after W warm-up steps.  Per case
and caller: us per call (the best round; all rounds listed), achieved GB/s = (K + V of the Sk visible tokens once per KV
head + q + out) / time, and its share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth).  The outputs of `this` and
`copy+fa` are compared on the timed inputs.  Prints one JSON line with the card's name, power limit and SM clocks.
Synthetic, seeded fp16 data.  Writes nothing in the tree.
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

PEAK_GBPS = 3350.0
LAYERS = 8
MODELS = {"Llama-3-8B": (32, 8, 128), "Qwen2-7B": (28, 4, 128), "Qwen2-0.5B": (14, 2, 64)}
CASES = [(m, "FT", h, c) for m in MODELS for h in (1024, 4096, 8192) for c in (17, 64, 128, 512)] + \
        [(m, "BTHD", 16384 - c, c) for m in MODELS for c in (17, 32, 64)]


def clocks(index):
    """Current and maximum SM clock in MHz (read-only NVML queries); None where NVML is unavailable."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        return {"sm_mhz": pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM),
                "sm_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)}
    except Exception:  # noqa: BLE001
        return {"sm_mhz": None, "sm_max_mhz": None}


def copy_history(kc, vc, xk, xv, start, layout):
    """The caller's keys / values for flash_attn_func: tinychat's chunk branch for FT caches, the cache views for BTHD."""
    import torch
    B, S, Hkv, D = xk.shape
    if layout == "BTHD":
        return kc[:B, :start + S], vc[:B, :start + S]
    keys = kc[:B, :, :, 0:start].permute(0, 3, 1, 2, 4).reshape(B, start, Hkv, D).contiguous()
    values = vc[:B, :, 0:start].transpose(2, 1).reshape(B, start, Hkv, D).contiguous()
    return torch.cat((keys, xk), dim=1), torch.cat((values, xv), dim=1)


def run(args):
    import torch
    import llm_awq_b200 as P
    eng = P.engine()
    device = torch.device("cuda", 0)
    dtype = torch.float16
    try:
        import flash_attn
        from flash_attn import flash_attn_func as fa_func
        fa_version = flash_attn.__version__
    except Exception:  # noqa: BLE001
        fa_func = fa_version = None
    g = torch.Generator(device=device).manual_seed(0)
    results = []
    card = card_info(0)
    clk_before = clocks(0)
    for model, layout, hist, Sq in CASES:
        H, Hkv, D = MODELS[model]
        B, Sk = 1, hist + Sq
        Lmax = Sk + 256  # the caches are longer than the context, as tinychat's are
        layers = []
        for _ in range(LAYERS):
            K = torch.randn(B, Lmax, Hkv, D, generator=g, device=device).to(dtype)
            V = torch.randn(B, Lmax, Hkv, D, generator=g, device=device).to(dtype)
            if layout == "FT":
                kc, vc = K.view(B, Lmax, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous(), V.permute(0, 2, 1, 3).contiguous()
            else:
                kc, vc = K, V
            q = torch.randn(B, Sq, H, D, generator=g, device=device).to(dtype)
            xk, xv = K[:, hist:Sk].contiguous(), V[:, hist:Sk].contiguous()  # the chunk's k / v, already stored
            pre = copy_history(kc, vc, xk, xv, hist, layout) if layout == "FT" else None
            layers.append((q, kc, vc, xk, xv, pre))
            del K, V

        def this(x):
            return eng.kv_cache_attention(x[0], x[1], x[2], Sk)

        def route(x):
            k, v = copy_history(x[1], x[2], x[3], x[4], hist, layout)
            return eng.flash_attn_func(x[0], k, v, 0.0, None, True)

        impls = {"this": lambda: [this(x) for x in layers], "copy+fa": lambda: [route(x) for x in layers]}
        if layout == "FT":
            impls["fa_only"] = lambda: [eng.flash_attn_func(x[0], x[5][0], x[5][1], 0.0, None, True) for x in layers]
        if fa_func is not None:
            if layout == "FT":
                impls["flash_attn"] = lambda: [fa_func(x[0], x[5][0], x[5][1], 0.0, None, True) for x in layers]
            else:
                impls["flash_attn"] = lambda: [fa_func(x[0], x[1][:, :Sk], x[2][:, :Sk], 0.0, None, True) for x in layers]
        graphs, outs, errors = {}, {}, {}
        for key, fn in impls.items():
            try:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    fn()
                side.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=side):
                    outs[key] = fn()
                graphs[key] = gr
            except Exception as e:  # noqa: BLE001  (a backend that cannot take the shape is reported, not timed)
                errors[key] = f"{type(e).__name__}: {str(e).splitlines()[0][:160]}"
        times = {k: [] for k in graphs}
        for _ in range(3):  # alternate the callers
            for key, gr in graphs.items():
                ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
                times[key].append(ms * 1e3 / (args.steps * LAYERS))
        err = None
        if "this" in outs and "copy+fa" in outs:  # the graphs' own outputs, after their last replay
            torch.cuda.synchronize()
            err = 0.0
            for a, b in zip(outs["this"], outs["copy+fa"]):
                a, b = a.double(), b.double()
                num = (a - b).transpose(1, 2).flatten(2).norm(dim=-1)  # per (batch, head) over rows and columns
                den = b.transpose(1, 2).flatten(2).norm(dim=-1).clamp_min(1e-30)
                err = max(err, float((num / den).max()))
        nbytes = 2 * (2 * B * Sk * Hkv * D + 2 * B * Sq * H * D)
        row = {"case": f"{model} {layout} history={hist} Sq={Sq}", "model": model, "layout": layout, "H": H, "Hkv": Hkv,
               "head_dim": D, "batch": B, "Sq": Sq, "Sk": Sk, "causal": True, "bytes": nbytes,
               "max_rel_err_this_vs_copy_fa": err, "impls": {}}
        for key, ts in times.items():
            us = min(ts)
            row["impls"][key] = {"us_per_call": us, "us_runs": ts, "gbps": nbytes / us / 1e3,
                                 "frac_hbm": nbytes / us / 1e3 / PEAK_GBPS}
        for key, e in errors.items():
            row["impls"][key] = {"error": e}
        results.append(row)
        del layers, graphs, outs, impls
        torch.cuda.empty_cache()
    line = {"metric": "attention of a prefill chunk over a KV cache, one call per layer in a CUDA graph, 1xH100",
            "unit": "us per call", "steps": args.steps, "warmup": args.warmup, "layers": LAYERS, "dtype": "fp16",
            "data": "synthetic", "flash_attn_version": fa_version, "torch_version": torch.__version__,
            "peaks": {"hbm_gbps": PEAK_GBPS, "source": "H100 SXM data sheet"}, "card": card,
            "clocks_before": clk_before, "clocks_after": clocks(0), "cases": results}
    print(json.dumps(line))
    for r in results:
        parts = []
        for k, v in r["impls"].items():
            parts.append(f"{k} {v['us_per_call']:7.1f} us {v['frac_hbm']:4.2f} [" +
                         " ".join(f"{t:.1f}" for t in v["us_runs"]) + "]" if "us_per_call" in v else f"{k} n/a")
        print(f"{r['case']:<44} err {r['max_rel_err_this_vs_copy_fa']:.1e} " + " | ".join(parts), file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_kv_cache_attention.py runs on one GPU")
    run(args)


if __name__ == "__main__":
    main()
