#!/usr/bin/env python
"""Benchmark of RoPE + the KV-cache store of a chunk (tinychat's chunked prefill and long_forward's decode: every layer,
every chunk, between the qkv linear and attention) on 1 x H100.

    python bench_rope_kv_store.py [--steps K] [--warmup W]

Callers, timed on the same inputs in the same process, alternating, three rounds each:
  this            rope_kv_store(qkv, freqs, cache_k, cache_v, start_pos): one launch
  composed        tinychat's code over this build's ops: fused_rope_with_pos_forward_func on q, then on k, then the
                  stores (FT: transpose of v, permute + contiguous of k, two slice assignments; BTHD: two slice
                  assignments)
  this+attn       `this`, then kv_cache_attention(q, cache_k, cache_v, start_pos + S)
  composed+attn   `composed`, then the same kv_cache_attention call
A step is one call per layer, every layer with its own qkv, caches and output (8 layers, more than the 50 MB L2),
captured in a CUDA graph and timed with CUDA events, K steps after W warm-up steps.  Per case and caller: us per call
(the best round; all rounds listed).  For `this` and `composed`: achieved GB/s of the algorithmic bytes (qkv read once,
rotated q, k and v written once, the angles read once) and its share of 3.35 TB/s (H100 SXM data sheet HBM3
bandwidth).  The outputs (q, both caches, attention) of `this` and `composed` are compared bit for bit on the timed
inputs.  Prints one JSON line with the card's name, power limit and SM clocks.  Synthetic, seeded fp16 data, batch 1.
Writes nothing in the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import timed_steps  # noqa: E402  (the timing helper of the main benchmark)
from bench_kv_cache_attention import clocks  # noqa: E402
from bench_siglip import card_info  # noqa: E402

PEAK_GBPS = 3350.0
LAYERS = 8
MODELS = {"Llama-3-8B": (32, 8, 128), "Qwen2-7B": (28, 4, 128), "Qwen2-0.5B": (14, 2, 64)}
CASES = [(m, "FT", h, c) for m in MODELS for h in (1024, 8192) for c in (17, 128, 512, 2048)] + \
        [(m, "BTHD", 16383, 1) for m in MODELS] + [(m, "BTHD", 16384 - c, c) for m in MODELS for c in (17, 64)]


def composed(eng, xqkv, freqs, kc, vc, start, H, Hkv, layout):
    """tinychat's code between the qkv linear and attention (fused_attn.py, short_forward's prefill branch for FT
    caches, long_forward for BTHD caches)."""
    B, S, _, D = xqkv.shape
    xq = eng.fused_rope_with_pos_forward_func(xqkv[:, :, :H], freqs, True)
    xk = eng.fused_rope_with_pos_forward_func(xqkv[:, :, H:H + Hkv], freqs, True)
    xv = xqkv[:, :, H + Hkv:]
    if layout == "FT":
        vc[:B, :, start:start + S, :] = xv.transpose(2, 1)
        kc[:B, :, :, start:start + S, :] = xk.reshape(B, S, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous()
    else:
        vc[:B, start:start + S] = xv
        kc[:B, start:start + S] = xk
    return xq


def run(args):
    import torch
    import llm_awq_b200 as P
    eng = P.engine()
    device = torch.device("cuda", 0)
    dtype = torch.float16
    g = torch.Generator(device=device).manual_seed(0)
    results = []
    card = card_info(0)
    clk_before = clocks(0)
    all_identical = True
    for model, layout, hist, S in CASES:
        H, Hkv, D = MODELS[model]
        B, Lmax = 1, hist + S + 256
        nh = H + 2 * Hkv
        # batch 1: tinychat's freqs slice [S, 1, 1, D] is read per (token, batch row) by fused_rope_with_pos
        freqs = (torch.rand(S, 1, 1, D, generator=g, device=device) * 100.0).contiguous()
        arms = {}
        for arm in ("this", "composed"):
            layers = []
            for i in range(LAYERS):
                gi = torch.Generator(device=device).manual_seed(1000 * i + S)
                qkv = torch.randn(B, S, nh, D, generator=gi, device=device).to(dtype)
                if layout == "FT":
                    kc = torch.randn(B, Hkv, D // 8, Lmax, 8, generator=gi, device=device).to(dtype)
                    vc = torch.randn(B, Hkv, Lmax, D, generator=gi, device=device).to(dtype)
                else:
                    kc = torch.randn(B, Lmax, Hkv, D, generator=gi, device=device).to(dtype)
                    vc = torch.randn(B, Lmax, Hkv, D, generator=gi, device=device).to(dtype)
                layers.append((qkv, kc, vc))
            arms[arm] = layers
        # `this` rotates q in place: every replay rotates it again, so each timed call works on fresh-looking bytes
        # of the same size; the bit comparison below runs once on pristine copies.
        src = {arm: [(x[0].clone(), x[1].clone(), x[2].clone()) for x in layers] for arm, layers in arms.items()}

        def this_fn(attn):
            def fn():
                outs = []
                for qkv, kc, vc in arms["this"]:
                    q = eng.rope_kv_store(qkv, freqs, kc, vc, hist)
                    outs.append(eng.kv_cache_attention(q, kc, vc, hist + S) if attn else q)
                return outs
            return fn

        def composed_fn(attn):
            def fn():
                outs = []
                for qkv, kc, vc in arms["composed"]:
                    q = composed(eng, qkv, freqs, kc, vc, hist, H, Hkv, layout)
                    outs.append(eng.kv_cache_attention(q, kc, vc, hist + S) if attn else q)
                return outs
            return fn

        impls = {"this": this_fn(False), "composed": composed_fn(False), "this+attn": this_fn(True),
                 "composed+attn": composed_fn(True)}
        graphs, outs = {}, {}
        for key, fn in impls.items():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                fn()
            side.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=side):
                outs[key] = fn()
            graphs[key] = gr
        times = {k: [] for k in graphs}
        for _ in range(3):  # alternate the callers
            for key, gr in graphs.items():
                ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
                times[key].append(ms * 1e3 / (args.steps * LAYERS))
        # bit comparison on the timed inputs: both arms restored to the same pristine bytes, one replay each
        identical = True
        for key in ("this+attn", "composed+attn"):
            arm = key.split("+")[0]
            for (qkv, kc, vc), (q0, k0, v0) in zip(arms[arm], src[arm]):
                qkv.copy_(q0), kc.copy_(k0), vc.copy_(v0)
            graphs[key].replay()
        torch.cuda.synchronize()
        # rotated q: in place in `this`'s qkv; `composed` leaves qkv as it was, so its own graph's q output is current
        for (qa, ka, va), (_, kb, vb), qb in zip(arms["this"], arms["composed"], outs["composed"]):
            identical &= torch.equal(qa[:, :, :H].contiguous().view(torch.int16), qb.contiguous().view(torch.int16))
            identical &= torch.equal(ka.view(torch.int16), kb.view(torch.int16)) and torch.equal(va.view(torch.int16), vb.view(torch.int16))
        for oa, ob in zip(outs["this+attn"], outs["composed+attn"]):
            identical &= torch.equal(oa.view(torch.int16), ob.view(torch.int16))
        all_identical &= identical
        nbytes = 2 * B * S * nh * D * 2 + S * D * 4
        row = {"case": f"{model} {layout} start={hist} S={S}", "model": model, "layout": layout, "H": H, "Hkv": Hkv,
               "head_dim": D, "batch": B, "S": S, "start_pos": hist, "bytes": nbytes, "bit_identical": identical,
               "impls": {}}
        for key, ts in times.items():
            us = min(ts)
            row["impls"][key] = {"us_per_call": us, "us_runs": ts}
            if "+" not in key:
                row["impls"][key].update({"gbps": nbytes / us / 1e3, "frac_hbm": nbytes / us / 1e3 / PEAK_GBPS})
        results.append(row)
        del arms, src, graphs, outs, impls
        torch.cuda.empty_cache()
    line = {"metric": "RoPE + KV-cache store of a chunk, one call per layer in a CUDA graph, 1xH100",
            "unit": "us per call", "steps": args.steps, "warmup": args.warmup, "layers": LAYERS, "dtype": "fp16",
            "data": "synthetic", "torch_version": torch.__version__, "bit_identical": all_identical,
            "peaks": {"hbm_gbps": PEAK_GBPS, "source": "H100 SXM data sheet"}, "card": card,
            "clocks_before": clk_before, "clocks_after": clocks(0), "cases": results}
    print(json.dumps(line))
    for r in results:
        parts = []
        for k, v in r["impls"].items():
            extra = f" {v['frac_hbm']:4.2f}" if "frac_hbm" in v else ""
            parts.append(f"{k} {v['us_per_call']:6.1f} us{extra} [" + " ".join(f"{t:.1f}" for t in v["us_runs"]) + "]")
        print(f"{r['case']:<40} {'same' if r['bit_identical'] else 'DIFF'} " + " | ".join(parts), file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_rope_kv_store.py runs on one GPU")
    run(args)


if __name__ == "__main__":
    main()
