"""What the RMSNorm prologues (b200awq_w4a16_norm_linear, b200awq_w4a16_norm_mlp_front) do to a decode chain on one H100.

    python bench_norm_prologue.py --steps K --warmup W

Per workload, a chain of 32 decoder layers with their own weights, each layer in tinychat's launch order without the
attention itself (the o projection reads a fixed attention output), captured in one CUDA graph per variant:
    composed: rmsnorm -> qkv (+ bias) -> o (+ residual) -> rmsnorm -> mlp_front -> down (+ residual)
    fused:    norm_qkv (+ bias)       -> o (+ residual) -> norm_mlp_front       -> down (+ residual)
Workloads: Llama-3-8B fp16, Qwen2-7B fp16 (q/k/v bias), Qwen2-0.5B fp16 (small layers: the decode plan may split k
over a cluster), Llama-3-8B bf16 at one token and fp16 at four tokens (both on the ring kernel); each with programmatic
dependent launch on and off.  The two variants' graphs are replayed round by round in turn; each figure is the median
over the rounds, with the rounds' range.  The final residual stream and each layer's last q/k/v and MLP front outputs of
the two chains must be bit-identical (checked in the same run).  Prints the card's name and power limit, and one JSON
line."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_linear_epilogue import graph_of, rand_layer  # noqa: E402
from bench_siglip import card_info  # noqa: E402

LAYERS = 32
ROUNDS = 7
# name: (hidden, q/k/v outputs, intermediate, q/k/v bias, dtype, tokens)
WORKLOADS = {"Llama-3-8B fp16 m=1": (4096, 6144, 14336, False, "f16", 1),
             "Qwen2-7B fp16 m=1": (3584, 4608, 18944, True, "f16", 1),
             "Qwen2-0.5B fp16 m=1": (896, 1152, 4864, True, "f16", 1),
             "Llama-3-8B bf16 m=1": (4096, 6144, 14336, False, "bf16", 1),
             "Llama-3-8B fp16 m=4": (4096, 6144, 14336, False, "f16", 4)}


def layer_set(torch, hidden, nqkv, inter, bias, T, g):
    L = {"qkv": rand_layer(torch, nqkv, hidden, g), "o": rand_layer(torch, hidden, hidden, g),
         "gate": rand_layer(torch, inter, hidden, g), "up": rand_layer(torch, inter, hidden, g),
         "down": rand_layer(torch, hidden, inter, g)}
    L = {k: tuple(t.to(T) if t.dtype == torch.float16 else t for t in v) for k, v in L.items()}
    dev = g.device
    L["bias"] = (0.5 * torch.randn(nqkv, generator=g, device=dev)).to(T) if bias else None
    L["g1"] = (1 + 0.1 * torch.randn(hidden, generator=g, device=dev)).to(T)
    L["g2"] = (1 + 0.1 * torch.randn(hidden, generator=g, device=dev)).to(T)
    return L


def time_alternating(torch, graphs, steps, warmup):
    """{name: [ms per replay of each round]}; the graphs are replayed round by round in turn."""
    for g in graphs.values():
        for _ in range(warmup):
            g.replay()
    torch.cuda.synchronize()
    per = {name: [] for name in graphs}
    for _ in range(ROUNDS):
        for name, g in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            per[name].append(e0.elapsed_time(e1) / steps)
    return per


def workload(torch, eng, name, pdl, steps, warmup):
    hidden, nqkv, inter, bias, dt, m = WORKLOADS[name]
    T = torch.float16 if dt == "f16" else torch.bfloat16
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(7)
    layers = [layer_set(torch, hidden, nqkv, inter, bias, T, g) for _ in range(LAYERS)]
    x0 = (4 * torch.randn(m, hidden, generator=g, device=dev)).to(T)
    att = torch.randn(m, hidden, generator=g, device=dev).to(T)   # stands in for the attention output
    eps = 1e-6

    def step(fused):
        h, outs = x0, []
        for L in layers:
            if fused:
                qkv = eng.rmsnorm_w4a16_linear_forward_cuda(h, L["g1"], eps, *L["qkv"], 128, bias=L["bias"])
            else:
                a = torch.empty_like(h)
                eng.layernorm_forward_cuda(h, L["g1"], a, eps)
                qkv = eng.w4a16_linear_forward_cuda(a, *L["qkv"], 128, bias=L["bias"])
            h = eng.w4a16_linear_forward_cuda(att, *L["o"], 128, residual=h)
            if fused:
                f = eng.rmsnorm_mlp_front_forward_cuda(h, L["g2"], eps, *L["gate"], *L["up"])
            else:
                a2 = torch.empty_like(h)
                eng.layernorm_forward_cuda(h, L["g2"], a2, eps)
                f = eng.mlp_front_forward_cuda(a2, *L["gate"], *L["up"])
            h = eng.w4a16_linear_forward_cuda(f, *L["down"], 128, residual=h)
            outs += [qkv, f]
        return [h] + outs

    old = eng.set_pdl(pdl)
    try:
        st = torch.cuda.Stream()
        g_c, y_c = graph_of(torch, lambda: step(False), st)
        g_f, y_f = graph_of(torch, lambda: step(True), st)
    finally:
        eng.set_pdl(old)
    g_c.replay()
    g_f.replay()
    torch.cuda.synchronize()
    identical = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(y_c, y_f))
    per = time_alternating(torch, {"composed": g_c, "fused": g_f}, steps, warmup)
    del g_c, g_f, layers
    torch.cuda.empty_cache()
    us = {k: [round(v * 1e3 / LAYERS, 2) for v in runs] for k, runs in per.items()}
    med = {k: round(statistics.median(v), 2) for k, v in us.items()}
    return {"workload": name, "pdl": pdl, "layers": LAYERS, "bit_identical": identical,
            "us_per_layer": med, "us_per_layer_range": {k: [min(v), max(v)] for k, v in us.items()},
            "fused_saves_us_per_layer": round(med["composed"] - med["fused"], 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_norm_prologue.py needs a CUDA device")
    import llm_awq_b200 as P
    eng = P.engine()
    card = card_info(0)
    card["name"] = card["name"] or torch.cuda.get_device_name(0)
    print(card)
    rows = []
    for name in WORKLOADS:
        for pdl in (True, False):
            r = workload(torch, eng, name, pdl, args.steps, args.warmup)
            rows.append(r)
            print(f"{name:22s} pdl={int(pdl)}  composed {r['us_per_layer']['composed']:7.2f} us/layer "
                  f"{r['us_per_layer_range']['composed']}  fused {r['us_per_layer']['fused']:7.2f} us/layer "
                  f"{r['us_per_layer_range']['fused']}  saves {r['fused_saves_us_per_layer']:+.2f}  "
                  f"bit-identical {r['bit_identical']}", flush=True)
    print(json.dumps({"bench": "norm_prologue", "card": card, "steps": args.steps, "rounds": ROUNDS, "results": rows}))
    if not all(r["bit_identical"] for r in rows):
        raise SystemExit("a fused chain's output differs from the composed chain's")


if __name__ == "__main__":
    main()
