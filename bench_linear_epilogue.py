"""Cost and gain of the W4A16 bias / residual epilogue (b200awq_w4a16_linear) on one H100.

    python bench_linear_epilogue.py --steps K --warmup W

1. Decode chain, batch 1, fp16, in tinychat's order per decoder layer, every layer with its own weights and its own
   FasterTransformer KV cache (context 1024 and 8192), captured in one CUDA graph per chain:
     today: rmsnorm -> q, k, v (+ torch bias adds for Qwen2) -> single_query_attention -> o -> torch add (residual)
            -> rmsnorm -> mlp_front -> down -> torch add (residual)
     fused: the same with the bias and the residual adds in the linears' epilogues.
   Qwen2-7B (28 layers, q / k / v bias) and Llama-3-8B (32 layers, no bias).  The two chains' outputs must be
   bit-identical (checked in the same run); reported as us per token.
2. Per shape, one token: a graph of 32 launches with distinct weights (beyond L2), plain against the same with the
   epilogue, and against plain + a PyTorch add: the epilogue's own cost and what it replaces.
3. Prefill, 2048 tokens: o_proj and down_proj with the residual, against the GEMM + a PyTorch add.
Timed graph replays of the variants alternate round by round; each figure is the median over rounds.  Prints the
card's name, power limit and SM clocks, and one JSON line."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_kv_cache_attention import clocks  # noqa: E402
from bench_siglip import card_info  # noqa: E402

# hidden, heads, kv heads, intermediate, layers, q/k/v bias, rope base
MODELS = {"Qwen2-7B": (3584, 28, 4, 18944, 28, True, 1000000.0),
          "Llama-3-8B": (4096, 32, 8, 14336, 32, False, 500000.0)}
HD = 128
ROUNDS = 5


def rand_layer(torch, n, k, g):
    """Packed int4 weights, scales and scaled zeros of one [n, k] layer (WQLinear's buffers), generated on the device."""
    dev = g.device
    qw = torch.randint(-32768, 32768, (n // 4, k), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
    rows = -(-(k // 128) // 8) * 8
    s = torch.zeros(rows, n, device=dev, dtype=torch.float16)
    s[:k // 128] = (0.004 + 0.012 * torch.rand(k // 128, n, generator=g, device=dev)).half()
    z = (-(s.float() * torch.randint(0, 16, (rows, n), generator=g, device=dev))).half()
    return qw, s, z


def graph_of(torch, fn, stream):
    """fn captured into a CUDA graph on `stream` (warmed up there first); returns (graph, its output)."""
    with torch.cuda.stream(stream):
        fn()
    stream.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        out = fn()
    return g, out


def time_alternating(torch, graphs, steps, warmup):
    """{name: median over ROUNDS of ms per replay}; the graphs are replayed round by round in turn."""
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
    return {name: (statistics.median(v), v) for name, v in per.items()}


def decode_chain(torch, eng, model, ctx, steps, warmup):
    hidden, heads, kvh, inter, nl, has_bias, base = MODELS[model]
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    kvd = kvh * HD
    layers = []
    for _ in range(nl):
        L = {name: rand_layer(torch, n, k, g) for name, n, k in
             (("q", hidden, hidden), ("k", kvd, hidden), ("v", kvd, hidden), ("o", hidden, hidden),
              ("gate", inter, hidden), ("up", inter, hidden), ("down", hidden, inter))}
        L["bias"] = {p: (0.5 * torch.randn(n, generator=g, device=dev)).half() if has_bias else None
                     for p, n in (("q", hidden), ("k", kvd), ("v", kvd))}
        L["g1"] = (1 + 0.1 * torch.randn(hidden, generator=g, device=dev)).half()
        L["g2"] = (1 + 0.1 * torch.randn(hidden, generator=g, device=dev)).half()
        L["kc"] = (0.5 * torch.randn(1, kvh, HD // 8, ctx + 16, 8, generator=g, device=dev)).half()
        L["vc"] = (0.5 * torch.randn(1, kvh, ctx + 16, HD, generator=g, device=dev)).half()
        layers.append(L)
    x0 = torch.randn(1, hidden, generator=g, device=dev).half()

    def gemv(a, w):
        return eng.gemv_forward_cuda_new(a, *w, 1, w[1].shape[1], a.shape[-1], 128)

    def linear(a, w, bias=None, residual=None):
        return eng.w4a16_linear_forward_cuda(a, *w, 128, bias=bias, residual=residual)

    def step(fused):
        h = x0
        for L in layers:
            a = torch.empty_like(h)
            eng.layernorm_forward_cuda(h, L["g1"], a, 1e-6)
            qkv = []
            for p in ("q", "k", "v"):
                b = L["bias"][p]
                if fused:
                    qkv.append(linear(a, L[p], bias=b))
                else:
                    t = gemv(a, L[p])
                    qkv.append(t + b if b is not None else t)
            q, k, v = qkv
            att = eng.single_query_attention(q.view(1, heads, HD), k.view(1, kvh, HD), v.view(1, kvh, HD), L["kc"], L["vc"],
                                             None, None, ctx, HD, base, 1.0, True)
            att = att.view(1, hidden)
            h = linear(att, L["o"], residual=h) if fused else h + gemv(att, L["o"])
            a2 = torch.empty_like(h)
            eng.layernorm_forward_cuda(h, L["g2"], a2, 1e-6)
            f = eng.mlp_front_forward_cuda(a2, *L["gate"], *L["up"])
            h = linear(f, L["down"], residual=h) if fused else h + gemv(f, L["down"])
        return h

    st = torch.cuda.Stream()
    g_today, y_today = graph_of(torch, lambda: step(False), st)
    g_fused, y_fused = graph_of(torch, lambda: step(True), st)
    g_today.replay()
    g_fused.replay()
    torch.cuda.synchronize()
    identical = torch.equal(y_today.view(torch.int16), y_fused.view(torch.int16))
    assert identical, f"{model} ctx {ctx}: the fused chain's output differs from today's"
    t = time_alternating(torch, {"today": g_today, "fused": g_fused}, steps, warmup)
    del g_today, g_fused, layers
    torch.cuda.empty_cache()
    return {"model": model, "context": ctx, "layers": nl, "bit_identical": identical,
            "us_per_token": {k: round(v[0] * 1e3, 1) for k, v in t.items()},
            "us_runs": {k: [round(x * 1e3, 1) for x in v[1]] for k, v in t.items()},
            "fused_vs_today": round(t["today"][0] / t["fused"][0] - 1.0, 4)}


# (name, n, k, operand): one-token shapes of the two models
SHAPES = [("Qwen2-7B q", 3584, 3584, "bias"), ("Qwen2-7B k/v", 512, 3584, "bias"),
          ("Qwen2-7B o", 3584, 3584, "residual"), ("Qwen2-7B down", 3584, 18944, "residual"),
          ("Llama-3-8B o", 4096, 4096, "residual"), ("Llama-3-8B down", 4096, 14336, "residual")]
CHAIN = 32


def per_shape(torch, eng, name, n, k, op, m, chain, steps, warmup):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(n + k)
    ws = [rand_layer(torch, n, k, g) for _ in range(chain)]
    x = torch.randn(m, k, generator=g, device=dev).half()
    operand = (torch.randn(n, generator=g, device=dev) if op == "bias" else 4 * torch.randn(m, n, generator=g, device=dev)).half()
    kw = {op: operand}

    def engine_call(w):
        if m < 8:
            return eng.gemv_forward_cuda_new(x, *w, m, n, k, 128)
        return eng.gemm_forward_cuda_new(x, *w)

    def plain():
        return [engine_call(w) for w in ws]

    def plain_add():
        return [engine_call(w) + operand if op == "bias" else operand + engine_call(w) for w in ws]

    def fused():
        return [eng.w4a16_linear_forward_cuda(x, *w, 128, **kw) for w in ws]

    st = torch.cuda.Stream()
    graphs, outs = {}, {}
    for label, fn in (("plain", plain), ("plain+torch_add", plain_add), ("fused", fused)):
        graphs[label], outs[label] = graph_of(torch, fn, st)
        graphs[label].replay()
    torch.cuda.synchronize()
    identical = all(torch.equal(a, b) for a, b in zip(outs["fused"], outs["plain+torch_add"]))
    assert identical, f"{name} m={m}: fused differs from plain + torch add"
    t = time_alternating(torch, graphs, steps, warmup)
    del graphs, ws
    torch.cuda.empty_cache()
    us = {label: round(v[0] * 1e3 / chain, 2) for label, v in t.items()}
    return {"shape": name, "m": m, "n": n, "k": k, "operand": op, "launches": chain, "bit_identical": identical,
            "us_per_launch": us, "epilogue_cost_us": round(us["fused"] - us["plain"], 2),
            "saved_vs_torch_add_us": round(us["plain+torch_add"] - us["fused"], 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_linear_epilogue.py runs on one GPU")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_linear_epilogue.py needs a CUDA device")
    import llm_awq_b200 as P
    eng = P.engine()
    torch.cuda.set_device(0)
    card, clk0 = card_info(0), clocks(0)
    out = {"card": card, "clocks_before": clk0, "steps": args.steps, "warmup": args.warmup, "rounds": ROUNDS}
    with torch.no_grad():
        out["decode_chain"] = []
        for model in MODELS:
            for ctx in (1024, 8192):
                r = decode_chain(torch, eng, model, ctx, args.steps, args.warmup)
                out["decode_chain"].append(r)
                print(f"{model:<11} ctx {ctx:5d}: today {r['us_per_token']['today']:8.1f} us/token, fused "
                      f"{r['us_per_token']['fused']:8.1f} ({100 * r['fused_vs_today']:+.2f} % tokens/s), bit-identical",
                      file=sys.stderr)
        out["per_shape"] = []
        for name, n, k, op in SHAPES:
            r = per_shape(torch, eng, name, n, k, op, 1, CHAIN, args.steps, args.warmup)
            out["per_shape"].append(r)
            print(f"{name:<16} m=1 {op:<8}: {r['us_per_launch']} us per launch", file=sys.stderr)
        out["prefill"] = []
        for name, n, k, op in SHAPES:
            if op != "residual":
                continue
            r = per_shape(torch, eng, name, n, k, op, 2048, 8, max(2, args.steps // 4), 1)
            out["prefill"].append(r)
            print(f"{name:<16} m=2048 {op:<8}: {r['us_per_launch']} us per launch", file=sys.stderr)
    out["clocks_after"] = clocks(0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
