#!/usr/bin/env python
"""Benchmark of whole W8A8 vision-encoder layers, attention included, with the residual stream in PyTorch (composed)
and in the GEMM epilogue (fused), on 1 x H100.

    python bench_vision_encoder.py [--steps K] [--warmup W] [--rounds R]

A step is every encoder layer of a tower as tinychat runs it: LN-quant -> qkv -> attention -> quant -> out (+ residual)
-> LN-quant -> fc1 -> gelu-quant -> fc2 (+ residual), through `awq_inference_engine`.
  * SigLIP-so400m-patch14-448 (NVILA, tinychat/modules/fused_siglipdecoder.py): 27 layers, hidden 1152, inter 4304,
    16 heads x 72, 1024 tokens per image, attention through flash_attn_func on views of the qkv output; the
    residual is `residual + out`.
  * InternViT-300M-448px (InternVL3, tinychat/modules/fused_internencoder.py): 24 layers, hidden 1024, inter 4096,
    16 heads x 64, 1025 tokens per tile, attention through flash_attn_varlen_qkvpacked_func; the residual is
    `residual + out * ls`.
Each at 1 and 8 images / tiles, every layer's weights distinct.  The composed route is today's GEMM entry followed by
the PyTorch mul / add; the fused route passes `residual=` (and `layer_scale=`) to w8a8_linear_forward_cuda.  Both run
as CUDA graphs, alternated over R rounds in this process (K timed steps after W warm-up steps each, CUDA events).
The out + fc2 chains alone (every layer's two residual-carrying linears, nothing else) are timed three ways: the plain
GEMM, the GEMM plus the PyTorch ops, and the fused launch; their difference per launch is the epilogue's cost.
Kernels per step are counted by torch.profiler on one eager step per route, after the timed rounds.  The last step's
outputs of the two routes are compared bit for bit; the script fails if they differ.  Prints one JSON line with the
card's name and power limit, read in the same run.  Synthetic, seeded data; writes nothing.
"""
import argparse
import json
import statistics
import subprocess

TOWERS = {
    "siglip": dict(name="SigLIP-so400m-patch14-448", layers=27, hidden=1152, inter=4304, heads=16, tokens=1024,
                   layer_scale=False),
    "internvit": dict(name="InternViT-300M-448px", layers=24, hidden=1024, inter=4096, heads=16, tokens=1025,
                      layer_scale=True),
}


def card_info():
    """Name and power limit of GPU 0 (read-only queries)."""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"unavailable": repr(e)[:200]}


def make_layers(torch, cfg, device, seed):
    g = torch.Generator(device=device).manual_seed(seed)
    H, I = cfg["hidden"], cfg["inter"]
    layers = []
    for _ in range(cfg["layers"]):
        lay = {}
        for nm, (n, k) in {"qkv": (3 * H, H), "out": (H, H), "fc1": (I, H), "fc2": (H, I)}.items():
            lay[nm] = (torch.randint(-127, 128, (n, k), generator=g, device=device, dtype=torch.int8),
                       (0.0005 + 0.002 * torch.rand(n, generator=g, device=device)).half(),
                       (0.1 * torch.randn(n, generator=g, device=device)).half())
        for ln in ("ln1", "ln2"):
            lay[ln] = ((1 + 0.1 * torch.randn(H, generator=g, device=device)).half(),
                       (0.1 * torch.randn(H, generator=g, device=device)).half())
        if cfg["layer_scale"]:
            lay["ls1"] = (0.1 * torch.randn(H, generator=g, device=device)).half()
            lay["ls2"] = (0.1 * torch.randn(H, generator=g, device=device)).half()
        layers.append(lay)
    return layers


def residual_linear(torch, eng, lay, nm, q, s, residual, ls, fused):
    """tinychat's out / fc2 linear and the residual after it: `residual + out (* ls)`."""
    w, ws, b = lay[nm]
    out = torch.empty(q.shape[0], w.shape[0], dtype=torch.float16, device=q.device)
    if fused:
        eng.w8a8_linear_forward_cuda(q, w, ws, s, out, bias=b, layer_scale=ls, residual=residual)
        return out
    eng.w8a8_gemm_fuse_bias_forward_cuda(q, w, ws, s, out, b)
    return residual + (out if ls is None else out * ls)


def encoder_layer(torch, eng, cfg, lay, h, images, fused):
    M, H = h.shape
    I, heads, T = cfg["inter"], cfg["heads"], cfg["tokens"]
    D = H // heads
    dev = h.device
    qH = torch.empty(M, H, dtype=torch.int8, device=dev)
    s = torch.empty(M, dtype=torch.float16, device=dev)
    eng.rms_norm_general(qH, h, lay["ln1"][0], lay["ln1"][1], s, 1e-6, True)
    qkv = torch.empty(M, 3 * H, dtype=torch.float16, device=dev)
    eng.w8a8_gemm_fuse_bias_forward_cuda(qH, *lay["qkv"][:2], s, qkv, lay["qkv"][2])
    if cfg["layer_scale"]:  # InternViT: packed qkv, uniform cu_seqlens
        cu = torch.arange(0, (images + 1) * T, step=T, dtype=torch.int32, device=dev)
        attn = eng.flash_attn_varlen_qkvpacked_func(qkv.view(M, 3, heads, D), cu, T, 0.0, softmax_scale=None, causal=False)
    else:                   # SigLIP: views of the qkv output
        q, k, v = qkv.split([H, H, H], dim=-1)
        shp = (images, T, heads, D)
        attn = eng.flash_attn_func(q.reshape(shp), k.reshape(shp), v.reshape(shp), softmax_scale=None, causal=False)
    eng.invoke_quant(qH, attn.reshape(M, H), s)
    h = residual_linear(torch, eng, lay, "out", qH, s, h, lay.get("ls1"), fused)
    eng.rms_norm_general(qH, h, lay["ln2"][0], lay["ln2"][1], s, 1e-6, True)
    fc1 = torch.empty(M, I, dtype=torch.float16, device=dev)
    eng.w8a8_gemm_fuse_bias_forward_cuda(qH, *lay["fc1"][:2], s, fc1, lay["fc1"][2])
    qI = torch.empty(M, I, dtype=torch.int8, device=dev)
    eng.gelu_and_quant(qI, fc1, s, torch.empty(M * I, dtype=torch.float16, device=dev))
    return residual_linear(torch, eng, lay, "fc2", qI, s, h, lay.get("ls2"), fused)


def run_case(torch, P, cfg, layers, images, args):
    eng = P.engine()
    dev = torch.device("cuda", 0)
    M, H = cfg["tokens"] * images, cfg["hidden"]
    g = torch.Generator(device=dev).manual_seed(images)
    x = (2 * torch.randn(M, H, generator=g, device=dev)).half()
    qH = torch.randint(-127, 128, (M, H), generator=g, device=dev, dtype=torch.int8)
    qI = torch.randint(-127, 128, (M, cfg["inter"]), generator=g, device=dev, dtype=torch.int8)
    s = (0.002 + 0.01 * torch.rand(M, generator=g, device=dev)).half()

    def step(fused):
        h = x
        for lay in layers:
            h = encoder_layer(torch, eng, cfg, lay, h, images, fused)
        return h

    def chain(mode):  # every layer's out and fc2 linears with their residuals, nothing else
        h = x
        for lay in layers:
            for nm, q, ls in (("out", qH, lay.get("ls1")), ("fc2", qI, lay.get("ls2"))):
                if mode == "gemm":
                    w, ws, b = lay[nm]
                    out = torch.empty(M, H, dtype=torch.float16, device=dev)
                    eng.w8a8_gemm_fuse_bias_forward_cuda(q, w, ws, s, out, b)
                    h = out
                else:
                    h = residual_linear(torch, eng, lay, nm, q, s, h, ls, mode == "fused")
        return h

    def graph_of(fn):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            out = fn()
        return gr, out

    graphs = {"composed": graph_of(lambda: step(False)), "fused": graph_of(lambda: step(True)),
              "chain_gemm": graph_of(lambda: chain("gemm")), "chain_composed": graph_of(lambda: chain("composed")),
              "chain_fused": graph_of(lambda: chain("fused"))}
    per_round = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for k, (gr, _) in graphs.items():
            for _ in range(args.warmup):
                gr.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            per_round[k].append(e0.elapsed_time(e1) * 1e3 / args.steps)  # us per step

    graphs["composed"][0].replay()
    graphs["fused"][0].replay()
    torch.cuda.synchronize()
    a, b = graphs["composed"][1], graphs["fused"][1]
    identical = bool(torch.equal(a.view(torch.int16), b.view(torch.int16)))
    n_diff = int((a.view(torch.int16) != b.view(torch.int16)).sum().item())
    finite = bool(torch.isfinite(a).all().item())

    kernels = {}
    for route, fused in (("composed", False), ("fused", True)):
        step(fused)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step(fused)
            torch.cuda.synchronize()
        kernels[route] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                             and not e.name.startswith(("Memcpy", "Memset")))

    def summary(v):
        return {"median": statistics.median(v), "min": min(v), "max": max(v), "rounds": v}

    L = cfg["layers"]
    res = {"tokens": M, "images": images}
    for route in ("composed", "fused"):
        t = summary(per_round[route])
        res[route] = {"us_per_step": t, "images_per_s": images * 1e6 / t["median"], "kernels_per_step": kernels[route]}
    med_c, med_f = res["composed"]["us_per_step"]["median"], res["fused"]["us_per_step"]["median"]
    spread = max(max(per_round[r]) - min(per_round[r]) for r in ("composed", "fused"))
    res["fused_vs_composed"] = {"speedup": med_c / med_f, "saved_us_per_step": med_c - med_f,
                                "round_spread_us": spread,
                                "fused_not_slower": med_f <= med_c + spread}
    chains = {k: summary(per_round["chain_" + k]) for k in ("gemm", "composed", "fused")}
    n_launch = 2 * L
    res["out_fc2_chains"] = {
        "launches": n_launch,
        "us_per_linear": {k: v["median"] / n_launch for k, v in chains.items()},
        "epilogue_cost_us_per_launch": (chains["fused"]["median"] - chains["gemm"]["median"]) / n_launch,
        "torch_ops_cost_us_per_launch": (chains["composed"]["median"] - chains["gemm"]["median"]) / n_launch,
        "rounds_us_per_chain": {k: v["rounds"] for k, v in chains.items()},
    }
    res["outputs"] = {"bit_identical": identical, "elements_differing": n_diff, "finite": finite}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_vision_encoder.py runs on one GPU")
    import torch
    import llm_awq_b200 as P
    if not torch.cuda.is_available():
        raise SystemExit("bench_vision_encoder.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = card_info()
    results = {}
    for i, (key, cfg) in enumerate(TOWERS.items()):
        layers = make_layers(torch, cfg, dev, seed=100 + i)
        for images in (1, 8):
            results[f"{key}_{images}"] = run_case(torch, P, cfg, layers, images, args)
        del layers
        torch.cuda.empty_cache()
    ok = all(r["outputs"]["bit_identical"] and r["outputs"]["finite"] for r in results.values())
    line = {"metric": "W8A8 vision-encoder step, residual epilogue fused vs composed, 1xH100",
            "value": results["siglip_8"]["fused_vs_composed"]["speedup"], "unit": "x (SigLIP, 8 images)",
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
            "higher_is_better": True, "data": "synthetic", "card": card,
            "towers": {k: {kk: v for kk, v in cfg.items()} for k, cfg in TOWERS.items()},
            "outputs_bit_identical": ok, "cases": results}
    print(json.dumps(line))
    if not ok:
        raise SystemExit("the fused and composed routes' outputs differ")


if __name__ == "__main__":
    main()
