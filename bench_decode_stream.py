#!/usr/bin/env python
"""Where the one-token W4A16 decode step spends its time: Llama-3-8B (the `bench.py` headline workload) taken apart.

    python bench_decode_stream.py [--steps K] [--warmup W] [--lib PATH] [--json FILE]

Every figure is a CUDA graph of C-ABI launches (include/b200awq.h) replayed K times and timed with CUDA events, as in
bench.py, with programmatic dependent launch on.  Weights are synthetic and distinct per layer (bench.build_model),
so every weight byte is an HBM read.  Rows:
  step        the 160 launches of one token in model order (bench.py's `value`)
  long only   the same step with only gate, up and down (96 launches): the byte-bound launches
  short only  the same step with only qkv and o (64 launches): the launches whose weights fit a CTA's look-ahead
  chain NxK   32 distinct layers of one shape back to back, per launch
  ceiling     the same bytes as a long chain in ONE launch (no launch boundary): 196608 x 4096 (373 quad rows per
              CTA) and 131072 x 14336 (k split over 2-CTA clusters, 125 row blocks per CTA)
each at the decode kernel's ring depth chosen from the shape and capped at 3 and 4 slots (B200AWQ_DECODE_SLOTS, the
library's test seam).  Bytes are bench.py's algorithmic bytes (packed weights, scales, zeros, x, y); `frac` is the
share of the H100 SXM data-sheet 3.35 TB/s.  The card name, power limit and median SM clock come from NVML in the same
run.  `--lib` times another build of libb200awq.so (for example the parent commit's) through the same code.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402  (shapes, synthetic weights, algorithmic bytes, clock sampler)

CEILINGS = ((196608, 4096), (131072, 14336))
SLOTS = (0, 3, 4)  # 0: the ring depth chosen from the shape


def load_lib(path):
    L = ctypes.CDLL(path)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.b200awq_w4a16_gemv.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    L.b200awq_w4a16_gemv.restype = ci
    L.b200awq_strerror.argtypes = [ci]
    L.b200awq_strerror.restype = ctypes.c_char_p
    L.b200awq_reload_config.restype = None
    return L


def card_info(index):
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit_w": None, "nvml": repr(e)[:120]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--lib", default=None, help="libb200awq.so to time (default: this tree's build)")
    ap.add_argument("--json", default=None, help="also write the result record to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_stream.py needs a CUDA device")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    lib_path = args.lib or os.path.join(ROOT, "llm_awq_b200", "lib", "libb200awq.so")
    lib = load_lib(lib_path)
    cfg, G, dtype = bench.LLAMA3_8B, bench.G, torch.float16
    hbm = bench.read_peaks()["hbm"]
    sampler = bench.ClockSampler(0)
    windows = []

    model = bench.build_model(torch, cfg, dtype, device)
    ceil = [bench.build_model(torch, cfg, dtype, device, layers=1, projs=[("ceiling", K, N)])[0] for N, K in CEILINGS]
    g = torch.Generator(device=device).manual_seed(100)
    xs = {K: torch.randn(1, K, generator=g, device=device).to(dtype) for K in {m["K"] for m in model + ceil}}
    ys = {N: torch.empty(1, N, dtype=dtype, device=device) for N in {m["N"] for m in model + ceil}}
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def graph(layers):
        def launch_all():
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            for m in layers:
                rc = lib.b200awq_w4a16_gemv(p(xs[m["K"]]), p(m["qw"]), p(m["sc"]), p(m["sz"]), p(ys[m["N"]]), 1, m["N"],
                                            m["K"], G, 0, st)
                if rc != 0:
                    raise RuntimeError(lib.b200awq_strerror(rc).decode())
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            launch_all()
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            launch_all()
        return gr

    def measure(layers):
        gr = graph(layers)
        ms, w = bench.timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
        windows.append(w)
        us = ms * 1e3 / args.steps
        nbytes = sum(bench.alg_bytes(1, m["N"], m["K"]) for m in layers)
        return {"us": round(us, 2), "launches": len(layers), "us_per_launch": round(us / len(layers), 3),
                "gb_s": round(nbytes / us / 1e3, 1), "frac": round(nbytes / us / 1e3 / hbm, 4)}

    shapes = []
    for m in model[:5]:
        shapes.append((m["name"], m["N"], m["K"]))
    sampler.start()
    rows = {}
    for slots in SLOTS:
        os.environ["B200AWQ_DECODE_SLOTS"] = str(slots)
        lib.b200awq_reload_config()
        r = {}
        r["step"] = measure(model)
        r["step"]["tok_s"] = round(1e6 / r["step"]["us"], 1)
        r["long only"] = measure([m for m in model if m["name"] in ("gate", "up", "down")])
        r["short only"] = measure([m for m in model if m["name"] in ("qkv", "o")])
        if slots == 0:
            for name, N, K in shapes:
                if name == "up":
                    continue  # the same shape as gate
                r["chain %s %dx%d" % (name, N, K)] = measure([m for m in model if (m["N"], m["K"]) == (N, K)][:32])
        for m in ceil:
            r["ceiling %dx%d" % (m["N"], m["K"])] = measure([m])
        rows["default" if slots == 0 else "slots=%d" % slots] = r
    os.environ.pop("B200AWQ_DECODE_SLOTS")
    lib.b200awq_reload_config()
    clocks = sampler.stop(windows)
    rec = {"card": card_info(0), "clocks": clocks, "lib": os.path.relpath(lib_path, ROOT), "steps": args.steps,
           "warmup": args.warmup, "peak_hbm_gb_s": hbm, "rows": rows}

    print("%s, power limit %s W, median SM clock %s MHz" % (rec["card"]["name"], rec["card"]["power_limit_w"],
                                                           clocks.get("sm_mhz")))
    for plan, r in rows.items():
        print("[%s]" % plan)
        for k, v in r.items():
            extra = ("  %.1f tok/s" % v["tok_s"]) if "tok_s" in v else ""
            print("  %-26s %9.2f us  %4d launches  %7.3f us/launch  %7.1f GB/s  %.3f%s" % (
                k, v["us"], v["launches"], v["us_per_launch"], v["gb_s"], v["frac"], extra))
    print(json.dumps(rec))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
