#!/usr/bin/env python
"""Per-CTA trace of the launch boundaries of the one-token W4A16 decode step (Llama-3-8B, `bench.py`'s headline).

    python bench_decode_trace.py [--replays R] [--warmup W] [--lib PATH] [--json FILE]

Builds a trace variant of libb200awq.so (build.py's NVCC_FLAGS plus -DB200AWQ_DECODE_TRACE) into a temporary
directory, unless --lib names one already built that way.  In that build every CTA of w4a16_decode_kernel writes time
stamps (%globaltimer, %clock64, %smid) at: CTA start, first lap issued, held slots released, first refill issued, last
copy issued, dependency wait returned (consumer warp 0), last MAC (consumer warp 0) and last store (finisher).  The
product library contains none of this code.

The 160-launch step graph (bench_decode_stream.py's `step`) is replayed R times after W warm-up replays, and for every
boundary between launch L-1 and launch L of a step the script reports medians and p90s over CTAs and boundaries of
  last issue -> grid end      L-1's grid end minus each L-1 CTA's last copy issue (the ramp-down)
  grid end -> wait            each L CTA's wait return minus L-1's grid end (grid end = L-1's latest stamp)
  wait -> first refill        each L CTA's first refill issue minus its own wait return
  release before wait         share of L's CTAs that held slots and released them before their wait returned
grouped by the shape of L.  It also reports the smallest nonzero step of %globaltimer seen, and checks that the
per-SM handoff counters are back where they started after the synchronised replays.
"""
import argparse
import ctypes
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402  (shapes, synthetic weights)

EVENTS = ("start", "first_lap", "release", "refill", "last_issue", "wait", "last_mac", "last_store")
EV = {n: i for i, n in enumerate(EVENTS)}
REC = np.dtype([("g", "<u8"), ("c", "<u8"), ("layer", "<u8"), ("block", "<u4"), ("se", "<u4")])
MAX_SM = 256  # kDecMaxSm in w4a16_decode.cu


def build_trace_lib(out_dir):
    spec = importlib.util.spec_from_file_location("_b200awq_build", os.path.join(ROOT, "llm_awq_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    lib = os.path.join(out_dir, "libb200awq_trace.so")
    srcs = [os.path.join(b.CSRC, f) for f in b.KERNEL_SRCS]
    b._run([os.environ.get("NVCC", "nvcc")] + b.NVCC_FLAGS + ["-DB200AWQ_DECODE_TRACE", "-shared", "-o", lib] + srcs)
    return lib


def stats(v):
    v = np.asarray(v, dtype=np.float64) / 1e3  # ns -> us
    if v.size == 0:
        return None
    return {"median_us": round(float(np.median(v)), 3), "p90_us": round(float(np.percentile(v, 90)), 3), "n": int(v.size)}


def analyse(recs, model, grid):
    """recs: REC array of R replays.  Returns per-shape boundary statistics and the timer resolution."""
    ev = recs["se"] & 0xFF
    idx = {m["qw"].data_ptr(): i for i, m in enumerate(model)}
    lay = np.array([idx.get(int(p), -1) for p in recs["layer"]])
    if (lay < 0).any():
        raise RuntimeError("trace records of launches outside the step")
    nl = len(model)
    # t[e][layer, replay, block]: the r-th occurrence (in time) of event e of (layer, block) belongs to replay r
    reps = int(np.sum((ev == EV["start"]) & (lay == 0) & (recs["block"] == 0)))
    t = {e: np.full((nl, reps, grid), np.nan) for e in range(len(EVENTS))}
    order = np.lexsort((recs["g"], recs["block"], lay, ev))
    e_s, l_s, b_s, g_s = ev[order], lay[order], recs["block"][order], recs["g"][order].astype(np.float64)
    key = (e_s.astype(np.int64) * nl + l_s) * grid + b_s
    first = np.r_[0, np.flatnonzero(np.diff(key)) + 1]
    rank = np.arange(key.size) - np.repeat(first, np.diff(np.r_[first, key.size]))
    ok = rank < reps
    for e in range(len(EVENTS)):
        s = ok & (e_s == e)
        t[e][l_s[s], rank[s], b_s[s]] = g_s[s]
    end = np.nanmax(np.stack([t[EV["last_issue"]], t[EV["last_mac"]], t[EV["last_store"]]]), axis=0)
    grid_end = np.nanmax(end, axis=2)  # [layer, replay]
    out = {}
    for i in range(1, nl):
        name = model[i]["name"]
        r = out.setdefault(name, {"ramp": [], "to_wait": [], "to_refill": [], "held": 0, "released_early": 0})
        li = t[EV["last_issue"]][i - 1]
        r["ramp"].extend((grid_end[i - 1][:, None] - li)[~np.isnan(li)])
        w = t[EV["wait"]][i]
        r["to_wait"].extend((w - grid_end[i - 1][:, None])[~np.isnan(w)])
        rf = t[EV["refill"]][i]
        r["to_refill"].extend((rf - w)[~np.isnan(rf) & ~np.isnan(w)])
        rel = t[EV["release"]][i]
        r["held"] += int(np.sum(~np.isnan(rel)))
        r["released_early"] += int(np.sum(rel < w))
    res = {}
    for name, r in out.items():
        res[name] = {"last issue -> grid end": stats(r["ramp"]), "grid end -> wait": stats(r["to_wait"]),
                     "wait -> first refill": stats(r["to_refill"]), "held CTAs": r["held"],
                     "released before wait": r["released_early"]}
    g = np.unique(recs["g"])
    steps = np.diff(g)
    return res, int(steps[steps > 0].min()) if (steps > 0).any() else None, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--lib", default=None, help="a libb200awq.so built with -DB200AWQ_DECODE_TRACE (default: build one)")
    ap.add_argument("--json", default=None, help="also write the result record to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode_trace.py needs a CUDA device")
    import bench_decode_stream as bds
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    with tempfile.TemporaryDirectory() as tmp:
        lib_path = args.lib or build_trace_lib(tmp)
        lib = bds.load_lib(lib_path)
        read = lib.b200awq_decode_trace_read
        read.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        read.restype = ctypes.c_longlong

        cfg, G, dtype = bench.LLAMA3_8B, bench.G, torch.float16
        model = bench.build_model(torch, cfg, dtype, device)
        g = torch.Generator(device=device).manual_seed(100)
        xs = {K: torch.randn(1, K, generator=g, device=device).to(dtype) for K in {m["K"] for m in model}}
        ys = {N: torch.empty(1, N, dtype=dtype, device=device) for N in {m["N"] for m in model}}
        p = lambda t: ctypes.c_void_p(t.data_ptr())

        def launch_all():
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            for m in model:
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
        for _ in range(args.warmup):
            gr.replay()
        torch.cuda.synchronize()
        cap = 1 << 20
        buf = np.zeros(cap, dtype=REC)
        before = np.zeros(MAX_SM, dtype=np.uint32)
        read(buf.ctypes.data, 0, before.ctypes.data, 1)
        for _ in range(args.replays):
            gr.replay()
        torch.cuda.synchronize()
        after = np.zeros(MAX_SM, dtype=np.uint32)
        n = read(buf.ctypes.data, cap, after.ctypes.data, 1)
        if n < 0:
            raise RuntimeError("trace read-back failed")
        if n > cap:
            raise SystemExit("trace buffer overflow: %d records; use fewer --replays" % n)
        recs = buf[:n]
        grid = int(recs["block"].max()) + 1
        res, res_ns, reps = analyse(recs, model, grid)
        drift = {int(i): [int(before[i]), int(after[i])] for i in np.flatnonzero(before != after)}
        card = bds.card_info(0)
        rec = {"card": card, "lib": lib_path if args.lib else "trace build of this tree", "replays": reps,
               "records": int(n), "ctas_per_launch": grid, "globaltimer_step_ns": res_ns,
               "counters_nonzero_before": int(np.count_nonzero(before)), "counter_drift": drift, "boundaries": res}
    print("%s, power limit %s W; %d replays, %d records, smallest nonzero %%globaltimer step %s ns" % (
        card["name"], card["power_limit_w"], reps, n, res_ns))
    for name, r in res.items():
        print("[L = %s]  held CTAs %d, released before wait %d" % (name, r["held CTAs"], r["released before wait"]))
        for k in ("last issue -> grid end", "grid end -> wait", "wait -> first refill"):
            v = r[k]
            print("  %-24s %s" % (k, "-" if v is None else "median %7.3f us  p90 %7.3f us  (n %d)" % (
                v["median_us"], v["p90_us"], v["n"])))
    print("handoff counters: %s" % ("unchanged by the replays" if not drift else "DRIFT %s" % drift))
    print(json.dumps(rec))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1)
    if drift:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
