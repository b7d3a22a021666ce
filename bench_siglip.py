#!/usr/bin/env python
"""Benchmark of the W8A8 vision-tower ops: NVILA's SigLIP-so400m-patch14-448 tower on 1 x H100.

    python bench_siglip.py [--steps K] [--warmup W] [--dump-outputs DIR]

Prints one JSON line.  A step is 27 layers x {LN-quant, qkv+bias, quant, out+bias, LN-quant, fc1+bias, gelu-quant,
fc2+bias} over 1024 tokens per image (tinychat's QuantSiglipEncoder, seqlen 1024), timed at 1 and at 8 images as a
CUDA graph of C-ABI launches (include/b200awq.h), K steps after W warm-up steps, CUDA events.  Every layer's weights are
distinct (411 MB of int8 weights, beyond the 50 MB L2).  Per GEMM shape the line gives TOP/s against the dense INT8
data-sheet rate (1979 TOP/s) and bytes/s against 3.35 TB/s (ops 2MNK; bytes MK + NK + 2MN + 2(M + 2N)) and names the
bound.  With oracle/_ref/ref_awq_w8a8 built (oracle/build_ref_w8a8.py), `reference_on_gpu` times the reference's own
W8A8 kernels in the same step, eager on the legacy default stream, beside this repo launched the same way.
--dump-outputs DIR writes the last step's fc2 output (first 1024 tokens) and scales as DIR/<name>.npy (float32).
Synthetic, seeded data.  Writes nothing in the tree unless --dump-outputs points there.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import dump_outputs, timed_steps  # noqa: E402  (the timing and dump helpers of the main benchmark)

# ------------------------------------------------------------------------------------------ siglip (W8A8)
SIGLIP_SO400M = dict(name="SigLIP-so400m-patch14-448", hidden=1152, inter=4304, layers=27, tokens=1024)
INT8_TOPS = 1979.0  # H100 SXM data sheet, dense INT8 tensor-core rate (TOP/s)


def card_info(index):
    """Name and power limit of the card (read-only NVML queries); None where NVML is unavailable."""
    info = {"name": None, "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        name = pynvml.nvmlDeviceGetName(h)
        info["name"] = name.decode() if isinstance(name, bytes) else name
        info["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:  # noqa: BLE001
        pass
    return info


def run_siglip(args):
    """W8A8 ops of NVILA's SigLIP-so400m-patch14-448 vision tower (tinychat QuantSiglipEncoder, seqlen 1024).

    One step = 27 layers x {LN-quant, qkv+bias, quant, out+bias, LN-quant, fc1+bias, gelu-quant, fc2+bias} over
    1024 tokens per image, at 1 and at 8 images, every layer's weights distinct (411 MB of int8 weights: beyond L2).
    Attention (flash-attn), the residual adds and the projector are not part of the step: the quant step reads a
    fixed stand-in for the attention output and the second LN reads the out-projection's output."""
    import torch
    import llm_awq_b200 as P
    device = torch.device("cuda", 0)
    lib = P.lib()
    cfg = SIGLIP_SO400M
    H, I, L = cfg["hidden"], cfg["inter"], cfg["layers"]
    shapes = {"qkv": (3 * H, H), "out": (H, H), "fc1": (I, H), "fc2": (H, I)}
    g = torch.Generator(device=device).manual_seed(1152)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None

    def rnd(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device=device) * scale

    layers = []
    for _ in range(L):
        lay = {nm: dict(w=torch.randint(-127, 128, (n, k), generator=g, device=device, dtype=torch.int8),
                        ws=(0.002 + 0.01 * torch.rand(n, generator=g, device=device)).half(),
                        b=rnd(n, scale=0.1).half()) for nm, (n, k) in shapes.items()}
        for ln in ("ln1", "ln2"):
            lay[ln] = ((1 + 0.1 * rnd(H)).half(), (0.1 * rnd(H)).half())
        layers.append(lay)
    weights_bytes = sum(v["w"].numel() for lay in layers for k, v in lay.items() if k in shapes)

    def buffers(M):
        return dict(h=rnd(M, H).half(), attn=rnd(M, H).half(), qH=torch.empty(M, H, dtype=torch.int8, device=device),
                    qI=torch.empty(M, I, dtype=torch.int8, device=device), s=torch.empty(M, dtype=torch.float16, device=device),
                    y={nm: torch.empty(M, n, dtype=torch.float16, device=device) for nm, (n, k) in shapes.items()},
                    tmp=torch.empty(M, I, dtype=torch.float16, device=device))

    def check(rc):
        if rc != 0:
            raise RuntimeError(lib.b200awq_strerror(rc).decode())

    def step_abi(M, bf, only=None):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        s, y = bf["s"], bf["y"]

        def lin(lay, nm):
            n, k = shapes[nm]
            W_ = lay[nm]
            q = bf["qI"] if nm == "fc2" else bf["qH"]
            check(lib.b200awq_w8a8_gemm(p(q), p(W_["w"]), p(W_["ws"]), p(s), p(W_["b"]), p(y[nm]), M, n, k, st))
        for lay in layers:
            if only is not None:
                lin(lay, only)
                continue
            check(lib.b200awq_layernorm_quant(p(bf["h"]), p(lay["ln1"][0]), p(lay["ln1"][1]), p(bf["qH"]), p(s), M, H,
                                              ctypes.c_float(1e-6), 1, 0, st))
            lin(lay, "qkv")
            check(lib.b200awq_quant_per_token(p(bf["attn"]), p(bf["qH"]), p(s), M, H, 0, st))
            lin(lay, "out")
            check(lib.b200awq_layernorm_quant(p(y["out"]), p(lay["ln2"][0]), p(lay["ln2"][1]), p(bf["qH"]), p(s), M, H,
                                              ctypes.c_float(1e-6), 1, 0, st))
            lin(lay, "fc1")
            check(lib.b200awq_gelu_quant(p(y["fc1"]), p(bf["qI"]), p(s), p(bf["tmp"]), M, I, st))
            lin(lay, "fc2")

    def graph_of(fn):
        sg = torch.cuda.Stream()
        with torch.cuda.stream(sg):
            fn()
        sg.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fn()
        return gr

    ref = None
    if os.path.isdir(os.path.join(ROOT, "oracle", "_ref")):  # built by oracle/build_ref_w8a8.py
        try:
            sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
            import importlib
            ref = importlib.import_module("ref_awq_w8a8")
        except Exception as e:  # noqa: BLE001
            ref = repr(e)[:200]

    def step_ref(M, bf, only=None):
        qH, qI, s, y = bf["qH"], bf["qI"], bf["s"], bf["y"]

        def lin(lay, nm):
            W_ = lay[nm]
            ref.w8a8_gemm_fuse_bias_forward_cuda(qI if nm == "fc2" else qH, W_["w"], W_["ws"], s, y[nm], W_["b"])
        for lay in layers:
            if only is not None:
                lin(lay, only)
                continue
            ref.rms_norm_general(qH, bf["h"], lay["ln1"][0], lay["ln1"][1], s, 1e-6, True)
            lin(lay, "qkv")
            ref.invoke_quant(qH, bf["attn"], s)
            lin(lay, "out")
            ref.rms_norm_general(qH, y["out"], lay["ln2"][0], lay["ln2"][1], s, 1e-6, True)
            lin(lay, "fc1")
            ref.gelu_and_quant(qI, y["fc1"], s, bf["tmp"])
            lin(lay, "fc2")

    results, dumps = {}, {}
    for images in (1, 8):
        M = cfg["tokens"] * images
        bf = buffers(M)
        gr = graph_of(lambda: step_abi(M, bf))
        ms, _ = timed_steps(torch, None, device, gr.replay, args.steps, args.warmup)
        res = {"tokens": M, "us_per_step": ms * 1e3 / args.steps, "images_per_s": images * 1000.0 * args.steps / ms,
               "launches_per_step": 8 * L, "gemm": {}}
        kk = max(1, args.steps // 4)
        for nm, (n, k) in shapes.items():
            gg = graph_of(lambda nm=nm: step_abi(M, bf, only=nm))
            ms_g, _ = timed_steps(torch, None, device, gg.replay, kk, args.warmup)
            t = ms_g * 1e-3 / (kk * L)
            ops, byt = 2.0 * M * n * k, float(M * k + n * k + 2 * M * n + 2 * (M + 2 * n))
            bound = "tensor" if ops / (INT8_TOPS * 1e12) >= byt / 3.35e12 else "hbm"
            res["gemm"][nm] = {"M": M, "N": n, "K": k, "us": t * 1e6, "TOPs": ops / t / 1e12,
                               "frac_int8_peak": ops / t / 1e12 / INT8_TOPS, "GBps": byt / t / 1e9,
                               "frac_hbm": byt / t / 3.35e12, "bound": bound,
                               "bound_us": max(ops / (INT8_TOPS * 1e12), byt / 3.35e12) * 1e6}
        if ref is not None and not isinstance(ref, str):
            ke = max(1, args.steps // 4)
            with torch.cuda.stream(torch.cuda.default_stream()):
                ms_r, _ = timed_steps(torch, None, device, lambda: step_ref(M, bf), ke, args.warmup)
                ms_o, _ = timed_steps(torch, None, device, lambda: step_abi(M, bf), ke, args.warmup)
                per = {}
                for nm in shapes:
                    ms_rg, _ = timed_steps(torch, None, device, lambda nm=nm: step_ref(M, bf, only=nm), ke, args.warmup)
                    ms_og, _ = timed_steps(torch, None, device, lambda nm=nm: step_abi(M, bf, only=nm), ke, args.warmup)
                    per[nm] = {"reference_us": ms_rg * 1e3 / (ke * L), "this_repo_us": ms_og * 1e3 / (ke * L)}
            res["reference_on_gpu"] = {"eager_us_per_step": ms_r * 1e3 / ke, "this_repo_eager_us_per_step": ms_o * 1e3 / ke,
                                       "gemm_eager": per,
                                       "how": "ref_awq_w8a8 (oracle/build_ref_w8a8.py) entry points, plain launches on the legacy default stream; "
                                              "this repo's C ABI launched the same way beside it"}
        elif isinstance(ref, str):
            res["reference_on_gpu"] = {"unavailable": ref}
        gr.replay()  # the dumped outputs are those of one full step of this repo's kernels
        torch.cuda.synchronize()
        dumps[f"siglip_{images}img_fc2"] = bf["y"]["fc2"][:1024]
        dumps[f"siglip_{images}img_scales"] = bf["s"]
        results[f"{images}img"] = res

    if args.dump_outputs:
        dump_outputs(args.dump_outputs, dumps)
    one, eight = results["1img"], results["8img"]
    line = {"metric": "SigLIP-so400m W8A8 vision-tower ops, images/s at 8 images per step, 1xH100",
            "value": eight["images_per_s"], "unit": "images/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "higher_is_better": True, "dtype": "int8 x int8 -> fp16", "data": "synthetic",
            "config": {"workload": "NVILA SigLIP-so400m-patch14-448: 27 layers x {LN-quant, qkv+bias, quant, out+bias, LN-quant, "
                                   "fc1+bias, gelu-quant, fc2+bias}, 1024 tokens per image, C ABI in a CUDA graph",
                       "excluded": "attention (flash-attn), residual adds, projector",
                       "weights_bytes": weights_bytes, "l2": "411 MB of distinct int8 weights per step: beyond L2",
                       "peaks": {"int8_tops": INT8_TOPS, "hbm_tbps": 3.35, "source": "H100 SXM data sheet (700 W)"}},
            "card": card_info(0), "1_image": one, "8_images": eight}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1 is supported")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last step's outputs as DIR/<name>.npy (float32)")
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_siglip.py runs on one GPU")
    run_siglip(args)


if __name__ == "__main__":
    main()
