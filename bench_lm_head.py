"""The LM head on one H100: b200awq_lm_head against tinychat's current tail (cuBLAS through F.linear).

    python bench_lm_head.py --steps K --warmup W

Per case (the heads of Llama-3-8B, Qwen2-7B, Qwen2.5-1.5B and Qwen2-0.5B at m = 1 and m = 8 in fp16, and Llama-3-8B
in bf16), each arm captured in CUDA graphs:
    (a) plain:  lm_head_forward_cuda(x, W)                 against F.linear(x, W).float()
    (b) normed: lm_head_forward_cuda(x, W, gamma, eps)     against layernorm_forward_cuda + F.linear + .float()
    (c) (a) and (b), each followed by sample_next_token (greedy)
    (d) the last layer's down projection + residual (w4a16_linear_forward_cuda, k = 14336 for Llama-3-8B, 18944 for
        Qwen2-7B), then (b) + sampling: our tail with programmatic dependent launch on against off
The graphs of a case are replayed round by round in turn, three rounds; each figure is the median over the rounds, with
their range.  Each head is larger than the 50 MB L2, so every replay streams it from HBM.  The bytes of a call are the
weights, x and the fp32 logits, counted once; the share is those bytes over the time against 3.35 TB/s.  Our logits
are checked against torch's in the same run (same argmax on the rows where torch's top-two margin exceeds 1e-2).
Prints the card's name, power limit and SM clock, read in the same run, and one JSON line.  Writes nothing."""
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

ROUNDS = 3
HBM_BYTES_PER_S = 3.35e12
# name: (vocab, hidden, down projection's k)
HEADS = {"Llama-3-8B": (128256, 4096, 14336), "Qwen2-7B": (152064, 3584, 18944),
         "Qwen2.5-1.5B": (151936, 1536, 8960), "Qwen2-0.5B": (151936, 896, 4864)}
CASES = [(h, m, "f16") for h in HEADS for m in (1, 8)] + [("Llama-3-8B", 1, "bf16"), ("Llama-3-8B", 8, "bf16")]


def sm_clock_mhz(index):
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        return pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:  # noqa: BLE001
        return None


def time_alternating(torch, graphs, steps, warmup):
    """{name: [us per replay of each round]}; the graphs are replayed round by round in turn."""
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
            per[name].append(e0.elapsed_time(e1) * 1e3 / steps)
    return per


def case(torch, eng, name, m, dt, steps, warmup):
    import torch.nn.functional as F
    vocab, k, k_down = HEADS[name]
    T = torch.float16 if dt == "f16" else torch.bfloat16
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(vocab + k + m)
    W = (0.02 * torch.randn(vocab, k, generator=g, device=dev)).to(T)
    x = (2 * torch.randn(m, k, generator=g, device=dev)).to(T)
    gamma = (1 + 0.1 * torch.randn(k, generator=g, device=dev)).to(T)
    eps = 1e-6
    down = tuple(t.to(T) if t.dtype == torch.float16 else t for t in rand_layer(torch, k, k_down, g))
    act = (0.1 * torch.randn(m, k_down, generator=g, device=dev)).to(T)

    def ours_plain():
        return eng.lm_head_forward_cuda(x, W)

    def ours_norm(h=x):
        return eng.lm_head_forward_cuda(h, W, gamma, eps)

    def torch_plain():
        return F.linear(x, W).float()

    def torch_norm():
        xn = torch.empty_like(x)
        eng.layernorm_forward_cuda(x, gamma, xn, eps)
        return F.linear(xn, W).float()

    def sampled(fn):
        return lambda: eng.sample_next_token(fn(), None, 1.0, 1.0, 1.0, 0, True)

    def chain():
        h = eng.w4a16_linear_forward_cuda(act, *down, 128, residual=x)
        return eng.sample_next_token(ours_norm(h), None, 1.0, 1.0, 1.0, 0, True)

    fns = {"a_ours": ours_plain, "a_torch": torch_plain, "b_ours": ours_norm, "b_torch": torch_norm,
           "c_plain_ours": sampled(ours_plain), "c_plain_torch": sampled(torch_plain),
           "c_norm_ours": sampled(ours_norm), "c_norm_torch": sampled(torch_norm)}
    st = torch.cuda.Stream()
    graphs, outs = {}, {}
    for key, fn in fns.items():
        graphs[key], outs[key] = graph_of(torch, fn, st)
    for pdl in (True, False):
        old = eng.set_pdl(pdl)
        try:
            graphs[f"d_pdl{int(pdl)}"], outs[f"d_pdl{int(pdl)}"] = graph_of(torch, chain, st)
        finally:
            eng.set_pdl(old)
    for gr in graphs.values():
        gr.replay()
    torch.cuda.synchronize()
    agree = {}
    for arm in ("a", "b"):
        ref, got = outs[f"{arm}_torch"], outs[f"{arm}_ours"]
        top2 = ref.topk(2, dim=1).values
        safe = (top2[:, 0] - top2[:, 1]) > 1e-2
        agree[arm] = bool(torch.equal(got.argmax(1)[safe], ref.argmax(1)[safe]))
    agree["d_pdl_bits"] = bool(torch.equal(outs["d_pdl1"], outs["d_pdl0"]))
    per = time_alternating(torch, graphs, steps, warmup)
    del graphs, outs, W
    torch.cuda.empty_cache()
    nbytes = vocab * k * 2 + m * k * 2 + m * vocab * 4
    med = {key: round(statistics.median(v), 1) for key, v in per.items()}
    rng = {key: [round(min(v), 1), round(max(v), 1)] for key, v in per.items()}
    share = {key: round(nbytes / (med[key] * 1e-6) / HBM_BYTES_PER_S, 3) for key in ("a_ours", "a_torch", "b_ours", "b_torch")}
    rounds_faster = {arm: all(o < t for o, t in zip(per[f"{arm}_ours"], per[f"{arm}_torch"]))
                     for arm in ("a", "b", "c_plain", "c_norm")}
    return {"case": f"{name} {dt} m={m}", "vocab": vocab, "k": k, "m": m, "bytes": nbytes, "us": med, "us_range": rng,
            "share_of_3.35TBs": share, "ours_faster_every_round": rounds_faster, "checks": agree}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lm_head.py needs a CUDA device")
    import llm_awq_b200 as P
    eng = P.engine()
    card = card_info(0)
    card["name"] = card["name"] or torch.cuda.get_device_name(0)
    print(card, flush=True)
    rows, clocks = [], []
    for name, m, dt in CASES:
        r = case(torch, eng, name, m, dt, args.steps, args.warmup)
        clocks.append(sm_clock_mhz(0))
        rows.append(r)
        u, s = r["us"], r["share_of_3.35TBs"]
        print(f"{r['case']:26s} (a) ours {u['a_ours']:7.1f} us ({s['a_ours']:.2f})  torch {u['a_torch']:7.1f} us "
              f"({s['a_torch']:.2f}) | (b) ours {u['b_ours']:7.1f}  torch {u['b_torch']:7.1f} | (c) plain "
              f"{u['c_plain_ours']:7.1f} / {u['c_plain_torch']:7.1f}  norm {u['c_norm_ours']:7.1f} / "
              f"{u['c_norm_torch']:7.1f} | (d) pdl on {u['d_pdl1']:7.1f}  off {u['d_pdl0']:7.1f} | "
              f"ranges {r['us_range']} | {r['checks']}", flush=True)
    card["sm_clock_mhz_after_each_case"] = clocks
    print(json.dumps({"bench": "lm_head", "card": card, "steps": args.steps, "rounds": ROUNDS, "results": rows}))
    if not all(all(r["checks"].values()) for r in rows):
        raise SystemExit("a check failed")


if __name__ == "__main__":
    main()
