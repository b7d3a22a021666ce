#!/usr/bin/env python
"""Benchmark of the choice of the next token (tinychat's per-token block after the LM head) on 1 x H100.

    python bench_sampling.py [--steps K] [--warmup W]

Callers, timed on the same logits in the same process:
  chain       tinychat's block (stream_gen.py): transformers' TemperatureLogitsWarper, RepetitionPenaltyLogitsProcessor,
              TopPLogitsWarper and TopKLogitsWarper in a LogitsProcessorList (the restatement in
              tests/sampling_oracle.py when transformers cannot be imported), then argmax, or softmax + torch.multinomial
  this        sample_next_token, eager; when not greedy, after the torch.rand that draws its uniform (the Python mirror,
              llm_awq_b200.sampling)
  this_graph  the same calls captured in a CUDA graph (20 per graph), replayed
Batch 1, fp32 logits [1, 1, V] read as the view logits[:, -1, :], previous ids already on the device (tinychat's
torch.as_tensor copy and its int() synchronisation are not part of any caller).  Per case and caller: us per call over
K calls after W warm-up calls (CUDA events), and kernels per call (one profiled call, torch.profiler).  Greedy cases
also compare the chosen tokens.  Prints one JSON line with the card's name, power limit and SM clocks.  Synthetic,
seeded logits (N(0, 2^2)).  Writes nothing in the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_kv_cache_attention import clocks  # noqa: E402
from bench_siglip import card_info  # noqa: E402

VOCABS = (32000, 128256, 152064)
SETTINGS = {  # tinychat gen_params: temp, repeat_penalty, top_p, top_k
    "defaults": (0.2, 1.1, 0.95, 50),
    "full_vocab_top_p": (1.0, 1.0, 0.95, 0),
    "greedy": (0.0, 1.1, 0.95, 50),
}
N_PREV = (0, 512, 4096)
GRAPH_CALLS = 20


def chain_fn(torch, V, temp, penalty, top_p, top_k):
    """tinychat's per-token block as a function of (logits [1, S, V], output ids [1, n]) -> token tensor."""
    try:
        from transformers.generation import logits_process as lp
        procs = lp.LogitsProcessorList()
        if temp >= 1e-5 and temp != 1.0:
            procs.append(lp.TemperatureLogitsWarper(temp))
        if penalty > 1.0:
            procs.append(lp.RepetitionPenaltyLogitsProcessor(penalty))
        if 1e-8 <= top_p < 1.0:
            procs.append(lp.TopPLogitsWarper(top_p))
        procs.append(lp.TopKLogitsWarper(top_k if top_k > 0 else V))
        source = "transformers"
    except ImportError:
        import sampling_oracle as O

        def procs(ids, scores):
            return O.restate(scores, ids, temp if temp >= 1e-5 and temp != 1.0 else 1.0, penalty, top_p if top_p < 1.0 else 1.0,
                             top_k if top_k > 0 else V).to(scores.device)
        source = "restatement"
    greedy = temp < 1e-5 or top_p < 1e-8

    def run(logits, ids):
        last = procs(ids if penalty > 1.0 else None, logits[:, -1, :])[0]
        if greedy:
            return torch.argmax(last)
        return torch.multinomial(torch.softmax(last, dim=-1), num_samples=1)
    return run, source


def kernels_per_call(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sum(1 for n in names if not n.startswith(("Memcpy", "Memset")))


def time_us(torch, fn, steps, warmup, per=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / (steps * per)


def run(args):
    import torch
    from llm_awq_b200 import sampling as S
    device = torch.device("cuda", 0)
    card = card_info(0)
    clk_before = clocks(0)
    results = []
    for V in VOCABS:
        g = torch.Generator(device=device).manual_seed(V)
        logits = torch.randn(1, 1, V, generator=g, device=device) * 2
        for setting, (temp, penalty, top_p, top_k) in SETTINGS.items():
            for n_prev in N_PREV:
                ids = torch.randint(0, V, (1, n_prev), generator=g, device=device)
                chain, source = chain_fn(torch, V, temp, penalty, top_p, top_k)

                def this():
                    return S.sample_next_token(logits[:, -1, :], ids, temp, penalty, top_p, top_k, V)
                row = {"vocab": V, "setting": setting, "n_prev": n_prev, "chain_source": source}
                row["chain_kernels"] = kernels_per_call(torch, lambda: chain(logits, ids))
                row["this_kernels"] = kernels_per_call(torch, this)
                this()
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    this()
                torch.cuda.current_stream().wait_stream(s)
                with torch.cuda.graph(graph):
                    for _ in range(GRAPH_CALLS):
                        this()
                row["chain_us"] = time_us(torch, lambda: chain(logits, ids), args.steps, args.warmup)
                row["this_us"] = time_us(torch, this, args.steps, args.warmup)
                row["this_graph_us"] = time_us(torch, graph.replay, max(1, args.steps // GRAPH_CALLS),
                                               max(1, args.warmup // GRAPH_CALLS), per=GRAPH_CALLS)
                if setting == "greedy":
                    row["greedy_match"] = int(chain(logits, ids)) == int(this()[0])
                del graph
                results.append(row)
                print(f"{V:7d} {setting:17s} n_prev {n_prev:5d}  chain {row['chain_us']:8.1f} us "
                      f"({row['chain_kernels']:2d} kernels)  this {row['this_us']:6.1f} us ({row['this_kernels']} kernels)"
                      f"  graph {row['this_graph_us']:6.1f} us", file=sys.stderr)
    return {"bench": "sampling", "card": card, "clocks_before": clk_before, "clocks_after": clocks(0),
            "steps": args.steps, "warmup": args.warmup, "results": results}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py needs a CUDA device")
    print(json.dumps(run(args)))


if __name__ == "__main__":
    main()
