"""Restatement of tinychat's per-token logits chain (tinychat/stream_generators/stream_gen.py) and a float64 oracle of
the draw, shared by tests/test_sampling_cpu.py and tests/test_sampling_gpu.py.

`restate` is HF's four processors on CPU fp32 tensors, with two definitions the library makes: the top-p sort is
stable (ties ordered by index) and its cumulative sums are float64.  `draw` is the inverse CDF over float64
probabilities.  The kernel's probabilities are fp32 exponentials summed in fixed point, so near the top-p threshold it
may decide a token differently from `restate`: TOPP_BOUND bounds that band (DESIGN §3.12), and `safe_top_p` picks a
top_p whose threshold lies further than that from every token's cumulative probability, so that no token of a test
row falls in the band."""
import numpy as np
import torch

TOPP_BOUND = 1e-5   # |cumulative probability - (1 - top_p)| within which kernel and restatement may disagree
MIN_P = 1e-5        # the midpoint tests address only kept tokens of at least this probability


def thr_of(top_p):
    """fp32(1 - top_p) for the fp32 top_p the kernel receives."""
    return float(np.float32(1.0 - float(np.float32(top_p))))


def restate(scores, prev_ids=None, temperature=1.0, penalty=1.0, top_p=1.0, top_k=0):
    """fp32 [B, V] logits -> fp32 [B, V] processed scores, removed tokens at -inf.  prev_ids int64 [B, n] (ids outside
    [0, V) are ignored), or None."""
    x = scores.detach().to("cpu", torch.float32).clone()
    B, V = x.shape
    if temperature != 1.0:
        x = x / torch.tensor(temperature, dtype=torch.float32)
    if penalty > 1.0 and prev_ids is not None:
        p = torch.tensor(penalty, dtype=torch.float32)
        prev = prev_ids.detach().cpu()
        for b in range(B):
            ids = prev[b][(prev[b] >= 0) & (prev[b] < V)]
            if len(ids):
                g = x[b, ids]
                x[b, ids] = torch.where(g < 0, g * p, g / p)
    if top_p < 1.0:
        thr = thr_of(top_p)
        for b in range(B):
            order = torch.sort(x[b], stable=True).indices
            cum = torch.softmax(x[b].double(), 0)[order].cumsum(0)
            remove = cum <= thr
            remove[-1] = False
            x[b, order[remove]] = -float("inf")
    if 0 < top_k < V:
        kth = torch.topk(x, top_k, dim=-1).values[:, -1:]
        x = x.masked_fill(x < kth, -float("inf"))
    return x


def topp_margin(scores_row, top_p):
    """The smallest distance between the threshold and a token's float64 cumulative probability (ascending, stable)."""
    x = scores_row.detach().to("cpu", torch.float32)
    order = torch.sort(x, stable=True).indices
    cum = torch.softmax(x.double(), 0)[order].cumsum(0)
    return float((cum - thr_of(top_p)).abs().min())


def safe_top_p(scores_row, want):
    """A top_p near `want` whose threshold lies more than TOPP_BOUND from every cumulative probability of the row
    (`scores_row`: the values top-p sees, i.e. after temperature and penalty)."""
    x = scores_row.detach().to("cpu", torch.float32)
    cum = torch.softmax(x.double(), 0)[torch.sort(x, stable=True).indices].cumsum(0).numpy()
    edges = np.concatenate(([0.0], cum))
    gaps = edges[1:] - edges[:-1]
    mids = (edges[1:] + edges[:-1]) / 2
    ok = np.nonzero(gaps > 3 * TOPP_BOUND)[0]
    for i in ok[np.argsort(np.abs(mids[ok] - (1.0 - want)))]:
        top_p = float(np.float32(1.0 - mids[i]))
        if 0.0 < top_p < 1.0 and topp_margin(x, top_p) > TOPP_BOUND:
            return top_p
    raise AssertionError("no top_p with a safe margin near %g" % want)


def masses(x_row):
    """float64 exp(x - max) of a processed row (0 for -inf)."""
    x = x_row.detach().to("cpu").double()
    return torch.exp(x - x.max()).numpy()


def draw(x_row, u, greedy=False):
    """The token the chain picks from a processed row: the first maximum, or the inverse CDF at u."""
    if greedy:
        return int(torch.argmax(x_row))
    p = masses(x_row)
    cdf = np.cumsum(p)
    return int(np.searchsorted(cdf, u * cdf[-1], side="right"))


def midpoints(x_row):
    """(kept tokens of probability >= MIN_P in index order, the fp32 midpoints of their CDF intervals)."""
    p = masses(x_row)
    cdf = np.cumsum(p)
    S = cdf[-1]
    idx = np.nonzero(p / S >= MIN_P)[0]
    mid = ((cdf[idx] - p[idx] / 2) / S).astype(np.float32)
    return idx, mid
