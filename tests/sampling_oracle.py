"""Restatement of tinychat's per-token logits chain (tinychat/stream_generators/stream_gen.py) and a float64 oracle of
the draw, shared by the sampling tests (tests/test_sampling_*.py).

`restate` is HF's four processors on CPU fp32 tensors, with two definitions the library makes: the top-p sort is
stable (ties ordered by index) and its cumulative sums are float64.  `draw` is the inverse CDF over float64
probabilities.  The kernel's probabilities are fp32 exponentials summed in fixed point, so near the top-p threshold it
may decide a token differently from `restate`: TOPP_BOUND bounds that band (DESIGN §3.12), and `safe_top_p` picks a
top_p whose threshold lies further than that from every token's cumulative probability, so that no token of a test
row falls in the band.

DRAW_BOUND bounds the distance between an edge of the kernel's inverse CDF and the float64 edge.  The kernel draws
token j when W_j <= floor(u S) < W_j+1, with W_j the sum of the kept weights before j, S their total, and
w_i = rn(2^44 expf(fp32(x_i - max))).  Its lower edge of token j is W_j / S (the double product u S rounds by 2^-53
relative, negligible); the float64 edge is P_j / P over p_i = exp(x_i - max).  Per token, w_i = 2^44 p_i (1 + e_i) + r_i
with
  |e_i| <= 2^-22 + 2^-24 d_i: expf is within 2 ulp (CUDA's bound without fast math; an ulp is at most 2^-23 of the
          value), and fp32(x_i - max) is within 2^-24 d_i of d_i = max - x_i, which moves exp(-d_i) by 2^-24 d_i relative;
  |r_i| <= 1/2: the rounding to an integer (a weight below 2^-45 rounds to 0).
The error of W_j / S - P_j / P is at most (sum_i |e_i| p_i + n 2^-45) / P, with n the kept tokens (<= 2^18) and P >= 1
(the maximum weighs 1).  sum_i p_i d_i / P is the mean of d under the kept distribution, which is its entropy minus
ln P, so at most ln n.  Hence |W_j / S - P_j / P| <= 2^-22 + 2^-24 ln n + n 2^-45 (about 9.9e-7 at n = 2^18).  A
measured edge is the smallest fp32 u at or above the kernel's edge, at most one fp32 spacing below 1 (2^-24) above it.
The same terms bound the kernel's top-p decisions; TOPP_BOUND keeps a 10x margin over them."""
import math

import numpy as np
import torch

TOPP_BOUND = 1e-5   # |cumulative probability - (1 - top_p)| within which kernel and restatement may disagree
MIN_P = 1e-5        # the midpoint tests address only kept tokens of at least this probability
MAX_VOCAB = 2 ** 18         # B200AWQ_SAMPLE_MAX_VOCAB
EXPF_ULP = 2                # CUDA's maximum ulp error of expf (no fast math)
FIXED_POINT_BITS = 44       # weights are exp(x - max) in units of 2^-44
DRAW_BOUND = (EXPF_ULP * 2.0 ** -23 + 2.0 ** -24 * math.log(MAX_VOCAB) + MAX_VOCAB * 2.0 ** -(FIXED_POINT_BITS + 1)
              + 2.0 ** -24)

SAMPLE_CTAS = 8             # CTAs per row (one cluster)
SAMPLE_THREADS = 512        # threads per CTA


def slices(V):
    """The launcher's partition of a row of V keys over the cluster: [(start, stop)] of each CTA, some possibly empty.
    CTA r holds [r slice, min(V, (r + 1) slice)), slice = ceil(ceil(V / 8) / 32) 32."""
    per_cta = -(-V // SAMPLE_CTAS)
    s = -(-per_cta // 32) * 32
    return [(min(V, r * s), min(V, (r + 1) * s)) for r in range(SAMPLE_CTAS)]


def draw_chunk(n):
    """Keys per thread of a CTA's draw scan over its n keys: thread t scans [t chunk, (t + 1) chunk)."""
    return -(-n // SAMPLE_THREADS)


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


def topp_order(scores_row):
    """(the stable ascending order of a row's values, the float64 inclusive cumulative probability along it)."""
    x = scores_row.detach().to("cpu", torch.float32)
    order = torch.sort(x, stable=True).indices
    return order.numpy(), torch.softmax(x.double(), 0)[order].cumsum(0).numpy()


def topp_cut(cum, top_p):
    """How many tokens top-p removes, given `cum` from topp_order: the position in the ascending order of the first
    kept token (the last token is always kept)."""
    return min(int(np.searchsorted(cum, thr_of(top_p), side="right")), len(cum) - 1)


def topp_margin(scores_row, top_p):
    """The smallest distance between the threshold and a token's float64 cumulative probability (ascending, stable)."""
    return float(np.abs(topp_order(scores_row)[1] - thr_of(top_p)).min())


def safe_top_p(scores, want):
    """A top_p near `want` whose threshold lies more than TOPP_BOUND from every cumulative probability of each row
    (`scores`: one row or [B, V] rows of the values top-p sees, i.e. after temperature and penalty)."""
    rows = scores.reshape(-1, scores.shape[-1])
    cums = [topp_order(r)[1] for r in rows]
    edges = np.unique(np.concatenate([[0.0]] + cums))
    gaps = edges[1:] - edges[:-1]
    mids = (edges[1:] + edges[:-1]) / 2
    ok = np.nonzero(gaps > 3 * TOPP_BOUND)[0]
    for i in ok[np.argsort(np.abs(mids[ok] - (1.0 - want)))]:
        top_p = float(np.float32(1.0 - mids[i]))
        thr = thr_of(top_p)
        if 0.0 < top_p < 1.0 and all(np.abs(c - thr).min() > TOPP_BOUND for c in cums):
            return top_p
    raise AssertionError("no top_p with a safe margin near %g" % want)


def masses(x_row):
    """float64 exp(x - max) of a processed row (0 for -inf)."""
    x = x_row.detach().to("cpu").double()
    return torch.exp(x - x.max()).numpy()


def draw(x_row, u, greedy=False):
    """The token the chain picks from a processed row: the first maximum, or the inverse CDF at u (a number, or an
    array of them)."""
    if greedy:
        return int(torch.argmax(x_row))
    p = masses(x_row)
    cdf = np.cumsum(p)
    t = np.searchsorted(cdf, np.asarray(u, dtype=np.float64) * cdf[-1], side="right")
    return int(t) if t.ndim == 0 else t


def cdf_edges(x_row):
    """(the kept tokens of probability >= MIN_P after the first kept token, in index order; the float64 lower edge of
    each one's CDF interval, i.e. the probability of the kept tokens before it)."""
    p = masses(x_row)
    cdf = np.cumsum(p)
    S = cdf[-1]
    idx = np.nonzero(p / S >= MIN_P)[0]
    idx = idx[idx > np.nonzero(p > 0)[0][0]]
    return idx, (cdf[idx] - p[idx]) / S


def midpoints(x_row):
    """(kept tokens of probability >= MIN_P in index order, the fp32 midpoints of their CDF intervals)."""
    p = masses(x_row)
    cdf = np.cumsum(p)
    S = cdf[-1]
    idx = np.nonzero(p / S >= MIN_P)[0]
    mid = ((cdf[idx] - p[idx] / 2) / S).astype(np.float32)
    return idx, mid
