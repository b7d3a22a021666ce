"""b200awq_sample_next_token over its whole envelope, against the restatement and the float64 oracle
(tests/sampling_oracle.py).

Each row is one cluster of 8 CTAs, CTA r holding keys [r slice, min(V, (r + 1) slice)) (`O.slices`), and the grid holds
at most 65535 clusters, so a larger batch makes each cluster carry its state from one row to the next.  The tests put
the row maximum on every CTA's first and last key for vocabularies with short and empty last CTAs up to the bound
262144, run 2 * 65535 + 17 rows, cut tie groups that span all eight CTAs with top-p and top-k, and measure the two
numerical claims of DESIGN §3.12: the top-p band (TOPP_BOUND) and the edges of the draw's CDF (DRAW_BOUND)."""
import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import sampling_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VOCABS = [1, 2, 31, 33, 255, 257, 1000, 4097, 32064, 50257, 65024, 92544, 151936, 256000, 262143, 262144]
MAX_CLUSTERS = 65535
U1 = float(np.nextafter(np.float32(1), np.float32(0)))
INF = float("inf")
# temperature, penalty, top_p wanted (made safe per test), top_k
PROCS = {"off": (1.0, 1.0, 1.0, 0), "T_penalty": (0.7, 1.3, 1.0, 0), "defaults": (0.2, 1.1, 0.95, 50)}


def _call(logits, prev=None, T=1.0, pen=1.0, top_p=1.0, top_k=0, greedy=False, u=None):
    """Through the C ABI into a token buffer filled with -1, so that a row the kernel never writes shows up (a fresh
    tensor could hold an earlier call's tokens)."""
    B, V = logits.shape
    tokens = torch.full((B,), -1, dtype=torch.long, device=DEV)
    rc = P.lib().b200awq_sample_next_token(logits.data_ptr(), logits.stride(0), B, V,
                                           None if prev is None else prev.data_ptr(),
                                           0 if prev is None else prev.stride(0), 0 if prev is None else prev.shape[1],
                                           T, pen, top_p, top_k, int(greedy), None if greedy else u.data_ptr(),
                                           tokens.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    return tokens.cpu()


def _safe(x, prev, T, pen, want_p):
    return want_p if want_p >= 1.0 else O.safe_top_p(O.restate(x, prev, T, pen), want_p)


def _enumerate(x_row, prev_row, T, pen, top_p, k):
    """(processed row, kept tokens of probability >= MIN_P, what the kernel returns at their CDF midpoints) through a
    stride-0 batch of the same row."""
    proc = O.restate(x_row[None].cpu(), None if prev_row is None else prev_row[None].cpu(), T, pen, top_p, k)[0]
    idx, mid = O.midpoints(proc)
    got = []
    for s in range(0, len(mid), 8192):
        u = torch.from_numpy(mid[s:s + 8192]).to(DEV)
        n = len(u)
        prev = None if prev_row is None else prev_row[None].expand(n, -1)
        got.append(_call(x_row[None].expand(n, -1), prev, T, pen, top_p, k, u=u))
    return proc, idx, torch.cat(got).numpy()


def _prev_avoiding(x, keep, n, seed):
    """Penalised ids per row: the row's largest values other than `keep[b]` (so the penalty reorders the top), random
    ids, and ids outside [0, V)."""
    B, V = x.shape
    g = torch.Generator().manual_seed(seed)
    top = torch.topk(x, min(V, 24), dim=1).indices
    p = torch.randint(0, V, (B, n), generator=g)
    p[:, :top.shape[1]] = top
    p[:, -4:] = torch.tensor([-1, V, 2 ** 40, -(2 ** 40)])
    p[p == torch.as_tensor(keep)[:, None]] = -1
    return p


# ------------------------------------------------------------------------------------------------ partition geometry
@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("procs", list(PROCS))
def test_greedy_maximum_on_every_slice_edge(V, procs):
    """One row per placement of the maximum: each CTA's first and last key and V - 1.  The rows are contiguous, so for
    odd V they start off 16-byte alignment."""
    pos = sorted({V - 1} | {i for lo, hi in O.slices(V) if hi > lo for i in (lo, hi - 1)})
    B = len(pos)
    x = torch.randn(B, V, generator=torch.Generator().manual_seed(V)) * 0.5
    x[torch.arange(B), pos] = x.max(dim=1).values + 0.05
    T, pen, want_p, k = PROCS[procs]
    prev = _prev_avoiding(x, pos, 40, seed=V)
    top_p = _safe(x, prev, T, pen, want_p)
    want = O.restate(x, prev, T, pen, top_p, k).argmax(dim=1)
    assert want.tolist() == pos
    assert torch.equal(_call(x.to(DEV), prev.to(DEV), T, pen, top_p, k, greedy=True), want)


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("case", ["defaults", "full_vocab_top_p"])
def test_midpoints_at_every_partition(V, case):
    g = torch.Generator().manual_seed(V + 1)
    if case == "defaults":
        x = torch.randn(V, generator=g) * 0.5
        T, pen, want_p, k = PROCS["defaults"]
        prev = _prev_avoiding(x[None], [-1], 600, seed=V)[0]
    else:
        x = torch.randn(V, generator=g) * 3
        T, pen, want_p, k, prev = 1.0, 1.0, 0.95, 0, None
    top_p = _safe(x[None], None if prev is None else prev[None], T, pen, want_p)
    proc, idx, got = _enumerate(x.to(DEV), None if prev is None else prev.to(DEV), T, pen, top_p, k)
    assert np.array_equal(got, idx), (len(got), len(idx), np.nonzero(got != idx)[0][:5])


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("procs", list(PROCS))
def test_u_edges_and_odd_row_strides(V, procs):
    """Batch 3, contiguous rows: u = 0 returns the first kept token, u just below 1 the last, a midpoint its token."""
    x = torch.randn(3, V, generator=torch.Generator().manual_seed(V + 2))
    x[:, 0] = x[:, V - 1] = 6.0  # the first and last indices kept, with non-negligible mass
    if V >= 3:
        x[1, 0] = -INF
    T, pen, want_p, k = PROCS[procs]
    prev = _prev_avoiding(x, [0, V - 1, 0], 40, seed=V)
    prev[prev == V - 1] = -1
    top_p = _safe(x, prev, T, pen, want_p)
    proc = O.restate(x, prev, T, pen, top_p, k)
    mids = []
    for b in range(3):
        idx, mid = O.midpoints(proc[b])
        mids.append(float(mid[(b * len(mid)) // 3]))
    xd, pd = x.to(DEV), prev.to(DEV)
    for u in ([0.0] * 3, [U1] * 3, mids):
        want = [O.draw(proc[b], u[b]) for b in range(3)]
        assert _call(xd, pd, T, pen, top_p, k, u=torch.tensor(u, device=DEV)).tolist() == want, u
    if V >= 3:
        assert [O.draw(proc[b], 0.0) for b in range(3)] == [0, int(np.nonzero(O.masses(proc[1]) > 0)[0][0]), 0]
        assert [O.draw(proc[b], U1) for b in range(3)] == [V - 1] * 3


# ------------------------------------------------------------------------------------------------ more rows than clusters
def test_rows_beyond_the_grid_carry_no_state():
    """2 * 65535 + 17 rows: clusters 0-16 take three rows, the others two.  Row b reads base row b mod 61, so rows b and
    b + 65535 differ in penalised ids, tie placement and whether top-k runs; each row's u is the midpoint of one kept
    token of its base row."""
    R, V, B = 61, 1000, 2 * MAX_CLUSTERS + 17
    assert MAX_CLUSTERS % R != 0
    g = torch.Generator().manual_seed(61)
    scale = torch.linspace(0.25, 6.0, R)[torch.randperm(R, generator=g)][:, None]
    base = torch.round(torch.randn(R, V, generator=g) * scale * 4) / 4  # a 0.25 grid: ties at the cuts
    base_prev = torch.randint(-3, V + 3, (R, 32), generator=g)
    T, pen, k = 0.7, 1.2, 50
    top_p = O.safe_top_p(O.restate(base, base_prev, T, pen), 0.9)
    kept_p = torch.isfinite(O.restate(base, base_prev, T, pen, top_p)).sum(dim=1)
    assert (kept_p <= k).any() and (kept_p > k).any()
    proc = O.restate(base, base_prev, T, pen, top_p, k)
    kept = [O.midpoints(proc[r]) for r in range(R)]
    rows = torch.arange(B)
    r_of, j_of = (rows % R).numpy(), (rows // R).numpy()
    want = torch.tensor([int(kept[r][0][j % len(kept[r][0])]) for r, j in zip(r_of, j_of)])
    u = torch.tensor([float(kept[r][1][j % len(kept[r][0])]) for r, j in zip(r_of, j_of)], device=DEV)
    logits = base.to(DEV)[rows.to(DEV) % R]
    prev = base_prev.to(DEV)[rows.to(DEV) % R]
    got = _call(logits, prev, T, pen, top_p, k, False, u)
    bad = torch.nonzero(got != want)[:, 0]
    assert len(bad) == 0, (len(bad), bad[:8].tolist(), got[bad[:8]].tolist(), want[bad[:8]].tolist())
    want_g = proc.argmax(dim=1)[rows % R]
    assert torch.equal(_call(logits, prev, T, pen, top_p, k, True), want_g)
    del logits, prev

    # one row read through a stride-0 view by the same batch, tinychat's defaults
    V = 152064
    x = torch.randn(1, V, generator=g) * 0.5
    xp = torch.randint(0, V, (1, 600), generator=g)
    T, pen, _, k = PROCS["defaults"]
    top_p = O.safe_top_p(O.restate(x, xp, T, pen), 0.95)
    idx, mid = O.midpoints(O.restate(x, xp, T, pen, top_p, k)[0])
    assert len(idx) > 20
    j = (rows % len(idx)).numpy()
    got = _call(x.to(DEV).expand(B, -1), xp.to(DEV).expand(B, -1), T, pen, top_p, k, False,
                    torch.from_numpy(mid[j]).to(DEV))
    assert torch.equal(got, torch.from_numpy(idx[j]))


# ------------------------------------------------------------------------------------------------ tie groups across CTAs
def _tie_row(V, tie, seed):
    """About 4000 tokens at `tie` (every CTA's first and last key, the last key of draw thread 99 and the first of
    thread 100 in each CTA, the rest at random), 3 tokens at tie + 1 and the rest near tie - 6.  The ties hold most of
    the mass, so consecutive tie ranks lie ~2.3e-4 apart in cumulative probability."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, generator=g) * 0.5 + (tie - 6.0)
    perm = torch.randperm(V, generator=g).tolist()
    ties = set(perm[:3900])
    for lo, hi in O.slices(V):
        c = O.draw_chunk(hi - lo)
        ties |= {i for i in (lo, hi - 1, lo + 100 * c - 1, lo + 100 * c) if lo <= i < hi}
    above = [i for i in perm[3900:] if i not in ties][:3]
    ties = sorted(ties)
    x[ties] = tie
    x[above] = tie + 1.0
    return x, ties, above


def _tie_cuts(V, ties):
    """Tie ranks to cut at: 0, the first and last tie of CTAs 1, 4 and 7, the ties on both sides of draw thread 100's
    first key in CTA 3, and the last tie."""
    sl = O.slices(V)
    rank = {t: r for r, t in enumerate(ties)}
    cuts = {0, len(ties) - 1}
    for r in (1, 4, 7):
        lo, hi = sl[r]
        mine = [rank[t] for t in ties if lo <= t < hi]
        cuts |= {mine[0], mine[-1]}
    lo, hi = sl[3]
    c = O.draw_chunk(hi - lo)
    cuts |= {rank[lo + 100 * c - 1], rank[lo + 100 * c]}
    return sorted(cuts)


@pytest.mark.parametrize("V,tie,signed_zeros", [(151936, -0.5, False), (151936, 0.0, True), (262144, 0.0, True),
                                                (65024, 2.5, False)])
def test_topp_cut_inside_a_tie_group_spanning_all_ctas(V, tie, signed_zeros):
    x, ties, above = _tie_row(V, tie, seed=V)
    if signed_zeros:
        x[ties[1::2]] = -0.0
    order, cum = O.topp_order(x)
    nb = V - len(ties) - len(above)  # tokens below the ties come first in the ascending order
    assert sorted(order[nb:nb + len(ties)].tolist()) == ties
    xd = x.to(DEV)
    for c in _tie_cuts(V, ties):
        lo = cum[nb + c - 1] if nb + c > 0 else 0.0
        top_p = float(np.float32(1.0 - (lo + cum[nb + c]) / 2))
        assert O.topp_cut(cum, top_p) == nb + c and O.topp_margin(x, top_p) > O.TOPP_BOUND
        kept_ties = len(ties) - c
        a = len(above)
        for k in (0, a + kept_ties - 1, a + kept_ties, a + kept_ties + 1):
            proc, idx, got = _enumerate(xd, None, 1.0, 1.0, top_p, k)
            assert np.array_equal(got, idx), (c, k, len(got), len(idx), np.nonzero(got != idx)[0][:5])
            if k == 0:
                assert int(torch.isfinite(proc[ties]).sum()) == kept_ties
                assert np.array_equal(idx, np.sort(np.concatenate([ties[c:], above])))
        assert _call(xd[None], top_p=top_p, greedy=True).tolist() == [min(above)]


def test_all_equal_row_at_the_vocabulary_bound():
    """V = 262144 equal logits: every weight is exactly 2^44, the sum reaches 2^62 and the arithmetic is exact, so the
    cut and the draw must match the oracle for every u."""
    V = O.MAX_VOCAB
    x = torch.full((V,), 1.5)
    xd = x.to(DEV)
    u = torch.cat([torch.zeros(1), torch.rand(4093, generator=torch.Generator().manual_seed(5)),
                   torch.tensor([0.5, U1])])
    n = len(u)
    for want_c in (None, 1, 32767, 32768, 131071, 250000, V - 2, V - 1):
        if want_c is None:
            top_p = 1.0
        else:
            top_p = float(np.float32(1.0 - (want_c + 0.5) / V))
            assert O.topp_cut(O.topp_order(x)[1], top_p) == want_c
        proc = O.restate(x[None], top_p=top_p)[0]
        c = 0 if want_c is None else want_c
        assert int(torch.isfinite(proc).sum()) == V - c
        want = O.draw(proc, u.numpy())
        assert want[0] == c and want[-1] == V - 1
        got = _call(xd[None].expand(n, -1), top_p=top_p, u=u.to(DEV)).numpy()
        assert np.array_equal(got, want), (want_c, np.nonzero(got != want)[0][:5])
        assert _call(xd[None], top_p=top_p, greedy=True).tolist() == [c]
        for k in (1, V - c - 1, V - c):  # the k-th value is the tie value: every kept token stays
            assert _call(xd[None], top_p=top_p, top_k=k, u=u[-1:].to(DEV)).tolist() == [V - 1]


# ------------------------------------------------------------------------------------------------ top-k edges
def _topk_row(V, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "negative":  # every value, so the k-th, negative
        return -(torch.rand(V, generator=g) * 8 + 0.1), 0
    if kind == "signed_zero":  # a block of +0 / -0 under 20 positive values
        x = -2.0 - torch.rand(V, generator=g) * 6
        perm = torch.randperm(V, generator=g)
        x[perm[:20]] = 0.5 + torch.rand(20, generator=g) * 2.5
        zeros = perm[20:min(V, 2020)]
        x[zeros] = 0.0
        x[zeros[::2]] = -0.0
        return x, 20
    x = torch.full((V,), -INF)  # fewer finite entries than most top_k below
    x[torch.randperm(V, generator=g)[:40]] = torch.randn(40, generator=g) * 2
    return x, 0


@pytest.mark.parametrize("V", [4097, 151936])
@pytest.mark.parametrize("kind", ["negative", "signed_zero", "minus_inf"])
@pytest.mark.parametrize("want_p", [1.0, 0.9])
def test_topk_edges(V, kind, want_p):
    x, n_pos = _topk_row(V, kind, seed=V)
    top_p = _safe(x[None], None, 1.0, 1.0, want_p)
    kept_p = int(torch.isfinite(O.restate(x[None], top_p=top_p)).sum())
    finite = int(torch.isfinite(x).sum())
    ks = {kept_p - 1, kept_p, kept_p + 1, V - 1, V, 2 ** 31 - 1, finite - 1, finite + 1}
    if n_pos:
        ks |= {n_pos + 1, n_pos + 500}  # the k-th value is +0 or -0
    xd = x.to(DEV)
    for k in sorted(v for v in ks if v >= 1):
        proc, idx, got = _enumerate(xd, None, 1.0, 1.0, top_p, k)
        assert np.array_equal(got, idx), (k, len(got), len(idx), np.nonzero(got != idx)[0][:5])
        assert _call(xd[None], top_p=top_p, top_k=k, greedy=True).tolist() == [int(proc.argmax())], k


# ------------------------------------------------------------------------------------------------ the top-p band
@pytest.mark.parametrize("V", [32000, 152064, 262144])
@pytest.mark.parametrize("T", [1.0, 0.2])
def test_topp_band_measured(V, T):
    """Rows whose processed values ascend with the index, are distinct and lie within 25 of the maximum: every kept token
    weighs more than 0 in fixed point, so u = 0 returns the kernel's cut.  Every token it decides differently from the
    restatement must lie within TOPP_BOUND of the threshold."""
    g = torch.Generator().manual_seed(V + int(T * 10))
    step = 24.9 / V
    v = torch.linspace(-24.9, 0.0, V, dtype=torch.float64) + (torch.rand(V, generator=g, dtype=torch.float64) - 0.5) * \
        0.6 * step
    x = (v * T).float()[None]
    proc = O.restate(x, temperature=T)[0]
    assert bool((proc[1:] > proc[:-1]).all()) and float(proc[-1] - proc[0]) <= 25.0
    _, cum = O.topp_order(proc)
    rng = np.random.default_rng(V)
    near = cum[rng.integers(0, V - 1, 400)] + rng.uniform(-3e-6, 3e-6, 400)
    thrs = np.concatenate([rng.uniform(0.0, 1.0, 400), near])
    tops = sorted({float(np.float32(1.0 - t)) for t in thrs if 0.0 < float(np.float32(1.0 - t)) < 1.0})
    xd, u0 = x.to(DEV), torch.zeros(1, device=DEV)
    got = np.array([int(_call(xd, None, T, 1.0, p, 0, u=u0)) for p in tops])
    worst, disagree = 0.0, 0
    for p, c in zip(tops, got):
        thr, want = O.thr_of(p), O.topp_cut(cum, p)
        if c != want:
            lo, hi = min(c, want), max(c, want)
            d = float(np.abs(cum[lo:hi] - thr).max())
            assert d <= O.TOPP_BOUND, (p, int(c), want, d)
            disagree += hi - lo
            worst = max(worst, d)
    print(f"\ntop-p band V={V} T={T}: {len(tops)} top_p, {disagree} tokens decided differently, "
          f"largest |cum64 - thr| among them {worst:.3g}")


# ------------------------------------------------------------------------------------------------ the draw's CDF
def _bisect_edges(x_row, prev_row, T, pen, top_p, k):
    """The kernel's lower edge of each kept token of probability >= MIN_P (but the first), bisected in fp32 u with one
    stride-0 call per step; asserts the token is monotone in u over every u asked.  Returns (float64 edges, measured
    edges)."""
    proc = O.restate(x_row[None].cpu(), None if prev_row is None else prev_row[None].cpu(), T, pen, top_p, k)[0]
    idx, e64 = O.cdf_edges(proc)
    n = len(idx)
    f32 = lambda a: np.asarray(a, dtype=np.float32)  # noqa: E731
    lo = f32(np.maximum(e64 - O.MIN_P / 2, 0.0)).view(np.int32).astype(np.int64)
    hi = f32(e64 + O.MIN_P / 2).view(np.int32).astype(np.int64)
    xs = x_row[None].expand(n, -1)
    ps = None if prev_row is None else prev_row[None].expand(n, -1)
    asked_u, asked_t = [], []

    def run(bits):
        u = bits.astype(np.int32).view(np.float32)
        t = _call(xs, ps, T, pen, top_p, k, u=torch.from_numpy(u.copy()).to(DEV)).numpy()
        asked_u.append(u)
        asked_t.append(t)
        return t
    assert (run(lo) < idx).all() and (run(hi) == idx).all()
    while (hi - lo > 1).any():
        mid = (lo + hi) // 2
        up = run(mid) >= idx
        hi, lo = np.where(up, mid, hi), np.where(up, lo, mid)
    u, t = np.concatenate(asked_u), np.concatenate(asked_t)
    o = np.argsort(u, kind="stable")
    assert (np.diff(t[o]) >= 0).all(), "the token is not monotone in u"
    return e64, hi.astype(np.int32).view(np.float32).astype(np.float64)


def test_draw_edges_measured():
    """The kernel's CDF edges on permuted rows (each level once) lie within DRAW_BOUND of the float64 edges: tinychat's
    defaults over 40 rows, and full-vocabulary top-p over thousands of kept tokens."""
    worst, count = 0.0, 0
    g = torch.Generator().manual_seed(17)
    for V, case, rows in ((152064, "defaults", 40), (32000, "full_vocab_top_p", 1), (152064, "full_vocab_top_p", 1)):
        for _ in range(rows):
            levels = (torch.arange(V, dtype=torch.float32) - V / 2) * (12.0 / V)
            x = levels[torch.randperm(V, generator=g)]
            if case == "defaults":
                T, pen, want_p, k = PROCS["defaults"]
                prev = torch.randint(0, V, (600,), generator=g)
            else:
                T, pen, want_p, k, prev = 1.0, 1.0, 0.95, 0, None
            top_p = _safe(x[None], None if prev is None else prev[None], T, pen, want_p)
            e64, got = _bisect_edges(x.to(DEV), None if prev is None else prev.to(DEV), T, pen, top_p, k)
            dev = np.abs(got - e64)
            assert dev.max() <= O.DRAW_BOUND, (V, case, float(dev.max()))
            worst, count = max(worst, float(dev.max())), count + len(e64)
    assert count > 5000
    print(f"\ndraw edges: {count} edges, largest |measured - float64| {worst:.3g} (DRAW_BOUND {O.DRAW_BOUND:.3g})")
