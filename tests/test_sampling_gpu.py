"""b200awq_sample_next_token on the GPU against the restatement of tinychat's chain and the float64 inverse-CDF oracle
(tests/sampling_oracle.py).

Midpoint enumeration: a batch of rows that all read the same logits (a stride-0 view), each row's uniform at the
midpoint of one kept token's float64 CDF interval, must return every kept token exactly once, in index order.  That
checks the kept set and the draw order at once.  Every top_p here comes from `safe_top_p`, so no token's cumulative
probability lies within TOPP_BOUND of the threshold and none is excluded from the comparison; tokens of probability
below MIN_P (too narrow for an fp32 midpoint) are not addressed."""
import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import sampling_oracle as O
from llm_awq_b200 import sampling as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VOCABS = [32000, 128256, 152064]
INF = float("inf")


def _e():
    return P.engine()


def _call(logits, prev=None, T=1.0, pen=1.0, top_p=1.0, top_k=0, greedy=False, u=None):
    return _e().sample_next_token(logits, prev, T, pen, top_p, top_k, greedy, u)


def _rows(B, V, seed, scale=4.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, V, generator=g) * scale).to(DEV)


def _prev(B, V, n, seed):
    """ids with duplicates, 0, V - 1 and out-of-range ids."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randint(0, V, (B, n), generator=g)
    if n >= 8:
        p[:, :8] = torch.tensor([0, V - 1, -1, V, 2 ** 40, -(2 ** 40), 5, 5])
        p[:, 8:16] = p[:, 16:24]
    return p.to(DEV)


# ------------------------------------------------------------------------------------------------ greedy
@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T,pen,want_p,k", [(1.0, 1.0, 1.0, 0), (1.0, 1.1, 1.0, 0), (0.7, 1.3, 0.95, 50), (1.0, 1.5, 0.5, 7)])
def test_greedy_is_exact(V, B, T, pen, want_p, k):
    x = _rows(B, V, seed=V + B)
    prev = _prev(B, V, 600, seed=B)
    # the penalised ids hold the row maxima, so that the penalty decides the argmax
    idx = prev[:, 16:40].clamp(0, V - 1)
    x.scatter_(1, idx, (x.max(dim=1, keepdim=True).values + 0.05).expand_as(idx).contiguous())
    top_p = want_p
    if want_p < 1.0:
        top_p = min(O.safe_top_p(O.restate(x[b:b + 1], prev[b:b + 1], T, pen)[0], want_p) for b in range(B))
        assert all(O.topp_margin(O.restate(x[b:b + 1], prev[b:b + 1], T, pen)[0], top_p) > O.TOPP_BOUND for b in range(B))
    want = O.restate(x, prev, T, pen, top_p, k).argmax(dim=1)
    got = _call(x, prev, T, pen, top_p, k, greedy=True).cpu()
    assert torch.equal(got, want)


@pytest.mark.parametrize("V", VOCABS)
def test_greedy_ties_and_topp_removed_maximum(V):
    x = torch.full((3, V), -30.0, device=DEV)
    x[:, 5] = x[:, V - 1] = 4.0  # two tied maxima, ~1/2 of the mass each
    x[1, 0] = 4.0                # three in row 1
    assert _call(x, greedy=True).tolist() == [5, 0, 5]
    assert _call(x, top_k=1, greedy=True).tolist() == [5, 0, 5]  # ties at the top_k-th value are kept
    # thr = 0.6: in ascending (value, index) order a maximum whose inclusive cumulative mass is <= 0.6 is removed
    # (rows 0 and 2: index 5 at 1/2; row 1: index 0 at 1/3, index 5 at 2/3 stays)
    assert _call(x, top_p=0.4, greedy=True).tolist() == [V - 1, 5, V - 1]
    assert _call(x, top_p=0.6, greedy=True).tolist() == [5, 5, 5]  # row 1: thr 0.4 removes index 0 only
    assert _call(x, top_p=1e-7, greedy=True).tolist() == [V - 1] * 3  # thr rounds to 1: only the last is kept


# ------------------------------------------------------------------------------------------------ midpoint enumeration
def _enumerate(x_row, prev_row, T, pen, top_p, k, vocab_check=True):
    """Every kept token's midpoint through the kernel, on a stride-0 batch of the same row."""
    proc = O.restate(x_row[None], None if prev_row is None else prev_row[None], T, pen, top_p, k)[0]
    idx, mid = O.midpoints(proc)
    got = []
    for s in range(0, len(mid), 8192):
        u = torch.from_numpy(mid[s:s + 8192]).to(DEV)
        n = len(u)
        prev = None if prev_row is None else prev_row[None].expand(n, -1)
        got.append(_call(x_row[None].expand(n, -1), prev, T, pen, top_p, k, u=u).cpu())
    got = torch.cat(got).numpy()
    return proc, idx, got


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("case", ["defaults", "top_k_1", "topk_ties", "full_vocab_top_p"])
def test_midpoints_return_every_kept_token_once(V, case):
    g = torch.Generator().manual_seed(V)
    prev = _prev(1, V, 600, seed=V)[0]
    if case == "defaults":  # tinychat: temperature 0.2, penalty 1.1, top-p 0.95, top-k 50
        x = (torch.randn(V, generator=g) * 0.5).to(DEV)
        T, pen, want_p, k = 0.2, 1.1, 0.95, 50
    elif case == "top_k_1":
        x = (torch.randn(V, generator=g) * 2).to(DEV)
        T, pen, want_p, k = 0.7, 1.1, 0.95, 1
    elif case == "topk_ties":  # values on a coarse grid: the 50th largest value is shared by several tokens
        x = torch.round(torch.randn(V, generator=g) * 4).to(DEV)
        T, pen, want_p, k = 1.0, 1.0, 1.0, 50
    else:  # top-p alone over the whole vocabulary: thousands of kept tokens
        x = (torch.randn(V, generator=g) * 3).to(DEV)
        T, pen, want_p, k, prev = 1.0, 1.0, 0.95, 0, None
    top_p = want_p
    if want_p < 1.0:
        top_p = O.safe_top_p(O.restate(x[None], None if prev is None else prev[None], T, pen)[0], want_p)
    proc, idx, got = _enumerate(x, prev, T, pen, top_p, k)
    kept = np.nonzero(np.isfinite(proc.numpy()))[0]
    assert np.array_equal(got, idx), (len(got), len(idx), np.nonzero(got != idx)[0][:5])
    if case == "topk_ties":
        assert len(kept) > k
    if case == "full_vocab_top_p":
        assert len(kept) > 1000
        assert len(np.unique(got)) == len(idx)
    if case == "top_k_1":
        assert len(kept) == 1


@pytest.mark.parametrize("V", VOCABS)
def test_u_edges(V):
    """u = 0 returns the first kept index, u just below 1 the last."""
    x = _rows(3, V, seed=11, scale=1.0)
    x[:, 0] = x[:, V - 1] = 6.0  # first and last indices kept, with non-negligible mass
    x[1, 0] = -INF
    u0 = torch.zeros(3, device=DEV)
    u1 = torch.full((3,), float(np.nextafter(np.float32(1), np.float32(0))), device=DEV)
    for args in (dict(), dict(top_k=50), dict(T=0.2, pen=1.1, top_p=0.95, top_k=50)):
        top_p = args.get("top_p", 1.0)
        proc = O.restate(x, None, args.get("T", 1.0), 1.0, top_p, args.get("top_k", 0))
        first = [int(np.nonzero(O.masses(proc[b]) > 0)[0][0]) for b in range(3)]
        assert _call(x, u=u0, **args).tolist() == first
        assert _call(x, u=u1, **args).tolist() == [V - 1] * 3


# ------------------------------------------------------------------------------------------------ penalty, -inf, NaN
def _logit_for(value, T):
    """A logit whose fp32 x / T is exactly `value` (T == 1: the value itself), or None."""
    if T == 1.0:
        return value
    Tt = torch.tensor(T, dtype=torch.float32)
    c = value * Tt
    for _ in range(16):
        q = c / Tt
        if q == value:
            return c
        c = torch.nextafter(c, torch.tensor(INF if q < value else -INF))
    return None


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("T", [1.0, 0.7])
def test_penalty_is_bit_exact(V, T):
    """A penalised token a competes with an unpenalised token b whose processed value is the exact fp32 result of the
    penalty.  The first index wins a tie, so with b before a and with b after a the kernel's value is that result bit for
    bit.  The positive values are ones where x / penalty differs from x * fp32(1 / penalty)."""
    pen = 1.1
    Tt, pt = torch.tensor(T, dtype=torch.float32), torch.tensor(pen, dtype=torch.float32)
    xs = torch.rand(4096, generator=torch.Generator().manual_seed(1)) * 8 + 0.5
    ys = xs / Tt if T != 1.0 else xs
    pos = xs[ys / pt != ys * (1 / pt)][:4]
    checked = 0
    for xa in list(pos) + [-v for v in xs[:4]]:
        y = xa / Tt if T != 1.0 else xa
        want = y * pt if y < 0 else y / pt
        xb = _logit_for(want, T)
        if xb is None:
            continue
        for a, b in ((100, 50), (50, 100)):
            x = torch.full((1, V), -60.0)
            x[0, a], x[0, b] = xa, xb
            prev = torch.tensor([[a, a, V + 3]])
            assert O.restate(x, prev, T, pen).argmax(dim=1).item() == min(a, b)
            got = _call(x.to(DEV), prev.to(DEV), T, pen, greedy=True)
            assert got.item() == min(a, b), (float(xa), a, b)
            checked += 1
    assert checked >= 12


@pytest.mark.parametrize("V", VOCABS)
def test_minus_inf_entries_are_never_drawn(V):
    x = _rows(1, V, seed=5, scale=1.0)
    x[0, ::3] = -INF
    x[0, 1] = -INF
    u = torch.linspace(0, 0.9999, 4096, device=DEV)
    for args in (dict(), dict(top_p=0.95), dict(top_k=1000), dict(T=0.2, pen=1.1, top_p=0.95, top_k=50)):
        prev = torch.arange(0, 600, device=DEV)[None].expand(4096, -1)
        got = _call(x.expand(4096, -1), prev, u=u, **args).cpu()
        assert torch.isfinite(x[0].cpu()[got]).all(), args


@pytest.mark.parametrize("V", VOCABS)
def test_rows_outside_the_contract_get_an_id_in_range(V):
    x = torch.full((4, V), -INF, device=DEV)
    x[1] = float("nan")
    x[2, ::2] = float("nan")
    x[3, 7] = INF
    u = torch.tensor([0.0, 0.5, 0.99, 0.3], device=DEV)
    for args in (dict(), dict(top_p=0.9, top_k=50), dict(T=0.2, pen=1.1, top_p=0.95, top_k=50)):
        for greedy in (True, False):
            got = _call(x, torch.zeros(4, 3, dtype=torch.long, device=DEV), u=u, greedy=greedy, **args).cpu()
            assert ((got >= 0) & (got < V)).all(), (args, greedy, got)
            assert got[3] == 7


# ------------------------------------------------------------------------------------------------ determinism, graphs
def _default_call(x, prev, u):
    return _call(x, prev, 0.2, 1.1, 0.95, 50, u=u)


def test_repeated_calls_are_identical_and_one_launch_each():
    x = _rows(3, 128256, seed=9, scale=0.5)
    prev = _prev(3, 128256, 600, seed=9)
    u = torch.rand(3, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    first = _default_call(x, prev, u)
    for _ in range(20):
        n0 = P.lib().b200awq_launch_count()
        assert torch.equal(_default_call(x, prev, u), first)
        assert P.lib().b200awq_launch_count() - n0 == 1


@pytest.mark.parametrize("pdl", [True, False])
def test_graph_replay_matches_eager(pdl):
    """A graph of a producing kernel (the logits written right before the call) and the call, replayed with new logits
    and uniforms, gives the eager tokens, with PDL on and off."""
    V, B = 152064, 3
    src = _rows(B, V, seed=3, scale=0.5)
    logits = torch.empty_like(src)
    prev = _prev(B, V, 512, seed=3)
    u = torch.rand(B, device=DEV)
    old = _e().set_pdl(pdl)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            logits.copy_(src)
            _default_call(logits, prev, u)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            torch.mul(src, 1.0, out=logits)
            out = _default_call(logits, prev, u)
        for seed in range(4):
            src.copy_(_rows(B, V, seed=100 + seed, scale=0.5))
            u.copy_(torch.rand(B, device=DEV))
            logits.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, _default_call(src.clone(), prev, u.clone()))
    finally:
        _e().set_pdl(old)


# ------------------------------------------------------------------------------------------------ memory
def test_guard_bands_and_read_only_inputs():
    V, B, G = 128256, 3, 4096
    x = _rows(B, V, seed=4, scale=0.5)
    lbuf = torch.randn(G + B * (V + 64) + G, device=DEV)
    logits = lbuf[G:G + B * (V + 64)].view(B, V + 64)[:, :V]  # padded row stride
    logits.copy_(x)
    pbuf = torch.randint(-5, V + 5, (G + B * 700 + G,), device=DEV)
    prev = pbuf[G:G + B * 700].view(B, 700)[:, :600]
    ubuf = torch.rand(G + B + G, device=DEV)
    u = ubuf[G:G + B]
    tbuf = torch.full((G + B + G,), 0x5A5A5A5A5A5A5A5A, dtype=torch.long, device=DEV)
    before = [t.clone() for t in (lbuf, pbuf, ubuf, tbuf)]
    rc = P.lib().b200awq_sample_next_token(logits.data_ptr(), logits.stride(0), B, V, prev.data_ptr(), prev.stride(0), 600,
                                           0.2, 1.1, 0.95, 50, 0, u.data_ptr(), tbuf[G:].data_ptr(),
                                           torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    for a, b in zip((lbuf, pbuf, ubuf), before[:3]):
        assert torch.equal(a, b)
    assert torch.equal(tbuf[:G], before[3][:G]) and torch.equal(tbuf[G + B:], before[3][G + B:])
    assert torch.equal(tbuf[G:G + B], _default_call(x, prev.contiguous(), u))


# ------------------------------------------------------------------------------------------------ the Python mirror
def _stream_gen_block(logits, output_ids, temp, repeat_penalty, top_p, top_k, n_vocab, u):
    """tinychat's per-token block (stream_gen.py) restated on CPU, with the multinomial's uniform given."""
    if top_k <= 0:
        top_k = n_vocab
    T = temp if temp >= 1e-5 and temp != 1.0 else 1.0
    pen = repeat_penalty if repeat_penalty > 1.0 else 1.0
    p = top_p if 1e-8 <= top_p < 1.0 else 1.0
    x = O.restate(logits, output_ids if pen > 1.0 else None, T, pen, p, top_k)[0]
    greedy = temp < 1e-5 or top_p < 1e-8
    return O.draw(x, u, greedy=greedy), x


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("params", [
    dict(temp=0.2, repeat_penalty=1.1, top_p=0.95, top_k=50),  # tinychat's defaults
    dict(temp=0.0, repeat_penalty=1.1, top_p=0.95, top_k=50),  # greedy by temperature
    dict(temp=0.7, repeat_penalty=1.0, top_p=0.0, top_k=0),    # greedy by top_p
    dict(temp=1.0, repeat_penalty=1.0, top_p=1.0, top_k=0),    # no processor but top-k = n_vocab
    dict(temp=1.3, repeat_penalty=1.3, top_p=1.0, top_k=5),
])
def test_python_mirror_matches_stream_gen(V, params):
    x = (torch.randn(1, 3, V, generator=torch.Generator().manual_seed(V)) * 2).to(DEV)
    logits = x[:, -1, :]  # a row-strided view, as the generator passes it
    ids = _prev(1, V, 600, seed=2).clamp(0, V - 1)
    want_p = params["top_p"]
    if 1e-8 <= want_p < 1.0:
        T = params["temp"] if params["temp"] >= 1e-5 and params["temp"] != 1.0 else 1.0
        params = dict(params, top_p=O.safe_top_p(O.restate(logits, ids, T, params["repeat_penalty"])[0], want_p))
    for seed in range(8):
        gen = torch.Generator(device=DEV).manual_seed(seed)
        u = float(torch.rand(1, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV))
        want, proc = _stream_gen_block(logits, ids, n_vocab=V, u=u, **params)
        got = S.sample_next_token(logits, ids, n_vocab=V, generator=gen, **params)
        # a uniform closer to a CDF edge than the kernel's fixed-point rounding is not a comparison of the rule
        p = O.masses(proc)
        cdf = np.cumsum(p) / p.sum()
        if params["temp"] >= 1e-5 and params["top_p"] >= 1e-8 and np.min(np.abs(cdf - u)) < 1e-5:
            continue
        assert got.tolist() == [want], (seed, u)
