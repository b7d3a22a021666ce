"""CPU checks of b200awq_sample_next_token (tinychat's temperature, repetition penalty, top-p, top-k and the choice of
the next token, one launch): argument validation that returns before any device is touched, the restatement of the
chain (tests/sampling_oracle.py) pinned to transformers' own processors, and the oracle's own rules (stable ties,
penalty once per distinct id, inverse CDF)."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import sampling_oracle as O

SHAPE, ALIGN, DEVICE = -1, -3, -8
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every ABI case below returns first)
MAX_VOCAB = 262144


# ------------------------------------------------------------------------------------------------ ABI validation
def _call(logits=A, stride=128256, B=1, V=128256, prev=A, prev_stride=600, n_prev=600, T=0.2, pen=1.1, top_p=0.95,
          top_k=50, greedy=0, u=A, tokens=A):
    return P.lib().b200awq_sample_next_token(logits, stride, B, V, prev, prev_stride, n_prev, T, pen, top_p, top_k, greedy,
                                             u, tokens, None)


@pytest.mark.parametrize("kw,code", [
    (dict(B=-1), SHAPE), (dict(V=0), SHAPE), (dict(V=-5), SHAPE), (dict(V=MAX_VOCAB + 1), SHAPE), (dict(n_prev=-1), SHAPE),
    (dict(T=0.0), SHAPE), (dict(T=-0.5), SHAPE), (dict(T=float("inf")), SHAPE), (dict(T=float("nan")), SHAPE),
    (dict(pen=0.99), SHAPE), (dict(pen=0.0), SHAPE), (dict(pen=float("inf")), SHAPE), (dict(pen=float("nan")), SHAPE),
    (dict(top_p=0.0), SHAPE), (dict(top_p=-0.1), SHAPE), (dict(top_p=1.0001), SHAPE), (dict(top_p=float("nan")), SHAPE),
    (dict(top_k=-1), SHAPE), (dict(V=0, logits=None, tokens=None), SHAPE),
    (dict(logits=None), ALIGN), (dict(logits=A + 2), ALIGN), (dict(tokens=None), ALIGN), (dict(tokens=A + 4), ALIGN),
    (dict(u=None), ALIGN), (dict(u=A + 1), ALIGN), (dict(prev=None), ALIGN), (dict(prev=A + 4), ALIGN),
    (dict(B=0, tokens=None), ALIGN),
])
def test_rejected_before_any_device_work(kw, code):
    assert _call(**kw) == code, kw


@pytest.mark.parametrize("kw", [
    dict(B=0), dict(B=0, greedy=1, u=None), dict(B=0, n_prev=0, prev=None), dict(B=0, pen=1.0, prev=None),
])
def test_empty_batch_is_a_no_op(kw):
    """batch == 0 returns 0 after validation, before any device work (none is available here)."""
    assert _call(**kw) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
def test_envelope_edges_pass_validation():
    """Arguments at the envelope's edges stop at the device check, never at SHAPE / ALIGN: the vocabulary bound, one
    entry, the off values (top_p 1, top_k 0, penalty 1, temperature 1), pointers the call does not read left NULL."""
    for kw in (dict(V=MAX_VOCAB), dict(V=1), dict(V=152064), dict(top_p=1.0), dict(top_k=0), dict(top_k=10 ** 9),
               dict(pen=1.0, prev=None), dict(n_prev=0, prev=None), dict(greedy=1, u=None), dict(T=1e-30),
               dict(top_p=1e-30), dict(stride=0), dict(prev_stride=0), dict(B=2 ** 31 - 1)):
        assert _call(**kw) == DEVICE, kw


# ------------------------------------------------------------------------------------------------ the restatement
def _tie_free(B, V, seed, scale=2.0):
    """Rows that are random permutations of V evenly spaced, distinct fp32 levels in [-3 scale, 3 scale)."""
    g = torch.Generator().manual_seed(seed)
    levels = (torch.arange(V, dtype=torch.float32) - V / 2) * (6 * scale / V)
    x = torch.stack([levels[torch.randperm(V, generator=g)] for _ in range(B)])
    assert all(len(torch.unique(x[b])) == V for b in range(B))
    return x


def _hf():
    lp = pytest.importorskip("transformers.generation.logits_process")
    return lp


@pytest.mark.parametrize("V", [1000, 32000])
@pytest.mark.parametrize("T,pen,want_p,k", [(0.2, 1.1, 0.95, 50), (1.0, 1.0, 0.9, 0), (0.7, 1.3, 0.5, 7), (1.3, 1.0, 1.0, 3),
                                            (0.9, 1.2, 1.0, 0), (1.0, 1.0, 0.3, 1)])
def test_restatement_matches_transformers(V, T, pen, want_p, k):
    """On tie-free logits the restatement gives exactly what tinychat's LogitsProcessorList gives (CPU, fp32)."""
    lp = _hf()
    x = _tie_free(1, V, seed=V + k)
    g = torch.Generator().manual_seed(7)
    prev = torch.randint(0, V, (1, 600), generator=g)
    top_p = want_p
    if want_p < 1.0:
        top_p = O.safe_top_p(O.restate(x, prev, T, pen)[0], want_p)
    procs = lp.LogitsProcessorList()
    if T >= 1e-5 and T != 1.0:
        procs.append(lp.TemperatureLogitsWarper(T))
    if pen > 1.0:
        procs.append(lp.RepetitionPenaltyLogitsProcessor(pen))
    if 1e-8 <= top_p < 1.0:
        procs.append(lp.TopPLogitsWarper(top_p))
    if k > 0:
        procs.append(lp.TopKLogitsWarper(k))
    want = procs(prev, x.clone())
    got = O.restate(x, prev, T, pen, top_p, k)
    assert torch.equal(torch.isinf(want), torch.isinf(got))
    assert torch.equal(want, got)


def test_penalty_once_per_distinct_id_and_range():
    x = torch.tensor([[2.0, -2.0, 4.0, 1.0, -1.0]])
    prev = torch.tensor([[0, 0, 0, 1, 1, -1, 5, 2 ** 40, 4]])
    got = O.restate(x, prev, penalty=2.0)
    assert torch.equal(got, torch.tensor([[1.0, -4.0, 4.0, 1.0, -2.0]]))


def test_topp_ties_are_removed_in_index_order():
    """Two tied maxima of probability ~1/2 each: at thr 0.6 the lower index is removed, at thr 0.4 both stay."""
    x = torch.full((1, 10), -40.0)
    x[0, 3] = x[0, 7] = 5.0
    got = O.restate(x, top_p=0.4)
    assert torch.isinf(got[0, 3]) and got[0, 7] == 5.0
    assert O.draw(got[0], 0.0, greedy=True) == 7
    got = O.restate(x, top_p=0.6)
    assert got[0, 3] == 5.0 and got[0, 7] == 5.0
    assert O.draw(got[0], 0.0, greedy=True) == 3


def test_topk_keeps_ties_at_the_kth_value():
    x = torch.tensor([[1.0, 3.0, 2.0, 2.0, 0.0, 2.0]])
    got = O.restate(x, top_k=2)
    assert torch.equal(torch.isfinite(got), torch.tensor([[False, True, True, True, False, True]]))


def test_draw_is_the_inverse_cdf():
    x = torch.tensor([0.0, -float("inf"), np.log(3.0), 0.0])  # masses 1, 0, 3, 1: CDF 1/5, 1/5, 4/5, 1
    assert [O.draw(x, u) for u in (0.0, 0.19, 0.2, 0.5, 0.79, 0.8, 0.999)] == [0, 0, 2, 2, 2, 3, 3]
    idx, mid = O.midpoints(x)
    assert list(idx) == [0, 2, 3] and [O.draw(x, float(u)) for u in mid] == [0, 2, 3]


def test_safe_top_p_keeps_its_margin():
    x = torch.randn(32000, generator=torch.Generator().manual_seed(3)) * 4
    for want in (0.95, 0.5, 0.99):
        top_p = O.safe_top_p(x, want)
        assert abs(top_p - want) < 0.03 and O.topp_margin(x, top_p) > O.TOPP_BOUND
