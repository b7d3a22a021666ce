"""CPU pins of the helpers tests/test_sampling_envelope_gpu.py builds on (tests/sampling_oracle.py): the launcher's
partition of a row over the cluster, the top-p cut against the restatement, the draw's CDF edges, and the inputs of
DRAW_BOUND's derivation."""
import math

import numpy as np
import pytest
import torch

import sampling_oracle as O

SWEEP = [1, 2, 31, 33, 255, 257, 1000, 4097, 32064, 50257, 65024, 92544, 151936, 256000, 262143, 262144]


# ------------------------------------------------------------------------------------------------ partition geometry
@pytest.mark.parametrize("V,slice_,last", [
    (1, 32, (0, 1)), (33, 32, (32, 33)), (257, 64, (256, 257)), (32000, 4000, (28000, 32000)),
    (32064, 4032, (28224, 32064)), (151936, 19008, (133056, 151936)), (152064, 19008, (133056, 152064)),
    (262143, 32768, (229376, 262143)), (262144, 32768, (229376, 262144)),
])
def test_slices_by_hand(V, slice_, last):
    """slice = ceil(ceil(V / 8) / 32) 32; `last` is the last non-empty CTA's range (Phi-3's 32064 leaves 3840 keys to
    CTA 7, Qwen2-0.5B's 151936 leaves 18880)."""
    s = O.slices(V)
    assert s[0] == (0, min(V, slice_))
    assert [r for r in s if r[1] > r[0]][-1] == last


@pytest.mark.parametrize("V", SWEEP)
def test_slices_tile_the_row(V):
    s = O.slices(V)
    assert len(s) == O.SAMPLE_CTAS and s[0][0] == 0 and s[-1][1] == V
    assert all(a[1] == b[0] for a, b in zip(s, s[1:]))
    size = s[0][1] - s[0][0] if V > 32 else 32
    assert size % 32 == 0 and size * O.SAMPLE_CTAS >= V and (size - 32) * O.SAMPLE_CTAS < V
    assert all(hi - lo <= size for lo, hi in s)
    assert size * 4 + size // 8 <= 132 * 1024  # a CTA's keys and penalty flags: 132 KB at the vocabulary bound


def test_empty_ctas():
    assert [hi - lo for lo, hi in O.slices(33)] == [32, 1, 0, 0, 0, 0, 0, 0]
    assert [hi - lo for lo, hi in O.slices(257)] == [64, 64, 64, 64, 1, 0, 0, 0]
    assert [hi - lo for lo, hi in O.slices(1)] == [1, 0, 0, 0, 0, 0, 0, 0]


def test_draw_chunk():
    assert [O.draw_chunk(n) for n in (0, 1, 512, 513, 4000, 18880, 19008, 32768)] == [0, 1, 1, 2, 8, 37, 38, 64]


# ------------------------------------------------------------------------------------------------ the top-p cut
@pytest.mark.parametrize("seed", range(6))
def test_topp_cut_is_the_restatements_first_kept_token(seed):
    """On small ascending rows the cut is the index of restate's first kept token; on permuted rows it is that token's
    position in the stable ascending order."""
    g = torch.Generator().manual_seed(seed)
    V = 40
    asc = torch.sort(torch.randn(V, generator=g) * (1 + seed)).values
    asc[5:9] = asc[5]  # a tie group
    perm = torch.randperm(V, generator=g)
    for top_p in list(torch.rand(50, generator=g).tolist()) + [1e-9, 0.999999]:
        top_p = float(np.float32(top_p))
        if not 0.0 < top_p < 1.0:
            continue
        order, cum = O.topp_order(asc)
        assert np.array_equal(order, np.arange(V))
        cut = O.topp_cut(cum, top_p)
        kept = torch.isfinite(O.restate(asc[None], top_p=top_p)[0])
        assert int(torch.nonzero(kept)[0]) == cut and int(kept.sum()) == V - cut
        x = asc[perm]
        order, cum = O.topp_order(x)
        kept = torch.isfinite(O.restate(x[None], top_p=top_p)[0])
        assert set(order[cut:].tolist()) == set(torch.nonzero(kept)[:, 0].tolist())


def test_topp_cut_keeps_the_last_token():
    order, cum = O.topp_order(torch.tensor([0.0, 1.0, 2.0]))
    assert O.topp_cut(cum, float(np.float32(1e-9))) == 2


def test_safe_top_p_over_several_rows():
    x = torch.randn(5, 4000, generator=torch.Generator().manual_seed(2)) * torch.tensor([[0.5], [1], [2], [4], [8]])
    top_p = O.safe_top_p(x, 0.9)
    assert all(O.topp_margin(r, top_p) > O.TOPP_BOUND for r in x)


# ------------------------------------------------------------------------------------------------ the draw's CDF edges
def test_cdf_edges():
    x = torch.tensor([-float("inf"), 0.0, -float("inf"), np.log(3.0), 0.0])  # masses 0, 1, 0, 3, 1
    idx, e = O.cdf_edges(x)
    assert list(idx) == [3, 4] and np.allclose(e, [0.2, 0.8], rtol=0, atol=1e-15)
    assert list(O.draw(x, e + 1e-12)) == [3, 4] and list(O.draw(x, e - 1e-12)) == [1, 3]
    assert list(O.draw(x, np.array([0.0, 0.19, 0.2, 0.79, 0.8]))) == [1, 1, 3, 3, 4]


def test_draw_bound_derivation_inputs():
    """DRAW_BOUND = expf's 2 ulp (2^-22 relative) + 2^-24 ln n for the rounded x - max + n 2^-45 for the fixed point,
    at n = 2^18, + one fp32 spacing below 1 for the measured u."""
    assert O.MAX_VOCAB == 262144 and O.FIXED_POINT_BITS == 44 and O.EXPF_ULP == 2
    parts = [2.0 ** -22, 2.0 ** -24 * 18 * math.log(2), 2.0 ** -27, 2.0 ** -24]
    assert O.DRAW_BOUND == pytest.approx(sum(parts), rel=1e-12)
    assert 1.04e-6 < O.DRAW_BOUND < 1.06e-6 < O.TOPP_BOUND
    assert float(np.nextafter(np.float32(1), np.float32(0))) == 1 - 2.0 ** -24


@pytest.mark.parametrize("kind", ["flat", "spread", "two_levels", "one_hot"])
def test_mean_distance_from_the_maximum_is_at_most_ln_n(kind):
    """The lemma of the derivation: under p_i = exp(-d_i) / P with min d = 0, the mean of d is at most ln n."""
    g = torch.Generator().manual_seed(1)
    n = 262144
    d = {"flat": torch.zeros(n), "spread": torch.rand(n, generator=g) * 30,
         "two_levels": torch.cat([torch.zeros(1), torch.full((n - 1,), 8.0)]),
         "one_hot": torch.cat([torch.zeros(1), torch.full((n - 1,), 80.0)])}[kind].double()
    p = torch.exp(-d)
    assert float((p * d).sum() / p.sum()) <= math.log(n)


@pytest.mark.parametrize("spread", [2.0, 12.0, 30.0])
def test_fixed_point_cdf_emulation_within_the_bound(spread):
    """numpy's fp32 exp of fp32 (x - max), rounded to 2^-44 and summed in integers, as the kernel does: every CDF
    edge lies within DRAW_BOUND - 2^-24 of float64 (numpy's expf stands in for CUDA's, both within 2 ulp)."""
    V = 152064
    g = torch.Generator().manual_seed(int(spread))
    x = ((torch.arange(V, dtype=torch.float32) - V / 2) * (spread / V))[torch.randperm(V, generator=g)].numpy()
    d32 = (x - x.max()).astype(np.float32)
    w = np.rint(np.exp(d32).astype(np.float32).astype(np.float64) * 2.0 ** 44).astype(np.int64)
    W = np.concatenate([[0], np.cumsum(w)])
    p = np.exp(x.astype(np.float64) - float(x.max()))
    P64 = np.concatenate([[0.0], np.cumsum(p)])
    dev = np.abs(W[:-1] / float(W[-1]) - P64[:-1] / P64[-1]).max()
    assert dev <= O.DRAW_BOUND - 2.0 ** -24
