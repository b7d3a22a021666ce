"""The elementwise bound of tests/attention_bounds.py against numpy emulations of the kernels' arithmetic, on reduced
versions of every landscape the GPU file runs:

  * right: every element of the emulations stays within B, for one split, one split per tile (per 32 positions for
    the decode kernel) and random partitions, and so does the float64 oracle rounded to T;
  * not vacuous: on each dtype and kernel family some element reaches 1/4 of B.  On the short wgmma cases the output
    rounding alone gets there (B is then within about 2 ulp of T); the long case shows the accumulator term reached
    by the emulation's own error, beyond the rounded oracle's;
  * sharp: each one-line defect of the emulations breaks the bound somewhere."""
import numpy as np
import pytest
import torch

import attention_bounds as AB
import prefill_attention_oracle as PO

DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
R, N, D = 32, 640, 64      # wgmma: 32 rows (lo and hi halves of two warps), 5 key tiles
G, NP, DD = 8, 700, 128    # decode: 8 heads, 700 positions, D = 128 (1 / sqrt(D) inexact in fp32)


def _wgmma_case(kind, causal, seed):
    g = torch.Generator().manual_seed(seed)
    scale = AB.wgmma_scale(D)
    u = AB.level_units(D, scale)
    i = torch.arange(R).view(-1, 1)
    j = torch.arange(N).view(1, -1)
    vis = j <= i + N - R if causal else torch.ones(R, N, dtype=torch.bool)
    hi = [N - R + r if causal else N - 1 for r in range(R)]
    targets = [AB.needle_targets(0, h, N, AB.TILE, r) for r, h in enumerate(hi)]
    k = AB.make_k(kind, N, D, u, g)
    q = AB.make_q(kind, targets, N, D, g)
    v = AB.make_v(N, D, g)
    AB.check_exact(q, k, v)
    s = torch.where(vis, q @ k.T, torch.tensor(float("-inf"), dtype=torch.float64))
    return q, k, v, s, vis, scale


def _decode_case(kind, seed, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    scale = DD ** -0.5
    u = AB.level_units(DD, scale)
    targets = [AB.needle_targets(0, NP - 1, NP, 32, 3 * h + 1) for h in range(G)]
    k = AB.make_k(kind, NP, DD, u, g, shift)
    q = AB.make_q(kind, targets, NP, DD, g)
    v = AB.make_v(NP, DD, g)
    AB.check_exact(q, k, v)
    return q, k, v, q @ k.T, torch.ones(G, NP, dtype=torch.bool), scale


def _partitions(n, step, seed):
    """One split, one per `step` keys, and three random partitions on `step` edges."""
    cuts = list(range(0, n, step))[1:]
    out = [[0, n], [0] + cuts + [n]]
    rng = np.random.default_rng(seed)
    for k in (1, 2, 3):
        out.append([0] + sorted(rng.choice(cuts, size=min(k, len(cuts)), replace=False).tolist()) + [n])
    return out


WGMMA_CASES = [(kind, causal) for kind in AB.KINDS for causal in (False, True)]
DECODE_CASES = [(kind, shift) for shift in (0.0, AB.TOP) for kind in AB.KINDS]  # TOP: the top above exp's range


def _worst(got, O, B):
    return float(AB.ratio(torch.from_numpy(np.asarray(got, np.float64)), O, B).max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_wgmma_emulation_within_bound(dtype):
    top = 0.0
    for n, (kind, causal) in enumerate(WGMMA_CASES):
        q, k, v, s, vis, scale = _wgmma_case(kind, causal, 10 + n)
        O, B = AB.bound(s, vis, v, scale, dtype, "wgmma")
        want = PO.prefill_attention(q.view(1, R, 1, D), k.view(1, N, 1, D), v.view(1, N, 1, D), causal, scale)[0, :, 0]
        assert np.allclose(O.numpy(), want, rtol=1e-12, atol=1e-12), kind
        assert _worst(O.to(dtype).to(torch.float64), O, B) <= 1.0, f"{kind}: the oracle rounded to T"
        for edges in _partitions(N, AB.TILE, n):
            r = _worst(AB.emulate_wgmma(s.numpy(), v.numpy(), scale, dtype, edges), O, B)
            assert r <= 1.0, f"{kind} causal={causal} splits {edges}: err / B = {r:.3f}"
            top = max(top, r)
    print(f"wgmma emulation {dtype}: largest err / B {top:.3f}")
    assert top >= 0.25, f"the bound is loose everywhere: largest err / B {top:.3f}"


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_emulation_within_bound(dtype):
    top = 0.0
    for n, (kind, shift) in enumerate(DECODE_CASES):
        q, k, v, s, vis, scale = _decode_case(kind, 40 + n, shift)
        O, B = AB.bound(s, vis, v, scale, dtype, "decode")
        want = PO.prefill_attention(q.view(1, 1, G, DD), k.view(1, NP, 1, DD), v.view(1, NP, 1, DD), False, scale)[0, 0]
        assert np.allclose(O.numpy(), want, rtol=1e-12, atol=1e-12), kind
        assert _worst(O.to(dtype).to(torch.float64), O, B) <= 1.0, f"{kind}: the oracle rounded to T"
        for edges in _partitions(NP, 32, n):
            r = _worst(AB.emulate_decode(s.numpy(), v.numpy(), DD, dtype, edges), O, B)
            assert r <= 1.0, f"{kind} shift={shift} chunks {edges}: err / B = {r:.3f}"
            top = max(top, r)
    print(f"decode emulation {dtype}: largest err / B {top:.3f}")
    assert top >= 0.25, f"the bound is loose everywhere: largest err / B {top:.3f}"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("defect", AB.WGMMA_DEFECTS)
def test_wgmma_defect_breaks_bound(defect, dtype):
    worst = 0.0
    for n, (kind, causal) in enumerate(WGMMA_CASES):
        _, _, v, s, vis, scale = _wgmma_case(kind, causal, 10 + n)
        O, B = AB.bound(s, vis, v, scale, dtype, "wgmma")
        for edges in _partitions(N, AB.TILE, n)[1:]:
            worst = max(worst, _worst(AB.emulate_wgmma(s.numpy(), v.numpy(), scale, dtype, edges, defect), O, B))
    assert worst > 1.0, f"{defect}: no element outside the bound (largest err / B {worst:.3f})"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("defect", AB.DECODE_DEFECTS)
def test_decode_defect_breaks_bound(defect, dtype):
    worst = 0.0
    for n, (kind, shift) in enumerate(DECODE_CASES):
        _, _, v, s, vis, scale = _decode_case(kind, 40 + n, shift)
        O, B = AB.bound(s, vis, v, scale, dtype, "decode")
        for edges in _partitions(NP, 32, n)[1:]:
            worst = max(worst, _worst(AB.emulate_decode(s.numpy(), v.numpy(), DD, dtype, edges, defect), O, B))
    assert worst > 1.0, f"{defect}: no element outside the bound (largest err / B {worst:.3f})"


def test_landscapes_stretch_the_softmax():
    """The staircase's first rescale factor is below 2^-126 (flushed), descending puts most fp16 p below 2^-14,
    the tiles landscape has tile maxima more than 126 log2 units below the top, ties are exact ties."""
    scale = AB.wgmma_scale(D)
    c = AB.scale_log2(scale)
    g = torch.Generator().manual_seed(1)
    u = AB.level_units(D, scale)
    for kind in AB.KINDS:
        k = AB.make_k(kind, 2048, D, u, g)
        q = AB.make_q(kind, [AB.needle_targets(0, 2047, 2048, AB.TILE, r) for r in range(4)], 2048, D, g)
        AB.check_exact(q, k)
        s = (q @ k.T) * c  # log2 units
        tmax = s.view(4, -1, AB.TILE).amax(-1)
        M = s.amax(-1, keepdim=True)
        if kind == "staircase":
            assert float((tmax[:, 1] - tmax[:, 0]).min()) > 126
            assert bool((tmax[:, 1:] > tmax[:, :-1]).all())
        elif kind == "descending":
            assert float(((s - M) < -14).double().mean()) > 0.9 and float(((s - M) < -25).double().mean()) > 0.5
        elif kind == "needles":
            top2 = s.topk(2, -1).values
            assert float((top2[:, 0] - top2[:, 1]).min()) > 12
        elif kind == "tiles":
            assert float((M - tmax).max()) > 126 and bool((tmax[:, 0] < M[:, 0]).all())
        else:
            assert bool((tmax == M).all())
        assert float(M.abs().max()) < 24, kind


@pytest.mark.parametrize("dtype", DTYPES)
def test_wgmma_emulation_long_key_range(dtype):
    """64 key tiles (512 k16 steps): the accumulator term 2^-21 n16 A is 2^-12 A, half a u of fp16.  The emulation
    loses the model's whole budget at every step, toward 0, and stays within B.  On the descending landscape the
    weight sits at key 0, so |acc| is large from the first step: there, on the constant V channel, the emulation's
    error before the output's rounding reaches at least half of the accumulator term (in bf16 the rounding of P to
    T adds more)."""
    n, rows, C = 64 * AB.TILE, 16, 8
    scale = AB.wgmma_scale(D)
    u = AB.level_units(D, scale)
    reach = 0.0
    for m, kind in enumerate(AB.KINDS):
        g = torch.Generator().manual_seed(70 + m)
        targets = [AB.needle_targets(0, n - 1, n, AB.TILE, 37 * r) for r in range(rows)]
        k = AB.make_k(kind, n, D, u, g)
        q = AB.make_q(kind, targets, n, D, g)
        v = AB.make_v(n, D, g)[:, -C:]
        s = q @ k.T
        vis = torch.ones(rows, n, dtype=torch.bool)
        O, B, A, acc = AB.bound(s, vis, v, scale, dtype, "wgmma", parts=True)
        assert float((acc / A).max()) == 2.0 ** -12
        for edges in ([0, n], [0, 17 * AB.TILE, 40 * AB.TILE, n]):
            pre = AB.emulate_wgmma(s.numpy(), v.numpy(), scale, dtype, edges, rounded=False)
            r = float(AB.ratio(torch.from_numpy(pre).to(dtype).to(torch.float64), O, B).max())
            assert r <= 1.0, f"{kind} splits {edges}: err / B = {r:.3f}"
            if kind == "descending":
                reach = max(reach, float(((torch.from_numpy(pre) - O).abs() / acc)[:, -1].max()))
    print(f"long key range {dtype}: error before rounding / accumulator term on the constant channel {reach:.3f}")
    assert reach >= 0.5, reach
