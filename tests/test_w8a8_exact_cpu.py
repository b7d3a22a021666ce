"""The admissible-output model of oracle/w8a8_oracle.py without a GPU: the exact fp32 steps against libm, the fp16 /
bf16 roundings against torch, the kernels' thread geometry and summation order against hand-worked tables and a
scalar loop, the monotone shortcut against full enumeration, and the bounds against real hardware -- the reference's
own invoke_quant / gelu_and_quant outputs stored in tests/golden/reference_kernels_w8a8.npz lie inside them."""
import ctypes
import ctypes.util
import itertools
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

import w8a8_cases as W
from oracle import w8a8_oracle as O

F16, F32, F64 = np.float16, np.float32, np.float64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kernels_w8a8.npz")
TORCH_T = {"f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _libm_fmaf():
    f = ctypes.CDLL(ctypes.util.find_library("m")).fmaf
    f.argtypes = [ctypes.c_float] * 3
    f.restype = ctypes.c_float
    return f


def _flush(v):
    return 0.0 * np.sign(v) if abs(v) < 2.0 ** -126 else v


def _fma_cases():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(F32)
    b = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(F32)
    c = (rng.standard_normal(3000) * np.exp2(rng.integers(-40, 40, 3000))).astype(F32)
    adv = []
    for k in range(1, 24):            # a * b = 1 + 2^-k exactly; c pushes it onto or just off a float32 midpoint
        x = F32(1 + 2.0 ** -k)
        for cc in (-2.0 ** -24, 2.0 ** -24, -2.0 ** -48, 2.0 ** -48, -1.0, 2.0 ** -25):
            adv.append((x, F32(1), F32(cc)))
    for cc in (2.0 ** -60, -2.0 ** -60, 2.0 ** -100):   # a * b = 1 + 2^-11 + 2^-24, a float32 midpoint, plus a hair
        adv.append((F32(1 + 2.0 ** -12), F32(1 + 2.0 ** -12), F32(cc)))
    for e in range(-30, 30):          # cancellation: a * b - c with c the float32 rounding of a * b
        x, y = F32(1 + 3 * 2.0 ** -23) * F32(2.0 ** e), F32(1 - 5 * 2.0 ** -24)
        adv.append((x, y, -F32(F64(x) * F64(y))))
    for m in (1.0, 1.5, 1.999):       # results below 2^-126 that must flush, and just above
        adv.append((F32(m * 2.0 ** -70), F32(2.0 ** -60), F32(0)))
        adv.append((F32(m * 2.0 ** -63), F32(2.0 ** -63), F32(-2.0 ** -126)))
        adv.append((F32(2.0 ** -63), F32(2.0 ** -63), F32(m * 2.0 ** -126)))
    adv.append((F32(1e-39), F32(1e30), F32(1)))       # subnormal input: flushed before the product
    aa, bb, cc = (np.array(t, F32) for t in zip(*adv))
    return np.concatenate([a, aa]), np.concatenate([b, bb]), np.concatenate([c, cc])


def test_fma_ftz_matches_libm_fmaf():
    fmaf = _libm_fmaf()
    a, b, c = _fma_cases()
    got = O.fma_ftz(a, b, c)
    fa, fb, fc = O.ftz(a), O.ftz(b), O.ftz(c)
    want = np.array([_flush(fmaf(float(x), float(y), float(z))) for x, y, z in zip(fa, fb, fc)], F32)
    np.testing.assert_array_equal(got.view(np.uint32) & 0x7FFFFFFF, want.view(np.uint32) & 0x7FFFFFFF)
    # float64 then a cast (two roundings) is wrong on some of these, so they really test the single rounding
    twice = O.ftz((fa.astype(F64) * fb + fc).astype(F32))
    assert (twice != want).any()


def test_add_mul_match_exact_rationals():
    rng = np.random.default_rng(2)
    a = (rng.standard_normal(500) * np.exp2(rng.integers(-30, 30, 500))).astype(F32)
    b = (rng.standard_normal(500) * np.exp2(rng.integers(-30, 30, 500))).astype(F32)
    for op, f in ((O.add_ftz, lambda x, y: x + y), (O.mul_ftz, lambda x, y: x * y), (O.sub_ftz, lambda x, y: x - y)):
        got = op(a, b)
        for x, y, g in zip(a, b, got):
            want = _nearest_f32(f(Fraction(float(x)), Fraction(float(y))))
            assert Fraction(float(g)) == want, (op.__name__, x, y, g)


def _nearest_f32(v):
    r = F32(float(v))
    cands = [r, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf))]
    dist = [abs(Fraction(float(c)) - v) for c in cands]
    best = min(dist)
    win = [c for c, d in zip(cands, dist) if d == best]
    win = min(win, key=lambda c: int(np.array(c, F32).view(np.uint32)) & 1)     # ties: even mantissa
    return Fraction(float(_flush(float(win))))


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_roundings_match_torch(tag):
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(20000) * np.exp2(rng.integers(-30, 20, 20000))).astype(F32)
    x = np.concatenate([x, np.array([65519.99, 65520, 3.4e38, -3.4e38, np.inf, 2.0 ** -25, 6e-8, 0.0], F32)])
    want = torch.from_numpy(x).to(TORCH_T[tag]).float().numpy()
    with np.errstate(over="ignore"):
        np.testing.assert_array_equal(O.round_t(x, tag), want)
    if tag == "f16":                  # float64 -> fp16 in one rounding, checked against the exact nearest
        y = rng.standard_normal(3000) * np.exp2(rng.integers(-26, 12, 3000))
        y = np.concatenate([y, [1 + 2.0 ** -11 + 2.0 ** -40, 1 + 2.0 ** -11, 1 - 2.0 ** -12 - 2.0 ** -50]])
        got = O.rn16(y)
        for v, g in zip(y, got):
            grid = [F16(g), np.nextafter(F16(g), F16(np.inf)), np.nextafter(F16(g), F16(-np.inf))]
            assert abs(Fraction(float(g)) - Fraction(float(v))) <= min(abs(Fraction(float(c)) - Fraction(float(v)))
                                                                      for c in grid if np.isfinite(c))


# (n, access width) -> threads per row and chunks per thread, worked by hand from row_threads and chunks_per_thread
GEOMETRY = [(8, 8, 32, 1), (256, 8, 32, 1), (264, 8, 64, 1), (8192, 8, 1024, 1), (8200, 8, 544, 2),
            (16384, 8, 1024, 2), (16392, 8, 704, 3), (24576, 8, 1024, 3), (24584, 8, 800, 4), (32768, 8, 1024, 4),
            (1, 1, 32, 1), (31, 1, 32, 1), (1024, 1, 1024, 1), (1025, 1, 544, 2), (2048, 1, 1024, 2),
            (2049, 1, 704, 3), (3072, 1, 1024, 3), (3073, 1, 800, 4), (4096, 1, 1024, 4), (4097, 1, 832, 5),
            (5120, 1, 1024, 5), (5121, 1, 864, 6), (6144, 1, 1024, 6), (6145, 1, 896, 7), (7168, 1, 1024, 7),
            (7169, 1, 928, 8), (8191, 1, 1024, 8), (8192, 1, 1024, 8)]


@pytest.mark.parametrize("n,vec,threads,chunks", GEOMETRY)
def test_row_geometry(n, vec, threads, chunks):
    assert O.row_threads(n // vec) == threads
    assert -(-(n // vec) // threads) == chunks and O.row_fits(n, vec)


def test_row_width_choice_and_limits():
    assert O.row_vec(1152) == 8 and O.row_vec(1001) == 1 and O.row_vec(1152, aligned=False) == 1
    assert O.row_fits(32768, 8) and not O.row_fits(32776, 8)
    assert O.row_fits(8192, 1) and not O.row_fits(8193, 1)


def _scalar_ln_sums(row, vec):
    """layernorm_quant_kernel's statistics with one scalar loop per thread and per shuffle, as the kernel spells it."""
    n = len(row)
    nc, thr = n // vec, O.row_threads(n // vec)
    chunks = {8: 4, 1: 8}[vec]
    s, q = [F32(0)] * thr, [F32(0)] * thr
    for t in range(thr):
        for j in range(chunks):
            ci = t + j * thr
            if ci < nc:
                for e in range(vec):
                    v = row[ci * vec + e]
                    s[t] = O.add_ftz(s[t], v)[()]
                    q[t] = O.fma_ftz(v, v, q[t])[()]

    def shuffle_reduce(vals):
        vals = list(vals)
        for o in (16, 8, 4, 2, 1):
            vals = [O.add_ftz(vals[i], vals[i ^ o])[()] for i in range(32)]
        return vals[0]
    nw = thr // 32
    outs = []
    for part in (s, q):
        red = [shuffle_reduce(part[32 * w:32 * w + 32]) for w in range(nw)] + [F32(0)] * (32 - nw)
        outs.append(shuffle_reduce(red))
    return outs


@pytest.mark.parametrize("n,vec", [(37, 1), (1025, 1), (8200, 8), (4104, 8)])
def test_ln_sums_match_scalar_loop(n, vec):
    rng = np.random.default_rng(n)
    x = (rng.standard_normal((2, n)) * [[1.0], [300.0]] + [[0.0], [1000.0]]).astype(F16).astype(F32)
    s, q = O.ln_sums(x, vec)
    for r in range(2):
        ss, qq = _scalar_ln_sums(x[r], vec)
        assert s[r] == ss and q[r] == qq


def test_quant_bounds_equal_enumeration():
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((50, 24)) * np.exp(rng.standard_normal((50, 1)))).astype(F16).astype(F32)
    b = O.quant_per_token_bounds(x)
    amax = np.abs(x).max(axis=1)
    ilo, ihi = O.div_approx(F32(127), amax)
    for r in range(50):
        invs = [ilo[r]]
        while invs[-1] < ihi[r]:
            invs.append(np.nextafter(invs[-1], F32(np.inf)))
        codes = O.cvt_s8(np.stack([O.mul_ftz(x[r], i) for i in invs]))
        np.testing.assert_array_equal(codes.min(axis=0), b["lo"][r])
        np.testing.assert_array_equal(codes.max(axis=0), b["hi"][r])


def test_gelu_bounds_equal_enumeration():
    x = np.concatenate([np.linspace(-6, 6, 4001), np.linspace(-1e-3, 1e-3, 97)]).astype(F16)
    inner, h = O.gelu_front_f16(x)
    t_lo, t_hi = O.tanh_range(inner.astype(F32))
    b = O.gelu_quant_bounds(x[None, :])
    for i in range(len(x)):
        ts = [t_lo[i]]
        while ts[-1] < t_hi[i]:
            ts.append(np.nextafter(ts[-1], F16(np.inf)))
        gs = O.gelu_tail_f16(np.full(len(ts), h[i]), np.array(ts, F16))
        assert gs.min() == b["g_lo"][0, i] and gs.max() == b["g_hi"][0, i]


def test_layernorm_bounds_contain_enumeration():
    """Every combination of the div.approx candidates for mean and E[x^2], every float32 rstd the bound allows and
    every 127 / amax candidate gives codes inside the corner-evaluated sets, and on rows without cancellation reaches
    their ends on most elements."""
    rng = np.random.default_rng(5)
    for tag in ("f16", "bf16"):
        x = (rng.standard_normal((6, 40)) * 2 + [[0], [0], [30], [0], [100], [0.01]]).astype(F32)
        x = O.round_t(x, tag)
        x[3] = O.round_t(np.full(40, 100.0, F32), tag)
        gm, bt = O.round_t(1 + 0.2 * rng.standard_normal(40), tag), O.round_t(0.1 * rng.standard_normal(40), tag)
        b = O.layernorm_quant_bounds(x, gm, bt, 1e-6, tag)
        s, q = O.ln_sums(x, 8)
        k = range(-2, 3)
        for r in range(6):
            seen = []
            for dm, dq in itertools.product(k, k):
                mean = O.steps32(O.div_approx(s[r], F32(40))[0], 2 + dm)
                sqn = O.steps32(O.div_approx(q[r], F32(40))[0], 2 + dq)
                ve = O.add_ftz(O.fma_ftz(-mean, mean, sqn), F32(1e-6))
                rlo, rhi = O.rsqrt_approx(ve)
                if np.isnan(rlo):
                    continue
                rs = [rlo]
                while rs[-1] < rhi:
                    rs.append(np.nextafter(rs[-1], F32(np.inf)))
                for rstd in rs:
                    y = O.fma_ftz(O.mul_ftz(O.sub_ftz(x[r], mean), rstd), gm, bt)
                    amax = max(np.abs(O.round_t(y, tag)).max(), O.round_t(np.array([1e-6], F32), tag)[0])
                    ilo, ihi = O.div_approx(F32(127), amax)
                    for inv in (ilo, ihi):
                        seen.append(O.cvt_s8(O.mul_ftz(y, inv)))
            if not seen:
                assert b["deg"][r]
                continue
            seen = np.stack(seen)
            assert (seen.min(axis=0) >= b["lo"][r]).all() and (seen.max(axis=0) <= b["hi"][r]).all(), (tag, r)
            if r in (0, 1, 5):        # no cancellation: the box adds nothing the enumeration does not reach
                assert np.mean((seen.min(axis=0) == b["lo"][r]) & (seen.max(axis=0) == b["hi"][r])) > 0.9


def test_layernorm_constant_row_takes_the_nan_branch():
    """A constant row of 100: var = fma(-mean, mean, sq / n) is below -eps for some div.approx candidates, where the
    kernel's rstd is NaN, its codes 0 and its amax the floor rn_T(1e-6)."""
    x = np.full((1, 64), 100.0, F32)
    b = O.layernorm_quant_bounds(x, np.ones(64, F32), None, 1e-6, "f16")
    assert b["deg"][0]
    assert b["d_lo"][0] == b["d_hi"][0] == F16(F32(F16(1e-6)) / 127)
    assert O.admissible_rows(np.zeros((1, 64)), np.array([b["d_lo"][0]]), b)[0]


def test_div_approx_outside_its_range():
    lo, hi = O.div_approx(np.array([127, 1, 0, np.inf, 127], F32), np.array([2.0 ** 127, np.inf, 0, np.inf, 1e-39], F32))
    np.testing.assert_array_equal(lo[:2], [0, 0])
    assert np.isnan(lo[2]) and np.isnan(lo[3]) and lo[4] == np.inf      # 0 / 0, inf / inf; a flushed divisor is 0
    lo, hi = O.div_approx(F32(3), F32(7))
    assert O.steps32(lo, 4) == hi and lo < F32(3 / 7) < hi


def test_gemm_epilogue_single_rounding():
    """The fused-bias epilogue rounds fma(p, as, b) once: on these operands float64 followed by a cast to float32
    rounds twice, and the fp16 result moves."""
    rng = np.random.default_rng(6)
    acc = rng.integers(-2 ** 20, 2 ** 20, (400, 64))
    ws, a, bias = W.gen_scales(64, 1).numpy(), W.gen_scales(400, 2).numpy(), W.gen_bias(64, 3).numpy()
    y = O.gemm_exact(acc, ws, a, bias)
    p = O.mul_ftz(acc.astype(F32), ws.astype(F32)[None, :])
    want = O.fma_ftz(p, a.astype(F32)[:, None], bias.astype(F32)[None, :])
    np.testing.assert_array_equal(y, want.astype(F16))
    fmaf = _libm_fmaf()
    for i, j in [(0, 0), (13, 7), (399, 63)]:
        assert F16(F32(fmaf(float(p[i, j]), float(F32(a[i])), float(F32(bias[j]))))) == y[i, j]


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_reference_quant_inside_admissible_sets(gold, tag, MN):
    M, N = MN
    key = f"{tag}_{M}x{N}"
    x = W.act_rows(M, N, TORCH_T[tag], seed=M + N).float().numpy()
    b = O.quant_per_token_bounds(x)
    q = gold[f"quant_q_{key}"]
    lo, hi = b["lo"].reshape(-1)[::W.ROW_SAMPLE], b["hi"].reshape(-1)[::W.ROW_SAMPLE]
    assert ((q >= lo) & (q <= hi)).all()
    s = gold[f"quant_s_{key}"].view(F16)
    assert ((s >= b["s_lo"]) & (s <= b["s_hi"])).all()


@pytest.mark.parametrize("MN", W.ROW_SHAPES)
def test_reference_gelu_inside_admissible_sets(gold, MN):
    M, N = MN
    key = f"f16_{M}x{N}"
    b = O.gelu_quant_bounds(W.gelu_rows(M, N, seed=7 * M + N).numpy())
    smp = lambda a: a.reshape(-1)[::W.ROW_SAMPLE]
    q, g = gold[f"gelu_q_{key}"], gold[f"gelu_t_{key}"].view(F16)
    assert ((q >= smp(b["lo"])) & (q <= smp(b["hi"]))).all()
    O.assert_between(g, smp(b["g_lo"]), smp(b["g_hi"]), "gelu")
    s = gold[f"gelu_s_{key}"].view(F16)
    assert ((s >= b["s_lo"]) & (s <= b["s_hi"])).all()
