"""Elementwise error bounds for the attention kernels on inputs whose scores are exact.  Shared by
tests/test_attention_bounds_cpu.py (the bound against numpy emulations of the kernels' arithmetic) and
tests/test_attention_bounds_gpu.py (the bound against the kernels).

Inputs.  q lies in 2^-2 Z with |q| <= 4 and k in 2^-4 Z with |k| <= 8, so every product q_c k_c is a multiple of 2^-6
of size <= 32 and every partial sum of q . k (|s| <= 32 D <= 2^13) is exact in fp32 whatever the order: the S = Q K^T
wgmma, the decode kernel's fp32 dot products and the float64 oracle see the same raw scores.  V lies in 2^-2 Z with
|v| <= 4; its last channel is a constant, so that any mismatch between the numerator and the row sum l shows there.
Channels: the first D / 2 are "level" channels (q = 4, k sums to the key's level), then r x nb code channels
(needles: key j carries +-8 per bit of j, the row's q +-4 per bit of its target), then noise (q in +-0.5, k in +-1).
Landscapes, given as exponents in log2 units, u log2 units per unit of level:
  * staircase: the level rises at every 128-key tile edge, by more than 126 after tile 0 (ex2.approx.ftz flushes that
    rescale factor to 0), and the last tile is the top;
  * descending: the top at key 0, then -60 sqrt(j / N): in fp16 most p are subnormal or 0;
  * needles: flat noise, each row's target key 12 above and every other key at least 12 below;
  * tiles: every 128-key tile at its own random level down to 170 below the top (split maxima far apart, combine
    weights that underflow); the top tile is never tile 0;
  * ties: one key per tile, with the same K row everywhere, at the top, the others at least 0.25 level units lower:
    rescale factors and combine weights of exactly 1.
The top sits near exponent 0, which keeps |scale_log2 * m| small: see the term for -m * c below.  `shift` moves it:
the decode kernel also runs with the top above the range of exp (scores > 88 natural units), where a combine weight
taken without subtracting the max overflows.

The bound |O_kernel - O| <= B, O the float64 attention, per element (row i, channel d), with p_ij = exp(scale (s_ij -
M_i)), l_i = sum_j p_ij, A_id = sum_j p_ij |v_jd| / l_i (the attention of |V|), u_T = 2^-11 (fp16) / 2^-8 (bf16),
u = 2^-24:

  B = 1/2 ulp_T(|O| + E) + E            the one rounding of the output to T (prefill_attention.cu:227,
                                        splitkv_attention.cu:252/321/351, attention.cu:298/324)
  E = sum_j p_ij delta_ij (|v_jd| + |O_id|) / l_i  (1 + 2^-10)   relative errors of p_ij common to the numerator and
                                        l (each moves O by at most delta (|v| + |O|)), with the slack for second order
    + 2 u_T A                           wgmma kernels: P rounded to T for O += P V, l summed from the fp32 p
                                        (attention_wgmma.cuh:126-131); 0 for the decode kernel, which keeps p in fp32
    + 2^-21 n16 A                       wgmma kernels: the P V accumulator.  Model, not documented by NVIDIA: each
                                        k16 step returns the exact sum within 2^-21 (|acc| + sum |products|), about
                                        2 fp32 ulps of max(|acc|, sum |products|), truncation included; n16 = 8 x the
                                        tiles of the key range, as if all of a row's keys ran in one CTA.  16384 keys:
                                        2^-11 A, one u of fp16
    + 2^-25 sum_visible |v_jd| / l_i    fp16 wgmma kernels: p below 2^-14 is subnormal in fp16, below 2^-25 it is 0
    + 2^-124 n (max |v| + |O|) / l_i    p and rescale factors below 2^-126 flushed (ex2.approx.ftz)

delta_ij, wgmma kernels (c = scale_log2 in fp32, cs = c s in log2 units, t = key j's tile, T tiles, cm_t = the row's
running maximum of cs after tile t, ln2 u per log2 unit of argument rounding):
    ln2 u (|cs_ij| (1 + 3 (T - t)) + 3 sum_{t' >= t} |cm_t'| + 4 |cs_ij - cM_i| + 3 |cM_i|)
        nb = -m c rounded (attention_wgmma.cuh:119-120), common to a tile, and the FFMA roundings of p's argument and
        of each later rescale's argument (:121, :126-127); any split's running max lies between s_ij and cm_t'.  The
        4 |cs - cM| covers scale_log2 = fp32(scale * fp32(log2 e)) against scale log2 e (prefill_attention.cu:268),
        3 |cM| the combine's weight (splitkv_attention.cu:299-302)
  + 2^-21 (T - t + 2)                   ex2.approx of p, of each later rescale factor and of the combine weight
  + u (23 + 2 (T - t) + 2 T)            l: the 16 pair sums of a tile and the quad reduction (:128, :200-206); per
                                        later tile the FMA l * alpha + sum (:133) and O's rescale (:136-137); the
                                        combine's fp32 FMAs over <= T splits (splitkv_attention.cu:304, :317); 1 / l
                                        and the product (:246-253)
delta_ij, decode kernel (x = scale s in natural units, M_i the row max): x rounded, times fp32 log2 e rounded, and
__expf (attention.cu:225), the fp32 1 / sqrt(D) and the score's rounding (:189), the chunk max and the combine weight
(:321):
    4 2^-21 + u (6 |x_ij - M_i| + 9 |x_ij| + 9 |M_i|) + u (n / 8 + 128)
  the last term for the fp32 sums of p and p v (<= n / 8 FMAs per thread, 32 position rows, 8 warps, 64 splits).

The roundings of -m c and of the rescale arguments are derived per key from the running maxima; with the top near 0
they stay below 2^-14 relative.  Nothing in B is fitted to kernel output."""
import math

import numpy as np
import torch

TILE = 128
LOG2E = 1.4426950408889634
U32 = 2.0 ** -24
UT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
MANT = {torch.float16: 10, torch.bfloat16: 7}
EMIN = {torch.float16: -14, torch.bfloat16: -126}
KINDS = ("staircase", "descending", "needles", "tiles", "ties")
TOP = 7.8  # |level| bound: with +-1/16 of noise per channel k stays within +-8


def f32(x):
    """Rounds a float64 value or array to fp32 (as float64)."""
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def wgmma_scale(D):
    """softmax_scale for the wgmma entries: about 24 log2 units per level unit (level raw score = 2 D x level), an
    fp32 value so that the oracle and the kernel start from the same number."""
    return float(np.float32(24.0 / (2 * D * LOG2E)))


def scale_log2(scale):
    """The kernels' c = fp32(scale * fp32(log2 e)) (prefill_attention.cu:268, splitkv_attention.cu:423)."""
    return float(np.float32(np.float32(scale) * np.float32(LOG2E)))


def level_units(D, scale):
    """log2 units per level unit: the level's raw score is 4 x (D / 2) x level."""
    return 2 * D * scale * LOG2E


def code_bits(n):
    return max(4, math.ceil(math.log2(max(n, 2))))


def code_repeat(D, nbits):
    """Channels per code bit: the codes take at most D / 2 - 4 channels, and the level that offsets them stays
    within TOP."""
    r = min((D // 2 - 4) // nbits, int(D * TOP / (16 * (nbits - 1))))
    assert r >= 1, (D, nbits)
    return r


# ------------------------------------------------------------------------------------------------ landscapes
def key_levels(kind, n, u, gen, shift=0.0):
    """Level (raw score / (2 D)) of each of n keys, float64 [n], and the tie keys (a list of indices)."""
    T = -(-n // TILE)
    t = torch.arange(n) // TILE
    q16 = lambda e: torch.round(torch.as_tensor(e, dtype=torch.float64) / u * 16) / 16  # log2 units -> levels
    ties = []
    if kind == "staircase":
        jump = q16(136.0) + 1 / 16
        step = min(1.0, (TOP - float(jump)) / max(T - 1, 1)) if T > 1 else 0.0
        lev = -(T - 1 - t).to(torch.float64) * step
        lev = torch.where(t == 0, lev - jump, lev) if T > 1 else lev
    elif kind == "descending":
        lev = q16(-60.0 * torch.sqrt(torch.arange(n, dtype=torch.float64) / n))
    elif kind == "needles":
        lev = torch.zeros(n, dtype=torch.float64)  # the code offset is added by `make_k`
    elif kind == "tiles":
        tl = -torch.randint(0, int(170 / u * 16) + 1, (T,), generator=gen).to(torch.float64) / 16
        top = int(torch.randint(1 if T > 1 else 0, T, (1,), generator=gen))
        tl[top] = 0.0
        lev = tl[t] - torch.randint(0, 9, (n,), generator=gen).to(torch.float64) / 16
    elif kind == "ties":
        lev = -0.25 - torch.randint(0, 13, (n,), generator=gen).to(torch.float64) / 16
        off = torch.randint(0, TILE, (T,), generator=gen)
        ties = [min(n - 1, k * TILE + int(off[k])) for k in range(T)]
        lev[ties] = 0.0
    else:
        raise ValueError(kind)
    return (lev + shift).clamp(-TOP, TOP), ties


def make_k(kind, n, D, u, gen, shift=0.0):
    """K [n, D] float64 of one (batch row, KV head)."""
    nb = code_bits(n)
    r = code_repeat(D, nb)
    nl = D // 2
    lev, ties = key_levels(kind, n, u, gen, shift)
    if kind == "needles":  # flat: the target's codes 32 r nb, less 32 r (nb - 1), score 32 r raw above the level
        lev = lev - torch.round(torch.tensor(32.0 * r * (nb - 1) / (2 * D)) * 16 * nl) / (16 * nl)
    units = torch.round(lev * 16 * nl).to(torch.long)  # level in 1/16 steps of one channel
    c = torch.arange(nl)
    k = torch.zeros(n, D, dtype=torch.float64)
    k[:, :nl] = ((units.view(-1, 1) // nl) + (c.view(1, -1) < (units.view(-1, 1) % nl))).to(torch.float64) / 16
    k[:, :nl] += torch.randint(-1, 2, (n, nl), generator=gen).to(torch.float64) / 16
    bits = ((torch.arange(n).view(-1, 1) >> torch.arange(nb).view(1, -1)) & 1).to(torch.float64) * 2 - 1
    k[:, nl:nl + r * nb] = 8 * bits.repeat(1, r)
    k[:, nl + r * nb:] = torch.randint(-16, 17, (n, D - nl - r * nb), generator=gen).to(torch.float64) / 16
    for j in ties[1:]:
        k[j] = k[ties[0]]
    return k


def make_q(kind, targets, n, D, gen):
    """q [rows, D] float64 for rows whose needle targets are `targets` (ignored unless kind is needles)."""
    rows = len(targets)
    nb = code_bits(n)
    r = code_repeat(D, nb)
    nl = D // 2
    q = torch.zeros(rows, D, dtype=torch.float64)
    q[:, :nl] = 4
    if kind == "needles":
        t = torch.as_tensor(targets, dtype=torch.long).clamp(min=0)
        bits = ((t.view(-1, 1) >> torch.arange(nb).view(1, -1)) & 1).to(torch.float64) * 2 - 1
        q[:, nl:nl + r * nb] = 4 * bits.repeat(1, r)
    q[:, nl + r * nb:] = torch.randint(-2, 3, (rows, D - nl - r * nb), generator=gen).to(torch.float64) / 4
    return q


def make_v(n, D, gen):
    """V [n, D] float64: multiples of 1/4 in [-4, 4], the last channel 1.75 throughout."""
    v = torch.randint(-16, 17, (n, D), generator=gen).to(torch.float64) / 4
    v[:, -1] = 1.75
    return v


def needle_targets(lo, hi, n, edge, slot):
    """A needle key for a row that sees keys lo .. hi: candidate `slot` (cyclic) of its horizon, the key before,
    key lo, key 0, the last key, and the first and last key of every `edge`-key block, among the keys it sees."""
    if hi < lo:
        return -1
    cand = [hi, hi - 1, lo, 0, n - 1]
    for e in range(0, n, edge):
        cand += [e, e + edge - 1]
    seen = []
    for x in cand:
        if lo <= x <= hi and x not in seen:
            seen.append(x)
    return seen[slot % len(seen)]


def check_exact(*ts):
    """Every value is exact in fp16 and in bf16."""
    for x in ts:
        for dt in (torch.float16, torch.bfloat16):
            assert torch.equal(x.to(dt).to(torch.float64), x), f"not exact in {dt}"


# ------------------------------------------------------------------------------------------------ the bound
def ulp_t(x, dtype):
    """One unit in the last place of T at |x| (float64), subnormals included."""
    _, e = torch.frexp(x.abs().to(torch.float64))
    return torch.pow(2.0, (e - 1).clamp(min=EMIN[dtype]) - MANT[dtype]).to(torch.float64)


def bound(s, vis, v, scale, dtype, family, n_keys=None, parts=False):
    """(O, B) float64 [..., R, C] for raw scores s [..., R, N] (exact), visibility vis [..., R, N] and V [..., N, C]
    (T values); family "wgmma" (flash_attn_func, the varlen entry, kv_cache_attention) or "decode"
    (single_query_attention, scale 1 / sqrt(D)).  n_keys: the key range whose tiles a row's CTA may run (default N).
    Rows that see no key: O = 0, B = 0 (the kernels write zeros).  parts: also A and the accumulator term of E."""
    N = s.shape[-1]
    n_keys = N if n_keys is None else n_keys
    dev = s.device
    x = torch.where(vis, s * scale, torch.tensor(float("-inf"), dtype=torch.float64, device=dev))
    M = x.amax(-1, keepdim=True)
    seen = torch.isfinite(M)
    M = torch.where(seen, M, torch.zeros_like(M))
    p = torch.exp(x - M)
    l = p.sum(-1, keepdim=True)
    li = torch.where(l > 0, 1 / l, torch.zeros_like(l))
    av = v.abs()
    O = (p @ v) * li
    A = (p @ av) * li
    j = torch.arange(N, device=dev)
    if family == "wgmma":
        c = scale_log2(scale)
        T = -(-n_keys // TILE)
        tj = (j // TILE).to(torch.float64)
        cs = torch.where(vis, s * c, torch.zeros_like(s))
        cx = torch.where(vis, s * c, torch.tensor(float("-inf"), dtype=torch.float64, device=dev))
        pad = T * TILE - N
        if pad:
            cx = torch.nn.functional.pad(cx, (0, pad), value=float("-inf"))
        tmax = cx.view(*cx.shape[:-1], T, TILE).amax(-1)
        cm = torch.cummax(tmax, -1).values
        cm = torch.where(torch.isfinite(cm), cm.abs(), torch.zeros_like(cm))
        suf = cm.flip(-1).cumsum(-1).flip(-1)  # sum over t' >= t of |cm_t'|
        cM = (M * c / scale).abs()
        delta = (math.log(2) * U32 * (cs.abs() * (1 + 3 * (T - tj)) + 3 * suf[..., (j // TILE)]
                                      + 4 * (cs - M * c / scale).abs() + 3 * cM)
                 + 2.0 ** -21 * (T - tj + 2) + U32 * (23 + 2 * (T - tj) + 2 * T))
    else:
        delta = 4 * 2.0 ** -21 + U32 * (6 * (s * scale - M).abs() + 9 * (s * scale).abs() + 9 * M.abs()) \
            + U32 * (n_keys / 8 + 128)
        delta = torch.where(vis, delta, torch.zeros_like(delta))
    pd = p * delta
    E = ((pd @ av) * li + O.abs() * (pd.sum(-1, keepdim=True) * li)) * (1 + 2.0 ** -10)
    vmax = av.amax(-2, keepdim=True)
    E = E + 2.0 ** -124 * n_keys * (vmax + O.abs()) * li
    acc = 2.0 ** -21 * 8 * (-(-n_keys // TILE)) * A if family == "wgmma" else torch.zeros_like(A)
    if family == "wgmma":
        E = E + 2 * UT[dtype] * A + acc
        if dtype == torch.float16:
            E = E + 2.0 ** -25 * (vis.to(torch.float64) @ av) * li
    B = torch.where(seen, 0.5 * ulp_t(O.abs() + E, dtype) + E, torch.zeros_like(E))
    return (O, B, A, acc) if parts else (O, B)


def ratio(got, O, B):
    """err / B elementwise: inf where B = 0 and err > 0, and wherever the output is NaN."""
    got = got.to(torch.float64)
    err = (got - O).abs()
    r = torch.where(B > 0, err / torch.where(B > 0, B, torch.ones_like(B)), torch.where(err > 0, math.inf, 0.0))
    return torch.where(torch.isnan(got) | torch.isnan(r), torch.full_like(r, math.inf), r)


# ------------------------------------------------------------------------------------------------ emulations (numpy)
def _rn_t(x, dtype):
    if dtype == torch.float16:
        return x.astype(np.float16).astype(np.float64)
    return torch.from_numpy(x.astype(np.float32)).to(torch.bfloat16).to(torch.float64).numpy()


def _fma(a, b, c):
    return f32(np.asarray(a, dtype=np.float64) * b + c)


def _ex2(x, sign=1.0):
    """ex2.approx.ftz.f32 as exp2 rounded to fp32, perturbed by sign * 2^-22 relative, subnormals flushed."""
    y = f32(f32(np.exp2(x)) * (1 + sign * 2.0 ** -22))
    return np.where(np.abs(y) < 2.0 ** -126, 0.0, y)


def _expf(x, sign=1.0):
    """__expf: ex2.approx.f32 of x * fp32(log2 e)."""
    y = f32(np.exp2(f32(x * float(np.float32(LOG2E))))) * (1 + sign * 2.0 ** -22)
    return f32(y)


def _acc_step(exact, mag):
    """One k16 step under the bound's accumulator model, every loss toward 0: the fp32 value nearest to exact -
    sign(exact) 2^-21 mag that is no further than 2^-21 mag from exact."""
    budget = 2.0 ** -21 * mag
    r = np.asarray(exact - np.sign(exact) * budget, np.float32)
    over = np.abs(r.astype(np.float64) - exact) > budget
    r = np.where(over, np.nextafter(r, np.asarray(exact, np.float32)), r)
    return r.astype(np.float64)


WGMMA_DEFECTS = ("hi_not_rescaled", "l_not_rescaled", "alpha_prev_max", "no_quad_max", "combine_next_max", "no_log2e")


def emulate_wgmma(s, v, scale, dtype, edges, defect=None, rounded=True):
    """The wgmma kernels' softmax and P V for one (batch row, head): raw scores s [R, N] (exact, -inf masked), V [N,
    C] (T values), split edges (multiples of 128 from 0 to N) -> output [R, C] (T values; rounded=False: the fp32
    value before the output's rounding).  Row r is a "hi" row when r % 16 >= 8; key j of a tile belongs to thread
    (j % 8) // 2, and so does channel d's accumulator."""
    with np.errstate(all="ignore"):
        out = _emulate_wgmma(np.asarray(s, np.float64), np.asarray(v, np.float64), scale, dtype, edges, defect)
    return _rn_t(out, dtype) if rounded else out


def _emulate_wgmma(s, v, scale, dtype, edges, defect):
    R, N = s.shape
    C = v.shape[1]
    c = scale_log2(scale) if defect != "no_log2e" else float(np.float32(scale))
    thr_k = (np.arange(TILE) % 8) // 2
    thr_c = (np.arange(C) % 8) // 2
    hi = (np.arange(R) % 16) >= 8
    key_sign = np.where((np.arange(N + TILE) * 2654435761 >> 7) & 1, 1.0, -1.0)
    parts = []
    for e0, e1 in zip(edges[:-1], edges[1:]):
        m = np.full((R, 4), -np.inf)
        l = np.zeros((R, 4))
        o = np.zeros((R, C))
        for k0 in range(e0, e1, TILE):
            sc = np.full((R, TILE), -np.inf)
            sc[:, :min(TILE, N - k0)] = s[:, k0:k0 + TILE]
            vt = np.zeros((TILE, C))
            vt[:min(TILE, N - k0)] = v[k0:k0 + TILE]
            mx = np.stack([np.maximum(m[:, t], sc[:, thr_k == t].max(1)) for t in range(4)], 1)
            if defect != "no_quad_max":
                mx = np.repeat(mx.max(1, keepdims=True), 4, 1)
            nb = np.where(mx == -np.inf, 0.0, -f32(mx * c))
            nb_a = nb if defect != "alpha_prev_max" else np.where(m == -np.inf, 0.0, -f32(m * c))
            alpha = _ex2(_fma(m, c, nb_a))
            m = mx
            p = _ex2(_fma(sc, c, nb[:, thr_k]), key_sign[k0:k0 + TILE])
            pairs = f32(p[:, 0::2] + p[:, 1::2]).reshape(R, 16, 4)  # pair k of thread t: keys 8 k + 2 t, + 1
            sm = np.zeros((R, 4))
            for k in range(16):
                sm = f32(sm + pairs[:, k])
            l = f32(l + sm) if defect == "l_not_rescaled" else _fma(l, alpha, sm)
            a_c = alpha[:, thr_c]
            if defect == "hi_not_rescaled":
                a_c = np.where(hi[:, None], 1.0, a_c)
            o = f32(o * a_c)
            pt = _rn_t(p, dtype)
            for kk in range(TILE // 16):
                prod = pt[:, 16 * kk:16 * kk + 16, None] * vt[None, 16 * kk:16 * kk + 16]
                exact = o + prod.sum(1)
                mag = np.abs(o) + np.abs(prod).sum(1)
                o = _acc_step(exact, mag)
        lq = f32(l + l[:, [1, 0, 3, 2]])
        lq = f32(lq + lq[:, [2, 3, 0, 1]])
        parts.append((o, m[:, 0], lq[:, 0]))
    if len(parts) == 1:
        o, _, l = parts[0]
        inv = np.where(l > 0, f32(1 / np.where(l > 0, l, 1)), 0.0)
        return f32(o * inv[:, None])
    ms = np.stack([p[1] for p in parts])
    M = ms.max(0)
    nb = np.where(M == -np.inf, 0.0, -f32(M * c))
    S = len(parts)
    den = np.zeros(R)
    x = np.zeros((R, C))
    for sp in range(S):
        mw = ms[(sp + 1) % S] if defect == "combine_next_max" else ms[sp]
        w = _ex2(_fma(mw, c, nb))
        den = _fma(w, parts[sp][2], den)
        x = _fma(w[:, None], parts[sp][0], x)
    inv = np.where(den > 0, f32(1 / np.where(den > 0, den, 1)), 0.0)
    return f32(x * inv[:, None])


DECODE_DEFECTS = ("decode_no_max",)


def emulate_decode(raw, v, D, dtype, edges, defect=None):
    """single_query_attention's chunked softmax and combine for the G heads of one KV head: raw scores q . k [G, n]
    (exact), V [n, C] (T values), chunk edges (multiples of 32 from 0 to n) -> output [G, C] (T values)."""
    with np.errstate(all="ignore"):
        return _emulate_decode(np.asarray(raw, np.float64), np.asarray(v, np.float64), D, dtype, edges, defect)


def _emulate_decode(raw, v, D, dtype, edges, defect):
    G, n = raw.shape
    C = v.shape[1]
    s = f32(raw * float(np.float32(1 / np.float32(np.sqrt(np.float32(D))))))
    rows = 256 // (D // 8)
    sign = np.where((np.arange(n) * 2654435761 >> 7) & 1, 1.0, -1.0)
    parts = []
    for p0, p1 in zip(edges[:-1], edges[1:]):
        sc = s[:, p0:p1]
        m = np.maximum(sc.max(1), -np.float32(3.4028234663852886e38))
        e = _expf(f32(sc - m[:, None]), sign[p0:p1])
        k = p1 - p0
        th = np.zeros((G, 256))
        for i in range(0, k, 256):  # thread tid sums positions tid, tid + 256, ...
            blk = np.zeros((G, 256))
            blk[:, :min(256, k - i)] = e[:, i:i + 256]
            th = f32(th + blk)
        w = th.reshape(G, 8, 32)
        for o_ in (16, 8, 4, 2, 1):
            w = f32(w + w[:, :, np.arange(32) ^ o_])
        l = np.zeros(G)
        for wi in range(8):
            l = f32(l + w[:, wi, 0])
        acc = np.zeros((G, rows, C))
        for i in range(0, k, rows):  # position row r takes positions p0 + r, + rows, ... in order
            blk = min(rows, k - i)
            acc[:, :blk] = _fma(e[:, i:i + blk, None], v[None, p0 + i:p0 + i + blk], acc[:, :blk])
        o = np.zeros((G, C))
        for r in range(rows):
            o = f32(o + acc[:, r])
        parts.append((o, m, l))
    if len(parts) == 1:
        o, _, l = parts[0]
        return _rn_t(f32(o / l[:, None]), dtype)
    M = np.max([p[1] for p in parts], 0)
    num = np.zeros((G, C))
    den = np.zeros(G)
    for o, m, l in parts:
        w = _expf(f32(m)) if defect == "decode_no_max" else _expf(f32(m - M))
        num = _fma(w[:, None], o, num)
        den = _fma(w, l, den)
    return _rn_t(f32(num / den[:, None]), dtype)
