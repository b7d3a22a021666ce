"""Known-answer inputs for the attention kernels, with exact expected outputs.  Shared by tests/test_attention_exact_cpu.py
and tests/test_attention_exact_gpu.py.

Visibility probe (which keys each output row sees).  q = 0, so every score is exactly 0 and every visible key has
p = 1 (exact in fp16, bf16 and fp32); K is random and finite.  In probe block beta, V[b, j, g, c] = w[b, g] when
j == beta * D + c, else 0, with w a distinct power of two per (batch row, KV head).  Output [b, i, h, c] is then
w[b, h // G] / n_i when key beta * D + c is visible to row i (n_i keys visible), and 0 when it is not.  The expected
values are not derived here: they are the existing float64 oracles' outputs on the same inputs, rounded to T.  The check
is exact zeros where the oracle gives 0 and one ulp of T elsewhere (the kernels compute 1 / l in fp32 and combine
splits).  A key seen that should not be, a key missed, a key counted twice, or a read from another batch row or KV head
turns 0 into w / n, w / n into 0 or 2 w / n, or w into another power of two.  Run over every block of the key range
(and one past it, where a cache has slots past the keys in use), the check covers every (row, head, key), so every
split and tile boundary is covered wherever a planner puts it.

Pointer probe (which K and V rows each row reads).  Key j of (batch row b, KV head g) carries the +-1 code of
j ^ mask[b, g] over `nbits` channels spread over all D / 8 column blocks; the other K channels are random.  Row i of
head h picks a visible target t with q = beta * code(t) in the code channels and 0 elsewhere, so every other key scores
at least 2 beta * scale per Hamming unit below it.  With 2 beta * scale >= 32 the target's p is exactly 1 and all other
keys together weigh below e^-32 * nbits, so the output is V[b, t, h // G, :] bit for bit (V holds integers in
+-[1, 8]).  A wrong K address moves the argmax to another key, a wrong (b, g) reads another code or value, and a wrong
packed row <-> head map returns another head's target.

Targets are chosen from the visible keys that the oracle reports (the visibility probe), never from a restated mask."""
import math

import torch

MANT = {torch.float16: 10, torch.bfloat16: 7}
EMIN = {torch.float16: -14, torch.bfloat16: -126}
TILE = 128  # key tile of the kernels: targets sit on both sides of its edges


# ------------------------------------------------------------------------------------------------ visibility probe
def weights(rows, kv_heads, exp0=0, device="cpu"):
    """w [rows, kv_heads] float64: 2^(exp0 + b * kv_heads + g), a distinct power of two per (batch row, KV head)."""
    assert rows * kv_heads <= 8, "at most 8 distinct powers keep every w / n far from the ends of fp16's range"
    e = exp0 + torch.arange(rows * kv_heads, dtype=torch.float64, device=device).view(rows, kv_heads)
    return torch.pow(2.0, e)


def visibility_values(w, n_keys, D, beta):
    """V [rows, n_keys, Hkv, D] float64 of probe block beta: V[b, beta * D + c, g, c] = w[b, g]."""
    rows, hkv = w.shape
    v = torch.zeros(rows, n_keys, hkv, D, dtype=torch.float64, device=w.device)
    c = torch.arange(D, device=w.device)
    j = beta * D + c
    keep = j < n_keys
    v[:, j[keep], :, c[keep]] = w.unsqueeze(0).expand(int(keep.sum()), rows, hkv)
    return v


def all_blocks(n_keys, D, past=0):
    """Every probe block of keys [0, n_keys), then `past` more (slots past the keys in use)."""
    return list(range(-(-n_keys // D) + past))


def sampled_blocks(n_keys, D, first, last, every):
    """Block 0, the blocks of keys first .. last - 1 (say the causal horizons), and every `every`-th block."""
    n = -(-n_keys // D)
    return sorted({0, n - 1} | set(range(first // D, min(n, -(-last // D)))) | set(range(0, n, every)))


def visibility_expected(oracle, w, n_keys, D, blocks, dtype, group=16):
    """Yields (beta, want, exact) for each probe block: `exact` is the float64 oracle output [B, S, H, D] on block
    beta's V, `want` that rounded to `dtype`.  `oracle(V)` takes V [rows, n_keys, Hkv, C] with C a multiple of D and
    returns [B, S, H, C]; every output channel depends on its own V channel only, so `group` blocks go through one
    oracle call, their V's side by side."""
    for s in range(0, len(blocks), group):
        part = blocks[s:s + group]
        out = oracle(torch.cat([visibility_values(w, n_keys, D, b) for b in part], dim=-1))
        for n, beta in enumerate(part):
            exact = out[..., n * D:(n + 1) * D]
            yield beta, exact.to(dtype), exact


# ------------------------------------------------------------------------------------------------ pointer probe
def code_channels(D, nbits):
    """Channel of code bit k: column block k % (D / 8), element k // (D / 8), so consecutive bits sit in different
    8-column blocks of the FT K layout [D / 8][L][8]."""
    nblk = D // 8
    assert nbits <= D
    return torch.tensor([(k % nblk) * 8 + k // nblk for k in range(nbits)], dtype=torch.long)


def code_bits(n_keys):
    return max(4, math.ceil(math.log2(max(n_keys, 2))))


def masks(rows, kv_heads, nbits):
    """A distinct mask per (batch row, KV head) below 2^nbits: odd multiples are a bijection modulo 2^nbits."""
    i = torch.arange(rows * kv_heads, dtype=torch.long).view(rows, kv_heads)
    return (i * 0x9E5 + 0x35) % (1 << nbits)


def codes(idx, nbits):
    """+-1 float64 [..., nbits]: bit k of idx -> +1 when set."""
    k = torch.arange(nbits, device=idx.device)
    return ((idx.unsqueeze(-1) >> k) & 1).to(torch.float64) * 2 - 1


def random_keys(rows, n_keys, kv_heads, D, gen, device="cpu"):
    """K [rows, n_keys, Hkv, D] float64: random multiples of 1/8 in [-4, 4] (exact in fp16 and bf16)."""
    return (torch.randint(-32, 33, (rows, n_keys, kv_heads, D), generator=gen).to(torch.float64) / 8).to(device)


def pointer_keys(rows, n_keys, kv_heads, D, nbits, gen, device="cpu"):
    """K [rows, n_keys, Hkv, D] float64: the code of j ^ mask[b, g] in the code channels, `random_keys` elsewhere."""
    K = random_keys(rows, n_keys, kv_heads, D, gen, device)
    j = torch.arange(n_keys, device=device).view(1, n_keys, 1)
    m = masks(rows, kv_heads, nbits).to(device).view(rows, 1, kv_heads)
    K[..., code_channels(D, nbits).to(device)] = codes(j ^ m, nbits)
    return K


def pointer_values(rows, n_keys, kv_heads, D, gen, device="cpu"):
    """V [rows, n_keys, Hkv, D] float64: random integers in +-[1, 8]."""
    mag = torch.randint(1, 9, (rows, n_keys, kv_heads, D), generator=gen)
    sign = torch.randint(0, 2, (rows, n_keys, kv_heads, D), generator=gen) * 2 - 1
    return (mag * sign).to(torch.float64).to(device)


def pointer_queries(targets, kv_heads, D, nbits, beta):
    """q [B, S, H, D] float64: row (b, i, h) holds beta * code(targets[b, i, h] ^ mask[b, h // G]) in the code
    channels, 0 elsewhere; 0 throughout where the target is -1 (a row that sees no key)."""
    B, S, H = targets.shape
    dev = targets.device
    m = masks(B, kv_heads, nbits).to(dev).repeat_interleave(H // kv_heads, dim=1).view(B, 1, H)
    q = torch.zeros(B, S, H, D, dtype=torch.float64, device=dev)
    q[..., code_channels(D, nbits).to(dev)] = beta * codes(targets.clamp(min=0) ^ m, nbits)
    return q * (targets >= 0).unsqueeze(-1)


def choose_targets(visible, seed):
    """targets [B, S, H] from visible [B, S, H, N] (bool, from the oracle): per row one of its last visible key (the
    horizon), the one before, its first visible key, key 0, the last key, the keys on both sides of the tile edge below
    its horizon and of the first tile edge, and four random keys, among those it sees; the G heads of a row take
    different candidates while there are enough.  -1 where a row sees no key."""
    B, S, H, N = visible.shape
    dev = visible.device
    ar = torch.arange(N, device=dev)
    any_ = visible.any(-1)
    hi = torch.where(visible, ar, -1).amax(-1)
    lo = torch.where(visible, ar, N).amin(-1)
    edge = hi // TILE * TILE
    g = torch.Generator().manual_seed(seed)
    span = (hi - lo + 1).clamp(min=1)
    rnd = [lo + (torch.randint(0, 1 << 30, (B, S, 1), generator=g).to(dev) % span) for _ in range(4)]  # one per row
    const = lambda v: torch.full_like(hi, v)
    cand = torch.stack([hi, hi - 1, lo, const(0), const(N - 1), edge, edge - 1, const(TILE - 1), const(TILE)] + rnd, -1)
    cand = cand.clamp(0, N - 1)
    first = torch.ones_like(cand, dtype=torch.bool)  # each key once, so that consecutive picks differ
    for k in range(1, cand.shape[-1]):
        first[..., k] = (cand[..., k:k + 1] != cand[..., :k]).all(-1)
    ok = torch.gather(visible, -1, cand) & first & any_.unsqueeze(-1)
    n_ok = ok.sum(-1)
    b, i, h = (torch.arange(x, device=dev) for x in (B, S, H))
    pick = (h.view(1, 1, H) + 3 * i.view(1, S, 1) + 5 * b.view(B, 1, 1)) % n_ok.clamp(min=1)
    rank = ok.cumsum(-1) - 1
    sel = (ok & (rank == pick.unsqueeze(-1))).to(torch.long).argmax(-1)
    return torch.where(any_, torch.gather(cand, -1, sel.unsqueeze(-1)).squeeze(-1), -1)


def gather_targets(V, targets, kv_heads):
    """V[b, targets[b, i, h], h // G, :] as [B, S, H, D] (0 where the target is -1): the pointer probe's answer."""
    B, S, H = targets.shape
    kv = (torch.arange(H, device=V.device) // (H // kv_heads)).view(1, 1, H).expand(B, S, H)
    bb = torch.arange(B, device=V.device).view(B, 1, 1).expand(B, S, H)
    out = V[bb, targets.clamp(min=0), kv]
    return out * (targets >= 0).unsqueeze(-1)


# ------------------------------------------------------------------------------------------------ oracles
def ft_k_cache(K):
    """Logical keys [B, L, Hkv, D] as tinychat's FasterTransformer K cache [B, Hkv, D / 8, L, 8]."""
    B, L, Hkv, D = K.shape
    return K.reshape(B, L, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous()


def single_query_step(q, k, v, K, V, t, rot_dim, dtype_name, lps=None, base=10000.0, scale=1.0, neox=True):
    """oracle/layer_oracle.single_query_attention on one decode step: q [B, H, D], k / v [B, Hkv, D], cache slots as
    logical K / V [B, L, Hkv, D] (copied, never changed) -> [B, 1, H, D] float64 (T values)."""
    import numpy as np
    from oracle import layer_oracle as LO
    f64 = lambda x: np.array(x.detach().cpu().to(torch.float64).numpy())
    kc = f64(ft_k_cache(K))
    vc = f64(V.permute(0, 2, 1, 3))
    out = LO.single_query_attention(f64(q), f64(k), f64(v), kc, vc, t, rot_dim, base, scale, neox, dtype_name,
                                    length_per_sample=lps)
    return torch.from_numpy(out).to(q.device).unsqueeze(1)


def single_query_visibility_oracle(k, K, t, D, H, dtype_name, lps=None):
    """oracle(V) of `visibility_expected` for one single_query_attention step with RoPE over the whole head: V are the
    cache slots [B, L, Hkv, C]; the step's input v is slot t_b % L of V, and that cache slot holds 0 beforehand (the
    kernel must take the step's value from its input).  q = 0 in every head, so the oracle's output is the same for
    the G heads of a KV head: it is evaluated once per KV head."""
    B, L, Hkv, _ = K.shape
    ts = [int(lps[b]) if lps is not None else int(t) for b in range(B)]

    def oracle(V):
        outs = []
        for c in range(0, V.shape[-1], D):
            Vc = V[..., c:c + D].clone()
            v = torch.stack([Vc[b, ts[b] % L] for b in range(B)])
            for b in range(B):
                Vc[b, ts[b] % L] = 0
            q0 = torch.zeros(B, Hkv, D, dtype=torch.float64, device=V.device)
            outs.append(single_query_step(q0, k, v, K, Vc, t, D, dtype_name, lps))
        return torch.cat(outs, -1).repeat_interleave(H // Hkv, dim=2)
    return oracle


def single_query_step_inputs(Ktrue, Vtrue, t, lps=None):
    """The pointer probe's step: k / v = the keys and values of slot t_b % L; the caches hold, in that slot, another
    key's code and the negated value (the kernel must never read the slot it writes)."""
    B, L = Ktrue.shape[:2]
    ts = [int(lps[b]) if lps is not None else int(t) for b in range(B)]
    K, V = Ktrue.clone(), Vtrue.clone()
    k = torch.stack([Ktrue[b, ts[b] % L] for b in range(B)])
    v = torch.stack([Vtrue[b, ts[b] % L] for b in range(B)])
    for b in range(B):
        s = ts[b] % L
        K[b, s] = Ktrue[b, (s + 1) % L]
        V[b, s] = -Vtrue[b, s]
    return k, v, K, V


# ------------------------------------------------------------------------------------------------ checker
def ulp(x, dtype):
    """One unit in the last place of T at |x| (float64), subnormals included."""
    _, e = torch.frexp(x.abs().to(torch.float64))
    return torch.pow(2.0, (e - 1).clamp(min=EMIN[dtype]) - MANT[dtype]).to(torch.float64)


def violations(got, want, dtype, ulps=1, limit=8):
    """Entries of got [B, S, H, C] that break the probe's rule against want (T values of the rounded oracle): exactly
    +-0 where want is 0, within `ulps` ulp of T elsewhere (0: the same value).  Returns (count, the first `limit` (None:
    all) as (b, i, h, c, got, want))."""
    g, w = got.to(torch.float64), want.to(torch.float64)
    bad = torch.where(w == 0, g != 0, ~((g - w).abs() <= ulps * ulp(w, dtype)))
    n = int(bad.sum())
    if n == 0:
        return 0, []
    idx = bad.nonzero() if limit is None else bad.nonzero()[:limit]
    return n, [tuple(int(v) for v in r) + (float(g[tuple(r)]), float(w[tuple(r)])) for r in idx.tolist()]
