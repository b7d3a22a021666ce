"""CPU checks of the known-answer attention probes of tests/attention_exact.py: the float64 oracles, rounded to T, pass
the checker; outputs with one injected defect each are rejected; the pointer construction returns V[target] bit for
bit through the oracles."""
import pytest
import torch

import attention_exact as AE
import prefill_attention_oracle as PO

DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
NAME = {torch.float16: "f16", torch.bfloat16: "bf16"}


def _prefill_oracle(q, K, causal, scale):
    return lambda V: PO.prefill_attention_torch(q, K, V, causal, scale)


def _probe(oracle, w, n_keys, D, dtype, past=0):
    """(want, exact) over all probe blocks, side by side: [B, S, H, blocks * D]."""
    blocks = AE.all_blocks(n_keys, D, past)
    res = list(AE.visibility_expected(oracle, w, n_keys, D, blocks, dtype))
    assert [r[0] for r in res] == blocks
    return torch.cat([r[1] for r in res], -1), torch.cat([r[2] for r in res], -1)


def _fixed_case(causal, Sq=40, Sk=300, B=2, H=4, Hkv=2, D=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(B, Sq, H, D, dtype=torch.float64)
    K = AE.random_keys(B, Sk, Hkv, D, g)
    return q, K, AE.weights(B, Hkv)


def _kernel_like(exact, w, kv_of_head, dtype):
    """What a kernel computes from the probe: w / n in fp32 for each visible key, then rounded to T."""
    n = (exact != 0).sum(-1, keepdim=True).clamp(min=1).to(torch.float32)
    ww = w[:, kv_of_head].to(torch.float32).unsqueeze(1).unsqueeze(-1)
    return torch.where(exact != 0, ww / n, torch.zeros((), dtype=torch.float32)).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Sq,Sk,causal", [(40, 300, True), (40, 300, False), (300, 40, True), (128, 129, True)])
def test_oracle_passes_checker(Sq, Sk, causal, dtype):
    """Every visible key shows up once per row, as w / n_i; a kernel's fp32 w / n rounded to T is within the one ulp."""
    H, Hkv, D = 4, 2, 64
    q, K, w = _fixed_case(causal, Sq, Sk, H=H, Hkv=Hkv, D=D)
    want, exact = _probe(_prefill_oracle(q, K, causal, D ** -0.5), w, Sk, D, dtype)
    assert AE.violations(want, want, dtype) == (0, [])
    kv = torch.arange(H) // (H // Hkv)
    assert AE.violations(_kernel_like(exact, w, kv, dtype), want, dtype)[0] == 0
    n = (exact != 0).sum(-1)
    assert int(n.max()) <= Sk and (exact.sum(-1)[n > 0] / w[:, kv].unsqueeze(1).expand_as(n)[n > 0] - 1).abs().max() < 1e-12
    if causal and Sq > Sk:
        assert int(n[:, :Sq - Sk].sum()) == 0 and int((exact[:, :Sq - Sk] != 0).sum()) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_query_oracle_passes_checker(dtype):
    """Wrapped ring, per-sample lengths (one row before the wrap): every slot the step attends to shows up once."""
    B, H, Hkv, D, L = 2, 6, 2, 64, 150
    lps = [70, 400]
    g = torch.Generator().manual_seed(1)
    K = AE.random_keys(B, L, Hkv, D, g)
    k = AE.random_keys(B, 1, Hkv, D, g)[:, 0]
    w = AE.weights(B, Hkv)
    want, exact = _probe(AE.single_query_visibility_oracle(k, K, 0, D, H, NAME[dtype], lps), w, L, D, dtype)
    n = (exact != 0).sum(-1)
    assert n[0].unique().tolist() == [lps[0] + 1] and n[1].unique().tolist() == [L]
    kv = torch.arange(H) // (H // Hkv)
    assert AE.violations(_kernel_like(exact, w, kv, dtype), want, dtype)[0] == 0


# ------------------------------------------------------------------------------------------------ injected defects
def _rejects(fake, want, dtype):
    n, rep = AE.violations(fake, want, dtype)
    assert n > 0 and rep, "defect not reported"
    return rep


@pytest.mark.parametrize("dtype", DTYPES)
def test_rejects_row_seeing_horizon_plus_one(dtype):
    """Row i of a causal chunk sees one key more: exactly what row i + 1 sees."""
    q, K, w = _fixed_case(True)
    want, _ = _probe(_prefill_oracle(q, K, True, 0.125), w, 300, 64, dtype)
    fake = want.clone()
    fake[1, 17] = want[1, 18]
    rep = _rejects(fake, want, dtype)
    assert {r[:2] for r in rep} == {(1, 17)}


def _drop_or_repeat(K, V, j, repeat):
    """Key j removed, or present twice."""
    idx = list(range(j)) + [j] * (2 if repeat else 0) + list(range(j + 1, K.shape[1]))
    return K[:, idx], V[:, idx]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("key,repeat", [(64 + 128, False), (256, True), (128, True)], ids=["missed_mid_tile", "twice_256", "twice_128"])
def test_rejects_missed_or_repeated_key(key, repeat, dtype):
    """One row misses a key in the middle of a tile, or counts a key at a tile (split) boundary twice."""
    D, Sk = 64, 300
    q, K, w = _fixed_case(False, Sk=Sk, D=D)
    oracle = _prefill_oracle(q, K, False, D ** -0.5)
    want, _ = _probe(oracle, w, Sk, D, dtype)
    Vall = torch.cat([AE.visibility_values(w, Sk, D, b) for b in AE.all_blocks(Sk, D)], -1)
    K2, V2 = _drop_or_repeat(K, Vall, key, repeat)
    bad = PO.prefill_attention_torch(q, K2, V2, False, D ** -0.5).to(dtype)
    fake = want.clone()
    fake[0, 5] = bad[0, 5]
    n, rep = AE.violations(fake, want, dtype, limit=None)
    assert n > 0 and {r[:2] for r in rep} == {(0, 5)}
    assert any(r[3] == key for r in rep)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rejects_head_reading_neighbour_kv_head(dtype):
    q, K, w = _fixed_case(True, H=4, Hkv=2)
    want, _ = _probe(_prefill_oracle(q, K, True, 0.125), w, 300, 64, dtype)
    fake = want.clone()
    fake[:, :, 1] = want[:, :, 2]  # head 1 (KV head 0) with KV head 1's values
    assert {r[2] for r in _rejects(fake, want, dtype)} == {1}


def _pointer_case(B, Sq, Sk, H, Hkv, D, causal, seed, counts=False):
    g = torch.Generator().manual_seed(seed)
    nbits = AE.code_bits(Sk)
    K = AE.pointer_keys(B, Sk, Hkv, D, nbits, g)
    V = AE.pointer_values(B, Sk, Hkv, D, g)
    w = AE.weights(B, Hkv)
    q0 = torch.zeros(B, Sq, H, D, dtype=torch.float64)
    _, exact = _probe(_prefill_oracle(q0, K, causal, 1.0), w, Sk, D, torch.float16)
    targets = AE.choose_targets(exact[..., :Sk] != 0, seed)
    res = AE.pointer_queries(targets, Hkv, D, nbits, 16.0), K, V, targets
    return res + ((exact != 0).sum(-1),) if counts else res


@pytest.mark.parametrize("dtype", DTYPES)
def test_rejects_batch_row_reading_neighbours_k(dtype):
    B, Sq, Sk, H, Hkv, D = 2, 20, 300, 4, 2, 64
    q, K, V, _ = _pointer_case(B, Sq, Sk, H, Hkv, D, True, 3)
    want = PO.prefill_attention_torch(q, K, V, True, 1.0).to(dtype)
    K2 = K.clone()
    K2[0] = K[1]
    fake = want.clone()
    fake[0] = PO.prefill_attention_torch(q, K2, V, True, 1.0).to(dtype)[0]
    n, rep = AE.violations(fake, want, dtype, ulps=0)
    assert n > 0 and {r[0] for r in rep} == {0}


@pytest.mark.parametrize("dtype", DTYPES)
def test_rejects_packed_row_written_to_neighbouring_head(dtype):
    B, Sq, Sk, H, Hkv, D = 1, 16, 300, 8, 2, 64
    q, K, V, _ = _pointer_case(B, Sq, Sk, H, Hkv, D, True, 4)
    want = PO.prefill_attention_torch(q, K, V, True, 1.0).to(dtype)
    fake = want.clone()
    fake[0, 9, 3] = want[0, 9, 2]
    n, rep = AE.violations(fake, want, dtype, ulps=0)
    assert n > 0 and {r[:3] for r in rep} == {(0, 9, 3)}


# ------------------------------------------------------------------------------------------------ pointer construction
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,Sq,Sk,H,Hkv,D,causal", [(2, 40, 300, 14, 2, 64, True), (2, 300, 40, 4, 2, 64, True),
                                                    (1, 8, 1100, 5, 1, 128, False), (2, 3, 129, 8, 2, 72, True)])
def test_pointer_returns_target_value(B, Sq, Sk, H, Hkv, D, causal, dtype):
    """Through the float64 oracle, rounded to T: V[b, target, h // G] bit for bit, 0 for rows that see no key."""
    q, K, V, targets, n = _pointer_case(B, Sq, Sk, H, Hkv, D, causal, Sq + Sk, counts=True)
    got = PO.prefill_attention_torch(q, K, V, causal, 1.0).to(dtype)
    assert torch.equal(got, AE.gather_targets(V, targets, Hkv).to(dtype))
    assert bool((targets >= 0).any())
    if causal and Sq > Sk:
        assert bool((targets[:, :Sq - Sk] < 0).all()) and bool((targets[:, Sq - Sk:] >= 0).all())
    # the G heads of a row pick different keys wherever the row sees enough of them
    G = H // Hkv
    for b, i, hk in ((b, i, hk) for b in range(B) for i in range(Sq) for hk in range(Hkv)):
        if int(n[b, i, hk * G]) >= 16:
            assert len(set(targets[b, i, hk * G:(hk + 1) * G].tolist())) >= min(G, 5), (b, i, hk)


@pytest.mark.parametrize("dtype", DTYPES)
def test_pointer_varlen_returns_target_value(dtype):
    lengths = [0, 1, 127, 128, 129, 300]
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    T, H, D = cu[-1], 3, 64
    g = torch.Generator().manual_seed(7)
    nbits = AE.code_bits(T)
    K = AE.pointer_keys(1, T, H, D, nbits, g)
    V = AE.pointer_values(1, T, H, D, g)
    w = AE.weights(1, H)
    def orc(q, V_):  # the packed oracle returns D channels: one probe block per call
        return torch.cat([torch.from_numpy(PO.prefill_attention(q[0], K[0], V_[0, ..., c:c + D], True, 1.0, cu_seqlens=cu))
                          for c in range(0, V_.shape[-1], D)], -1).unsqueeze(0)
    q0 = torch.zeros(1, T, H, D, dtype=torch.float64)
    _, exact = _probe(lambda V_: orc(q0, V_), w, T, D, dtype)
    vis = exact[..., :T] != 0
    for s in range(len(lengths)):  # no row sees a key of another sequence
        rows = slice(cu[s], cu[s + 1])
        assert not bool(vis[0, rows, :, :cu[s]].any()) and not bool(vis[0, rows, :, cu[s + 1]:].any())
    targets = AE.choose_targets(vis, 7)
    q = AE.pointer_queries(targets, H, D, nbits, 16.0)
    assert torch.equal(orc(q, V).to(dtype), AE.gather_targets(V, targets, H).to(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D,t,lps", [(64, 90, None), (128, 260, None), (48, 0, [0, 3, 330])])
def test_pointer_single_query_returns_target_value(D, t, lps, dtype):
    """single_query_attention's oracle with the stale slot: the step's own value when the target is the current
    position, V[target] otherwise (ring of 200 slots: 260 and 330 wrap)."""
    B, H, Hkv, L = (2, 14, 2, 200) if lps is None else (3, 4, 1, 200)
    g = torch.Generator().manual_seed(D + t)
    nbits = AE.code_bits(L)
    Kt = AE.pointer_keys(B, L, Hkv, D, nbits, g)
    Vt = AE.pointer_values(B, L, Hkv, D, g)
    kin = AE.random_keys(B, 1, Hkv, D, g)[:, 0]
    _, exact = _probe(AE.single_query_visibility_oracle(kin, Kt, t, D, H, NAME[dtype], lps), AE.weights(B, Hkv), L, D,
                      dtype)
    targets = AE.choose_targets(exact[..., :L] != 0, D)
    assert bool((targets >= 0).all())
    k, v, K, V = AE.single_query_step_inputs(Kt, Vt, t, lps)
    q = AE.pointer_queries(targets, Hkv, D, nbits, float(round(16 * D ** 0.5)))[:, 0]
    got = AE.single_query_step(q, k, v, K, V, t, 0, NAME[dtype], lps).to(dtype)
    assert torch.equal(got, AE.gather_targets(Vt, targets, Hkv).to(dtype))
