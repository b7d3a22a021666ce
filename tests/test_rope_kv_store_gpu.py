"""GPU tests of `awq_inference_engine.rope_kv_store` and its C ABI b200awq_rope_kv_store: RoPE of a chunk's q and k
heads in the fused qkv output, q rotated in place, rotated k and v stored into tinychat's KV caches, one launch.

The yardstick is the composed route this entry replaces: this build's fused_rope_with_pos_forward_func(x.transpose(0,
1), freqs, True) on the q and k heads, one batch row at a time, then tinychat's own stores (`_tinychat_store` of
tests/test_kv_cache_attention_cpu.py for the FT caches, slice assignment for the BTHD caches).  The new entry must
match it bit for bit; caches and outputs are compared as 16-bit patterns, so poisoned NaNs compare too."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from guard_bands import Op, guarded_call, _code, _p, _st
from kernel_trace import trace
from test_kv_cache_attention_cpu import FT, BTHD, _tinychat_chunk_kv, _tinychat_store
from test_rope_kv_store_cpu import cache_shapes, poisoned

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
LAYOUTS = [pytest.param(FT, id="ft"), pytest.param(BTHD, id="bthd")]
MODELS = [pytest.param((32, 8, 128), id="llama3_8b"), pytest.param((28, 4, 128), id="qwen2_7b"),
          pytest.param((14, 2, 64), id="qwen2_0_5b"), pytest.param((8, 8, 128), id="g1"),
          pytest.param((8, 2, 256), id="d256")]
TOL = {torch.float16: 2e-3, torch.bfloat16: 8e-3}


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def precompute_freqs(dim, positions, theta=500000.0):
    """tinychat's precompute_freqs table (tinychat/models/llama.py) restated, rows `positions` only, as [S, D] fp32:
    inverse frequencies theta ** -(2i / dim), angles position * inverse frequency, the two halves equal."""
    inv = 1.0 / (theta ** (torch.arange(0, dim, 2).float() / dim))
    f = torch.einsum("i , j -> i j", positions.float(), inv)
    return torch.cat((f, f), dim=-1).contiguous().to(DEV)


def random_freqs(S, D, seed):
    """Random angles in [-40, 40) whose two halves differ."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(S, D, generator=g, device=DEV) * 80.0 - 40.0


def _rope(eng, x, freqs):
    """x [B, S, h, D] rotated through fused_rope_with_pos_forward_func(..., True) one batch row at a time (its angles
    are per (token, batch row); tinychat's table slice holds one row of angles per token)."""
    return torch.cat([eng.fused_rope_with_pos_forward_func(x[b:b + 1].transpose(0, 1), freqs, True).transpose(0, 1)
                      for b in range(x.shape[0])])


def composed(eng, qkv, freqs, kc, vc, H, Hkv, start):
    """The composed route: rotated q (returned) and tinychat's stores into kc / vc (in place)."""
    B, S = qkv.shape[:2]
    xq, xk = _rope(eng, qkv[:, :, :H], freqs), _rope(eng, qkv[:, :, H:H + Hkv], freqs)
    xv = qkv[:, :, H + Hkv:]
    if kc.dim() == 5:
        _tinychat_store(kc, vc, xk, xv, start)
    else:
        kc[:B, start:start + S] = xk
        vc[:B, start:start + S] = xv
    return xq


def _caches(layout, rows, Hkv, D, L, dtype):
    ks, vs = cache_shapes(layout, rows, Hkv, D, L)
    return poisoned(ks, dtype, DEV), poisoned(vs, dtype, DEV)


def _check_case(eng, qkv, freqs, kc0, vc0, H, Hkv, start):
    """The new entry against the composed route on the same inputs and caches."""
    want_k, want_v = kc0.clone(), vc0.clone()
    want_q = composed(eng, qkv, freqs, want_k, want_v, H, Hkv, start)
    x, kc, vc = qkv.clone(), kc0.clone(), vc0.clone()
    q = eng.rope_kv_store(x, freqs, kc, vc, start)
    assert q.data_ptr() == x.data_ptr() and q.shape == want_q.shape
    assert _same(q, want_q), "rotated q"
    assert _same(kc, want_k) and _same(vc, want_v), "caches"
    assert _same(x[:, :, H:], qkv[:, :, H:]), "k / v heads of qkv changed"


# ------------------------------------------------------------------------------------------------ sweep
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_sweep_matches_composed_route(model, layout, dtype):
    """S in {1, 2, 7, 8, 9, 17, 128, 1000}, start_pos 0, 1, a mid value and max_len - S, batch 1 and 2 of 3 cache rows,
    random angles and tinychat's table at positions up to 131072; poisoned caches."""
    eng = P.engine()
    H, Hkv, D = model
    L = 1100
    kc0, vc0 = _caches(layout, 3, Hkv, D, L, dtype)
    for i, S in enumerate((1, 2, 7, 8, 9, 17, 128, 1000)):
        for start in sorted({0, 1, (L - S) // 2, L - S}):
            for B in (1, 2):
                qkv = _rand((B, S, H + 2 * Hkv, D), dtype, 7 * i + start + B)
                for table in (False, True):
                    if table:
                        freqs = precompute_freqs(D, torch.arange(131072 - L + start, 131072 - L + start + S))
                    else:
                        freqs = random_freqs(S, D, i + start)
                    _check_case(eng, qkv, freqs, kc0, vc0, H, Hkv, start)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("H,Hkv,D", [(4, 1, 72), (6, 2, 8), (71, 1, 64), (3, 1, 40)])
def test_other_head_dims_and_ratios(H, Hkv, D, layout, dtype):
    """head_dim % 16 == 8 (8-byte pieces), head_dim 8, Falcon's G = 71."""
    eng = P.engine()
    L = 64
    kc0, vc0 = _caches(layout, 2, Hkv, D, L, dtype)
    for S, start in ((1, 0), (9, 5), (17, 47), (64, 0)):
        qkv = _rand((2, S, H + 2 * Hkv, D), dtype, S + D)
        _check_case(eng, qkv, random_freqs(S, D, S), kc0, vc0, H, Hkv, start)


# ------------------------------------------------------------------------------------------------ strides and tails
def _abi(v, layout, B, S, H, Hkv, D, L, start, strides, dtype):
    st = (ctypes.c_longlong * 3)(*strides)
    return P.lib().b200awq_rope_kv_store(_p(v["qkv"]), _p(v["freqs"]), _p(v["kc"]), _p(v["vc"]), layout, B, S, H, Hkv, D, L,
                                         start, st, _code(dtype), _st())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("B,S,start,L,H,Hkv,D", [(2, 17, 3, 40, 8, 2, 128), (1, 9, 0, 9, 14, 2, 64), (2, 1, 30, 31, 4, 4, 64),
                                                 (1, 3, 7, 12, 4, 1, 72), (2, 13, 5, 20, 4, 2, 256)])
def test_guard_bands(B, S, start, L, H, Hkv, D, layout, dtype):
    """qkv and both caches (updated in place) and freqs (read only) between guard bands; token counts that are not a
    multiple of the 8-token tile; the plain call's results match the composed route."""
    eng = P.engine()
    nh = H + 2 * Hkv
    qkv = _rand((B, S, nh, D), dtype, S * D + start)
    freqs = random_freqs(S, D, S)
    kc0, vc0 = _caches(layout, B + 1, Hkv, D, L, dtype)
    ops = {"qkv": Op("io", qkv), "freqs": Op("in", freqs), "kc": Op("io", kc0), "vc": Op("io", vc0)}
    strides = (S * nh * D, nh * D, D)
    plain = guarded_call(lambda v: _abi(v, layout, B, S, H, Hkv, D, L, start, strides, dtype), ops)
    want_k, want_v = kc0.clone(), vc0.clone()
    want_q = composed(eng, qkv, freqs, want_k, want_v, H, Hkv, start)
    assert _same(plain["qkv"][:, :, :H], want_q) and _same(plain["qkv"][:, :, H:], qkv[:, :, H:])
    assert _same(plain["kc"], want_k) and _same(plain["vc"], want_v)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_padded_batch_and_token_strides(layout):
    """qkv as a view of a larger buffer (padded token and batch strides): the result equals the dense call's, and the
    padding is not touched."""
    eng = P.engine()
    dtype, B, S, H, Hkv, D, L, start = torch.float16, 2, 19, 8, 2, 128, 64, 11
    nh = H + 2 * Hkv
    big = torch.full((B + 1, S + 5, nh + 1, D), float("nan"), dtype=dtype, device=DEV)
    view = big[:B, :S, :nh]
    view.copy_(_rand((B, S, nh, D), dtype, 3))
    assert view.stride(1) == (nh + 1) * D and view.stride(0) == (S + 5) * (nh + 1) * D
    dense = view.contiguous()
    outside = big.clone()
    outside[:B, :S, :nh] = 0
    freqs = random_freqs(S, D, 4)
    kc0, vc0 = _caches(layout, B, Hkv, D, L, dtype)
    kc, vc, kd, vd = kc0.clone(), vc0.clone(), kc0.clone(), vc0.clone()
    q = eng.rope_kv_store(view, freqs, kc, vc, start)
    qd = eng.rope_kv_store(dense, freqs, kd, vd, start)
    assert _same(q, qd) and _same(kc, kd) and _same(vc, vd)
    after = big.clone()
    after[:B, :S, :nh] = 0
    assert _same(after, outside)


def test_misaligned_pointers_and_strides_are_rejected():
    eng = P.engine()
    dtype, B, S, H, Hkv, D, L = torch.float16, 1, 9, 8, 2, 64, 32
    nh = H + 2 * Hkv
    kc, vc = _caches(FT, B, Hkv, D, L, dtype)
    freqs = random_freqs(S, D, 1)
    flat = _rand((B * S * nh * D + 64,), dtype, 2)
    k0, v0 = kc.clone(), vc.clone()
    for off, tok in ((4, nh * D), (0, nh * D + 4)):
        x = flat.as_strided((B, S, nh, D), (S * tok, tok, D, 1), off)
        with pytest.raises(RuntimeError):
            eng.rope_kv_store(x, freqs, kc, vc, 0)
    misaligned_f = torch.zeros(S * D + 1, device=DEV)[1:]
    with pytest.raises(RuntimeError):
        eng.rope_kv_store(flat[:B * S * nh * D].view(B, S, nh, D), misaligned_f, kc, vc, 0)
    lib = P.lib()
    x = flat[:B * S * nh * D].view(B, S, nh, D)
    ok = (ctypes.c_longlong * 3)(S * nh * D, nh * D, D)
    bad = (ctypes.c_longlong * 3)(S * nh * D, nh * D, D + 4)
    args = lambda q, f, k, v, st: lib.b200awq_rope_kv_store(q, f, k, v, FT, B, S, H, Hkv, D, L, 0, st, 0, _st())  # noqa: E731
    assert args(x.data_ptr() + 8, freqs.data_ptr(), kc.data_ptr(), vc.data_ptr(), ok) == -3
    assert args(x.data_ptr(), freqs.data_ptr() + 4, kc.data_ptr(), vc.data_ptr(), ok) == -3
    assert args(x.data_ptr(), freqs.data_ptr(), kc.data_ptr() + 2, vc.data_ptr(), ok) == -3
    assert args(x.data_ptr(), freqs.data_ptr(), kc.data_ptr(), vc.data_ptr() + 8, ok) == -3
    assert args(x.data_ptr(), freqs.data_ptr(), kc.data_ptr(), vc.data_ptr(), bad) == -3
    torch.cuda.synchronize()
    assert _same(kc, k0) and _same(vc, v0)


# ------------------------------------------------------------------------------------------------ launches
def test_launch_count():
    eng = P.engine()
    dtype, H, Hkv, D, L = torch.float16, 8, 2, 64, 64
    kc, vc = _caches(FT, 2, Hkv, D, L, dtype)
    for B, S, n in ((2, 17, 1), (1, 1, 1), (0, 5, 0), (2, 0, 0)):
        qkv = _rand((B, S, H + 2 * Hkv, D), dtype, 1) if B * S else torch.empty(B, S, H + 2 * Hkv, D, dtype=dtype, device=DEV)
        before = eng.launch_count()
        q = eng.rope_kv_store(qkv, random_freqs(S, D, 2) if S else torch.empty(0, device=DEV), kc, vc, 3)
        assert eng.launch_count() - before == n, (B, S)
        assert q.shape == (B, S, H, D)


def traced_call(B, S, layout):
    """kernel_trace builder: one rope_kv_store call of a chunk, with tinychat's [S, 1, 1, D] freqs slice."""
    H, Hkv, D, L = 32, 8, 128, 2048
    kc, vc = _caches(layout, B, Hkv, D, L, torch.float16)
    qkv = torch.randn(B, S, H + 2 * Hkv, D, device=DEV).half()
    freqs = torch.rand(S, 1, 1, D, device=DEV)
    return lambda: P.engine().rope_kv_store(qkv, freqs, kc, vc, 100)


def test_one_kernel_per_call():
    """Each call runs exactly one kernel, the rope_kv_store kernel, and no copy or fill."""
    cases = {"ft_s17": (1, 17, FT), "ft_s512_b2": (2, 512, FT), "bthd_s1": (1, 1, BTHD), "bthd_s64": (2, 64, BTHD)}
    for name, rec in zip(cases, trace("test_rope_kv_store_gpu:traced_call", cases.values(), per_process=8)):
        assert len(rec.names) == 1 and "rope_kv_store_kernel" in rec.names[0], (name, rec.names)


# ------------------------------------------------------------------------------------------------ tinychat, multi-round
def _unpatched_ft(eng, xqkv, freqs, ck, cv, start, H, Hkv):
    """short_forward's chunk branch as tinychat has it: rope twice, the stores, the history copies, flash_attn_func."""
    xq, xk, xv = _rope(eng, xqkv[:, :, :H], freqs), _rope(eng, xqkv[:, :, H:H + Hkv], freqs), xqkv[:, :, H + Hkv:]
    keys, values = _tinychat_chunk_kv(ck, cv, xk, xv, start)
    _tinychat_store(ck, cv, xk, xv, start)
    return eng.flash_attn_func(xq, keys, values, causal=True)


def _kv_patch(eng, xqkv, freqs, ck, cv, start, H, Hkv):
    """The kv_cache_attention patch (INTEGRATION.md §5): rope twice and the stores in PyTorch, then the cache read in
    place."""
    B, S = xqkv.shape[:2]
    xq = composed(eng, xqkv, freqs, ck, cv, H, Hkv, start)
    return eng.kv_cache_attention(xq, ck[:B], cv[:B], start + S)


def _rope_kv_patch(eng, xqkv, freqs, ck, cv, start):
    """The rope_kv_store patch (INTEGRATION.md §5), both cache layouts."""
    B, S = xqkv.shape[:2]
    xq = eng.rope_kv_store(xqkv, freqs, ck, cv, start)
    return eng.kv_cache_attention(xq, ck[:B], cv[:B], start + S)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Hkv,D", [pytest.param(32, 8, 128, id="llama3_8b"), pytest.param(28, 4, 128, id="qwen2_7b")])
def test_tinychat_multi_round_ft(H, Hkv, D, dtype):
    """short_forward with FT caches: a prefill of 1000 and chunks of 17, 64 and 300 through the three routes, then 5
    decode steps through single_query_attention.  The patched route's caches equal the unpatched route's byte for byte
    and its outputs equal the kv_cache_attention patch's bit for bit, and the unpatched copy + flash_attn_func route's
    within the attention tolerance."""
    eng = P.engine()
    B, L = 2, 1500
    caches = {r: (torch.zeros(B, Hkv, D // 8, L, 8, dtype=dtype, device=DEV), torch.zeros(B, Hkv, L, D, dtype=dtype, device=DEV))
              for r in ("new", "kv", "unpatched")}
    start = 0
    for i, S in enumerate((1000, 17, 64, 300)):
        xqkv = _rand((B, S, H + 2 * Hkv, D), dtype, 60 + i)
        freqs = precompute_freqs(D, torch.arange(start, start + S))
        new = _rope_kv_patch(eng, xqkv.clone(), freqs, *caches["new"], start)
        kv = _kv_patch(eng, xqkv.clone(), freqs, *caches["kv"], start, H, Hkv)
        ref = _unpatched_ft(eng, xqkv.clone(), freqs, *caches["unpatched"], start, H, Hkv)
        assert _same(new, kv), f"chunk {i}"
        for r in ("kv", "unpatched"):
            assert _same(caches["new"][0], caches[r][0]) and _same(caches["new"][1], caches[r][1]), (i, r)
        for b in range(B):
            for h in range(H):
                w = ref[b, :, h].double()
                assert float((new[b, :, h].double() - w).norm()) <= TOL[dtype] * float(w.norm()), (i, b, h)
        start += S
    for step in range(5):  # decode: single_query_attention rotates and stores the step itself
        xqkv = _rand((B, 1, H + 2 * Hkv, D), dtype, 90 + step)
        q, k, v = xqkv[:, 0, :H], xqkv[:, 0, H:H + Hkv], xqkv[:, 0, H + Hkv:]
        outs = [eng.single_query_attention(q, k, v, *caches[r], None, None, start, D, 500000.0, 1.0, True)
                for r in ("new", "unpatched")]
        assert _same(outs[0], outs[1]), f"decode step {step}"
        assert _same(caches["new"][0], caches["unpatched"][0]) and _same(caches["new"][1], caches["unpatched"][1])
        start += 1


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Hkv,D", [pytest.param(32, 8, 128, id="llama3_8b"), pytest.param(14, 2, 64, id="qwen2_0_5b")])
def test_tinychat_multi_round_bthd(H, Hkv, D, dtype):
    """long_forward with [B, Lmax, Hkv, D] caches: a prefill of 9000 in chunks of 4096, 4096 and 808, then 4 decode
    steps of one token, each through the patched route (rope_kv_store + kv_cache_attention), the kv_cache_attention
    patch and the unpatched route (rope twice, the stores, flash_attn_func over the cache views)."""
    eng = P.engine()
    B, L = 1, 9100
    caches = {r: (torch.zeros(B, L, Hkv, D, dtype=dtype, device=DEV), torch.zeros(B, L, Hkv, D, dtype=dtype, device=DEV))
              for r in ("new", "kv", "unpatched")}
    start = 0
    for i, S in enumerate((4096, 4096, 808, 1, 1, 1, 1)):
        xqkv = _rand((B, S, H + 2 * Hkv, D), dtype, 70 + i)
        freqs = precompute_freqs(D, torch.arange(start, start + S))
        new = _rope_kv_patch(eng, xqkv.clone(), freqs, *caches["new"], start)
        kv = _kv_patch(eng, xqkv.clone(), freqs, *caches["kv"], start, H, Hkv)
        ck, cv = caches["unpatched"]
        xq = composed(eng, xqkv.clone(), freqs, ck, cv, H, Hkv, start)
        ref = eng.flash_attn_func(xq, ck[:B, :start + S], cv[:B, :start + S], causal=True)
        assert _same(new, kv), f"step {i}"
        for r in ("kv", "unpatched"):
            assert _same(caches["new"][0], caches[r][0]) and _same(caches["new"][1], caches[r][1]), (i, r)
        for b in range(B):
            for h in range(H):
                w = ref[b, :, h].double()
                assert float((new[b, :, h].double() - w).norm()) <= TOL[dtype] * float(w.norm()), (i, b, h)
        start += S


# ------------------------------------------------------------------------------------------------ graphs, PDL, streams
def _attention_block(eng, x, res, wq, wo, bias, ck, cv, freqs, start, H, Hkv, D):
    """qkv linear with bias -> rope_kv_store -> kv_cache_attention -> o linear with the residual: four launches."""
    B, S, _ = x.shape
    xqkv = eng.w4a16_linear_forward_cuda(x, *wq, 128, bias, None).view(B, S, H + 2 * Hkv, D)
    q = eng.rope_kv_store(xqkv, freqs, ck, cv, start)
    o = eng.kv_cache_attention(q, ck[:B], cv[:B], start + S)
    return eng.w4a16_linear_forward_cuda(o.view(B, S, H * D), *wo, 128, None, res)


@pytest.mark.parametrize("pdl", [True, False], ids=["pdl", "no_pdl"])
def test_graph_stream_and_determinism(pdl):
    """Qwen2-0.5B's attention block of 17 tokens after 100 in the FT caches, captured in a CUDA graph and replayed over
    new inputs: bit-identical to eager calls (outputs and caches), with PDL on and off; repeated eager calls and a call
    on a side stream agree."""
    eng = P.engine()
    dtype, B, S, H, Hkv, D, L, start = torch.float16, 1, 17, 14, 2, 64, 256, 100
    hidden, nqkv = H * D, (H + 2 * Hkv) * D
    wq = gen_layer(nqkv, hidden, dtype, seed=1, device=DEV)
    wo = gen_layer(hidden, hidden, dtype, seed=2, device=DEV)
    bias = _rand((nqkv,), dtype, 3, 0.1)
    ck0 = _rand((B, Hkv, D // 8, L, 8), dtype, 4)
    cv0 = _rand((B, Hkv, L, D), dtype, 5)
    x, res = _rand((B, S, hidden), dtype, 6), _rand((B, S, hidden), dtype, 7)
    freqs = precompute_freqs(D, torch.arange(start, start + S))
    ck, cv = ck0.clone(), cv0.clone()
    prev = eng.set_pdl(pdl)
    try:
        def eager():
            ck.copy_(ck0), cv.copy_(cv0)
            out = _attention_block(eng, x, res, wq, wo, bias, ck, cv, freqs, start, H, Hkv, D)
            torch.cuda.synchronize()
            return out.clone(), ck.clone(), cv.clone()

        first = eager()
        for _ in range(2):
            again = eager()
            assert all(_same(a, b) for a, b in zip(again, first))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ck.copy_(ck0), cv.copy_(cv0)
            on_side = _attention_block(eng, x, res, wq, wo, bias, ck, cv, freqs, start, H, Hkv, D)
        side.synchronize()
        assert _same(on_side, first[0]) and _same(ck, first[1]) and _same(cv, first[2])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _attention_block(eng, x, res, wq, wo, bias, ck, cv, freqs, start, H, Hkv, D)  # warm-up on the capture stream
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            out = _attention_block(eng, x, res, wq, wo, bias, ck, cv, freqs, start, H, Hkv, D)
        for seed in (11, 12, 13):
            x.copy_(_rand((B, S, hidden), dtype, seed))
            res.copy_(_rand((B, S, hidden), dtype, seed + 100))
            ck.copy_(ck0), cv.copy_(cv0)
            gr.replay()
            torch.cuda.synchronize()
            got = (out.clone(), ck.clone(), cv.clone())
            want = eager()
            assert all(_same(a, b) for a, b in zip(got, want)), seed
    finally:
        eng.set_pdl(prev)


# ------------------------------------------------------------------------------------------------ rejected inputs
@pytest.mark.parametrize("what", ["fp32", "dtype_mix", "device_mix", "past_max_len", "negative_start", "batch", "d_not_8",
                                  "ratio", "freqs_size", "freqs_dtype", "freqs_noncontiguous", "cpu_tensor", "few_heads",
                                  "qkv_last_dim_strided", "v_shape"])
def test_rejected_inputs_raise(what):
    eng = P.engine()
    dtype, B, S, H, Hkv, D, L = torch.float16, 1, 5, 8, 2, 64, 32
    qkv = _rand((B, S, H + 2 * Hkv, D), dtype, 1)
    kc, vc = _caches(FT, B, Hkv, D, L, dtype)
    freqs = random_freqs(S, D, 1)
    args = [qkv, freqs, kc, vc, 3]
    if what == "fp32":
        args[0], args[2], args[3] = qkv.float(), kc.float(), vc.float()
    elif what == "dtype_mix":
        args[2] = kc.bfloat16()
    elif what == "device_mix":
        args[1] = freqs.cpu()
    elif what == "past_max_len":
        args[4] = L - S + 1
    elif what == "negative_start":
        args[4] = -1
    elif what == "batch":
        args[0] = _rand((B + 1, S, H + 2 * Hkv, D), dtype, 1)
    elif what == "d_not_8":
        args[0] = _rand((B, S, H + 2 * Hkv, 12), dtype, 1)
        args[1] = random_freqs(S, 12, 1)
        args[2], args[3] = _caches(BTHD, B, Hkv, 12, L, dtype)
    elif what == "ratio":
        args[0] = _rand((B, S, 7 + 2 * Hkv, D), dtype, 1)
    elif what == "freqs_size":
        args[1] = random_freqs(S + 1, D, 1)
    elif what == "freqs_dtype":
        args[1] = freqs.half()
    elif what == "freqs_noncontiguous":
        args[1] = random_freqs(D, S, 1).t()
    elif what == "cpu_tensor":
        args[0] = qkv.cpu()
    elif what == "few_heads":
        args[0] = _rand((B, S, 2 * Hkv, D), dtype, 1)
    elif what == "qkv_last_dim_strided":
        args[0] = _rand((B, S, H + 2 * Hkv, 2 * D), dtype, 1)[..., ::2]
    else:
        args[3] = vc[:, :, :L - 1].contiguous()
    k0, v0 = kc.clone(), vc.clone()
    with pytest.raises(RuntimeError):
        eng.rope_kv_store(*args)
    torch.cuda.synchronize()
    assert _same(kc, k0) and _same(vc, v0)
