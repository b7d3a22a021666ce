"""CPU checks of attention over a KV cache read in place (b200awq_kv_cache_attention): argument validation that returns
before any device is touched, the workspace bound against every split plan the launcher can pick, and the
de-interleaving of tinychat's FasterTransformer K cache that the GPU tests use to build their float64 reference.

The helpers here (`ft_keys`, `ft_values`, `plan`) are shared with tests/test_kv_cache_attention_gpu.py."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P

SHAPE, ALIGN, DTYPE, WORKSPACE, DEVICE = -1, -3, -4, -6, -8
FT, BTHD = 0, 1
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every case below returns first)
COUNTERS = 4096  # the workspace's counter block at offset 0 (kAttentionCounters u32)
MAX_SMS = 256


# ------------------------------------------------------------------------------------------------ shared helpers
def ft_keys(k_cache, n):
    """Keys 0 .. n - 1 of an FT cache [B, Hkv, D / 8, L, 8] as [B, n, Hkv, D], indexed as oracle/layer_oracle.py
    reads the cache: key j of KV head h is k_cache[b, h][:, j, :] with its D / 8 pieces of 8 in order."""
    B, Hkv, C, _, _ = k_cache.shape
    out = torch.empty(B, n, Hkv, C * 8, dtype=k_cache.dtype, device=k_cache.device)
    for b in range(B):
        for h in range(Hkv):
            out[b, :, h] = k_cache[b, h][:, :n, :].transpose(0, 1).reshape(n, C * 8)
    return out


def ft_values(v_cache, n):
    """Values 0 .. n - 1 of a cache [B, Hkv, L, D] as [B, n, Hkv, D]."""
    return v_cache[:, :, :n].transpose(1, 2)


def max_splits(rows):
    return (192 * 1024 // 4 - rows) // (2 * rows)


def plan(cells, n_tiles, sms, rows):
    """(splits, tiles per split) as splitkv_attention.cu's plan_splits picks them for `rows` packed rows per cell."""
    splits, tps = 1, n_tiles
    if n_tiles < 2 or cells > COUNTERS:
        return splits, tps
    cap = min(n_tiles, -(-sms // cells), max_splits(rows))
    best = n_tiles * -(-cells // sms)
    for sp in range(2, cap + 1):
        t = -(-n_tiles // sp)
        used = -(-n_tiles // t)
        cost = -(-(cells * used) // sms) * t
        if cost < best:
            best, splits, tps = cost, used, t
    return splits, tps


def cells_of(B, Sq, H, Hkv):
    """(cells, packed rows per cell) of a kv_cache_attention launch: row tiles of 128 packed rows x KV heads x batch."""
    R = Sq * (H // Hkv)
    return -(-R // 128) * B * Hkv, min(R, 128)


# ------------------------------------------------------------------------------------------------ ABI validation
def _call(layout=FT, B=1, Sq=17, Sk=4096, L=8192, H=32, Hkv=8, D=128, scale=None, dtype=0, q=A, k=A, v=A, out=A,
          q_st=None, ws=None, ws_bytes=None, causal=1):
    lib = P.lib()
    st = (Sq * H * D, H * D, D) if q_st is None else q_st
    need = lib.b200awq_kv_cache_attention_workspace_bytes(layout, B, Sq, Sk, H, Hkv, D)
    qs = None if st == "null" else (ctypes.c_longlong * 3)(*st)
    return lib.b200awq_kv_cache_attention(q, k, v, out, layout, B, Sq, Sk, L, H, Hkv, D, qs,
                                          ctypes.c_float(D ** -0.5 if scale is None else scale), causal, dtype,
                                          A if ws is None else ws, need if ws_bytes is None else ws_bytes, None)


@pytest.mark.parametrize("kw,code", [
    (dict(layout=2), SHAPE), (dict(layout=-1), SHAPE),
    (dict(Sk=8193, L=8192), SHAPE), (dict(L=0, Sk=0), SHAPE), (dict(Sk=-1), SHAPE), (dict(Sq=-1), SHAPE),
    (dict(B=-1), SHAPE),
    (dict(D=72), SHAPE), (dict(D=96), SHAPE), (dict(D=256), SHAPE),
    (dict(H=32, Hkv=6), SHAPE), (dict(Hkv=0), SHAPE),
    (dict(scale=0.0), SHAPE), (dict(scale=-0.1), SHAPE), (dict(scale=float("inf")), SHAPE),
    (dict(scale=float("nan")), SHAPE),
    (dict(dtype=2), DTYPE),
    (dict(q=None), ALIGN), (dict(k=None), ALIGN), (dict(v=None), ALIGN), (dict(out=None), ALIGN),
    (dict(q=A + 2), ALIGN), (dict(k=A + 8), ALIGN), (dict(v=A + 4), ALIGN), (dict(out=A + 8), ALIGN),
    (dict(q_st=(4096, 4100, 128)), ALIGN), (dict(q_st="null"), ALIGN),
    (dict(ws=A + 4), ALIGN),
    (dict(ws_bytes=16), WORKSPACE), (dict(ws=0, ws_bytes=0, Sq=1, Sk=100000, L=100000), WORKSPACE),
    (dict(ws=0, ws_bytes=64, Sk=128), WORKSPACE),
])
def test_rejected_before_any_device_work(kw, code):
    for layout in (kw["layout"],) if "layout" in kw else (FT, BTHD):
        assert _call(**dict(kw, layout=layout)) == code


@pytest.mark.parametrize("kw", [dict(B=0), dict(Sq=0), dict(B=0, Sq=0, Sk=0)])
def test_empty_calls_are_no_ops(kw):
    """batch == 0 or seqlen_q == 0 returns 0 after validation, before any device work (none is available here)."""
    for layout in (FT, BTHD):
        assert _call(layout=layout, **kw) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
def test_envelope_edges_pass_validation():
    """Shapes at the envelope's edges stop at the device check (B200AWQ_ERR_DEVICE), never at SHAPE / ALIGN /
    WORKSPACE: any seqlen_q, seqlen_k 0 or max_len, Falcon's G = 71."""
    for kw in (dict(Sq=1), dict(Sq=512), dict(Sq=4096, Sk=8192), dict(Sk=0), dict(Sk=8192), dict(Sq=2, H=71, Hkv=1, D=64),
               dict(Sq=100, Sk=10), dict(B=8, Sq=1, Sk=131072, L=131072), dict(causal=0)):
        for layout in (FT, BTHD):
            assert _call(layout=layout, **kw) == DEVICE, (layout, kw)


# ------------------------------------------------------------------------------------------------ workspace bound
def _ws(layout, B, Sq, Sk, H, Hkv, D):
    return P.lib().b200awq_kv_cache_attention_workspace_bytes(layout, B, Sq, Sk, H, Hkv, D)


SHAPES = [(B, Sq, Sk, H, Hkv, D)
          for (H, Hkv, D) in ((32, 8, 128), (28, 4, 128), (14, 2, 64), (8, 1, 128), (64, 1, 64), (4, 4, 64))
          for B in (1, 3)
          for Sq in (1, 17, 65, 129, 512, 1000)
          for Sk in (1, 128, 129, 4100, 131072)]


def test_workspace_bound_covers_every_plan_and_is_zero_exactly_without_splits():
    """For every SM count up to 256 the plan's partials fit the bound; the bound is 0 exactly when no SM count up to
    256 gives a plan of more than one split; both layouts share the bound."""
    for B, Sq, Sk, H, Hkv, D in SHAPES:
        cells, rows = cells_of(B, Sq, H, Hkv)
        n_tiles = -(-Sk // 128)
        bound = _ws(FT, B, Sq, Sk, H, Hkv, D)
        assert bound == _ws(BTHD, B, Sq, Sk, H, Hkv, D)
        worst = max(plan(cells, n_tiles, sms, rows)[0] for sms in range(1, MAX_SMS + 1))
        if worst == 1:
            assert bound == 0, (B, Sq, Sk, H, Hkv, D)
        else:
            assert bound >= COUNTERS * 4 + cells * worst * rows * (D + 2) * 4, (B, Sq, Sk, H, Hkv, D)


def test_workspace_is_zero_outside_the_envelope():
    assert _ws(2, 1, 1, 4096, 32, 8, 128) == 0
    assert _ws(FT, 0, 1, 4096, 32, 8, 128) == 0
    assert _ws(FT, 1, 0, 4096, 32, 8, 128) == 0
    assert _ws(FT, 1, 1, 4096, 32, 8, 72) == 0
    assert _ws(FT, 1, 1, 4096, 32, 6, 128) == 0


# ------------------------------------------------------------------------------------------------ FT de-interleave
def _tinychat_chunk_kv(cache_k, cache_v, xk, xv, start_pos):
    """A restatement of tinychat's chunk-prefill branch (short_forward with chunk_prefilling): the history copied out
    of the caches with permute / transpose + reshape, then the chunk's own k / v appended."""
    bsz, seqlen, Hkv, D = xk.shape
    keys = cache_k[:bsz, :, :, 0:start_pos, :].permute(0, 3, 1, 2, 4).reshape(bsz, start_pos, Hkv, D).contiguous()
    values = cache_v[:bsz, :, 0:start_pos, :].transpose(2, 1).reshape(bsz, start_pos, Hkv, D).contiguous()
    return torch.cat((keys, xk), dim=1), torch.cat((values, xv), dim=1)


def _tinychat_store(cache_k, cache_v, xk, xv, start_pos):
    """The branch's store of the chunk into the decode caches."""
    bsz, seqlen, Hkv, D = xk.shape
    cache_v[:bsz, :, start_pos:start_pos + seqlen, :] = xv.transpose(2, 1)
    cache_k[:bsz, :, :, start_pos:start_pos + seqlen, :] = \
        xk.reshape(bsz, seqlen, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous()


@pytest.mark.parametrize("B,Hkv,D,L,start,seqlen", [(1, 8, 128, 64, 20, 7), (2, 2, 64, 40, 0, 16), (3, 4, 128, 300, 129, 30)])
def test_ft_helpers_agree_with_tinychat_chunk_code(B, Hkv, D, L, start, seqlen):
    g = torch.Generator().manual_seed(B * 100 + start)
    cache_k = torch.randn(B + 1, Hkv, D // 8, L, 8, generator=g)
    cache_v = torch.randn(B + 1, Hkv, L, D, generator=g)
    xk = torch.randn(B, seqlen, Hkv, D, generator=g)
    xv = torch.randn(B, seqlen, Hkv, D, generator=g)
    want_k, want_v = _tinychat_chunk_kv(cache_k, cache_v, xk, xv, start)
    _tinychat_store(cache_k, cache_v, xk, xv, start)
    n = start + seqlen
    assert torch.equal(ft_keys(cache_k[:B], n), want_k)
    assert torch.equal(ft_values(cache_v[:B], n), want_v)
