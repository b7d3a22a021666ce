"""CPU checks of b200awq_rope_kv_store (RoPE of a chunk's q / k with the store of k / v into a KV cache): argument
validation that returns before any device is touched, and the kernel body (llm_awq_b200/csrc/rope_kv_store.cuh, shared
host/device) walked on the CPU by tests/host_harness/rope_kv_store_host.cpp against a numpy restatement of tinychat's
cache stores, in both cache layouts.

The restatement (`tinychat_store`), the poisoned caches and the byte checker (`store_mismatch`) are shared with
tests/test_rope_kv_store_gpu.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import llm_awq_b200 as P

SHAPE, ALIGN, DTYPE, DEVICE = -1, -3, -4, -8
FT, BTHD = 0, 1
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every ABI case below returns first)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
POISON = (float("nan"), float("inf"), -float("inf"), 65504.0, -65504.0)


# ------------------------------------------------------------------------------------------------ shared helpers
def cache_shapes(layout, rows, Hkv, D, L):
    if layout == FT:
        return (rows, Hkv, D // 8, L, 8), (rows, Hkv, L, D)
    return (rows, L, Hkv, D), (rows, L, Hkv, D)


def poisoned(shape, dtype, device="cpu"):
    """A cache filled with NaN, +-inf and +-65504 in turn."""
    pat = torch.tensor(POISON, device=device).to(dtype)
    n = int(np.prod(shape))
    return pat[torch.arange(n, device=device) % len(POISON)].view(shape).clone()


def tinychat_store(layout, k_cache, v_cache, xk, xv, start_pos):
    """tinychat's store of a chunk's rotated k and its v ([B, S, Hkv, D] each) into cache slots [start_pos, start_pos +
    S) of rows [0, B), restated in numpy on the raw 16-bit patterns (so NaNs compare too).  FT: short_forward's
    `cache_v[:bsz, :, start_pos:start_pos + seqlen, :] = xv.transpose(2, 1)` and `cache_k[:bsz, :, :, start_pos:start_pos
    + seqlen, :] = xk.reshape(bsz, seqlen, Hkv, D // 8, 8).permute(0, 2, 3, 1, 4)`; BTHD: long_forward's `cache_k[:bsz,
    start_pos:start_pos + seqlen] = xk` and the same for v.  Arrays are changed in place."""
    B, S, Hkv, D = xk.shape
    if layout == FT:
        v_cache[:B, :, start_pos:start_pos + S, :] = xv.transpose(0, 2, 1, 3)
        k_cache[:B, :, :, start_pos:start_pos + S, :] = xk.reshape(B, S, Hkv, D // 8, 8).transpose(0, 2, 3, 1, 4)
    else:
        k_cache[:B, start_pos:start_pos + S] = xk
        v_cache[:B, start_pos:start_pos + S] = xv


def bits(t):
    """The 16-bit patterns of a tensor as a numpy array (a copy)."""
    return t.detach().cpu().contiguous().view(torch.int16).numpy().copy()


def store_mismatch(got_k, got_v, want_k, want_v):
    """None when both caches hold the expected bits everywhere, else a description of the first difference."""
    for name, got, want in (("k_cache", got_k, want_k), ("v_cache", got_v, want_v)):
        if got.shape != want.shape:
            return f"{name}: shape {got.shape} != {want.shape}"
        bad = np.argwhere(got != want)
        if len(bad):
            return f"{name}: {len(bad)} elements differ, first at {tuple(bad[0])}"
    return None


# ------------------------------------------------------------------------------------------------ ABI validation
def _call(layout=FT, B=1, S=17, H=32, Hkv=8, D=128, L=8192, start=100, dtype=0, qkv=A, freqs=A, k=A, v=A, st=None):
    nh = H + 2 * Hkv
    s = (S * nh * D, nh * D, D) if st is None else st
    strides = None if s == "null" else (ctypes.c_longlong * 3)(*s)
    return P.lib().b200awq_rope_kv_store(qkv, freqs, k, v, layout, B, S, H, Hkv, D, L, start, strides, dtype, None)


@pytest.mark.parametrize("kw,code", [
    (dict(dtype=2), DTYPE), (dict(dtype=-1), DTYPE), (dict(dtype=2, layout=5, qkv=None), DTYPE),
    (dict(layout=2), SHAPE), (dict(layout=-1), SHAPE),
    (dict(B=-1), SHAPE), (dict(S=-1), SHAPE), (dict(H=0), SHAPE), (dict(Hkv=0), SHAPE), (dict(H=32, Hkv=6), SHAPE),
    (dict(D=0), SHAPE), (dict(D=4), SHAPE), (dict(D=12), SHAPE), (dict(D=100), SHAPE), (dict(D=264), SHAPE),
    (dict(L=0, start=0, S=0), SHAPE), (dict(start=-1), SHAPE), (dict(start=8192 - 16, S=17), SHAPE),
    (dict(start=2 ** 31 - 1, S=2, L=2 ** 31 - 1), SHAPE), (dict(D=12, qkv=None), SHAPE),
    (dict(qkv=None), ALIGN), (dict(freqs=None), ALIGN), (dict(k=None), ALIGN), (dict(v=None), ALIGN),
    (dict(qkv=A + 8), ALIGN), (dict(freqs=A + 4), ALIGN), (dict(k=A + 2), ALIGN), (dict(v=A + 8), ALIGN),
    (dict(st=(17 * 48 * 128 + 4, 48 * 128, 128)), ALIGN), (dict(st=(17 * 48 * 128, 48 * 128 + 2, 128)), ALIGN),
    (dict(st=(17 * 48 * 128, 48 * 128, 132)), ALIGN), (dict(st="null"), ALIGN), (dict(st="null", B=0), ALIGN),
])
def test_rejected_before_any_device_work(kw, code):
    for layout in (kw["layout"],) if "layout" in kw else (FT, BTHD):
        assert _call(**dict(kw, layout=layout)) == code, kw


@pytest.mark.parametrize("kw", [dict(B=0), dict(S=0), dict(B=0, S=0), dict(S=0, start=8192)])
def test_empty_calls_are_no_ops(kw):
    """batch == 0 or seqlen == 0 returns 0 after validation, before any device work (none is available here)."""
    for layout in (FT, BTHD):
        assert _call(layout=layout, **kw) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
def test_envelope_edges_pass_validation():
    """Shapes at the envelope's edges stop at the device check, never at SHAPE / ALIGN: head_dim 8, 72 and 256, G = 1
    and Falcon's 71, the last slot of the cache, one token."""
    for kw in (dict(D=8), dict(D=72), dict(D=256), dict(H=8, Hkv=8), dict(H=71, Hkv=1, D=64), dict(start=8192 - 17),
               dict(S=1, start=8191), dict(S=8192, start=0), dict(B=65536, S=1)):
        for layout in (FT, BTHD):
            assert _call(layout=layout, **kw) == DEVICE, (layout, kw)


# ------------------------------------------------------------------------------------------------ host harness
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h")):
        pytest.skip("needs g++ and the CUDA headers")
    so = str(tmp_path_factory.mktemp("rope_kv_store") / "rope_kv_store_host.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I" + CUDA_INC,
                    "-I" + os.path.join(ROOT, "llm_awq_b200", "csrc"),
                    os.path.join(ROOT, "tests", "host_harness", "rope_kv_store_host.cpp"), "-o", so], check=True)
    lib = ctypes.CDLL(so)
    vp, ci, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    lib.rope_kv_store_host.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, ll, ll, ll, ci, ci]
    lib.rope_kv_store_host.restype = ci
    return lib


def host_run(lib, qkv, freqs, kc, vc, layout, H, start, tile_log2=3):
    B, S, nh, D = qkv.shape
    Hkv = (nh - H) // 2
    L = kc.shape[3] if layout == FT else kc.shape[1]
    dt = {torch.float16: 0, torch.bfloat16: 1}[qkv.dtype]
    return lib.rope_kv_store_host(qkv.data_ptr(), freqs.data_ptr(), kc.data_ptr(), vc.data_ptr(), layout, B, S, H, Hkv, D,
                                  L, start, qkv.stride(0), qkv.stride(1), qkv.stride(2), dt, tile_log2)


def padded_qkv(B, S, nh, D, dtype, seed, pad=(0, 0, 0)):
    """[B, S, nh, D] of seeded data as a view with padded head, token and batch strides (pads in elements, multiples
    of 8); the padding holds NaN."""
    g = torch.Generator().manual_seed(seed)
    full = torch.full((B, S + pad[0], nh + pad[1], D + pad[2]), float("nan")).to(dtype)
    view = full[:, :S, :nh, :D]
    view.copy_(torch.randn(B, S, nh, D, generator=g).to(dtype))
    return full, view


def rotate64(x, freqs):
    """fused_rope_with_pos' rotation of x [B, S, h, D] in float64 with angles freqs [S, D]."""
    D = x.shape[-1]
    rot = np.concatenate([-x[..., D // 2:], x[..., :D // 2]], axis=-1)
    f = freqs[None, :, None, :]
    return x * np.cos(f) + rot * np.sin(f)


def ulp_close(got, want64, dtype):
    """One rounding of the fp32 rotation against float64: within 2 ulp of T (the host's sincosf is not the device's)."""
    ulp = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}[dtype]
    g = got.double().numpy()
    return bool(np.all(np.abs(g - want64) <= 2 * ulp * np.maximum(np.abs(want64), 2.0 ** -14) + 1e-6))


HOST_CASES = [  # layout, B, rows, S, start, L, H, Hkv, D
    (FT, 1, 1, 1, 0, 16, 4, 1, 64), (FT, 2, 3, 7, 5, 20, 8, 2, 128), (FT, 2, 3, 17, 3, 24, 4, 4, 64),
    (FT, 1, 2, 9, 0, 9, 6, 2, 72), (FT, 3, 3, 8, 1, 12, 2, 1, 256), (FT, 1, 1, 20, 30, 50, 7, 1, 40),
    (BTHD, 1, 1, 1, 15, 16, 4, 1, 64), (BTHD, 2, 3, 7, 5, 20, 8, 2, 128), (BTHD, 2, 2, 17, 0, 17, 4, 4, 64),
    (BTHD, 1, 2, 9, 3, 16, 6, 2, 72), (BTHD, 3, 4, 8, 1, 12, 2, 1, 256), (BTHD, 1, 1, 3, 2, 8, 3, 1, 24),
]


def _host_case(harness, case, dtype, zero_angles, tile_log2=3, pad=(0, 0, 0)):
    layout, B, rows, S, start, L, H, Hkv, D = case
    nh = H + 2 * Hkv
    _, qkv = padded_qkv(B, S, nh, D, dtype, seed=S * 31 + D + start, pad=pad)
    qkv0 = qkv.clone()
    g = torch.Generator().manual_seed(D + S)
    freqs = torch.zeros(S, D) if zero_angles else (torch.rand(S, D, generator=g) * 12.0 - 6.0)
    ks, vs = cache_shapes(layout, rows, Hkv, D, L)
    kc, vc = poisoned(ks, dtype), poisoned(vs, dtype)
    want_k, want_v = bits(kc), bits(vc)
    used = host_run(harness, qkv, freqs, kc, vc, layout, H, start, tile_log2)
    assert used == (8 if D % 16 == 0 else 4)
    assert torch.equal(qkv[:, :, H:].view(torch.int16), qkv0[:, :, H:].view(torch.int16))  # k and v heads unchanged
    return layout, B, S, start, H, Hkv, D, qkv, qkv0, freqs, kc, vc, want_k, want_v


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", HOST_CASES)
def test_host_walk_zero_angles_is_tinychats_store_exactly(harness, case, dtype):
    """With every angle 0 the rotation is exact: q is unchanged and the caches hold exactly what tinychat's store of the
    raw k / v writes, every other slot and row keeping its poison, bit for bit."""
    layout, B, S, start, H, Hkv, D, qkv, qkv0, _, kc, vc, want_k, want_v = _host_case(harness, case, dtype, True)
    assert torch.equal(qkv.view(torch.int16), qkv0.view(torch.int16))
    xk, xv = bits(qkv0[:, :, H:H + Hkv]), bits(qkv0[:, :, H + Hkv:])
    tinychat_store(layout, want_k, want_v, xk, xv, start)
    assert store_mismatch(bits(kc), bits(vc), want_k, want_v) is None


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", HOST_CASES)
def test_host_walk_random_angles(harness, case, dtype):
    """Random angles whose two halves differ: rotated q and the stored k are the float64 rotation within rounding, v
    is stored exactly, and nothing outside the chunk's slots and rows changes."""
    layout, B, S, start, H, Hkv, D, qkv, qkv0, freqs, kc, vc, want_k, want_v = _host_case(harness, case, dtype, False)
    f = freqs.double().numpy()
    assert ulp_close(qkv[:, :, :H], rotate64(qkv0[:, :, :H].double().numpy(), f), dtype)
    # where the restatement stores: the stored k read back from there, every other element keeps its poison
    mask_k, mask_v = np.zeros(want_k.shape, bool), np.zeros(want_v.shape, bool)
    tinychat_store(layout, mask_k, mask_v, np.ones((B, S, Hkv, D), bool), np.ones((B, S, Hkv, D), bool), start)
    stored = kc.numpy()[mask_k] if dtype == torch.float16 else kc.view(torch.int16).numpy()[mask_k]
    ids = np.zeros(want_k.shape, np.int64)
    tinychat_store(layout, ids, np.zeros(want_v.shape, np.int64), np.arange(B * S * Hkv * D).reshape(B, S, Hkv, D),
                   np.zeros((B, S, Hkv, D), np.int64), start)
    got_k = torch.from_numpy(stored[np.argsort(ids[mask_k])].copy())
    got_k = (got_k if dtype == torch.float16 else got_k.view(torch.bfloat16)).view(B, S, Hkv, D)
    assert ulp_close(got_k, rotate64(qkv0[:, :, H:H + Hkv].double().numpy(), f), dtype)
    assert np.array_equal(bits(kc)[~mask_k], want_k[~mask_k])
    tinychat_store(layout, want_k, want_v, bits(qkv0[:, :, H:H + Hkv]), bits(qkv0[:, :, H + Hkv:]), start)
    assert np.array_equal(bits(vc), want_v)


@pytest.mark.parametrize("tile_log2", [0, 1, 2, 3])
@pytest.mark.parametrize("pad", [(0, 0, 0), (3, 2, 8)], ids=["dense", "padded"])
def test_host_walk_tile_and_strides_do_not_matter(harness, tile_log2, pad):
    """The same bits for every token tile the launcher can pick and for padded token / head strides."""
    case = (FT, 2, 3, 11, 4, 32, 8, 2, 128)
    results = []
    for lg in (3, tile_log2):
        r = _host_case(harness, case, torch.float16, False, tile_log2=lg, pad=pad if lg == tile_log2 else (0, 0, 0))
        results.append((bits(r[7]), bits(r[10]), bits(r[11])))
    for a, b in zip(*results):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ the checker itself
def _wrong_store(layout, k_cache, v_cache, xk, xv, start_pos, defect):
    B, S, Hkv, D = xk.shape
    if defect == "ft_pos_block_swapped":
        # k_cache[b, h, pos, d / 8, d % 8] in a [.., max_len, D / 8, 8] reading of the same bytes
        kv = k_cache.reshape(k_cache.shape[0], Hkv, k_cache.shape[3], D // 8, 8)
        kv[:B, :, start_pos:start_pos + S] = xk.reshape(B, S, Hkv, D // 8, 8).transpose(0, 2, 1, 3, 4)
        v_cache[:B, :, start_pos:start_pos + S, :] = xv.transpose(0, 2, 1, 3)
        return
    assert defect == "one_slot_past_the_end"
    tinychat_store(layout, k_cache, v_cache, xk, xv, start_pos)
    tinychat_store(layout, k_cache, v_cache, xk[:, -1:], xv[:, -1:], start_pos + S)


@pytest.mark.parametrize("layout,defect", [(FT, "ft_pos_block_swapped"), (FT, "one_slot_past_the_end"),
                                           (BTHD, "one_slot_past_the_end")])
def test_checker_flags_wrong_stores(layout, defect):
    B, S, start, L, Hkv, D = 2, 9, 3, 16, 2, 64
    g = np.random.default_rng(5)
    ks, vs = cache_shapes(layout, 3, Hkv, D, L)
    k0, v0 = bits(poisoned(ks, torch.float16)), bits(poisoned(vs, torch.float16))
    xk = g.integers(0, 2 ** 14, (B, S, Hkv, D)).astype(np.int16)
    xv = g.integers(0, 2 ** 14, (B, S, Hkv, D)).astype(np.int16)
    want_k, want_v = k0.copy(), v0.copy()
    tinychat_store(layout, want_k, want_v, xk, xv, start)
    got_k, got_v = k0.copy(), v0.copy()
    tinychat_store(layout, got_k, got_v, xk, xv, start)
    assert store_mismatch(got_k, got_v, want_k, want_v) is None
    got_k, got_v = k0.copy(), v0.copy()
    _wrong_store(layout, got_k, got_v, xk, xv, start, defect)
    assert store_mismatch(got_k, got_v, want_k, want_v) is not None
