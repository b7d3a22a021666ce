"""Which return code wins when a C entry gets two bad arguments at once.  Every call here returns before any launch:
it is rejected by argument validation, or it is an empty call.  The cases marked `dev` are decided by where the device
check sits among the argument checks; with a device they would get past it on stand-in pointers, so they run only
without one.  Single defects per entry are covered by the per-entry CPU tests."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P

SHAPE, GROUP, ALIGN, DTYPE, BATCH, WORKSPACE, DEVICE = -1, -2, -3, -4, -5, -6, -8
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced)
HAVE_GPU = torch.cuda.is_available()


def _strides(*s):
    return (ctypes.c_longlong * 3)(*s)


def gemv(m=1, n=4096, k=4096, group=128, dtype=0, x=A, qw=A, s=A, z=A, y=A):
    return P.lib().b200awq_w4a16_gemv(x, qw, s, z, y, m, n, k, group, dtype, None)


def gemm(m=64, n=4096, k=4096, group=128, dtype=0, x=A, qw=A, s=A, z=A, y=A):
    return P.lib().b200awq_w4a16_gemm(x, qw, s, z, y, m, n, k, group, dtype, None, 0, None)


def linear(m=1, n=4096, k=4096, group=128, dtype=0, x=A, qw=A, s=A, z=A, bias=A, res=A, y=A):
    return P.lib().b200awq_w4a16_linear(x, qw, s, z, bias, res, y, m, n, k, group, dtype, None)


def gemv_allreduce(m=1, n=4096, k=4096, group=128, dtype=0, x=A, qw=A, s=A, z=A, y=A):
    return P.lib().b200awq_w4a16_gemv_allreduce(x, qw, s, z, y, m, n, k, group, dtype, None, None)


def mlp_front(m=2, n=14336, k=4096, group=128, dtype=0, x=A, gq=A, gs=A, gz=A, uq=A, us=A, uz=A, y=A, ws=A,
              ws_bytes=None):
    lib = P.lib()
    need = lib.b200awq_w4a16_mlp_front_workspace_bytes(m, n, k) if ws_bytes is None else ws_bytes
    return lib.b200awq_w4a16_mlp_front(x, gq, gs, gz, uq, us, uz, y, m, n, k, group, dtype, ws, need, None)


def prefill(B=1, Sq=64, Sk=64, H=32, Hkv=8, D=128, scale=0.1, dtype=0, q=A, out=A, cu_q=None, cu_k=None, qs=None):
    st = _strides(Sq * H * D, H * D, D) if qs is None else _strides(*qs)
    kst = _strides(Sk * Hkv * D, Hkv * D, D)
    return P.lib().b200awq_prefill_attention(q, A, A, out, cu_q, cu_k, B, Sq, Sk, H, Hkv, D, st, kst, kst,
                                             ctypes.c_float(scale), 1, dtype, None)


def splitkv(B=1, Sq=1, Sk=4096, H=32, Hkv=8, D=128, scale=0.1, dtype=0, q=A, out=A, qs=None, ws=A, ws_bytes=None):
    lib = P.lib()
    st = _strides(Sq * H * D, H * D, D) if qs is None else _strides(*qs)
    kst = _strides(Sk * Hkv * D, Hkv * D, D)
    need = lib.b200awq_splitkv_attention_workspace_bytes(B, Sq, Sk, H, Hkv, D) if ws_bytes is None else ws_bytes
    return lib.b200awq_splitkv_attention(q, A, A, out, B, Sq, Sk, H, Hkv, D, st, kst, kst, ctypes.c_float(scale), 1,
                                         dtype, ws, need, None)


def kv_cache(layout=0, B=1, Sq=17, Sk=4096, L=8192, H=32, Hkv=8, D=128, scale=0.1, dtype=0, q=A, out=A, qs=None, ws=A,
             ws_bytes=None):
    lib = P.lib()
    st = _strides(Sq * H * D, H * D, D) if qs is None else _strides(*qs)
    need = (lib.b200awq_kv_cache_attention_workspace_bytes(layout, B, Sq, Sk, H, Hkv, D) if ws_bytes is None
            else ws_bytes)
    return lib.b200awq_kv_cache_attention(q, A, A, out, layout, B, Sq, Sk, L, H, Hkv, D, st, ctypes.c_float(scale), 1,
                                          dtype, ws, need, None)


BAD_QS = (4096 * 128, 4096, 132)  # a stride that is not a multiple of 8 elements

CASES = [
    # (entry, two defects, winning code, decided by the device check's position)
    (gemv, dict(dtype=2, x=None), DTYPE, False),
    (gemv, dict(group=64, m=0), GROUP, False),
    (gemv, dict(n=4100, x=A + 2), SHAPE, False),
    (gemv, dict(k=0, y=None), SHAPE, False),
    (gemv, dict(m=8, x=None), ALIGN, False),            # pointers before the batch envelope
    (gemv, dict(m=8), DEVICE, True),                    # the device before the batch envelope
    (gemm, dict(dtype=2, group=64), DTYPE, False),
    (gemm, dict(group=64, k=100), GROUP, False),
    (gemm, dict(m=0, qw=None), SHAPE, False),
    (gemm, dict(n=4100, z=A + 8), SHAPE, False),
    (gemm, dict(n=520, s=None), ALIGN, False),          # pointers before n % 128
    (gemm, dict(n=520), DEVICE, True),                  # the device before n % 128
    (linear, dict(dtype=2, bias=A + 2), DTYPE, False),
    (linear, dict(k=0, res=A + 4), SHAPE, False),
    (linear, dict(x=None, bias=A + 2), ALIGN, False),
    (linear, dict(m=8, n=520, bias=A + 2), ALIGN, False),  # bias / residual before the GEMM envelope ...
    (linear, dict(m=8, n=520, res=None), SHAPE, False),    # ... and the GEMM envelope before the device
    (gemv_allreduce, dict(dtype=2, x=None), DTYPE, False),
    (gemv_allreduce, dict(x=None, m=9), ALIGN, False),
    (gemv_allreduce, dict(m=9), DEVICE, True),          # the device before the batch and the peers
    (mlp_front, dict(dtype=2, uq=None), DTYPE, False),
    (mlp_front, dict(m=0, uq=None), SHAPE, False),
    (mlp_front, dict(gq=None, uq=None), ALIGN, False),
    (mlp_front, dict(uq=None, m=8, n=520), DEVICE, True),  # the device before the up weights and n % 128
    (mlp_front, dict(ws=None, ws_bytes=0, us=A + 2), DEVICE, True),  # ... and before the workspace
    (prefill, dict(dtype=2, q=None), DTYPE, False),
    (prefill, dict(dtype=2, D=96), DTYPE, False),
    (prefill, dict(D=96, qs=BAD_QS), SHAPE, False),
    (prefill, dict(scale=0.0, q=None), SHAPE, False),
    (prefill, dict(Hkv=0, cu_q=A), SHAPE, False),
    (prefill, dict(cu_q=A, qs=BAD_QS), ALIGN, False),
    (prefill, dict(B=0, D=96), SHAPE, False),           # an empty call is validated all the same
    (prefill, dict(B=0, out=A + 2), ALIGN, False),
    (splitkv, dict(dtype=2, q=None), DTYPE, False),
    (splitkv, dict(Sq=17, qs=BAD_QS), SHAPE, False),    # Sq * G = 68 > 64
    (splitkv, dict(Hkv=0, ws_bytes=16), SHAPE, False),
    (splitkv, dict(D=72, ws=A + 4), SHAPE, False),
    (splitkv, dict(qs=BAD_QS, ws_bytes=16), ALIGN, False),
    (splitkv, dict(ws=A + 4, ws_bytes=16), ALIGN, False),
    (splitkv, dict(B=0, ws=None, ws_bytes=64), WORKSPACE, False),
    (kv_cache, dict(dtype=2, layout=2), DTYPE, False),
    (kv_cache, dict(layout=2, q=None), SHAPE, False),
    (kv_cache, dict(Sk=8193, qs=BAD_QS), SHAPE, False),
    (kv_cache, dict(Hkv=0, ws_bytes=16), SHAPE, False),
    (kv_cache, dict(qs=BAD_QS, ws_bytes=16), ALIGN, False),
    (kv_cache, dict(ws=A + 4, ws_bytes=16), ALIGN, False),
    (kv_cache, dict(B=0, ws=None, ws_bytes=64), WORKSPACE, False),
    (kv_cache, dict(Sq=0, D=96), SHAPE, False),
]


@pytest.mark.parametrize("entry,kw,code,dev", CASES, ids=[f"{c[0].__name__}-{i}" for i, c in enumerate(CASES)])
def test_precedence_of_two_defects(entry, kw, code, dev):
    if dev and HAVE_GPU:
        pytest.skip("with a device this call would get past the device check on stand-in pointers")
    before = P.lib().b200awq_launch_count()
    assert entry(**kw) == code
    assert P.lib().b200awq_launch_count() == before


@pytest.mark.parametrize("entry,kw", [(prefill, {}), (splitkv, {}), (kv_cache, dict(layout=0)), (kv_cache, dict(layout=1))])
@pytest.mark.parametrize("empty", [dict(B=0), dict(Sq=0)])
def test_empty_calls(entry, kw, empty):
    """An empty call launches nothing.  The two flash-attn entries check the device first, so without one they return
    B200AWQ_ERR_DEVICE; kv_cache_attention returns 0 before the device check."""
    kw = dict(kw, **empty)
    before = P.lib().b200awq_launch_count()
    assert entry(**kw) == (0 if HAVE_GPU or entry is kv_cache else DEVICE)
    assert P.lib().b200awq_launch_count() == before
