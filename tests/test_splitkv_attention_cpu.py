"""CPU checks of the split-key attention entry (b200awq_splitkv_attention): argument validation that returns before any
device is touched, and the workspace bound."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P

SHAPE, ALIGN, DTYPE, WORKSPACE, DEVICE = -1, -3, -4, -6, -8
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every case below is rejected first)


def _call(B=1, Sq=1, Sk=4096, H=32, Hkv=8, D=128, scale=None, dtype=0, q=A, k=A, v=A, out=A, q_st=None, ws=None,
          ws_bytes=None):
    lib = P.lib()
    st = (Sq * H * D, H * D, D) if q_st is None else q_st
    kst = (Sk * Hkv * D, Hkv * D, D)
    need = lib.b200awq_splitkv_attention_workspace_bytes(B, Sq, Sk, H, Hkv, D)
    arr = lambda s: (ctypes.c_longlong * 3)(*s)
    return lib.b200awq_splitkv_attention(q, k, v, out, B, Sq, Sk, H, Hkv, D, arr(st), arr(kst), arr(kst),
                                         ctypes.c_float(D ** -0.5 if scale is None else scale), 1, dtype,
                                         A if ws is None else ws, need if ws_bytes is None else ws_bytes, None)


@pytest.mark.parametrize("kw,code", [
    (dict(D=72), SHAPE), (dict(D=96), SHAPE), (dict(D=256), SHAPE),
    (dict(Sq=17, H=32, Hkv=8), SHAPE),            # Sq * G = 68 > 64
    (dict(Sq=2, H=71, Hkv=1, D=64), SHAPE),       # Falcon's G = 71
    (dict(H=32, Hkv=6), SHAPE),                   # uneven head ratio
    (dict(scale=0.0), SHAPE), (dict(scale=-0.1), SHAPE), (dict(scale=float("inf")), SHAPE),
    (dict(scale=float("nan")), SHAPE),
    (dict(dtype=2), DTYPE),
    (dict(q=A + 2), ALIGN), (dict(k=A + 8), ALIGN), (dict(out=None), ALIGN),
    (dict(q_st=(4096, 4100, 132)), ALIGN),        # strides must be multiples of 8 elements
    (dict(ws=A + 4), ALIGN),
    (dict(ws_bytes=16), WORKSPACE), (dict(ws=0, ws_bytes=0, Sk=100000), WORKSPACE),
])
def test_rejected_before_any_device_work(kw, code):
    assert _call(**kw) == code


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
def test_envelope_edges_are_accepted_by_validation():
    """Shapes at the envelope's edges pass validation and stop at the device check (B200AWQ_ERR_DEVICE), never at
    SHAPE / ALIGN / WORKSPACE.  Only without a device: the addresses are stand-ins (the GPU tests run these shapes)."""
    for kw in (dict(Sq=16, H=32, Hkv=8), dict(Sq=64, H=4, Hkv=4, D=64), dict(Sq=1, H=64, Hkv=1), dict(Sk=1),
               dict(Sk=131072, B=8)):
        assert _call(**kw) == DEVICE, kw


def _ws(B, Sq, Sk, H, Hkv, D):
    return P.lib().b200awq_splitkv_attention_workspace_bytes(B, Sq, Sk, H, Hkv, D)


def test_workspace_is_zero_outside_the_envelope_and_for_one_tile():
    assert _ws(1, 1, 128, 32, 8, 128) == 0          # one key tile: always one split, written directly
    assert _ws(1, 1, 1, 32, 8, 128) == 0
    assert _ws(1, 17, 4096, 32, 8, 128) == 0        # Sq * G > 64
    assert _ws(1, 1, 4096, 32, 8, 72) == 0
    assert _ws(0, 1, 4096, 32, 8, 128) == 0
    assert _ws(1, 1, 129, 32, 8, 128) > 0
    # more (batch, KV head) cells than the counter block holds: always one split, written directly
    assert _ws(512, 1, 4096, 32, 8, 128) > 0 and _ws(513, 1, 4096, 32, 8, 128) == 0


def test_workspace_is_monotone():
    """Within the shapes that can split (at most 4096 (batch, KV head) cells, the counter block's size)."""
    base = dict(B=1, Sq=1, Sk=16384, H=32, Hkv=8, D=128)
    sweeps = {"B": [1, 2, 3, 5, 8, 16, 64, 511, 512], "Sq": [1, 2, 3, 4, 8], "Sk": [129, 256, 1000, 4100, 16384, 131072, 1 << 20],
              "H": [8, 16, 24, 32, 64], "D": [64, 128]}
    for name, values in sweeps.items():
        sizes = [_ws(**dict(base, **{name: x})) for x in values]
        assert sizes == sorted(sizes), (name, sizes)


@pytest.mark.parametrize("B,Sq,Sk,H,Hkv,D", [(1, 1, 16384, 32, 8, 128), (8, 1, 32768, 32, 8, 128), (1, 1, 131072, 14, 2, 64),
                                             (1, 8, 16384, 32, 8, 128), (3, 64, 4100, 1, 1, 64), (1, 1, 1 << 20, 64, 1, 128),
                                             (4096, 1, 4096, 8, 1, 128)])
def test_workspace_covers_the_largest_split_count(B, Sq, Sk, H, Hkv, D):
    """The split rule takes at most ceil(sms / cells) splits of at least one 128-key tile, for any SM count up to 256:
    the workspace must hold the counters and the partials of the largest such plan."""
    cells, tiles, rows = B * Hkv, -(-Sk // 128), Sq * (H // Hkv)
    assert cells <= 4096
    worst = max(min(tiles, -(-sms // cells)) * cells for sms in range(1, 257))
    assert _ws(B, Sq, Sk, H, Hkv, D) >= 4096 * 4 + worst * rows * (D + 2) * 4
