"""CPU checks of attention over many queries: the float64 definition (tests/prefill_attention_oracle.py) against the
reference's own prefill-branch attention and torch, the C ABI's argument validation, and the extension's flash-attn
signatures."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import prefill_attention_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYER = np.load(os.path.join(ROOT, "tests", "golden", "reference_layer_ops.npz"))


@pytest.mark.parametrize("idx", range(3))
def test_oracle_matches_reference_prefill_attention(idx):
    """tinychat's prefill branch (fused_attn.py:290-304: causal, grouped-query) on the stored rotated q / k and v."""
    S, H, Hkv, D = (int(x) for x in LAYER[f"a{idx}_cfg"][:4])
    got = PO.prefill_attention(LAYER[f"a{idx}_rq"], LAYER[f"a{idx}_rk"], LAYER[f"a{idx}_xv"], True, 1.0 / math.sqrt(D))
    np.testing.assert_allclose(got, LAYER[f"a{idx}_out"], rtol=0, atol=1e-12)


def _torch_ref(q, k, v, causal, scale):
    """torch float64 SDPA on [B, H, S, D], grouped-query by repetition, bottom-right causal through causal_lower_right."""
    from torch.nn.attention.bias import causal_lower_right
    G = q.shape[2] // k.shape[2]
    qt, kt, vt = (torch.from_numpy(x).transpose(1, 2) for x in (q, k, v))
    kt, vt = kt.repeat_interleave(G, 1), vt.repeat_interleave(G, 1)
    mask = causal_lower_right(q.shape[1], k.shape[1]) if causal else None
    o = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=scale)
    return o.transpose(1, 2).numpy()


@pytest.mark.parametrize("causal,Sq,Sk,scale", [(False, 37, 53, None), (True, 40, 40, None), (True, 17, 90, None),
                                                (True, 64, 64, 0.3), (False, 5, 5, 2.0)])
def test_oracle_matches_torch(causal, Sq, Sk, scale):
    rng = np.random.default_rng(Sq * 100 + Sk)
    q, k, v = rng.standard_normal((2, Sq, 6, 16)), rng.standard_normal((2, Sk, 2, 16)), rng.standard_normal((2, Sk, 2, 16))
    sc = scale if scale is not None else 16 ** -0.5
    np.testing.assert_allclose(PO.prefill_attention(q, k, v, causal, sc), _torch_ref(q, k, v, causal, sc), rtol=0, atol=1e-12)
    # the float64 torch form used for the large GPU cases is the same computation
    tq, tk, tv = (torch.from_numpy(x) for x in (q, k, v))
    np.testing.assert_allclose(PO.prefill_attention_torch(tq, tk, tv, causal, sc).numpy(), PO.prefill_attention(q, k, v, causal, sc),
                               rtol=0, atol=1e-12)


def test_oracle_rows_that_see_no_key_are_zero():
    rng = np.random.default_rng(1)
    q, k, v = rng.standard_normal((1, 30, 2, 8)), rng.standard_normal((1, 20, 2, 8)), rng.standard_normal((1, 20, 2, 8))
    o = PO.prefill_attention(q, k, v, True, 0.5)
    assert np.all(o[:, :10] == 0) and np.all(np.any(o[:, 10:] != 0, axis=-1))
    ot = PO.prefill_attention_torch(*(torch.from_numpy(x) for x in (q, k, v)), True, 0.5).numpy()
    np.testing.assert_allclose(ot, o, rtol=0, atol=1e-12)


@pytest.mark.parametrize("causal", [False, True])
def test_oracle_varlen_is_per_sequence(causal):
    """Packed sequences, including an empty one and one of length 1."""
    rng = np.random.default_rng(7)
    lengths = [3, 0, 1, 12, 5]
    cu = np.concatenate([[0], np.cumsum(lengths)])
    q, k, v = (rng.standard_normal((cu[-1], 4, 16)) for _ in range(3))
    got = PO.prefill_attention(q, k, v, causal, 0.25, cu_seqlens=cu)
    for b, L in enumerate(lengths):
        s = slice(cu[b], cu[b + 1])
        if L:
            want = _torch_ref(q[None, s], k[None, s], v[None, s], causal, 0.25)[0]
            np.testing.assert_allclose(got[s], want, rtol=0, atol=1e-12)


def test_abi_rejects_bad_arguments_without_a_gpu():
    """Argument validation happens before anything touches the device."""
    lib = P.lib()
    buf = (ctypes.c_char * 64)()
    a = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    off = ctypes.c_void_p(a.value + 2)
    st = lambda *s: (ctypes.c_longlong * 3)(*s)
    good = st(4096 * 32 * 128, 32 * 128, 128)

    def call(q=a, out=a, cu_q=None, cu_k=None, H=32, Hkv=8, D=128, qs=good, dtype=0, scale=0.1):
        return lib.b200awq_prefill_attention(q, a, a, out, cu_q, cu_k, 1, 64, 64, H, Hkv, D, qs, good, good,
                                             ctypes.c_float(scale), 1, dtype, None)
    assert call(H=32, Hkv=5) == -1            # heads % kv_heads
    assert call(D=96) == -1                   # head sizes other than 64, 72, 128
    assert call(D=256) == -1
    assert call(scale=0.0) == -1 and call(scale=-0.1) == -1 and call(scale=float("inf")) == -1   # scale > 0
    assert call(q=None) == -3                 # null pointer
    assert call(out=off) == -3                # misaligned
    assert call(qs=st(4096 * 32 * 128, 32 * 128 + 4, 128)) == -3   # stride not a multiple of 8 elements
    assert call(cu_q=a) == -3                 # cu_seqlens for the queries only
    assert call(dtype=2) == -4                # fp32 / anything but fp16, bf16
    if not torch.cuda.is_available():
        assert call() != 0                    # no device -> error, never a silent CPU path


def test_extension_has_flash_attn_signatures():
    eng = P.engine()
    for name, params in (("flash_attn_func", "q, k, v, dropout_p=0.0, softmax_scale=None, causal=False"),
                         ("flash_attn_varlen_qkvpacked_func",
                          "qkv, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, causal=False")):
        fn = getattr(eng, name)
        sig = fn.__doc__.splitlines()[0]
        for p in params.split(", "):
            assert p.split("=")[0].strip() in sig, (name, p, sig)
    q = torch.zeros(1, 8, 2, 64, dtype=torch.float16)
    with pytest.raises(RuntimeError):
        eng.flash_attn_func(q, q, q)          # CPU tensors are rejected, not computed on the host
    with pytest.raises(TypeError):
        eng.flash_attn_func(q, q, q, window_size=(-1, -1))
