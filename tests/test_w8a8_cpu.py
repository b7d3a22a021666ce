"""W8A8 path without a GPU: the weight quantiser of the Python mirror and of the oracle against the reference's own
from_linear / from_qkv outputs (tests/golden/reference_w8a8_linear.npz), and the C ABI's argument checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from oracle import w8a8_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_w8a8_linear.npz")
DT = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def make_linear(w, b, dtype):
    lin = torch.nn.Linear(w.shape[1], w.shape[0], bias=b is not None).to(dtype).requires_grad_(False)
    lin.weight.copy_(torch.from_numpy(w).to(dtype))
    if b is not None:
        lin.bias.copy_(torch.from_numpy(b).to(dtype))
    return lin


@pytest.mark.parametrize("tag", list(DT))
@pytest.mark.parametrize("bias", [True, False])
def test_mirror_from_linear_matches_reference(gold, tag, bias):
    key = f"lin_{tag}_{'b' if bias else 'nb'}"
    w = gold[key + "_w"]
    lin = make_linear(w, gold[key + "_bias_in"] if bias else None, DT[tag])
    m = P.W8A8OF16LinearDynamicInputScale.from_linear(lin, device="cpu")
    assert m.weight.dtype == torch.int8 and tuple(m.weight.shape) == w.shape
    assert m.dequant_scale.dtype == torch.float16
    np.testing.assert_array_equal(m.weight.numpy(), gold[key + "_q"])
    np.testing.assert_array_equal(m.dequant_scale.numpy().view(np.uint16), gold[key + "_s"].view(np.uint16))
    np.testing.assert_array_equal(lin.weight.float().numpy(), w)  # the mirror leaves the layer alone
    if bias:
        np.testing.assert_array_equal(m.bias.numpy().view(np.uint16), gold[key + "_bias"].view(np.uint16))
    else:
        assert m.bias is None


@pytest.mark.parametrize("tag", list(DT))
def test_mirror_from_qkv_matches_reference(gold, tag):
    lins = [make_linear(gold[f"qkv_{tag}_w{i}"], gold[f"qkv_{tag}_b{i}"], DT[tag]) for i in range(3)]
    m = P.W8A8OF16LinearDynamicInputScale.from_qkv(*lins, device="cpu")
    np.testing.assert_array_equal(m.weight.numpy(), gold[f"qkv_{tag}_q"])
    np.testing.assert_array_equal(m.dequant_scale.numpy().view(np.uint16), gold[f"qkv_{tag}_s"].view(np.uint16))
    np.testing.assert_array_equal(m.bias.numpy().view(np.uint16), gold[f"qkv_{tag}_bias"].view(np.uint16))


@pytest.mark.parametrize("tag", list(DT))
def test_oracle_quantiser_matches_reference(gold, tag):
    for key in (f"lin_{tag}_b", f"lin_{tag}_nb"):
        q, s = O.quantize_weight(gold[key + "_w"], tag)
        np.testing.assert_array_equal(q, gold[key + "_q"])
        np.testing.assert_array_equal(s.view(np.uint16), gold[key + "_s"].view(np.uint16))
    w = np.concatenate([gold[f"qkv_{tag}_w{i}"] for i in range(3)])
    q, s = O.quantize_weight(w, tag)
    np.testing.assert_array_equal(q, gold[f"qkv_{tag}_q"])
    np.testing.assert_array_equal(s.view(np.uint16), gold[f"qkv_{tag}_s"].view(np.uint16))


def test_oracle_row_ops_basic_properties():
    x = np.array([[0.0] * 8, [1.0, -2.0, 0.5, 0, 0, 0, 0, 2.0]], np.float32)
    q, s = O.quant_per_token(x)
    assert (q[0] == 0).all() and s[0] == 0  # zero row: NaN codes become 0
    np.testing.assert_array_equal(q[1], [64, -127, 32, 0, 0, 0, 0, 127])
    np.testing.assert_array_equal(O.cvt_s8(np.array([0.5, 1.5, -2.5, 300, -300, np.nan], np.float32)),
                                  [0, 2, -2, 127, -128, 0])


# ------------------------------------------------------------------------------ C ABI argument checks (no device)
A = 1 << 20  # a 16-byte-aligned fake device address: every call below is rejected before any device access


def vp(v):
    return ctypes.c_void_p(v)


def test_abi_w8a8_gemm_rejects_bad_arguments():
    L = P.lib()
    g = lambda *a: L.b200awq_w8a8_gemm(*[vp(x) if isinstance(x, int) and x >= A else x for x in a])
    ok = (A, A, A, A, None, A)
    assert g(*ok, 64, 64, 24, None) == -1      # k % 16
    assert g(*ok, 64, 60, 64, None) == -1      # n % 8
    assert g(*ok, 0, 64, 64, None) == -1       # m < 1
    assert g(*ok, 64, 64, 8, None) == -1       # k < 16
    assert g(A + 8, A, A, A, None, A, 64, 64, 64, None) == -3   # misaligned x
    assert g(A, A + 4, A, A, None, A, 64, 64, 64, None) == -3   # misaligned w
    assert g(A, A, A, A, None, A + 2, 64, 64, 64, None) == -3   # misaligned y
    assert g(A, A, None, A, None, A, 64, 64, 64, None) == -3    # NULL wscales
    assert g(A, A, A, A + 1, None, A, 64, 64, 64, None) == -3   # odd ascales
    assert g(None, A, A, A, None, A, 64, 64, 64, None) == -3    # NULL x


def test_abi_w8a8_row_ops_reject_bad_arguments():
    L = P.lib()
    v = vp(A)
    assert L.b200awq_quant_per_token(v, v, v, 4, 64, 2, None) == -4              # fp32 / unknown dtype
    assert L.b200awq_quant_per_token(v, v, v, 4, 0, 0, None) == -1
    assert L.b200awq_quant_per_token(v, v, v, 4, 32769, 0, None) == -1           # longer than a row kernel holds
    assert L.b200awq_quant_per_token(None, v, v, 4, 64, 0, None) == -3
    assert L.b200awq_quant_per_token(v, None, v, 4, 64, 0, None) == -3
    assert L.b200awq_layernorm_quant(v, v, v, v, v, 4, 64, ctypes.c_float(1e-6), 1, 3, None) == -4
    assert L.b200awq_layernorm_quant(v, None, v, v, v, 4, 64, ctypes.c_float(1e-6), 1, 0, None) == -3
    assert L.b200awq_layernorm_quant(v, v, vp(A + 1), v, v, 4, 64, ctypes.c_float(1e-6), 1, 0, None) == -3
    assert L.b200awq_gelu_quant(v, v, v, None, 4, 64, None) == -3
    assert L.b200awq_gelu_quant(v, v, v, v, -1, 64, None) == -1
    assert L.b200awq_silu_and_mul(v, v, 4, 64, 5, None) == -4
    assert L.b200awq_silu_and_mul(v, v, 4, 0, 0, None) == -1
    assert L.b200awq_silu_and_mul(vp(A + 1), v, 4, 64, 0, None) == -3


def test_plugin_exposes_reference_w8a8_names():
    e = P.engine()
    for name in ("w8a8_gemm_forward_cuda", "w8a8_gemm_fuse_bias_forward_cuda", "invoke_quant", "rms_norm_general",
                 "silu_and_mul", "gelu_and_quant"):
        assert hasattr(e, name), name
    doc = e.rms_norm_general.__doc__
    assert "out" in doc and "use_per_token_quant: bool = True" in doc
