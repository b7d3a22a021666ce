"""CPU checks of the W4A16 linear with bias / residual epilogue (b200awq_w4a16_linear): argument rejections that return
before any device is touched, per route family (the GEMV envelope below 8 tokens, the GEMM envelope from 8), and the
Python surface, which computes nothing on the host."""
import inspect

import pytest
import torch

import llm_awq_b200 as P

SHAPE, GROUP, ALIGN, DTYPE, DEVICE = -1, -2, -3, -4, -8
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every case below returns first)


def _call(m=1, n=4096, k=4096, group=128, dtype=0, x=A, qw=A, s=A, z=A, bias=A, res=A, y=A):
    return P.lib().b200awq_w4a16_linear(x, qw, s, z, bias, res, y, m, n, k, group, dtype, None)


@pytest.mark.parametrize("kw,code", [
    (dict(dtype=2), DTYPE), (dict(group=64), GROUP),
    (dict(m=0), SHAPE), (dict(m=-1), SHAPE), (dict(n=4100), SHAPE), (dict(n=0), SHAPE), (dict(k=4000), SHAPE),
    (dict(k=0), SHAPE),
    (dict(m=8, n=520), SHAPE), (dict(m=64, n=4104), SHAPE), (dict(m=2048, n=4160, bias=None, res=None), SHAPE),
    (dict(x=None), ALIGN), (dict(qw=None), ALIGN), (dict(s=None), ALIGN), (dict(z=None), ALIGN), (dict(y=None), ALIGN),
    (dict(x=A + 2), ALIGN), (dict(y=A + 8), ALIGN),
    (dict(bias=A + 2), ALIGN), (dict(bias=A + 8), ALIGN), (dict(res=A + 4), ALIGN), (dict(res=A + 8, bias=None), ALIGN),
    (dict(m=2048, bias=A + 2), ALIGN), (dict(m=5, n=520, res=A + 6), ALIGN),
])
def test_rejected_before_any_device_work(kw, code):
    assert _call(**kw) == code


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
@pytest.mark.parametrize("kw", [
    dict(), dict(bias=None), dict(res=None), dict(bias=None, res=None),
    dict(m=7, n=520), dict(m=5, n=8, k=128), dict(m=8, n=128), dict(m=2048, n=3584, k=18944), dict(m=3, n=4104),
])
def test_envelope_edges_pass_validation(kw):
    """Shapes inside the envelopes, with or without either operand, stop at the device check: the GEMV routes take any
    n % 8 == 0 below 8 tokens, the GEMM routes n % 128 == 0 from 8."""
    assert _call(**kw) == DEVICE


def test_declared_and_exported():
    assert hasattr(P.lib(), "b200awq_w4a16_linear")
    assert b"aligned" in P.lib().b200awq_strerror(ALIGN)


def test_python_surface_computes_nothing_on_the_host():
    eng = P.engine()
    assert callable(eng.w4a16_linear_forward_cuda)
    m = P.WQLinear(4, 128, 256, 64, True, "cpu")
    assert list(inspect.signature(m.forward).parameters) == ["x", "residual"]
    x = torch.zeros(1, 256, dtype=torch.float16)
    with pytest.raises(RuntimeError):
        m(x)                                               # bias: the fused entry, which rejects CPU tensors
    with pytest.raises(RuntimeError):
        m(x, residual=torch.zeros(1, 64, dtype=torch.float16))
    with pytest.raises(RuntimeError):
        eng.w4a16_linear_forward_cuda(x, m.qweight, m.scales, m.scaled_zeros, 128, bias=m.bias)
