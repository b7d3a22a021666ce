"""CPU checks of the W8A8 linear with layer-scale / residual epilogue (b200awq_w8a8_linear): argument rejections that
return before any device is touched, shapes inside b200awq_w8a8_gemm's envelope reaching the device check, and the
Python surface, which computes nothing on the host."""
import inspect

import pytest
import torch

import llm_awq_b200 as P

SHAPE, ALIGN, DEVICE = -1, -3, -8
A = 1 << 24   # a 16-byte aligned stand-in address (never dereferenced: every case below returns first)
R = 1 << 28   # a second one, far from A: residual and y do not overlap


def _call(m=1024, n=1152, k=1152, x=A, w=A, ws=A, a=A, b=A, ls=A, res=R, y=A):
    return P.lib().b200awq_w8a8_linear(x, w, ws, a, b, ls, res, y, m, n, k, None)


@pytest.mark.parametrize("kw,code", [
    (dict(m=0), SHAPE), (dict(m=-1), SHAPE), (dict(n=4), SHAPE), (dict(n=1156), SHAPE), (dict(k=8), SHAPE),
    (dict(k=1160), SHAPE), (dict(n=0), SHAPE),
    (dict(x=None), ALIGN), (dict(w=None), ALIGN), (dict(ws=None), ALIGN), (dict(a=None), ALIGN), (dict(y=None), ALIGN),
    (dict(x=A + 8), ALIGN), (dict(w=A + 4), ALIGN), (dict(y=A + 2), ALIGN), (dict(ws=A + 1), ALIGN), (dict(b=A + 1), ALIGN),
    (dict(ls=A + 2), ALIGN), (dict(ls=A + 8, res=None), ALIGN), (dict(res=R + 4), ALIGN), (dict(res=R + 8, ls=None), ALIGN),
    (dict(res=A), ALIGN),                                          # residual is y
    (dict(res=A + 1024 * 1152 * 2 - 16), ALIGN),                   # residual starts inside y's last row
    (dict(res=A - 1024 * 1152 * 2 + 16, y=A), ALIGN),              # y starts inside the residual's last row
])
def test_rejected_before_any_device_work(kw, code):
    assert _call(**kw) == code


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
@pytest.mark.parametrize("kw", [
    dict(), dict(b=None), dict(ls=None), dict(res=None), dict(b=None, ls=None), dict(ls=None, res=None),
    dict(b=None, ls=None, res=None), dict(m=1, n=8, k=16), dict(m=8192, n=1152, k=4304), dict(m=8200, n=4304, k=1152),
    dict(ws=A + 2, a=A + 6, b=A + 10),                             # scales and bias need only 2-byte alignment
    dict(res=A + 1024 * 1152 * 2),                                 # residual right behind y: adjacent, not overlapping
    dict(res=A - 1024 * 1152 * 2),                                 # residual right before y
])
def test_envelope_reaches_the_device_check(kw):
    """Shapes inside b200awq_w8a8_gemm's envelope, with any of the three operands, stop at the device check."""
    assert _call(**kw) == DEVICE


def test_declared_and_exported():
    import os
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200awq.h")
    with open(header) as f:
        assert "int b200awq_w8a8_linear(" in f.read()
    assert hasattr(P.lib(), "b200awq_w8a8_linear")
    assert b"overlapping" in P.lib().b200awq_strerror(ALIGN)


def test_python_surface_computes_nothing_on_the_host():
    eng = P.engine()
    assert callable(eng.w8a8_linear_forward_cuda)
    lin = P.W8A8OF16LinearDynamicInputScale(64, 32, bias=True, device="cpu")
    params = list(inspect.signature(lin.forward).parameters)
    assert params == ["input_", "input_scale", "output_buffer", "residual", "layer_scale"]
    x = torch.zeros(4, 64, dtype=torch.int8)
    s = torch.ones(4, dtype=torch.float16)
    out = torch.zeros(4, 32, dtype=torch.float16)
    for kw in (dict(residual=torch.zeros(4, 32, dtype=torch.float16)), dict(layer_scale=torch.ones(32, dtype=torch.float16))):
        with pytest.raises(RuntimeError):
            lin(x, s, out, **kw)
    with pytest.raises(RuntimeError):
        eng.w8a8_linear_forward_cuda(x, lin.weight, lin.dequant_scale, s, out, bias=lin.bias,
                                     residual=torch.zeros(4, 32, dtype=torch.float16))
    assert torch.equal(out, torch.zeros(4, 32, dtype=torch.float16))
