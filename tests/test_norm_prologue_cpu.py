"""CPU checks of the RMSNorm prologue entries (b200awq_w4a16_norm_linear, b200awq_w4a16_norm_mlp_front): argument
rejections that return before any device is touched, the workspace size, the extension's argument checks, the Python
surface, which computes nothing on the host, and the row statistic's summation order (rmsnorm_stat.cuh) restated in numpy
against stored b200awq_rmsnorm outputs (tests/norm_order.py, tests/golden/rmsnorm_order.npz)."""
import inspect
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import norm_order as N

SHAPE, GROUP, ALIGN, DTYPE, WORKSPACE, DEVICE = -1, -2, -3, -4, -6, -8
A = 1 << 20  # a 16-byte aligned stand-in address (never dereferenced: every case below returns first)
BIG = 1 << 30


def _linear(m=1, n=4096, k=4096, group=128, dtype=0, x=A, gamma=A, eps=1e-6, qw=A, s=A, z=A, bias=A, y=A, ws=A, nb=BIG):
    return P.lib().b200awq_w4a16_norm_linear(x, gamma, eps, qw, s, z, bias, y, m, n, k, group, dtype, ws, nb, None)


def _front(m=1, n=14336, k=4096, group=128, dtype=0, x=A, gamma=A, eps=1e-6, up=A, y=A, ws=A, nb=BIG):
    return P.lib().b200awq_w4a16_norm_mlp_front(x, gamma, eps, A, A, A, up, A, A, y, m, n, k, group, dtype, ws, nb, None)


REJECTIONS = [
    (dict(dtype=2), DTYPE), (dict(group=64), GROUP),
    (dict(m=0), SHAPE), (dict(n=4100), SHAPE), (dict(k=4000), SHAPE), (dict(m=8, n=520), SHAPE),
    (dict(x=None), ALIGN), (dict(x=A + 2), ALIGN), (dict(y=A + 8), ALIGN),
    (dict(gamma=None), ALIGN), (dict(gamma=A + 2), ALIGN), (dict(gamma=A + 8), ALIGN),
    (dict(eps=float("nan")), SHAPE), (dict(eps=float("inf")), SHAPE), (dict(eps=-1e-6), SHAPE),
    (dict(ws=None), WORKSPACE), (dict(ws=A + 8), WORKSPACE), (dict(nb=0), WORKSPACE),
    # an argument the plain entry rejects is rejected first
    (dict(gamma=A + 2, dtype=2), DTYPE), (dict(eps=float("nan"), x=A + 2), ALIGN), (dict(ws=None, eps=-1.0), SHAPE),
]


@pytest.mark.parametrize("kw,code", REJECTIONS + [(dict(bias=A + 2), ALIGN), (dict(nb=4096 * 2 - 1), WORKSPACE),
                                                  (dict(m=3, nb=3 * 4096 * 2 - 16), WORKSPACE)])
def test_norm_linear_rejected_before_any_device_work(kw, code):
    assert _linear(**kw) == code


@pytest.mark.parametrize("kw,code", [(kw, c) for kw, c in REJECTIONS if "bias" not in kw] +
                         [(dict(up=None), ALIGN), (dict(up=A + 4), ALIGN),
                          (dict(nb=4096 * 2 + 2 * 14336 * 2 - 1), WORKSPACE), (dict(nb=4096 * 2), WORKSPACE)])
def test_norm_mlp_front_rejected_before_any_device_work(kw, code):
    assert _front(**kw) == code


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
@pytest.mark.parametrize("kw", [dict(), dict(bias=None), dict(eps=0.0), dict(m=7, n=520), dict(m=2048, n=3584, k=18944),
                                dict(nb=4096 * 2), dict(m=4, nb=4 * 4096 * 2)])
def test_norm_linear_envelope_passes_validation(kw):
    """Valid calls stop at the device check; norm_linear needs m k 2 bytes of workspace."""
    assert _linear(**kw) == DEVICE


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
@pytest.mark.parametrize("kw", [dict(), dict(m=5, n=520), dict(nb=4096 * 2 + 2 * 14336 * 2)])
def test_norm_mlp_front_envelope_passes_validation(kw):
    assert _front(**kw) == DEVICE


@pytest.mark.parametrize("m,n,k", [(1, 6144, 4096), (1, 14336, 4096), (4, 1152, 896), (2048, 10240, 8192), (3, 8, 128)])
def test_workspace_bytes(m, n, k):
    assert P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k) == m * k * 2 + 2 * m * n * 2


def test_workspace_bytes_of_empty_shapes():
    for m, n, k in [(0, 4096, 4096), (1, 0, 4096), (1, 4096, 0), (-1, 8, 128)]:
        assert P.lib().b200awq_w4a16_norm_workspace_bytes(m, n, k) == 0


def _layer(n=64, k=256, dtype=torch.float16, device="cpu"):
    m = P.WQLinear(4, 128, k, n, False, device, dtype=dtype)
    return m.qweight, m.scales, m.scaled_zeros


def test_extension_rejects_cpu_tensors_and_mismatches():
    eng = P.engine()
    x = torch.zeros(1, 256, dtype=torch.float16)
    g = torch.ones(256, dtype=torch.float16)
    W = _layer()
    with pytest.raises(RuntimeError, match="CUDA"):
        eng.rmsnorm_w4a16_linear_forward_cuda(x, g, 1e-6, *W, 128)
    with pytest.raises(RuntimeError, match="CUDA"):
        eng.rmsnorm_mlp_front_forward_cuda(x, g, 1e-6, *W, *W)
    with pytest.raises(RuntimeError):   # dtype mismatch of the weights' scales against in_feats
        eng.rmsnorm_w4a16_linear_forward_cuda(x.float(), g, 1e-6, *W, 128)
    with pytest.raises(TypeError):      # gamma and eps are required
        eng.rmsnorm_w4a16_linear_forward_cuda(x, *W, 128)


def test_python_surface_computes_nothing_on_the_host():
    from llm_awq_b200.fused_mlp import QuantLlamaMLP
    eng = P.engine()
    assert callable(eng.rmsnorm_w4a16_linear_forward_cuda) and callable(eng.rmsnorm_mlp_front_forward_cuda)
    lin = P.WQLinear(4, 128, 256, 64, True, "cpu")
    assert list(inspect.signature(lin.norm_forward).parameters) == ["x", "norm"]
    x = torch.zeros(1, 256, dtype=torch.float16)
    g = torch.ones(256, dtype=torch.float16)
    with pytest.raises(RuntimeError):
        lin.norm_forward(x, (g, 1e-6))
    mlp = QuantLlamaMLP(P.WQLinear(4, 128, 256, 512, False, "cpu"), P.WQLinear(4, 128, 512, 256, False, "cpu"),
                        P.WQLinear(4, 128, 256, 512, False, "cpu"))
    assert list(inspect.signature(mlp.forward).parameters) == ["x", "norm"]
    with pytest.raises(RuntimeError):
        mlp(x, norm=(g, 1e-6))
    with pytest.raises(RuntimeError):
        mlp(x)


# ------------------------------------------------------------------------------------------------ summation order
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rmsnorm_order.npz")


@pytest.mark.parametrize("n", N.WIDTHS)
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_restated_order_reproduces_the_stored_rmsnorm_bits(dtype, n):
    """The numpy restatement of rmsnorm_stat.cuh's order (tests/norm_order.py) reproduces every stored output row of
    b200awq_rmsnorm bit for bit, within rsqrtf's tolerance of the restated statistic."""
    stored = np.load(GOLDEN)[f"{dtype}_{n}"]
    x, g = N.inputs(n, dtype)
    for i, name in enumerate(N.ROWS):
        assert N.matches(x[i], g, stored[i], N.total_in_order(x[i]), dtype), f"{dtype} n={n} row {name}"


def test_stored_bits_tell_the_order_apart():
    """One accumulator over the whole row (the order a naive kernel would use) reproduces the stored bits of fewer
    rows: the stored rows pin the statistic's order, not only its value."""
    data = np.load(GOLDEN)
    missed = []
    for dtype in ("f16", "bf16"):
        for n in N.WIDTHS:
            x, g = N.inputs(n, dtype)
            stored = data[f"{dtype}_{n}"]
            missed += [(dtype, n, name) for i, name in enumerate(N.ROWS)
                       if not N.matches(x[i], g, stored[i], N.total_sequential(x[i]), dtype)]
    assert len(missed) >= 5, missed


def test_restated_pieces():
    """The butterfly of the restatement leaves the same sum in every lane, and chunk t + 256 j belongs to thread t."""
    s = np.arange(N.THREADS, dtype=np.float32)
    assert np.array_equal(N.butterfly(s), s.reshape(8, 32).sum(axis=1))
    sq = np.zeros(8 * N.THREADS * 2 + 8, dtype=np.float32)
    sq[8 * (N.THREADS + 5)] = 1.0       # chunk 261 = thread 5, round 1
    sq[8 * 2 * N.THREADS + 3] = 2.0     # chunk 512 = thread 0, round 2
    t = N.thread_sums(sq)
    assert t[5] == 1.0 and t[0] == 2.0 and t.sum() == 3.0
