"""CPU checks of the LM head (b200awq_lm_head, lm_head_forward_cuda): argument rejections that return before any device
is touched, a valid call without a device failing instead of computing on the host, the extension's argument checks,
and a self-test of the float64 oracle and its bound (tests/lm_head_oracle.py)."""
import numpy as np
import pytest
import torch

import llm_awq_b200 as P
import lm_head_oracle as O

SHAPE, ALIGN, DTYPE, BATCH, DEVICE = -1, -3, -4, -5, -8
A = 1 << 20          # 16-byte aligned stand-in addresses, far apart (never dereferenced: every case below returns first)
X, G, W, L = A, 2 * A, 1 << 32, 1 << 36


def _head(x=X, stride=4096, gamma=G, eps=1e-6, w=W, logits=L, m=1, vocab=128256, k=4096, dtype=0):
    return P.lib().b200awq_lm_head(x, stride, gamma, eps, w, logits, m, vocab, k, dtype, None)


REJECTIONS = [
    (dict(m=0), BATCH), (dict(m=9), BATCH), (dict(m=-1), BATCH),
    (dict(k=0, stride=8), SHAPE), (dict(k=4, stride=8), SHAPE), (dict(k=12, stride=16), SHAPE),
    (dict(k=8200, stride=8200), SHAPE), (dict(vocab=0), SHAPE), (dict(vocab=-3), SHAPE),
    (dict(dtype=7), DTYPE), (dict(dtype=2, m=0), DTYPE),
    (dict(x=None), ALIGN), (dict(x=X + 2), ALIGN), (dict(x=X + 8), ALIGN),
    (dict(w=None), ALIGN), (dict(w=W + 8), ALIGN),
    (dict(gamma=G + 2), ALIGN), (dict(gamma=G + 8), ALIGN),
    (dict(logits=None), ALIGN), (dict(logits=L + 4), ALIGN),
    (dict(stride=4095), SHAPE), (dict(stride=0), SHAPE), (dict(stride=4100), ALIGN), (dict(m=2, stride=4097), ALIGN),
    (dict(eps=-1e-6), SHAPE), (dict(eps=float("nan")), SHAPE), (dict(eps=float("inf")), SHAPE),
    # logits overlapping an input, by one element at either end
    (dict(logits=X + 4096 * 2 - 16), ALIGN), (dict(logits=X - 128256 * 4 + 16), ALIGN),
    (dict(m=2, stride=8192, logits=X + 8192 * 2 + 4096 * 2 - 16), ALIGN),
    (dict(logits=W + 128256 * 4096 * 2 - 16), ALIGN), (dict(logits=W - 16 * 4), ALIGN),
    (dict(logits=G), ALIGN), (dict(logits=G + 4096 * 2 - 16), ALIGN),
]


@pytest.mark.parametrize("kw,code", REJECTIONS)
def test_rejected_before_any_device_work(kw, code):
    assert _head(**kw) == code


@pytest.mark.skipif(torch.cuda.is_available(), reason="with a device these calls would launch on stand-in pointers")
@pytest.mark.parametrize("kw", [dict(), dict(gamma=None), dict(gamma=None, eps=float("nan")), dict(eps=0.0),
                                dict(m=8, stride=4096), dict(m=3, stride=5 * 4096), dict(k=8, stride=8, vocab=1),
                                dict(k=8192, stride=8192, vocab=262144, dtype=1),
                                # ends that touch without overlapping
                                dict(logits=X + 4096 * 2), dict(logits=X - 128256 * 4), dict(logits=G + 4096 * 2)])
def test_valid_call_without_device_is_an_error(kw):
    """Valid calls stop at the device check: there is no host path."""
    assert _head(**kw) == DEVICE


def _ext_call(**kw):
    e = P.engine()
    args = dict(hidden=torch.zeros(1, 64, dtype=torch.float16), weight=torch.zeros(32, 64, dtype=torch.float16))
    args.update(kw)
    return e.lm_head_forward_cuda(args.pop("hidden"), args.pop("weight"), **args)


@pytest.mark.parametrize("kw", [
    dict(),                                                                           # CPU tensors
    dict(weight=torch.zeros(32, 64, dtype=torch.bfloat16)),                          # dtype mismatch
    dict(gamma=torch.ones(64, dtype=torch.bfloat16)),
    dict(hidden=torch.zeros(1, 64, dtype=torch.float32), weight=torch.zeros(32, 64)),  # fp32
    dict(hidden=torch.zeros(1, 1, 64, dtype=torch.float16)),                          # rank
    dict(weight=torch.zeros(2, 32, 64, dtype=torch.float16)),
    dict(hidden=torch.zeros(9, 64, dtype=torch.float16)),                             # m > 8
    dict(weight=torch.zeros(32, 72, dtype=torch.float16)),                            # k mismatch
])
def test_extension_checks_raise(kw):
    with pytest.raises(RuntimeError):
        _ext_call(**kw)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the device-less path")
def test_extension_without_device_raises():
    with pytest.raises((RuntimeError, AssertionError)):
        _ext_call(hidden=torch.zeros(1, 64, dtype=torch.float16, device="cuda"))


# ------------------------------------------------------------------------------------------------ oracle self-test
def _case(m, vocab, k, bf16, seed):
    g = np.random.default_rng(seed)
    x = g.standard_normal((m, k)).astype(np.float32)
    w = (0.05 * g.standard_normal((vocab, k))).astype(np.float32)
    if bf16:
        rt = lambda a: (a.view(np.uint32) & 0xFFFF0000).view(np.float32)
    else:
        rt = lambda a: a.astype(np.float16).astype(np.float32)
    return rt(x), rt(w)


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("k", [8, 256, 896])
def test_emulated_kernel_order_meets_the_bound(k, bf16):
    x, w = _case(3, 40, k, bf16, k)
    got = O.emulate(x, w, bf16)
    assert not O.violations(got, x, w, bf16).any()


@pytest.mark.parametrize("bf16", [False, True])
def test_bound_rejects_wrong_logits(bf16):
    k = 896
    x, w = _case(2, 24, k, bf16, 5)
    good = O.emulate(x, w, bf16)
    assert not O.violations(good, x, w, bf16).any()
    # a neighbouring row's logit
    shifted = np.roll(good, 1, axis=1)
    assert O.violations(shifted, x, w, bf16).all(axis=0).sum() >= 20
    # one product dropped: the largest of each logit's sum
    prods = x[:, None, :].astype(np.float64) * w[None, :, :].astype(np.float64)
    j = np.abs(prods).argmax(axis=2)
    w_drop = np.repeat(w[None], 2, axis=0)
    for i in range(2):
        w_drop[i, np.arange(w.shape[0]), j[i]] = 0.0
    dropped = np.stack([O.emulate(x[i:i + 1], w_drop[i], bf16)[0] for i in range(2)])
    assert O.violations(dropped, x, w, bf16).all()
    # an fp32 value that is not one of T's
    off = good.copy()
    off[0, 0] = np.nextafter(off[0, 0], np.float32(np.inf))
    assert O.violations(off, x, w, bf16)[0, 0]


def test_bound_rejects_an_unwidened_fp16_overflow():
    """fp16 logits past the overflow threshold must be inf; the fp32 sum before the rounding is not a logit."""
    x = np.full((1, 8), 128.0, dtype=np.float32)
    w = np.full((3, 8), 80.0, dtype=np.float32)
    w[1] = -80.0
    w[2] = 0.5
    Y = O.oracle(x, w)[0]
    assert Y[0, 0] == 81920.0
    right = np.array([[np.inf, -np.inf, 512.0]], dtype=np.float32)
    assert not O.violations(right, x, w, False).any()
    assert (O.violations(O.emulate(x, w, False), x, w, False) == False).all()
    unwidened = np.array([[81920.0, -81920.0, 512.0]], dtype=np.float32)
    assert O.violations(unwidened, x, w, False)[0, :2].all()
    clamped = np.array([[65504.0, -65504.0, 512.0]], dtype=np.float32)
    assert O.violations(clamped, x, w, False)[0, :2].all()


def test_non_finite_rules():
    x = np.array([[1.0] * 8, [np.inf] + [1.0] * 7, [np.nan] + [1.0] * 7], dtype=np.float32)
    w = np.ones((2, 8), dtype=np.float32)
    w[1, 0] = 0.0
    Y = O.oracle(x, w)[0]
    got = np.array([[8.0, 7.0], [np.inf, np.nan], [np.nan, np.nan]], dtype=np.float32)
    assert np.isnan(Y[1, 1]) and Y[1, 0] == np.inf
    assert not O.violations(got, x, w, False).any()
    assert O.violations(np.array([[8.0, 7.0], [65504.0, np.nan], [np.nan, 0.0]], dtype=np.float32), x, w, False)[1:, :].sum() == 2


def test_roundings_and_spacing():
    assert O.roundings(8) == 13 and O.roundings(256) == 13 and O.roundings(4096) == 133 and O.roundings(8192) == 261
    assert O.t_spacing(np.array([1.0, 1.5, 2.0 ** -20, 0.0]), False).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -24, 2.0 ** -24]
    assert O.t_spacing(np.array([1.0, 2.0 ** -130]), True).tolist() == [2.0 ** -7, 2.0 ** -133]
