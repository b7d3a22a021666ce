"""The one-token decode kernel's per-SM handoff (DESIGN §3.1) changes only when weight copies are issued, never what is
computed.  Every case runs Llama-3-8B-shaped decode launches (qkv 6144 x 4096, o 4096 x 4096, gate / up 14336 x 4096,
down 4096 x 14336: every plan, including the k-split one) with programmatic dependent launch on, and compares the
outputs bit for bit with the same launches run with it off, where no two launches of a stream overlap.  Each case runs
twice: with gate and up as two plain GEMVs, and with the fused MLP front half (b200awq_w4a16_mlp_front: gate, up and
SiLU * mul in one decode launch, w4a16_decode_kernel<true, false>) between the second RMSNorm and down, the decode step
tinychat runs:
  * the decode step captured in a CUDA graph and replayed many times;
  * decode right after RMSNorm and right after decode attention;
  * two streams running decode chains at once (the counters then also count the other stream's producers);
  * a decode chain beside a long kernel on another stream (foreign CTAs on the same SMs)."""
import ctypes

import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer, gen_x

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = torch.float16
HID, INTER = 4096, 14336
SHAPES = {"qkv": (HID, 6144), "o": (HID, HID), "gate": (HID, INTER), "up": (HID, INTER), "down": (INTER, HID)}
MLP = ("gemv", "fused")   # gate and up as two GEMVs, or the fused MLP front half
# the outputs each layer keeps: the fused MLP front writes silu(gate) * up in place of the two products
OUTS = {"gemv": ("qkv", "o", "gate", "up", "down"), "fused": ("qkv", "o", "act", "down")}


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gemv(x, w, y):
    qw, s, z = w
    rc = P.lib().b200awq_w4a16_gemv(_p(x), _p(qw), _p(s), _p(z), _p(y), 1, y.shape[-1], x.shape[-1], 128, 0, _st())
    assert rc == 0, P.lib().b200awq_strerror(rc)


def _mlp_front(x, gate, up, y):
    """One fp16 token: the fused kernel, which needs no workspace."""
    rc = P.lib().b200awq_w4a16_mlp_front(_p(x), *map(_p, gate), *map(_p, up), _p(y), 1, y.shape[-1], x.shape[-1], 128, 0,
                                         None, 0, _st())
    assert rc == 0, P.lib().b200awq_strerror(rc)


def _rmsnorm(x, g, y):
    rc = P.lib().b200awq_rmsnorm(_p(x), _p(g), _p(y), 1, x.shape[-1], 1e-5, 0, _st())
    assert rc == 0, P.lib().b200awq_strerror(rc)


class Model:
    """`layers` decoder layers of linears (distinct weights) with RMSNorm between them, so that values stay in range:
    qkv after RMSNorm, o after qkv (decode after decode), then with mlp = "gemv" gate after RMSNorm and up after gate,
    with mlp = "fused" the MLP front after RMSNorm; down after RMSNorm."""

    def __init__(self, layers, seed, mlp="gemv"):
        self.mlp = mlp
        self.w = [{n: gen_layer(N, K, DT, seed=seed + 10 * l + i, device=DEV) for i, (n, (K, N)) in enumerate(SHAPES.items())}
                  for l in range(layers)]
        self.g = {n: (1.0 + 0.1 * gen_x(1, n, DT, seed=seed + n, device=DEV)).view(n) for n in (HID, INTER)}
        self.h0 = gen_x(1, HID, DT, seed=seed + 1, device=DEV)
        width = {n: N for n, (K, N) in SHAPES.items()} | {"act": INTER}
        self.bufs = [{n: torch.empty(1, width[n], dtype=DT, device=DEV) for n in OUTS[mlp]} for _ in self.w]
        self.norm = [{k: torch.empty(1, n, dtype=DT, device=DEV) for k, n in (("a", HID), ("m", HID), ("d", INTER))}
                     for _ in self.w]

    def run(self):
        h = self.h0
        for w, b, nb in zip(self.w, self.bufs, self.norm):
            _rmsnorm(h, self.g[HID], nb["a"])
            _gemv(nb["a"], w["qkv"], b["qkv"])
            _gemv(nb["a"], w["o"], b["o"])
            _rmsnorm(b["o"], self.g[HID], nb["m"])
            if self.mlp == "fused":
                _mlp_front(nb["m"], w["gate"], w["up"], b["act"])
            else:
                _gemv(nb["m"], w["gate"], b["gate"])
                _gemv(nb["m"], w["up"], b["up"])
            _rmsnorm(b["act" if self.mlp == "fused" else "up"], self.g[INTER], nb["d"])
            _gemv(nb["d"], w["down"], b["down"])
            h = b["down"]

    def outputs(self, names=None):
        return [t.clone() for b in self.bufs for n, t in b.items() if names is None or n in names]

    def clear(self):
        for b in self.bufs:
            for t in b.values():
                t.fill_(float("nan"))


def _pdl_off(fn):
    prev = P.lib().b200awq_set_pdl(0)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        P.lib().b200awq_set_pdl(prev)


def _same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.isfinite(y).all(), i
        assert torch.equal(x, y), i


def test_step_graph_replayed_matches_pdl_off():
    for mlp in MLP:
        _step_graph_replayed(mlp)


def _step_graph_replayed(mlp):
    m = Model(4, seed=100, mlp=mlp)
    _pdl_off(m.run)
    want = m.outputs()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        m.run()
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m.run()
    for _ in range(3):
        m.clear()
        for _ in range(20):
            g.replay()
        torch.cuda.synchronize()
        _same(want, m.outputs())


def test_decode_after_attention_matches_pdl_off():
    """o, and gate or the fused MLP front, right after decode attention."""
    for mlp in MLP:
        _decode_after_attention(mlp)


def _decode_after_attention(mlp):
    eng = P.engine()
    m = Model(2, seed=200, mlp=mlp)
    B, H, Hkv, D, L, t = 1, 32, 8, 128, 512, 300
    gq = torch.Generator().manual_seed(7)
    qkv = torch.randn(B, 1, H + 2 * Hkv, D, generator=gq).to(DT).to(DEV)
    kc0 = torch.randn(B, Hkv, D // 8, L, 8, generator=gq).to(DT).to(DEV)
    vc0 = torch.randn(B, Hkv, L, D, generator=gq).to(DT).to(DEV)

    def run():
        kc, vc = kc0.clone(), vc0.clone()
        outs = []
        for w, b in zip(m.w, m.bufs):
            att = eng.single_query_attention(qkv[:, 0, :H], qkv[:, 0, H:H + Hkv], qkv[:, 0, H + Hkv:], kc, vc, None, None,
                                             t, D, 500000.0, 1.0, True)
            _gemv(att.reshape(1, H * D), w["o"], b["o"])
            if mlp == "fused":
                _mlp_front(att.reshape(1, H * D), w["gate"], w["up"], b["act"])
            else:
                _gemv(att.reshape(1, H * D), w["gate"], b["gate"])
            outs.append(att)
        return outs

    names = ("o", "act" if mlp == "fused" else "gate")
    _pdl_off(run)
    want = m.outputs(names)
    for _ in range(5):
        m.clear()
        run()
        torch.cuda.synchronize()
        _same(want, m.outputs(names))


def test_two_streams_of_decode_chains_match_pdl_off():
    for mlp in MLP:
        _two_streams(mlp)


def _two_streams(mlp):
    a, b = Model(3, seed=300, mlp=mlp), Model(3, seed=400, mlp=mlp)
    _pdl_off(a.run)
    _pdl_off(b.run)
    want_a, want_b = a.outputs(), b.outputs()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(5):
        a.clear(), b.clear()
        torch.cuda.synchronize()
        for _ in range(4):
            with torch.cuda.stream(sa):
                a.run()
            with torch.cuda.stream(sb):
                b.run()
        torch.cuda.synchronize()
        _same(want_a, a.outputs())
        _same(want_b, b.outputs())


def test_decode_chain_beside_a_long_kernel_matches_pdl_off():
    for mlp in MLP:
        _beside_a_long_kernel(mlp)


def _beside_a_long_kernel(mlp):
    m = Model(4, seed=500, mlp=mlp)
    _pdl_off(m.run)
    want = m.outputs()
    big = torch.randn(8192, 8192, device=DEV, dtype=DT)
    side, main = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(3):
        m.clear()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            for _ in range(8):
                big @ big  # long tensor-core kernels on the same SMs
        with torch.cuda.stream(main):
            for _ in range(4):
                m.run()
        torch.cuda.synchronize()
        _same(want, m.outputs())
