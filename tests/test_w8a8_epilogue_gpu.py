"""The W8A8 linear with the vision towers' layer scale and residual in the GEMM's epilogue (b200awq_w8a8_linear,
awq_inference_engine.w8a8_linear_forward_cuda, W8A8OF16LinearDynamicInputScale.forward(..., residual, layer_scale)).

The contract is bit-identity with what tinychat's encoder layers do today: the W8A8 GEMM entry
(w8a8_gemm[_fuse_bias]_forward_cuda) followed by PyTorch's fp16 `out * ls` and then `residual + out`.  Every comparison
here is torch.equal on the 16-bit patterns.  Kernel names come from the profiler (tests/kernel_trace.py)."""
import ctypes
import json
import re

import pytest
import torch

import llm_awq_b200 as P
import w8a8_cases as W
from guard_bands import Op, guarded_call
from kernel_trace import trace

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = torch.float16
# (N, K) of the projections that carry a residual: out / fc2 of SigLIP-so400m and InternViT-300M (fc2's K = 4304 is a
# k tail), and (4304, 1152) for an N tail
SHAPES = [(1152, 1152), (1152, 4304), (1024, 1024), (1024, 4096), (4304, 1152)]
MS = (1, 7, 64, 127, 128, 129, 729, 1024, 1025, 8192)
COMBOS = [(b, ls, r) for b in (False, True) for ls in (False, True) for r in (False, True)]


def combo_id(c):
    return "+".join(nm for nm, on in zip(("bias", "ls", "res"), c) if on) or "plain"


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def epilogue_operands(M, N, seed):
    g = torch.Generator().manual_seed(seed)
    ls = (0.1 * torch.randn(N, generator=g)).half().to(DEV)
    res = (8 * torch.randn(M, N, generator=g)).half().to(DEV)
    return ls, res


def composed(x, w, ws, a, bias=None, ls=None, res=None):
    """Today's calls: the W8A8 GEMM entry, then tinychat's PyTorch ops in tinychat's order."""
    eng = P.engine()
    out = torch.empty(x.shape[0], w.shape[0], dtype=F16, device=x.device)
    if bias is None:
        eng.w8a8_gemm_forward_cuda(x, w, ws, a, out)
    else:
        eng.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, out, bias)
    if ls is not None:
        out = out * ls
    if res is not None:
        out = res + out
    return out


def via_abi(x, w, ws, a, bias=None, ls=None, res=None):
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=F16, device=x.device)
    rc = P.lib().b200awq_w8a8_linear(ptr(x), ptr(w), ptr(ws), ptr(a), ptr(bias), ptr(ls), ptr(res), ptr(y), M, N, K,
                                     stream())
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


def via_plugin(x, w, ws, a, bias=None, ls=None, res=None):
    y = torch.empty(x.shape[0], w.shape[0], dtype=F16, device=x.device)
    P.engine().w8a8_linear_forward_cuda(x, w, ws, a, y, bias=bias, layer_scale=ls, residual=res)
    return y


def via_module(x, w, ws, a, bias=None, ls=None, res=None):
    lin = P.W8A8OF16LinearDynamicInputScale(x.shape[1], w.shape[0], bias=bias is not None, device=DEV)
    lin.weight, lin.dequant_scale = w, ws
    if bias is not None:
        lin.bias = bias
    y = torch.empty(x.shape[0], w.shape[0], dtype=F16, device=x.device)
    lin(x, a, y, residual=res, layer_scale=ls)
    return y


ENTRIES = {"abi": via_abi, "plugin": via_plugin, "module": via_module}


def check_equal(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    gb, wb = got.view(torch.int16), want.view(torch.int16)
    if not torch.equal(gb, wb):
        bad = (gb != wb).nonzero()
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {bad.shape[0]} elements differ; first at {i}: {got[i].item()!r} vs {want[i].item()!r}")


# ------------------------------------------------------------------------------------------------ bit-identity
@pytest.mark.parametrize("NK", SHAPES, ids=lambda s: f"n{s[0]}_k{s[1]}")
def test_bit_identical_to_gemm_then_torch_ops(NK):
    N, K = NK
    for M in MS:
        x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
        ls, res = epilogue_operands(M, N, seed=M + N + K)
        for c in COMBOS:
            ops = dict(bias=b if c[0] else None, ls=ls if c[1] else None, res=res if c[2] else None)
            want = composed(x, w, ws, a, **ops)
            for name, fn in ENTRIES.items():
                check_equal(fn(x, w, ws, a, **ops), want, f"{name} M={M} N={N} K={K} {combo_id(c)}")


def test_extreme_operands():
    """Residuals of +-65504, +-0, +-inf and NaN; layer scales that are subnormal, overflow to inf, negative or zero;
    zero rows of activation codes (the GEMM gives +0, a negative layer scale -0).  inf, NaN and signed zeros must come
    out exactly as PyTorch's ops produce them."""
    M, N, K = 129, 1152, 1152
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    x[3] = 0
    x[64:70] = 0
    ls = torch.tensor([2.0 ** -24, -(2.0 ** -24), 2.0 ** -20, 3e-6, 65504.0, 30000.0, -65504.0, -1.5, -0.0, 0.0, 1.0, -1.0]
                      * (N // 12), dtype=F16)
    specials = torch.tensor([65504.0, -65504.0, 0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1.0], dtype=F16)
    res = specials.repeat(M * N // 8 + 1)[:M * N].view(M, N)
    res = res[torch.randperm(M, generator=torch.Generator().manual_seed(0))].contiguous()
    ls, res = ls.to(DEV), res.to(DEV)
    for c in COMBOS:
        ops = dict(bias=b if c[0] else None, ls=ls if c[1] else None, res=res if c[2] else None)
        want = composed(x, w, ws, a, **ops)
        if c[1] and not c[2]:
            assert torch.isinf(want).any() and (want.view(torch.int16) == -32768).any()   # the cases do arise
        for name, fn in ENTRIES.items():
            check_equal(fn(x, w, ws, a, **ops), want, f"{name} extremes {combo_id(c)}")


# ------------------------------------------------------------------------------------------------ launches
def traced_call(M, N, K, entry, combo):
    """kernel_trace builder: entry "linear" is w8a8_linear_forward_cuda with the combo's operands, "gemm" today's
    w8a8_gemm[_fuse_bias]_forward_cuda."""
    eng = P.engine()
    cb, cl, cr = combo
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    ls = torch.ones(N, dtype=F16, device=DEV)
    res = torch.ones(M, N, dtype=F16, device=DEV)
    y = torch.empty(M, N, dtype=F16, device=DEV)
    if entry == "linear":
        return lambda: eng.w8a8_linear_forward_cuda(x, w, ws, a, y, bias=b if cb else None, layer_scale=ls if cl else None,
                                                    residual=res if cr else None)
    if cb:
        return lambda: eng.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, y, b)
    return lambda: eng.w8a8_gemm_forward_cuda(x, w, ws, a, y)


def test_launches_pinned_by_kernel_name():
    """One launch per call and no other kernel.  Without layer scale and residual the entry launches today's kernel
    (the full name, template arguments included); with either, the epilogue instantiation of the same bias flag."""
    shapes = [(1, 1152, 1152), (129, 4304, 1152), (1025, 1024, 4096), (8192, 1152, 4304)]
    cases = [[M, N, K, entry, list(c)] for M, N, K in shapes for c in COMBOS for entry in ("linear", "gemm")
             if entry == "linear" or not (c[1] or c[2])]
    got = {json.dumps(c): (r.launches, r.names)
           for c, r in zip(cases, trace("test_w8a8_epilogue_gpu:traced_call", cases, per_process=16))}
    for M, N, K in shapes:
        for c in COMBOS:
            launches, names = got[json.dumps([M, N, K, "linear", list(c)])]
            assert launches == 1 and len(names) == 1, (M, N, K, c, launches, names)
            mt = re.search(r"w8a8_wgmma_kernel<(true|false)((?:, [^>]*)?)>", names[0])
            assert mt, names
            assert mt.group(1) == ("true" if c[0] else "false"), names
            epi = c[1] or c[2]
            assert (mt.group(2) == ", __half const*, __half const*") == epi and (mt.group(2) == "") != epi, names
            if not epi:
                l2, today = got[json.dumps([M, N, K, "gemm", list(c)])]
                assert today == names and l2 == 1, (today, names)


# ------------------------------------------------------------------------------------------------ whole layers
H_SIG, I_SIG, HEADS_SIG = 1152, 4304, 16
H_IV, I_IV, HEADS_IV = 1024, 4096, 16


def tower_layers(H, I, n_layers, seed, layer_scale):
    g = torch.Generator().manual_seed(seed)
    layers = []
    for _ in range(n_layers):
        lay = {}
        for nm, (n, k) in {"qkv": (3 * H, H), "out": (H, H), "fc1": (I, H), "fc2": (H, I)}.items():
            w = torch.randint(-127, 128, (n, k), generator=g, dtype=torch.int32).to(torch.int8)
            ws = (0.0005 + 0.002 * torch.rand(n, generator=g)).half()
            b = (0.1 * torch.randn(n, generator=g)).half()
            lay[nm] = [t.to(DEV) for t in (w, ws, b)]
        for ln in ("ln1", "ln2"):
            lay[ln] = [(1 + 0.1 * torch.randn(H, generator=g)).half().to(DEV), (0.1 * torch.randn(H, generator=g)).half().to(DEV)]
        if layer_scale:
            lay["ls1"] = (0.1 * torch.randn(H, generator=g)).half().to(DEV)
            lay["ls2"] = (0.1 * torch.randn(H, generator=g)).half().to(DEV)
        layers.append(lay)
    return layers


def _lin(eng, lay, nm, q, s, out, fused_res=None, fused_ls=None):
    w, ws, b = lay[nm]
    if fused_res is None and fused_ls is None:
        eng.w8a8_gemm_fuse_bias_forward_cuda(q, w, ws, s, out, b)
    else:
        eng.w8a8_linear_forward_cuda(q, w, ws, s, out, bias=b, layer_scale=fused_ls, residual=fused_res)


def siglip_layer(h, lay, bsz, seqlen, fused):
    """QuantSiglipEncoderLayer.forward (tinychat/modules/fused_siglipdecoder.py) with its attention and MLP."""
    eng = P.engine()
    M, H = h.shape
    qH = torch.empty(M, H, dtype=torch.int8, device=DEV)
    qI = torch.empty(M, I_SIG, dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=F16, device=DEV)
    residual = h
    eng.rms_norm_general(qH, h, lay["ln1"][0], lay["ln1"][1], s, 1e-6, True)
    qkv = torch.empty(M, 3 * H, dtype=F16, device=DEV)
    _lin(eng, lay, "qkv", qH, s, qkv)
    q, k, v = qkv.split([H, H, H], dim=-1)
    shp = (bsz, seqlen, HEADS_SIG, H // HEADS_SIG)
    attn = eng.flash_attn_func(q.reshape(shp), k.reshape(shp), v.reshape(shp), softmax_scale=None, causal=False)
    eng.invoke_quant(qH, attn.reshape(M, -1), s)
    out = torch.empty(M, H, dtype=F16, device=DEV)
    if fused:
        _lin(eng, lay, "out", qH, s, out, fused_res=residual)
        h = out
    else:
        _lin(eng, lay, "out", qH, s, out)
        h = residual + out
    residual = h
    eng.rms_norm_general(qH, h, lay["ln2"][0], lay["ln2"][1], s, 1e-6, True)
    fc1 = torch.empty(M, I_SIG, dtype=F16, device=DEV)
    _lin(eng, lay, "fc1", qH, s, fc1)
    eng.gelu_and_quant(qI, fc1, s, torch.empty(M * I_SIG, dtype=F16, device=DEV))
    out = torch.empty(M, H, dtype=F16, device=DEV)
    if fused:
        _lin(eng, lay, "fc2", qI, s, out, fused_res=residual)
        return out
    _lin(eng, lay, "fc2", qI, s, out)
    return residual + out


def internvit_layer(h, lay, bsz, seqlen, fused):
    """QuantInternVisionEncoderLayer.forward (tinychat/modules/fused_internencoder.py) with its attention and MLP."""
    eng = P.engine()
    M, H = h.shape
    D = H // HEADS_IV
    residual = h
    q1 = torch.empty(M, H, dtype=torch.int8, device=DEV)
    s1 = torch.empty(M, dtype=F16, device=DEV)
    eng.rms_norm_general(q1, h, lay["ln1"][0], lay["ln1"][1], s1, 1e-6, True)
    qkv = torch.empty(M, 3 * H, dtype=F16, device=DEV)
    _lin(eng, lay, "qkv", q1, s1, qkv)
    cu = torch.arange(0, (bsz + 1) * seqlen, step=seqlen, dtype=torch.int32, device=DEV)
    attn = eng.flash_attn_varlen_qkvpacked_func(qkv.view(M, 3, HEADS_IV, D), cu, seqlen, 0.0, softmax_scale=None,
                                                causal=False)
    attn = attn.reshape(M, H)
    qa = torch.empty_like(attn, dtype=torch.int8)
    sa = torch.empty(M, device=DEV, dtype=F16)
    eng.invoke_quant(qa, attn, sa)
    proj = torch.empty_like(attn)
    if fused:
        _lin(eng, lay, "out", qa, sa, proj, fused_res=residual, fused_ls=lay["ls1"])
        h = proj
    else:
        _lin(eng, lay, "out", qa, sa, proj)
        h = residual + proj * lay["ls1"]
    residual = h
    q2 = torch.empty(M, H, dtype=torch.int8, device=DEV)
    s2 = torch.empty(M, dtype=F16, device=DEV)
    eng.rms_norm_general(q2, h, lay["ln2"][0], lay["ln2"][1], s2, 1e-6, True)
    fc1 = torch.empty(M, I_IV, dtype=F16, device=DEV)
    _lin(eng, lay, "fc1", q2, s2, fc1)
    act = torch.empty_like(fc1, dtype=torch.int8)
    sact = torch.empty(M, device=DEV, dtype=F16)
    eng.gelu_and_quant(act, fc1, sact, torch.empty(M * I_IV, device=DEV, dtype=F16))
    fc2 = torch.empty(M, H, dtype=F16, device=DEV)
    if fused:
        _lin(eng, lay, "fc2", act, sact, fc2, fused_res=residual, fused_ls=lay["ls2"])
        return fc2
    _lin(eng, lay, "fc2", act, sact, fc2)
    return residual + fc2 * lay["ls2"]


TOWERS = {
    "siglip": (siglip_layer, H_SIG, I_SIG, 1024, 2, False),
    "internvit": (internvit_layer, H_IV, I_IV, 1025, 2, True),
}


@pytest.mark.parametrize("tower", list(TOWERS))
def test_two_chained_layers_bit_identical(tower):
    """Two encoder layers: the fused route (residual / layer scale in out and fc2) equals tinychat's PyTorch adds and
    muls, eager, replayed from a CUDA graph over new inputs, and on a side stream, with PDL on and off.  fc2's residual
    comes from the out projection's launch, and the next layer's LayerNorm reads fc2's output."""
    layer_fn, H, I, seqlen, bsz, ls = TOWERS[tower]
    layers = tower_layers(H, I, 2, seed=len(tower), layer_scale=ls)
    M = bsz * seqlen
    g = torch.Generator().manual_seed(7)
    inputs = [(2 * torch.randn(M, H, generator=g)).half().to(DEV) for _ in range(3)]

    def run(h, fused):
        for lay in layers:
            h = layer_fn(h, lay, bsz, seqlen, fused)
        return h

    want = [run(x, False) for x in inputs]
    assert all(torch.isfinite(w_).all() for w_ in want)
    lib = P.lib()
    for pdl in (True, False):
        prev = lib.b200awq_set_pdl(1 if pdl else 0)
        try:
            for i, x in enumerate(inputs):
                check_equal(run(x, True), want[i], f"{tower} eager pdl={pdl} input {i}")
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                y_side = run(inputs[1], True)
            torch.cuda.current_stream().wait_stream(side)
            check_equal(y_side, want[1], f"{tower} side stream pdl={pdl}")
            static_in = inputs[0].clone()
            with torch.cuda.stream(side):
                run(static_in, True)  # warm-up on the capture stream
            torch.cuda.current_stream().wait_stream(side)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                static_out = run(static_in, True)
            for i in (2, 0, 1):
                static_in.copy_(inputs[i])
                gr.replay()
                torch.cuda.synchronize()
                check_equal(static_out, want[i], f"{tower} graph replay pdl={pdl} input {i}")
        finally:
            lib.b200awq_set_pdl(prev)


# ------------------------------------------------------------------------------------------------ guard bands
@pytest.mark.parametrize("combo", [c for c in COMBOS if c[1] or c[2]], ids=combo_id)
@pytest.mark.parametrize("M,N,K", [(130, 4304, 1152), (5, 24, 48), (129, 136, 144), (65, 1160, 4304), (1025, 1024, 1024)])
def test_guard_bands(M, N, K, combo):
    """M / N tails: layer scale, residual and the other inputs unchanged, no guard byte written, and a read past the
    layer scale or residual would feed NaN in one run and zero in the other."""
    x, w, ws, a, b = W.gemm_inputs(M, N, K)
    ls, res = epilogue_operands(M, N, seed=M * N)
    ops = {"x": Op("in", x), "w": Op("in", w), "ws": Op("in", ws), "a": Op("in", a),
           "y": Op("out", shape=(M, N), dtype=F16)}
    if combo[0]:
        ops["b"] = Op("in", b)
    if combo[1]:
        ops["ls"] = Op("in", ls.cpu())
    if combo[2]:
        ops["r"] = Op("in", res.cpu())

    def call(v):
        return P.lib().b200awq_w8a8_linear(ptr(v["x"]), ptr(v["w"]), ptr(v["ws"]), ptr(v["a"]), ptr(v.get("b")),
                                           ptr(v.get("ls")), ptr(v.get("r")), ptr(v["y"]), M, N, K, stream())
    out = guarded_call(call, ops)
    want = composed(x.to(DEV), w.to(DEV), ws.to(DEV), a.to(DEV), b.to(DEV) if combo[0] else None,
                    ls if combo[1] else None, res if combo[2] else None)
    check_equal(out["y"], want, "guarded call")


# ------------------------------------------------------------------------------------------------ rejections
def test_bad_operands_raise():
    eng = P.engine()
    lib = P.lib()
    M, N, K = 64, 1152, 1152
    x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
    y = torch.empty(M, N, dtype=F16, device=DEV)
    buf = torch.zeros(M * N + 16, dtype=F16, device=DEV)
    big = torch.zeros(2 * M * N, dtype=F16, device=DEV)
    bad = [
        dict(residual=buf[1:1 + M * N].view(M, N)),                        # misaligned view
        dict(layer_scale=buf[4:4 + N]),                                    # misaligned layer scale
        dict(residual=torch.zeros(M, N + 8, dtype=F16, device=DEV)),       # wrong shape
        dict(residual=torch.zeros(M * N, dtype=F16, device=DEV)),          # wrong rank
        dict(residual=torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)),  # wrong dtype
        dict(layer_scale=torch.zeros(N, dtype=torch.float32, device=DEV)),
        dict(layer_scale=torch.zeros(N + 8, dtype=F16, device=DEV)),
        dict(layer_scale=torch.zeros(1, N, dtype=F16, device=DEV)),
        dict(residual=torch.zeros(M, N, dtype=F16)),                       # CPU tensors
        dict(layer_scale=torch.zeros(N, dtype=F16)),
        dict(residual=torch.zeros(N, M, dtype=F16, device=DEV).t()),       # not contiguous
        dict(layer_scale=torch.zeros(2 * N, dtype=F16, device=DEV)[::2]),
        dict(residual=y),                                                  # shares memory with out_feats
    ]
    for kw in bad:
        with pytest.raises(RuntimeError):
            eng.w8a8_linear_forward_cuda(x, w, ws, a, y, **kw)
    # out_feats and residual as overlapping views of one buffer
    with pytest.raises(RuntimeError):
        eng.w8a8_linear_forward_cuda(x, w, ws, a, big[:M * N].view(M, N), residual=big[M * N - 8:2 * M * N - 8].view(M, N))
    with pytest.raises(RuntimeError):
        eng.w8a8_linear_forward_cuda(x.float(), w, ws, a, y, residual=torch.zeros(M, N, dtype=F16, device=DEV))
    # the C ABI: misaligned, NULL where required, overlapping
    res = torch.zeros(M, N, dtype=F16, device=DEV)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    for args in ((p(x), p(w), p(ws), p(a), None, p(res, 2), None, p(y)),
                 (p(x), p(w), p(ws), p(a), None, None, p(res, 8), p(y)),
                 (p(x), p(w), None, p(a), None, None, p(res), p(y)),
                 (p(x), p(w), p(ws), p(a), None, None, p(res), None),
                 (p(x), p(w), p(ws), p(a), None, None, p(big, 16), p(big, 32))):
        assert lib.b200awq_w8a8_linear(*args, M, N, K, stream()) == -3
    c0 = eng.launch_count()
    eng.w8a8_linear_forward_cuda(x, w, ws, a, big[:M * N].view(M, N), residual=big[M * N:].view(M, N))  # adjacent: fine
    torch.cuda.synchronize()
    assert eng.launch_count() == c0 + 1
