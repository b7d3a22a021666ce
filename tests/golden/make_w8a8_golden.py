"""Generate tests/golden/reference_w8a8_linear.npz by running the REFERENCE's own W8A8 linear module on the CPU.

Needs an llm-awq checkout named by $AWQ_REFERENCE:

    AWQ_REFERENCE=<llm-awq checkout> python tests/golden/make_w8a8_golden.py

awq/quantize/w8a8_linear.py imports `awq_inference_engine` and `awq.utils.module` at import time; stub modules are
registered for them because only its weight quantiser is exercised here (no kernel is called).  The fixture pins
llm_awq_b200/w8a8_linear.py and oracle/w8a8_oracle.py::quantize_weight (tests/test_w8a8_cpu.py).
"""
import os
import sys
import types

import numpy as np
import torch

REF = os.environ["AWQ_REFERENCE"]
HERE = os.path.dirname(os.path.abspath(__file__))


def w8a8_linear_golden():
    """tests/golden/reference_w8a8_linear.npz: W8A8OF16LinearDynamicInputScale.from_linear / from_qkv of the reference
    (awq/quantize/w8a8_linear.py:140-211) on fp16, bf16 and fp32 layers, run on the CPU: its `.cuda()` calls and
    torch.cuda.current_device() are redirected to the CPU while it runs.  Pins llm_awq_b200/w8a8_linear.py and the
    quantiser of oracle/w8a8_oracle.py."""
    import importlib.util
    sys.modules.setdefault("awq_inference_engine", types.ModuleType("awq_inference_engine"))
    for name in ("awq", "awq.utils"):
        sys.modules.setdefault(name, types.ModuleType(name))
    um = types.ModuleType("awq.utils.module")
    um.set_op_by_name = lambda *a, **k: None
    sys.modules.setdefault("awq.utils.module", um)
    spec = importlib.util.spec_from_file_location("ref_w8a8_linear", os.path.join(REF, "awq/quantize/w8a8_linear.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    saved = (torch.Tensor.cuda, torch.nn.Module.cuda, torch.cuda.current_device)
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.cuda.current_device = lambda: "cpu"
    g = torch.Generator().manual_seed(8080)
    out = {}
    f = lambda t: t.detach().float().numpy().copy()  # a copy: from_linear divides fp32 weights in place
    try:
        for tag, dt in (("f16", torch.float16), ("bf16", torch.bfloat16), ("f32", torch.float32)):
            for bias in (True, False):
                N, K = 96, 256
                lin = torch.nn.Linear(K, N, bias=bias)
                with torch.no_grad():
                    lin.weight.copy_(torch.randn(N, K, generator=g) * 0.02)
                    lin.weight[3] = 0  # an all-zero row: the 1e-5 clamp
                    if bias:
                        lin.bias.copy_(torch.randn(N, generator=g) * 0.1)
                lin = lin.to(dt)
                key = f"lin_{tag}_{'b' if bias else 'nb'}"
                out[key + "_w"] = f(lin.weight)
                if bias:
                    out[key + "_bias_in"] = f(lin.bias)
                m = mod.W8A8OF16LinearDynamicInputScale.from_linear(lin)  # modifies lin.weight in place, as it does
                out[key + "_q"] = m.weight.numpy()
                out[key + "_s"] = m.dequant_scale.numpy()
                if bias:
                    out[key + "_bias"] = m.bias.detach().numpy()
            lins = []
            for n in (64, 32, 32):
                lin = torch.nn.Linear(K, n, bias=True)
                with torch.no_grad():
                    lin.weight.copy_(torch.randn(n, K, generator=g) * 0.03)
                    lin.bias.copy_(torch.randn(n, generator=g) * 0.1)
                lins.append(lin.to(dt))
            for i, lin in enumerate(lins):
                out[f"qkv_{tag}_w{i}"] = f(lin.weight)
                out[f"qkv_{tag}_b{i}"] = f(lin.bias)
            m = mod.W8A8OF16LinearDynamicInputScale.from_qkv(*lins)
            out[f"qkv_{tag}_q"] = m.weight.numpy()
            out[f"qkv_{tag}_s"] = m.dequant_scale.numpy()
            out[f"qkv_{tag}_bias"] = m.bias.detach().numpy()
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda, torch.cuda.current_device = saved
    path = os.path.join(HERE, "reference_w8a8_linear.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    w8a8_linear_golden()
