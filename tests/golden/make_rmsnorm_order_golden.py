"""Generate tests/golden/rmsnorm_order.npz: outputs of this project's b200awq_rmsnorm on an H100 for the rows of
tests/norm_order.py, stored as raw bits (uint16 [rows, n] per dtype and width, key "<dtype>_<n>").

    python tests/golden/make_rmsnorm_order_golden.py [OUT_DIR]      (default: tests/golden)

tests/test_norm_prologue_cpu.py reproduces them from the numpy restatement of the summation order, and
tests/test_norm_prologue_gpu.py checks that the kernels still produce them, so that the order rmsnorm.cu and the W4A16
RMSNorm prologues share (llm_awq_b200/csrc/rmsnorm_stat.cuh) cannot change without a test noticing."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import norm_order as N  # noqa: E402


def rmsnorm_bits(dt, n):
    import llm_awq_b200 as P
    T = torch.float16 if dt == "f16" else torch.bfloat16
    x, g = N.inputs(n, dt)
    xd, gd = torch.from_numpy(x).to(T).cuda(), torch.from_numpy(g).to(T).cuda()
    y = torch.full_like(xd, float("nan"))
    P.engine().layernorm_forward_cuda(xd, gd, y, N.EPS)
    torch.cuda.synchronize()
    return y.view(torch.int16).cpu().numpy().view(np.uint16)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else HERE
    data = {f"{dt}_{n}": rmsnorm_bits(dt, n) for dt in ("f16", "bf16") for n in N.WIDTHS}
    data["device"] = np.array(torch.cuda.get_device_name(0))
    np.savez_compressed(os.path.join(out, "rmsnorm_order.npz"), **data)
    print("wrote", os.path.join(out, "rmsnorm_order.npz"), sorted(data))


if __name__ == "__main__":
    main()
