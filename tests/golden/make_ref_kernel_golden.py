"""Generate tests/golden/reference_kernels_*.npz: outputs of the REFERENCE's own CUDA kernels on the GPU.

Needs a CUDA device and oracle/_ref/ref_awq_engine*.so (the reference's gemv / gemm / layernorm / RoPE kernels,
built by `AWQ_REFERENCE=<llm-awq checkout> python oracle/build_ref.py`):

    python tests/golden/make_ref_kernel_golden.py [OUT_DIR]      (default: tests/golden)

The inputs are the tests' own seeded CPU generators (tests/awq_testutil.py and the tests' helpers), so the tests
regenerate them bit for bit and compare this project's kernels with the stored reference outputs.  Large outputs
are stored as a fixed sample (token stride, element stride or head stride, recorded next to the data) to keep every
file well under 1 MB.  16-bit outputs are stored as their raw bits (uint16) and decoded by the tests.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle", "_ref")):
    if p not in sys.path:
        sys.path.insert(0, p)

from awq_testutil import gen_layer, gen_x  # noqa: E402
from test_gpu_parity import REF_CASES, ref_rows, ref_tokens  # noqa: E402
from test_layer_ops_gpu import LN_SAMPLE, ln_inputs  # noqa: E402
from test_zz_rope_neox_gpu import ROPE_HEADS, rope_ref_inputs  # noqa: E402

DEV = "cuda:0"
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}


def bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def gemm_gemv(ref):
    out = {}
    for tag, dtype in DTYPES.items():
        for (M, N, K) in REF_CASES:
            qw, s, z = gen_layer(N, K, dtype, seed=9, device=DEV)
            x = (gen_x(M, K, dtype, seed=10, device=DEV) * 0.25).contiguous()
            if M < 8:
                y = ref.gemv_forward_cuda_new(x, qw, s, z, M, N, K, 128)
            else:
                y = ref.gemm_forward_cuda_new(x, qw, s, z)
            torch.cuda.synchronize()
            y = y.view(M, N)[ref_tokens(M)][:, ref_rows(N)]
            out[f"{tag}_{M}x{N}x{K}"] = bits(y)
    return out


def layernorm(ref):
    out = {}
    for tag, dtype in DTYPES.items():
        x, gamma = ln_inputs(dtype, DEV)
        y = torch.empty_like(x)
        ref.layernorm_forward_cuda(x, gamma, y, 1e-6)
        torch.cuda.synchronize()
        out[tag] = bits(y.reshape(-1)[::LN_SAMPLE])
    return out


def rope(ref):
    out = {}
    for tag, dtype in DTYPES.items():
        dpos, q, k, dcache, D = rope_ref_inputs(dtype, DEV)
        ref.rotary_embedding_neox(dpos, q, k, D, dcache)
        torch.cuda.synchronize()
        H = q.shape[-2]
        out[f"{tag}_q"] = bits(q.reshape(-1, H, D)[:, ::ROPE_HEADS])
        out[f"{tag}_k"] = bits(k.reshape(-1, H, D)[:, ::ROPE_HEADS])
    return out


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    import ref_awq_engine as ref
    props = torch.cuda.get_device_properties(0)
    meta = dict(device=np.array(props.name), capability=np.array(f"{props.major}.{props.minor}"))
    for name, fn in (("gemm_gemv", gemm_gemv), ("layernorm", layernorm), ("rope", rope)):
        path = os.path.join(out_dir, f"reference_kernels_{name}.npz")
        np.savez_compressed(path, **fn(ref), **meta)
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
