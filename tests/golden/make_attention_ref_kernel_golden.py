"""Generate tests/golden/reference_kernels_attention.npz: outputs of the REFERENCE's own decode-attention kernel on the
GPU for the grouped-query ratios and head sizes of tests/attention_gqa_cases.py.

Needs a CUDA device and oracle/_ref/ref_awq_attention*.so (the reference's attention/ft_attention.cpp and
decoder_masked_multihead_attention.cu, built by `AWQ_REFERENCE=<llm-awq checkout> python oracle/build_ref_attention.py`):

    python tests/golden/make_attention_ref_kernel_golden.py [OUT_DIR]      (default: tests/golden)

The inputs are the tests' own seeded generators, so tests/test_attention_gqa_gpu.py regenerates them bit for bit.  Per
case and dtype the file holds, as raw 16-bit patterns, the output [B, H, D] (out_<dtype>_<case>) and the cache slot the
step wrote: k_cache[:, :, :, t % L] (kslot_...) and v_cache[:, :, t % L] (vslot_...).  When this project's plugin is
built, the largest difference from it in units in the last place is printed per case.
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

import attention_gqa_cases as C  # noqa: E402

DEV = "cuda:0"
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}


def bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def ulp(a, b):
    """Largest distance in units in the last place (sign-magnitude bits mapped to a monotone integer line)."""
    def line(t):
        x = t.contiguous().view(torch.int16).int()
        return torch.where(x < 0, -(x & 0x7FFF), x)
    return int((line(a) - line(b)).abs().max())


def attention(ref):
    out = {}
    try:
        import llm_awq_b200 as P
        eng = P.engine()
    except Exception:  # noqa: BLE001
        eng = None
    for tag, dtype in DTYPES.items():
        for case in C.REF_CASES:
            B, H, Hkv, D, L, t = case
            key = f"{tag}_{C.case_id(case)}"
            q, k, v, kc, vc = C.ref_case_inputs(case, dtype, DEV)
            o = ref.single_query_attention(q, k, v, kc, vc, None, None, t, D, C.ROPE_BASE, 1.0, True)
            torch.cuda.synchronize()
            out[f"out_{key}"], out[f"kslot_{key}"], out[f"vslot_{key}"] = bits(o), bits(kc[:, :, :, t % L]), bits(vc[:, :, t % L])
            if eng is not None:
                q, k, v, kc2, vc2 = C.ref_case_inputs(case, dtype, DEV)
                mine = eng.single_query_attention(q, k, v, kc2, vc2, None, None, t, D, C.ROPE_BASE, 1.0, True)
                torch.cuda.synchronize()
                rel = float((mine.double() - o.double()).norm() / o.double().norm())
                print(f"attention {key}: max {ulp(mine, o)} ulp, normwise {rel:.2e} from this project's output, "
                      f"k slot {ulp(kc2[:, :, :, t % L], kc[:, :, :, t % L])} ulp, v slot {ulp(vc2[:, :, t % L], vc[:, :, t % L])} ulp")
    return out


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    import ref_awq_attention as ref
    props = torch.cuda.get_device_properties(0)
    meta = dict(device=np.array(props.name), capability=np.array(f"{props.major}.{props.minor}"))
    path = os.path.join(out_dir, "reference_kernels_attention.npz")
    np.savez_compressed(path, **attention(ref), **meta)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
