"""Generate tests/golden/reference_kernels_w8a8.npz: outputs of the REFERENCE's own W8A8 CUDA kernels on the GPU.

Needs a CUDA device and oracle/_ref/ref_awq_w8a8*.so (the reference's w8a8/*.cu kernels, built by
`AWQ_REFERENCE=<llm-awq checkout> python oracle/build_ref_w8a8.py`):

    python tests/golden/make_w8a8_ref_kernel_golden.py [OUT_DIR]      (default: tests/golden)

The inputs are the tests' own seeded generators (tests/w8a8_cases.py), so tests/test_w8a8_gpu.py regenerates them bit
for bit and compares this project's kernels with the stored reference outputs.  Outputs are stored as a fixed sample
(rows / columns / element stride in tests/w8a8_cases.py) to stay under 1 MB; 16-bit outputs as their raw bits.
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

import w8a8_cases as W  # noqa: E402
from oracle import w8a8_oracle as WO  # noqa: E402

DEV = "cuda:0"
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}


def bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def w8a8(ref):
    """The reference's six W8A8 entry points.  GEMM outputs are stored only for shapes where the reference agrees
    with the exact oracle (gemm_ok_<shape> records the verdict); the row ops store sampled codes, every scale and,
    for gelu, the sampled fp16 GELU values.  The share of reference codes that differ from the oracle's is printed
    and stored (diff_<name>)."""
    out = {}
    for (M, N, K) in W.REF_GEMM:
        x, w, ws, a, b = W.gemm_inputs(M, N, K, DEV)
        rows, cols = W.sample_rows(M), np.arange(0, N, W.GEMM_COLS)
        for tag in ("nobias", "bias"):
            y = torch.empty(M, N, dtype=torch.float16, device=DEV)
            if tag == "bias":
                ref.w8a8_gemm_fuse_bias_forward_cuda(x, w, ws, a, y, b)
            else:
                ref.w8a8_gemm_forward_cuda(x, w, ws, a, y)
            torch.cuda.synchronize()
            ys = y.cpu().numpy()[rows]
            o = WO.gemm(x.cpu().numpy()[rows], w.cpu().numpy(), ws.cpu().numpy(), a.cpu().numpy()[rows],
                        b.cpu().numpy() if tag == "bias" else None)
            ulp = np.abs(ys.view(np.int16).astype(np.int32) - o.view(np.int16).astype(np.int32))
            ok = bool(ulp.max() <= (0 if tag == "nobias" else 1))
            key = f"{tag}_{M}x{N}x{K}"
            out[f"gemm_ok_{key}"] = np.array(ok)
            print(f"w8a8 gemm {key}: max {ulp.max()} ulp from the oracle -> {'stored' if ok else 'NOT stored'}")
            if ok:
                out[f"gemm_{key}"] = ys[:, cols].view(np.uint16)
    for tag, dtype in DTYPES.items():
        for (M, N) in W.ROW_SHAPES:
            key = f"{tag}_{M}x{N}"
            x = W.act_rows(M, N, dtype, seed=M + N, device=DEV)
            q = torch.empty(M, N, dtype=torch.int8, device=DEV)
            s = torch.empty(M, dtype=torch.float16, device=DEV)
            ref.invoke_quant(q, x, s)
            torch.cuda.synchronize()
            out[f"quant_q_{key}"], out[f"quant_s_{key}"] = q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], bits(s)
            oq, _ = WO.quant_per_token(x.float().cpu().numpy())
            out[f"diff_quant_{key}"] = np.array(np.mean(oq != q.cpu().numpy()))
            gamma, beta = W.ln_params(N, dtype, seed=N, device=DEV)
            q = torch.empty(M, N, dtype=torch.int8, device=DEV)
            s = torch.empty(M, dtype=torch.float16, device=DEV)
            ref.rms_norm_general(q, x, gamma, beta, s, W.LN_EPS, True)
            torch.cuda.synchronize()
            out[f"ln_q_{key}"], out[f"ln_s_{key}"] = q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], bits(s)
            oq, _ = WO.layernorm_quant(x.float().cpu().numpy(), gamma.float().cpu().numpy(), beta.float().cpu().numpy(),
                                       W.LN_EPS, tag)
            out[f"diff_ln_{key}"] = np.array(np.mean(oq != q.cpu().numpy()))
            q = torch.empty(M, N, dtype=torch.int8, device=DEV)
            s = torch.full((1,), 30.0, dtype=torch.float16, device=DEV)
            ref.rms_norm_general(q, x, gamma, beta, s, W.LN_EPS, False)
            torch.cuda.synchronize()
            out[f"lnt_q_{key}"] = q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE]
            y = ref.silu_and_mul(torch.cat([x, x.flip(0)], dim=1).contiguous())
            torch.cuda.synchronize()
            out[f"silu_{key}"] = bits(y.reshape(-1)[::W.ROW_SAMPLE])
    for (M, N) in W.ROW_SHAPES:
        key = f"f16_{M}x{N}"
        x = W.gelu_rows(M, N, seed=7 * M + N, device=DEV)
        q = torch.empty(M, N, dtype=torch.int8, device=DEV)
        s = torch.empty(M, dtype=torch.float16, device=DEV)
        tmp = torch.empty(M, N, dtype=torch.float16, device=DEV)
        ref.gelu_and_quant(q, x, s, tmp)
        torch.cuda.synchronize()
        out[f"gelu_q_{key}"], out[f"gelu_s_{key}"] = q.cpu().numpy().reshape(-1)[::W.ROW_SAMPLE], bits(s)
        out[f"gelu_t_{key}"] = bits(tmp.reshape(-1)[::W.ROW_SAMPLE])
        oq, _, _ = WO.gelu_quant(x.cpu().numpy())
        out[f"diff_gelu_{key}"] = np.array(np.mean(oq != q.cpu().numpy()))
    for k, v in out.items():
        if k.startswith("diff_"):
            print(f"w8a8 {k[5:]}: {100 * float(v):.4f} % of the reference's codes differ from the oracle's")
    return out


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    import ref_awq_w8a8 as ref
    props = torch.cuda.get_device_properties(0)
    meta = dict(device=np.array(props.name), capability=np.array(f"{props.major}.{props.minor}"))
    path = os.path.join(out_dir, "reference_kernels_w8a8.npz")
    np.savez_compressed(path, **w8a8(ref), **meta)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
