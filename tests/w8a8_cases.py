"""Seeded inputs of the W8A8 tests, shared with tests/golden/make_w8a8_ref_kernel_golden.py (which stores the reference
kernels' outputs on exactly these inputs)."""
import numpy as np
import torch

# (M, N, K) of the stored reference GEMM outputs: SigLIP-so400m (hidden 1152, qkv 3456, intermediate 4304) and
# InternViT-300M (hidden 1024, qkv 3072, intermediate 4096) projections at one image (729 / 1025 / 1024 tokens)
REF_GEMM = [(1024, 3456, 1152), (1024, 1152, 1152), (1024, 4304, 1152), (729, 1152, 4304),
            (1025, 3072, 1024), (1025, 4096, 1024), (1025, 1024, 4096)]
GEMM_ROWS = 127  # stored GEMM outputs: every GEMM_ROWS-th row and the last one, every GEMM_COLS-th column
GEMM_COLS = 5
ROW_SAMPLE = 31  # stored row-op outputs: every ROW_SAMPLE-th element (scales: all of them)
ROW_SHAPES = [(729, 1152), (257, 4304), (64, 1024)]  # (tokens, hidden) of the row-op goldens
LN_EPS = 1e-6


def gen_codes(rows, cols, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-128, 128, (rows, cols), generator=g, dtype=torch.int32).to(torch.int8)


def gen_scales(n, seed, lo=0.002, hi=0.02):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(n, generator=g)).half()


def gen_bias(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * 0.5).half()


def gemm_inputs(M, N, K, device="cpu"):
    x = gen_codes(M, K, seed=1000 + M)
    w = gen_codes(N, K, seed=2000 + N + K)
    ws, a = gen_scales(N, seed=3000 + N), gen_scales(M, seed=4000 + M)
    b = gen_bias(N, seed=5000 + N)
    return [t.to(device) for t in (x, w, ws, a, b)]


def sample_rows(M):
    return np.unique(np.concatenate([np.arange(0, M, GEMM_ROWS), [M - 1]]))


def act_rows(M, N, dtype, seed, device="cpu"):
    """Activation rows with a spread of magnitudes per token, one exactly-zero row and one row of tiny values."""
    g = torch.Generator().manual_seed(seed)
    mag = torch.exp(torch.randn(M, 1, generator=g))
    x = torch.randn(M, N, generator=g) * mag
    if M > 2:
        x[1] = 0
        x[2] = x[2] * 1e-4
    return x.to(dtype).to(device)


def ln_params(N, dtype, seed, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    gamma = (1 + 0.2 * torch.randn(N, generator=g)).to(dtype)
    beta = (0.1 * torch.randn(N, generator=g)).to(dtype)
    return gamma.to(device), beta.to(device)


def gelu_rows(M, N, seed, device="cpu"):
    """fp16 GELU inputs: mostly N(0, 2), one zero row and one row whose GELU stays below ~1e-3 (the reference's
    127 / amax overflows fp16 there and its codes saturate)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, N, generator=g) * 2
    if M > 2:
        x[1] = 0
        x[2] = torch.rand(N, generator=g) * 1e-3
    return x.half().to(device)
