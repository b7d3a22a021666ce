"""Further parity cases: Llama-2-70B TP=1 / TP=8-shard shapes over the whole
token sweep, the two known-answer tests SURVEY.md §8c(5) lists (all-ones weights, single non-zero group), the
persistent ring kernel's partition edge cases, and its determinism."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from oracle import w4a16_oracle as O
from awq_testutil import abi_call, dt_name, gen_layer, gen_x, np64, oracle_forward, rel_err
from test_gpu_parity import check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float16, torch.bfloat16]


def _call(x, qw, s, z, M, N, K, dtype):
    rc, y = abi_call(P.lib(), x, qw, s, z, M, N, K, dtype, "gemv" if M < 8 else "gemm")
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


# Llama-2-70B, TP = 1: fused qkv 8192 -> 10240, gate / up 8192 -> 28672, down 28672 -> 8192; TP = 8 o-proj shard
# 1024 -> 8192 (row-parallel: k is the sharded dimension) and the gate / up shard 8192 -> 3584
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 4, 7, 16, 64, 2048])
@pytest.mark.parametrize("N,K", [(10240, 8192), (28672, 8192), (8192, 28672), (8192, 1024), (3584, 8192)])
def test_llama2_70b_shapes_token_sweep(N, K, M, dtype):
    if N % 128 and M >= 8:
        pytest.skip("outside the reference GEMM envelope (N % 128)")   # none of the listed shapes
    qw, s, z = gen_layer(N, K, dtype, seed=N // 64 + K // 128, device=DEV)
    x = (gen_x(M, K, dtype, seed=M, device=DEV) * 0.5).contiguous()
    y = _call(x, qw, s, z, M, N, K, dtype)
    torch.cuda.synchronize()
    step = 257 if M >= 64 else 61
    rows = np.concatenate([np.arange(0, N, step), np.arange(N - 24, N)])
    check(y[:, rows], oracle_forward(x, qw, s, z, dtype, rows=rows), dtype)


# ------------------------------------------------------------------ known-answer tests (authored; §8c(5))
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 3, 8, 40, 300])
def test_kat_all_ones_weights(M, dtype):
    """q = 1 everywhere, s = 1, z = 0  =>  w~ = 1 exactly  =>  y[m, n] = sum_k x[m, k] for every n.  With small
    integer activations every partial sum is an integer below 2^11: EXACT in any accumulation order."""
    N, K = 512, 1024
    qw = torch.full((N // 4, K), 0x1111, dtype=torch.int16, device=DEV)
    rows = O.scale_rows(K)
    s = torch.zeros(rows, N, dtype=dtype, device=DEV)
    s[: K // 128] = 1.0
    z = torch.zeros(rows, N, dtype=dtype, device=DEV)
    g = torch.Generator().manual_seed(M)
    x = torch.randint(-3, 4, (M, K), generator=g).to(dtype).to(DEV)
    y = _call(x, qw, s, z, M, N, K, dtype)
    want = x.float().sum(dim=1, keepdim=True).expand(M, N).to(dtype)   # an exact integer, rounded once
    assert torch.equal(y, want)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 5, 12, 200])
@pytest.mark.parametrize("grp", [0, 3, 7])
def test_kat_single_nonzero_group(M, grp, dtype):
    """Scales and zeros are non-zero for ONE 128-k group only: the output must equal the contribution of that
    group alone (catches group <-> k mis-indexing, stale accumulators and padded-row reads)."""
    N, K = 384, 1024
    qw, s, z = gen_layer(N, K, dtype, seed=21, device=DEV)
    keep = torch.zeros(s.shape[0], 1, dtype=torch.bool, device=DEV)
    keep[grp] = True
    s1, z1 = torch.where(keep, s, torch.zeros_like(s)), torch.where(keep, z, torch.zeros_like(z))
    x = gen_x(M, K, dtype, seed=4, device=DEV)
    y = _call(x, qw, s1, z1, M, N, K, dtype)
    xk = torch.zeros_like(x)
    xk[:, grp * 128:(grp + 1) * 128] = x[:, grp * 128:(grp + 1) * 128]
    check(y, oracle_forward(xk, qw, s, z, dtype), dtype)
    # and the other groups really contribute nothing: activations outside the group do not matter, bit for bit
    y2 = _call(xk.contiguous(), qw, s1, z1, M, N, K, dtype)
    assert torch.equal(y, y2)


# ------------------------------------------------------------------ ring kernel: partition edge cases
@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 2, 4])
@pytest.mark.parametrize("N,K", [(8, 2048), (16, 4096), (1184, 2048), (1192, 2176), (2376, 4224), (4744, 2048),
                                 (296, 6144), (8, 128), (40, 1920)])
def test_ring_partition_edges(N, K, M, dtype):
    """Channel counts around multiples of an SM count (148 CTAs, 74 clusters: fewer octets than clusters, exactly
    one / two per cluster, an odd octet at the end), odd group counts (k split 8|9, 16|17), k below the split
    threshold, slots of fewer than 16 groups."""
    qw, s, z = gen_layer(N, K, dtype, seed=N + K, device=DEV)
    x = gen_x(M, K, dtype, seed=M + 1, device=DEV)
    y = _call(x, qw, s, z, M, N, K, dtype)
    check(y, oracle_forward(x, qw, s, z, dtype), dtype)


@pytest.mark.parametrize("slots", [0, 3])
@pytest.mark.parametrize("N,K,split", [(N, K, s) for (N, K) in [(8, 512), (24, 1024), (592, 4096), (600, 4096), (2376, 4224),
                                                                (4096, 4096), (1280, 8192), (4096, 14336), (4104, 11008),
                                                                (8192, 1024)] for s in (1, 2, 4) if K // 128 >= s])
def test_decode_kernel_splits_and_ring_depths(N, K, split, slots):
    """The one-token decode kernel with the k split forced to 1 / 2 / 4 CTAs per cluster and with the shallowest ring:
    quad-row counts below / around the CTA count, row blocks of 4 / 8 / 12 channels at the end of a CTA's range, pieces of
    fewer than 32 groups (k = 11008: 86 groups), k splits that leave odd group counts."""
    import os
    dtype = torch.float16
    os.environ["B200AWQ_DECODE_SPLIT"] = str(split)
    os.environ["B200AWQ_DECODE_SLOTS"] = str(slots)
    P.lib().b200awq_reload_config()
    try:
        qw, s, z = gen_layer(N, K, dtype, seed=N + K + split, device=DEV)
        x = gen_x(1, K, dtype, seed=split, device=DEV)
        y = _call(x, qw, s, z, 1, N, K, dtype)
        torch.cuda.synchronize()
        check(y, oracle_forward(x, qw, s, z, dtype), dtype)
        y2 = _call(x, qw, s, z, 1, N, K, dtype)
        assert torch.equal(y, y2)
    finally:
        os.environ.pop("B200AWQ_DECODE_SPLIT"), os.environ.pop("B200AWQ_DECODE_SLOTS")
        P.lib().b200awq_reload_config()


def test_decode_kernel_activation_ranges():
    """The digit decomposition of the activations: huge, tiny, mixed-magnitude and all-zero groups, negative zero,
    fp16 subnormals.  Exact digits => the result matches the float64 oracle to fp32 accumulation error."""
    N, K, dtype = 256, 1024, torch.float16
    qw, s, z = gen_layer(N, K, dtype, seed=77, device=DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, K, generator=g)
    x[0, 0:128] *= 3000.0                      # near the top of the fp16 range
    x[0, 128:256] *= 1e-4                      # small normals / subnormals
    x[0, 256:384] = 0.0                        # an all-zero group
    x[0, 384] = -0.0
    x[0, 385:512] *= 1e-7                      # flushes to fp16 subnormals / zero
    x[0, 512:640] = torch.where(torch.arange(128) % 2 == 0, torch.tensor(1000.0), torch.tensor(6e-5))  # 2^24 dynamic range
    x[0, 640] = 65504.0
    x = x.to(dtype).to(DEV)
    y = _call(x, qw, s, z, 1, N, K, dtype)
    torch.cuda.synchronize()
    want = oracle_forward(x, qw, s, z, dtype)
    assert np.isfinite(np64(y)).all()
    assert rel_err(np64(y), want) < 1e-3
    # group by group: only one group's activations non-zero -> tight relative check per group
    for grp in range(8):
        xk = torch.zeros_like(x)
        xk[:, grp * 128:(grp + 1) * 128] = x[:, grp * 128:(grp + 1) * 128]
        yk = _call(xk.contiguous(), qw, s, z, 1, N, K, dtype)
        wk = oracle_forward(xk, qw, s, z, dtype)
        if np.linalg.norm(wk) == 0:
            assert torch.count_nonzero(yk) == 0
        else:
            # normwise per group (the kernel uses q s + z unrounded: elementwise it differs from the oracle's
            # fp16-rounded w~ by ~2^-12 of the LARGEST term, not of the result)
            # (+ the fp16 subnormal quantum 2^-24 per element: group 3's outputs sit at the bottom of the fp16 range)
            assert np.linalg.norm(np64(yk) - wk) <= 1e-3 * np.linalg.norm(wk) + 6e-8 * np.sqrt(wk.size), grp


def test_decode_is_deterministic_and_rows_independent():
    N, K, dtype = 14336, 4096, torch.float16
    qw, s, z = gen_layer(N, K, dtype, seed=2, device=DEV)
    x = gen_x(4, K, dtype, seed=3, device=DEV)
    y1, y2 = _call(x, qw, s, z, 4, N, K, dtype), _call(x, qw, s, z, 4, N, K, dtype)
    assert torch.equal(y1, y2)
    for t in range(4):   # a token computed alone agrees with the same token inside a batch
        yt = _call(x[t:t + 1].contiguous(), qw, s, z, 1, N, K, dtype)
        assert rel_err(np64(yt), np64(y1[t:t + 1])) < 5e-4


def test_decode_chain_under_graph_replay_with_pdl():
    """A chain of dependent decode launches (y of one is x of the next) captured in a CUDA graph with programmatic
    dependent launch: the weight prefetch runs ahead of griddepcontrol.wait, the activations must not."""
    dtype, H = torch.float16, 2048
    layers = [gen_layer(H, H, dtype, seed=40 + i, device=DEV) for i in range(6)]
    x0 = (gen_x(1, H, dtype, seed=9, device=DEV) * 0.5).contiguous()
    bufs = [torch.empty(1, H, dtype=dtype, device=DEV) for _ in layers]
    lib = P.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def chain():
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        src = x0
        for (qw, s, z), dst in zip(layers, bufs):
            assert lib.b200awq_w4a16_gemv(p(src), p(qw), p(s), p(z), p(dst), 1, H, H, 128, 0, st) == 0
            src = dst
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        chain()
    side.synchronize()
    eager = [b.clone() for b in bufs]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        chain()
    for _ in range(5):
        for b in bufs:
            b.zero_()
        g.replay()
        torch.cuda.synchronize()
        for b, e in zip(bufs, eager):
            assert torch.equal(b, e)
    # against the oracle, layer by layer (each layer's input is the kernel's own previous output)
    src = x0
    for (qw, s, z), e in zip(layers, eager):
        check(e, oracle_forward(src, qw, s, z, dtype), dtype)
        src = e
