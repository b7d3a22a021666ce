"""Single-GPU loop-back of the fused decode GEMV + all-reduce kernel (`b200awq_w4a16_gemv_allreduce`,
include/b200awq.h): the `world` ranks are `world` launches on `world` streams of ONE device, each with its own
exchange buffer (plain device memory instead of NVLink peer mappings) and its own k-slice of the layer.  The protocol
is exactly the multi-GPU one -- every rank stores its fp32 partials with the call's epoch into every peer's buffer
and polls its own -- so world = 2, 4 and 8, several token counts, repeated calls (epoch advance), layers of different
widths sharing one exchange are all exercised on one GPU (the real NVLink run, incl.
CUDA-graph replay, is tests/test_tp_gpu.py -- a graph's branches are not GUARANTEED to run concurrently on one device,
and ranks that wait for each other must be).

All ranks' CTAs must be co-resident (they wait for each other).  The streaming kernel's grids here are small (<= 64 CTAs
per rank)."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer, gen_x, np64, oracle_forward, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class _Peers(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p * 8), ("epoch", ctypes.c_void_p), ("rank", ctypes.c_int),
                ("world", ctypes.c_int), ("cap_words", ctypes.c_int), ("n_max", ctypes.c_int)]


class LoopbackExchange:
    def __init__(self, world, max_tokens, n_max):
        self.world, self.cap = world, max_tokens * n_max
        self.data = [torch.zeros(2 * world * self.cap, dtype=torch.int64, device=DEV) for _ in range(world)]
        self.epoch = [torch.zeros(n_max // 8, dtype=torch.int32, device=DEV) for _ in range(world)]
        self.structs = []
        for r in range(world):
            p = _Peers()
            for q in range(world):
                p.data[q] = self.data[q].data_ptr()
            p.epoch = self.epoch[r].data_ptr()
            p.rank, p.world, p.cap_words, p.n_max = r, world, self.cap, n_max
            self.structs.append(p)
        self.streams = [torch.cuda.Stream() for _ in range(world)]

    def ptr(self, r):
        return ctypes.cast(ctypes.pointer(self.structs[r]), ctypes.c_void_p)


def _shards(qw, s, z, world):
    """Row-parallel shards (SURVEY.md §8e): contiguous int16 column slices of qweight, group rows of scales / zeros."""
    K = qw.shape[1]
    Kr = K // world
    out = []
    for r in range(world):
        g0, g1 = r * Kr // 128, (r + 1) * Kr // 128
        rows = -(-(g1 - g0) // 8) * 8
        sr = torch.zeros(rows, s.shape[1], dtype=s.dtype, device=DEV)
        zr = torch.zeros_like(sr)
        sr[: g1 - g0], zr[: g1 - g0] = s[g0:g1], z[g0:g1]
        out.append((qw[:, r * Kr:(r + 1) * Kr].contiguous(), sr, zr))
    return out


def _allreduce_call(ex, shards, xs, ys, M, N, Kr, current_stream=False):
    lib = P.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    main = torch.cuda.current_stream()
    for r in range(ex.world):
        st = ex.streams[r]
        st.wait_stream(main)
        with torch.cuda.stream(st):
            rc = lib.b200awq_w4a16_gemv_allreduce(p(xs[r]), p(shards[r][0]), p(shards[r][1]), p(shards[r][2]), p(ys[r]), M, N, Kr,
                                                  128, 0, ex.ptr(r), ctypes.c_void_p(st.cuda_stream))
        assert rc == 0, lib.b200awq_strerror(rc)
    for r in range(ex.world):
        main.wait_stream(ex.streams[r])


@pytest.mark.parametrize("world", [2, 4, 8])
def test_fused_gemv_allreduce_loopback(world):
    dtype, N, Kr = torch.float16, 256, 256
    K = Kr * world
    qw, s, z = gen_layer(N, K, dtype, seed=world, device=DEV)
    shards = _shards(qw, s, z, world)
    ex = LoopbackExchange(world, 8, 512)                     # sized for a wider layer than this one (n_max 512)
    for it, M in enumerate([1, 3, 1, 8, 2, 1]):                  # token count varies call to call: epochs per row block
        x = gen_x(M, K, dtype, seed=10 + it, device=DEV)
        xs = [x[:, r * Kr:(r + 1) * Kr].contiguous() for r in range(world)]
        ys = [torch.empty(M, N, dtype=dtype, device=DEV) for _ in range(world)]
        _allreduce_call(ex, shards, xs, ys, M, N, Kr)
        torch.cuda.synchronize()
        want = oracle_forward(x, qw, s, z, dtype)
        assert rel_err(np64(ys[0]), want) < 1e-3
        for r in range(1, world):
            assert torch.equal(ys[r], ys[0])                     # every rank holds the same bits


def test_fused_gemv_allreduce_loopback_two_widths_share_one_exchange():
    """o_proj-like and down_proj-like layers of DIFFERENT n through one exchange, interleaved (ADVICE r1: the slot of
    a word and its epoch counter share the row block as key, so this is legal), plus the capacity checks."""
    dtype, world = torch.float16, 2
    ex = LoopbackExchange(world, 4, 512)
    layers = []
    for N, Kr, seed in ((512, 128, 1), (256, 384, 2)):
        qw, s, z = gen_layer(N, Kr * world, dtype, seed=seed, device=DEV)
        layers.append((N, Kr, qw, s, z, _shards(qw, s, z, world)))
    for it in range(6):
        N, Kr, qw, s, z, shards = layers[it % 2]
        M = 1 + it % 3
        x = gen_x(M, Kr * world, dtype, seed=it, device=DEV)
        xs = [x[:, r * Kr:(r + 1) * Kr].contiguous() for r in range(world)]
        ys = [torch.empty(M, N, dtype=dtype, device=DEV) for _ in range(world)]
        _allreduce_call(ex, shards, xs, ys, M, N, Kr)
        torch.cuda.synchronize()
        assert rel_err(np64(ys[0]), oracle_forward(x, qw, s, z, dtype)) < 1e-3 and torch.equal(ys[0], ys[1])
    lib = P.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    N, Kr, qw, s, z, shards = layers[0]
    x = gen_x(8, Kr, dtype, seed=1, device=DEV)
    y = torch.empty(8, N, dtype=dtype, device=DEV)
    a = (p(x), p(shards[0][0]), p(shards[0][1]), p(shards[0][2]), p(y))
    assert lib.b200awq_w4a16_gemv_allreduce(*a, 8, N, Kr, 128, 0, ex.ptr(0), None) == -9      # 8 tokens > capacity 4
    assert lib.b200awq_w4a16_gemv_allreduce(*a, 1, 1024, Kr, 128, 0, ex.ptr(0), None) == -9   # n > n_max
    assert lib.b200awq_w4a16_gemv_allreduce(*a, 1, N, Kr, 128, 0, None, None) == -9           # no peers
