"""Tensor-parallel sharding in packed space (llm_awq_b200/tp.py): shard algebra against the oracle,
and the row-parallel all-reduce path with world_size 2 and 4 gloo processes on CPU.  The local product in
the CPU processes is the ORACLE standing in for the kernel (test harness only — the product module has
no CPU path; on the GPU tests/test_gpu_parity.py::test_tp_* run the same modules on the kernels)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import llm_awq_b200 as P
from llm_awq_b200 import tp
from oracle import w4a16_oracle as O
from awq_testutil import gen_layer, gen_x, np64, oracle_forward


def _full(N, K, dtype=torch.float16, bias=False, seed=0):
    m = P.WQLinear(4, 128, K, N, bias, "cpu", dtype=dtype)
    m.qweight, m.scales, m.scaled_zeros = gen_layer(N, K, dtype, seed=seed)
    if bias:
        m.bias = torch.randn(N, generator=torch.Generator().manual_seed(seed + 100)).to(dtype)
    return m


@pytest.mark.parametrize("world", [2, 4, 8])
def test_column_shards_concatenate_to_the_full_output(world):
    N, K = 256, 512
    full = _full(N, K, bias=True)
    x = gen_x(3, K)
    y = oracle_forward(x, full.qweight, full.scales, full.scaled_zeros, torch.float16)
    parts = []
    for r in range(world):
        qw, s, z, b = tp.shard_column(full.qweight, full.scales, full.scaled_zeros, full.bias, r, world)
        assert qw.shape == (N // world // 4, K) and s.shape == (full.scales.shape[0], N // world) and b.shape == (N // world,)
        parts.append(oracle_forward(x, qw, s, z, torch.float16))
    assert np.array_equal(np.concatenate(parts, axis=1), y)      # bit-identical: same operands, same order


@pytest.mark.parametrize("world,K", [(2, 512), (4, 1024), (8, 3584 * 8)])
def test_row_shards_sum_to_the_full_output(world, K):
    N = 64
    if K // world % 128:
        pytest.skip("shape not shardable")
    full = _full(N, K)
    x = gen_x(2, K)
    y = oracle_forward(x, full.qweight, full.scales, full.scaled_zeros, torch.float16)
    acc = np.zeros_like(y)
    k = K // world
    for r in range(world):
        qw, s, z = tp.shard_row(full.qweight, full.scales, full.scaled_zeros, r, world)
        assert qw.shape == (N // 4, k) and s.shape[0] == O.scale_rows(k) and s.shape[0] % 8 == 0
        assert torch.equal(s[k // 128:], torch.zeros_like(s[k // 128:]))
        acc += oracle_forward(x[:, r * k:(r + 1) * k], qw, s, z, torch.float16)
    assert np.allclose(acc, y, rtol=1e-12, atol=1e-12)


def test_fused_qkv_shards_by_head_block():
    hd, qh, kvh, K, world = 16, 8, 2, 256, 2
    q_out, kv_out = qh * hd, kvh * hd
    full = _full(q_out + 2 * kv_out, K, bias=True)
    x = gen_x(1, K)
    y = oracle_forward(x, full.qweight, full.scales, full.scaled_zeros, torch.float16)
    for r in range(world):
        qw, s, z, b = tp.shard_fused_qkv(full.qweight, full.scales, full.scaled_zeros, full.bias, q_out, kv_out, r, world)
        yr = oracle_forward(x, qw, s, z, torch.float16)
        ql, kl = q_out // world, kv_out // world
        want = np.concatenate([y[:, r * ql:(r + 1) * ql], y[:, q_out + r * kl:q_out + (r + 1) * kl],
                               y[:, q_out + kv_out + r * kl:q_out + kv_out + (r + 1) * kl]], axis=1)
        assert np.array_equal(yr, want)
        assert torch.equal(b, torch.cat([full.bias[r * ql:(r + 1) * ql], full.bias[q_out + r * kl:q_out + (r + 1) * kl],
                                         full.bias[q_out + kv_out + r * kl:q_out + kv_out + (r + 1) * kl]]))


def test_unshardable_shapes_are_rejected():
    full = _full(72, 384)
    with pytest.raises(ValueError):
        tp.shard_column(full.qweight, full.scales, full.scaled_zeros, None, 0, 4)     # 18 channels per rank
    with pytest.raises(ValueError):
        tp.shard_row(full.qweight, full.scales, full.scaled_zeros, 0, 2)              # 192 k per rank


# ------------------------------------------------------------------ world_size 2 and 4 gloo runs of the modules
def _oracle_local_forward(self, x):
    """Test stand-in for the kernel inside the CPU worker processes."""
    y = O.wq_linear_forward(np64(x), self.qweight.numpy(), np64(self.scales), np64(self.scaled_zeros),
                            bias=None if self.bias is None else np64(self.bias))
    return torch.from_numpy(y).to(torch.float32)


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    P.WQLinear.forward = _oracle_local_forward
    hidden, inter = 256, 512
    up = _full(inter, hidden, seed=1)
    down = _full(hidden, inter, bias=True, seed=2)
    col = tp.ColumnParallelWQLinear(up, rank, world)
    row = tp.RowParallelWQLinear(down, rank, world)
    x = gen_x(3, hidden).float()
    h = col(x)                                   # [3, inter / world], no communication
    y = row(h.to(torch.float16).float())         # local product + ONE all-reduce + bias
    torch.save(y, os.path.join(out_dir, f"y{rank}.pt"))
    # prefill-sized token count: the chunked compute / all-reduce overlap path gives the same tensor as one all-reduce
    xb = gen_x(700, hidden, seed=5).float()
    hb = col(xb).to(torch.float16).float()
    row.overlap_min_tokens, row.overlap_chunks = 512, 4
    y_over = row(hb)
    row.overlap_chunks = 1
    y_one = row(hb)
    assert y_over.shape == y_one.shape == (700, hidden)
    # two ranks: a + b in either order is the same float; more ranks: the ring's summation order may differ per chunk
    assert torch.equal(y_over, y_one) if world == 2 else torch.allclose(y_over, y_one, rtol=1e-5, atol=1e-5)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_column_then_row_parallel_mlp_gloo(world, tmp_path):
    port = 29500 + os.getpid() % 400 + world
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    ys = [torch.load(os.path.join(tmp_path, f"y{r}.pt")) for r in range(world)]
    assert all(torch.equal(ys[0], y) for y in ys[1:])   # every rank holds the reduced result
    hidden, inter = 256, 512
    up = _full(inter, hidden, seed=1)
    down = _full(hidden, inter, bias=True, seed=2)
    x = gen_x(3, hidden).float()
    h = O.wq_linear_forward(np64(x), up.qweight.numpy(), np64(up.scales), np64(up.scaled_zeros))
    h = torch.from_numpy(h).to(torch.float16)
    y = O.wq_linear_forward(np64(h), down.qweight.numpy(), np64(down.scales), np64(down.scaled_zeros), bias=np64(down.bias))
    assert np.allclose(ys[0].double().numpy(), y, rtol=1e-5, atol=1e-5)
