"""Tensor-parallel sharding of a WQLinear in PACKED space + the one all-reduce (SURVEY.md §8e).

The reference has no tensor parallelism (only accelerate layer placement, awq/utils/parallel.py);
this is the new work BASELINE.json's north_star asks for: column-parallel qkv / gate / up,
row-parallel o / down, and a single sum all-reduce on the row-parallel output.

Why slicing the packed tensors is legal (closed form of pack_intweight, qmodule.py:26-65):
  * the packing interleaves 4 output channels and is local to 64-k tiles, so
    - a column-parallel (output-channel) shard is a contiguous block of ROWS of `qweight`
      (granularity 4 channels; we require 8, the GEMV envelope) and of COLUMNS of scales/zeros;
    - a row-parallel (input-channel) shard is a contiguous block of int16 COLUMNS of `qweight`
      at 64-granularity; scales/zeros rows follow at group (128) granularity and are re-padded
      to a multiple of 8 rows like calculate_zeros_width does (qmodule.py:11-23).
One process per GPU; the collective is torch.distributed (NCCL over NVLink on GPUs, gloo in
the CPU tests).  The local product is always the sm_90a kernel: there is no CPU fallback.
"""
import torch
import torch.nn as nn

from .qmodule import WQLinear, calculate_zeros_width


def _check_div(value, parts, gran, what):
    if value % parts or (value // parts) % gran:
        raise ValueError(f"{what}={value} cannot be split {parts} ways at granularity {gran}")
    return value // parts


def shard_column(qweight, scales, scaled_zeros, bias, rank, world, gran=8):
    """Output-channel shard `rank` of `world`: rows of qweight, columns of scales / zeros / bias."""
    N = qweight.shape[0] * 4
    n = _check_div(N, world, gran, "out_features")
    lo = rank * n
    return (qweight[lo // 4:(lo + n) // 4].contiguous(), scales[:, lo:lo + n].contiguous(),
            scaled_zeros[:, lo:lo + n].contiguous(), None if bias is None else bias[lo:lo + n].contiguous())


def shard_row(qweight, scales, scaled_zeros, rank, world, group_size=128):
    """Input-channel shard `rank` of `world`: int16 columns of qweight, group rows of scales / zeros
    (re-padded to a multiple of 8 rows)."""
    K = qweight.shape[1]
    k = _check_div(K, world, max(group_size, 64), "in_features")
    lo = rank * k
    g0, ng = lo // group_size, k // group_size
    rows = calculate_zeros_width(k, group_size) * 8
    s = scales.new_zeros(rows, scales.shape[1])
    z = scaled_zeros.new_zeros(rows, scaled_zeros.shape[1])
    s[:ng] = scales[g0:g0 + ng]
    z[:ng] = scaled_zeros[g0:g0 + ng]
    return qweight[:, lo:lo + k].contiguous(), s, z


def shard_fused_qkv(qweight, scales, scaled_zeros, bias, q_out, kv_out, rank, world):
    """Fused [q; k; v] (tinychat/modules/fused_attn.py:566-594 concatenates along out_features):
    shard q, k and v separately by head block, then re-concatenate per rank."""
    parts, lo = [], 0
    for n in (q_out, kv_out, kv_out):
        sl = slice(lo, lo + n)
        parts.append(shard_column(qweight[lo // 4:(lo + n) // 4], scales[:, sl], scaled_zeros[:, sl],
                                  None if bias is None else bias[sl], rank, world))
        lo += n
    cat = lambda i, dim: torch.cat([p[i] for p in parts], dim=dim).contiguous()
    return cat(0, 0), cat(1, 1), cat(2, 1), None if bias is None else cat(3, 0)


def _from_tensors(qweight, scales, scaled_zeros, bias, group_size):
    N, K = qweight.shape[0] * 4, qweight.shape[1]
    m = WQLinear(4, group_size, K, N, bias is not None, qweight.device, dtype=scales.dtype)
    # assign THROUGH the registered buffers (nn.Module.__setattr__ keeps them registered for Tensor values)
    m.qweight, m.scales, m.scaled_zeros = qweight, scales, scaled_zeros
    if bias is not None:
        m.bias = bias
    assert "qweight" in m._buffers and "scales" in m._buffers and "scaled_zeros" in m._buffers
    return m


class ColumnParallelWQLinear(nn.Module):
    """y_local = x @ W[rows of this rank]^T.  Input replicated, output sharded; no communication."""

    def __init__(self, full: WQLinear, rank, world, qkv_split=None):
        super().__init__()
        if qkv_split is None:
            t = shard_column(full.qweight, full.scales, full.scaled_zeros, full.bias, rank, world)
        else:
            t = shard_fused_qkv(full.qweight, full.scales, full.scaled_zeros, full.bias, *qkv_split, rank, world)
        self.local = _from_tensors(*t, full.group_size)

    def forward(self, x):
        return self.local(x)


class RowParallelWQLinear(nn.Module):
    """y = sum over ranks of x[:, k-slice of this rank] @ W[:, k-slice]^T: the local kernel, then ONE
    all-reduce(sum) of the [tokens, out_features] partials.  The bias is added after the reduction."""

    def __init__(self, full: WQLinear, rank, world, group=None):
        super().__init__()
        t = shard_row(full.qweight, full.scales, full.scaled_zeros, rank, world, full.group_size)
        self.local = _from_tensors(*t, None, full.group_size)
        # a registered buffer, so that .to() / .cuda() / state_dict() carry it like the reference's WQLinear.bias
        self.register_buffer("bias", None if full.bias is None else full.bias.detach().clone())
        self.group = group
        self.world = world

    # Prefill: the [tokens, out_features] partial is tens of MB (33.5 MB at 2048 x 8192 fp16) and its all-reduce is
    # bandwidth-bound, so the row-parallel GEMM is chunked along the TOKEN dimension and the all-reduce of chunk i is
    # issued asynchronously (NCCL runs it on the process group's own stream over NVLink) while the tensor-core kernel of
    # chunk i + 1 runs on the compute stream (SURVEY.md §8e).  Chunks are row ranges of ONE output tensor, so the result
    # is the same tensor the unchunked path produces; every rank issues the same chunk sequence.
    overlap_min_tokens = 512     # below this the all-reduce is latency-bound and one call is better
    overlap_chunks = 4

    def forward(self, x_local):
        m = x_local.numel() // x_local.shape[-1]
        if self.world > 1 and m >= self.overlap_min_tokens and self.overlap_chunks > 1:
            return self._forward_overlapped(x_local, m)
        y = self.local(x_local)
        if self.world > 1:
            torch.distributed.all_reduce(y, op=torch.distributed.ReduceOp.SUM, group=self.group)
        return y + self.bias if self.bias is not None else y

    def _forward_overlapped(self, x_local, m):
        x2 = x_local.reshape(m, x_local.shape[-1])
        step = -(-m // self.overlap_chunks)
        step = -(-step // 128) * 128                      # whole 128-token tiles of the tensor-core kernel
        parts, works = [], []
        for lo in range(0, m, step):
            yc = self.local(x2[lo:lo + step])            # compute stream
            works.append(torch.distributed.all_reduce(yc, op=torch.distributed.ReduceOp.SUM, group=self.group, async_op=True))
            parts.append(yc)
        for w in works:
            w.wait()                                      # the compute stream waits for the collective's stream
        y = torch.cat(parts, dim=0).reshape(*x_local.shape[:-1], parts[0].shape[-1])
        return y + self.bias if self.bias is not None else y


class PeerExchange:
    """Symmetric (peer-mapped over NVLink) buffers for the fused GEMV + all-reduce kernel
    (`b200awq_w4a16_gemv_allreduce`, include/b200awq.h).  One instance can serve every row-parallel layer
    of a model: all ranks must issue the same sequence of calls.  Allocation uses
    torch.distributed._symmetric_memory (CUDA VMM peer mappings); plumbing only, no kernels."""

    def __init__(self, max_tokens, max_out_features, group=None):
        import ctypes
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        group = group or dist.group.WORLD
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if self.world > 8:
            raise ValueError("the fused exchange supports at most 8 ranks")
        dev = torch.device("cuda", torch.cuda.current_device())
        if max_out_features % 8:
            raise ValueError("max_out_features must be a multiple of 8")
        self.max_tokens, self.max_out_features = max_tokens, max_out_features
        self.cap_words = max_tokens * max_out_features
        # 8-byte words {fp32 partial, epoch}; int64 zeros == epoch 0 everywhere
        self.data = symm_mem.empty(2 * self.world * self.cap_words, dtype=torch.int64, device=dev)
        self.data.zero_()
        self.epoch = torch.zeros(max_out_features // 8, dtype=torch.int32, device=dev)
        hd = symm_mem.rendezvous(self.data, group.group_name)
        torch.cuda.synchronize()
        dist.barrier(group)          # every rank's buffer is zero before anybody's first call

        class _Peers(ctypes.Structure):
            _fields_ = [("data", ctypes.c_void_p * 8), ("epoch", ctypes.c_void_p), ("rank", ctypes.c_int),
                        ("world", ctypes.c_int), ("cap_words", ctypes.c_int), ("n_max", ctypes.c_int)]
        p = _Peers()
        for r in range(self.world):
            p.data[r] = int(hd.buffer_ptrs[r])
        p.epoch = self.epoch.data_ptr()
        p.rank, p.world, p.cap_words, p.n_max = self.rank, self.world, self.cap_words, max_out_features
        self._struct, self._handles = p, (hd,)
        self.ptr = ctypes.cast(ctypes.pointer(p), ctypes.c_void_p)


class FusedRowParallelWQLinear(RowParallelWQLinear):
    """Row-parallel layer whose decode path (tokens <= 8) is ONE kernel: local GEMV + the sum over ranks
    through NVLink peer memory.  Larger token counts use the local kernel + one NCCL all-reduce."""

    def __init__(self, full: WQLinear, rank, world, exchange: PeerExchange, group=None):
        super().__init__(full, rank, world, group)
        self.exchange = exchange

    def forward(self, x_local):
        import ctypes
        from .engine import lib
        m = x_local.numel() // x_local.shape[-1]
        loc = self.local
        ex = self.exchange
        if self.world == 1 or m > 8 or m > ex.max_tokens or loc.out_features > ex.max_out_features:
            return super().forward(x_local)      # outside what the exchange buffers hold: local kernel + NCCL
        x = x_local if x_local.is_contiguous() else x_local.contiguous()
        y = torch.empty(*x.shape[:-1], loc.out_features, dtype=x.dtype, device=x.device)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        rc = lib().b200awq_w4a16_gemv_allreduce(p(x), p(loc.qweight), p(loc.scales), p(loc.scaled_zeros), p(y), m,
                                                loc.out_features, loc.in_features, loc.group_size,
                                                0 if x.dtype == torch.float16 else 1, self.exchange.ptr,
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc == -1:                       # shape outside the fused envelope: local kernel + NCCL
            return super().forward(x_local)
        if rc != 0:
            raise RuntimeError(lib().b200awq_strerror(rc).decode())
        return y + self.bias if self.bias is not None else y
