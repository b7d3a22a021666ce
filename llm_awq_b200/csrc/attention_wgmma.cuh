// Shared by the sm_90a attention kernels (prefill_attention.cu, splitkv_attention.cu): the consumer pipeline (online
// softmax, tile loop, row sums) and the 4-D tensor map over [batch][tokens][heads][head_dim].  Their S = Q K^T is
// wgmma_ss (Q and K rows from shared memory) and their O += P V is wgmma_rs with P in registers and V transposed, both
// from tma_wgmma.cuh.
#pragma once
#include "tma_wgmma.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <typename T>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  if constexpr (!TypeTraits<T>::kIsBf16) return h2_as_u32(__floats2half2_rn(lo, hi));
  else return b2_as_u32(__floats2bfloat162_rn(lo, hi));
}

// ---------------------------------------------------------------- consumer pipeline
// One consumer warpgroup owns 64 query rows: thread (g = lane / 4, t = lane % 4) of warp w holds rows 16 w + g (lo) and
// + 8 (hi).  S element i of a 128-key tile is key 8 (i >> 2) + 2 t + (i & 1), row hi when i & 2; O has this layout over
// columns.  K / V tiles arrive in a ring of kStages stages: full[s] (TMA -> consumers), empty[s] (consumer warps ->
// producer).

// Online softmax of one tile's S: the running max m of the raw scores, p = exp2(scale_log2 * (s - m)) as one FFMA and
// one ex2, P rounded to T into the A fragments of the 8 k16 steps of O += P V, the partial row sums l of the fp32 p,
// and O and l rescaled by exp2(scale_log2 * (m_old - m)).  A row that has seen no key yet keeps m = -inf: its
// probabilities are exp2(-inf) = 0 and nothing is rescaled.
template <typename T, int N>
__device__ __forceinline__ void online_softmax(const float (&sc)[64], uint32_t (&pa)[8][4], float (&o)[N], float& m_lo,
                                               float& m_hi, float& l_lo, float& l_hi, float scale_log2) {
  float mx_lo = m_lo, mx_hi = m_hi;
#pragma unroll
  for (int i = 0; i < 64; i += 4) {
    mx_lo = fmaxf(mx_lo, fmaxf(sc[i], sc[i + 1]));
    mx_hi = fmaxf(mx_hi, fmaxf(sc[i + 2], sc[i + 3]));
  }
#pragma unroll
  for (int d = 1; d <= 2; d <<= 1) {
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, d));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, d));
  }
  const float nb_lo = mx_lo == -INFINITY ? 0.f : -mx_lo * scale_log2;
  const float nb_hi = mx_hi == -INFINITY ? 0.f : -mx_hi * scale_log2;
  const float alpha_lo = ex2(fmaf(m_lo, scale_log2, nb_lo)), alpha_hi = ex2(fmaf(m_hi, scale_log2, nb_hi));
  m_lo = mx_lo, m_hi = mx_hi;
  float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
  for (int i = 0; i < 64; i += 4) {
    const float p0 = ex2(fmaf(sc[i], scale_log2, nb_lo)), p1 = ex2(fmaf(sc[i + 1], scale_log2, nb_lo));
    const float p2 = ex2(fmaf(sc[i + 2], scale_log2, nb_hi)), p3 = ex2(fmaf(sc[i + 3], scale_log2, nb_hi));
    sum_lo += p0 + p1, sum_hi += p2 + p3;
    const int kk = i >> 3, half = (i >> 2) & 1;  // columns 8 (i / 4) + 2 t: k16 step i / 8, k + 8 when half
    pa[kk][2 * half] = pack2<T>(p0, p1);
    pa[kk][2 * half + 1] = pack2<T>(p2, p3);
  }
  l_lo = l_lo * alpha_lo + sum_lo, l_hi = l_hi * alpha_hi + sum_hi;
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    o[i] *= alpha_lo, o[i + 1] *= alpha_lo;
    o[i + 2] *= alpha_hi, o[i + 3] *= alpha_hi;
  }
}

// Turns of several consumer warpgroups at the tensor core, around each batch of wgmmas: first() before the first tile's
// wait, wait() before a batch, pass(last) after it.  A lone warpgroup takes no turns.
struct NoTurns {
  __device__ __forceinline__ void first() const {}
  __device__ __forceinline__ void wait() const {}
  __device__ __forceinline__ void pass(bool) const {}
};

// The consumer's loop over n_tiles tiles of the ring: Q K^T of tile 0, then per tile n the P V of n and the Q K^T of
// n + 1 as one batch (issue_pv(stage), issue_qk(stage)), stage n released once both have completed, and softmax(n + 1)
// (the kernel's mask, then online_softmax); then the P V of the last tile.
template <int kStages, int N, class Turns, class IssueQk, class IssuePv, class Softmax>
__device__ __forceinline__ void consume_tiles(int n_tiles, uint64_t* full, uint64_t* empty, int lane, float (&sc)[64],
                                              float (&o)[N], const Turns& turns, IssueQk issue_qk, IssuePv issue_pv,
                                              Softmax softmax) {
  if (n_tiles > 0) {
    turns.first();
    mbar_wait(&full[0], 0);
    turns.wait();
    wgmma_fence();
    issue_qk(0);
    wgmma_commit();
    turns.pass(false);
    wgmma_wait<0>();
    acc_fence(sc);
    softmax(0);
  }
  int s = 0;
  uint32_t ph = 0;
  for (int n = 0; n + 1 < n_tiles; ++n) {
    const int s1 = s + 1 == kStages ? 0 : s + 1;
    const uint32_t ph1 = s1 == 0 ? ph ^ 1 : ph;
    mbar_wait(&full[s1], ph1);
    turns.wait();
    wgmma_fence();
    issue_pv(s);
    issue_qk(s1);
    wgmma_commit();
    turns.pass(false);
    wgmma_wait<0>();
    acc_fence(o);
    acc_fence(sc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);  // tile n's K and V have been read
    softmax(n + 1);
    s = s1, ph = ph1;
  }
  if (n_tiles > 0) {
    turns.wait();
    wgmma_fence();
    issue_pv(s);
    wgmma_commit();
    turns.pass(true);
    wgmma_wait<0>();
    acc_fence(o);
  }
}

// The row sums l: each thread holds partial sums over its columns, the quad of threads that share a row adds them up
__device__ __forceinline__ void row_sums(float& l_lo, float& l_hi) {
#pragma unroll
  for (int d = 1; d <= 2; d <<= 1) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, d);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, d);
  }
}

// [batch][tokens][heads][head_dim] with element strides (batch, token, head) as a 4-D tensor map, box cw x rows
// (cw = 64: 128-byte swizzle, cw = 16: 32-byte swizzle)
template <typename T>
int encode_bthd(EncodeTiledFn enc, CUtensorMap* tm, const void* p, int head_dim, long long tokens, int heads, int batch,
                const long long st[3], int cw, int rows) {
  const size_t es = sizeof(T);
  cuuint64_t dims[4] = {(cuuint64_t)head_dim, (cuuint64_t)(tokens > 0 ? tokens : 1), (cuuint64_t)heads, (cuuint64_t)batch};
  cuuint64_t strides[3] = {(cuuint64_t)st[1] * es, (cuuint64_t)st[2] * es, (cuuint64_t)st[0] * es};
  cuuint32_t box[4] = {(cuuint32_t)cw, (cuuint32_t)rows, 1, 1};
  cuuint32_t ones[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, TypeTraits<T>::kIsBf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                   const_cast<void*>(p), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   cw == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : B200AWQ_ERR_DRIVER;
}

}  // namespace b200awq
