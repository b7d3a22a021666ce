// Shared by the sm_90a attention kernels (prefill_attention.cu, splitkv_attention.cu): the wgmma shapes of S = Q K^T
// and O += P V, the consumer pipeline (online softmax, tile loop, row sums) and the 4-D tensor map over
// [batch][tokens][heads][head_dim].
#pragma once
#include "tma_wgmma.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

// S[64 x 128] (+)= A[64 x 16] * B[16 x 128], both operands K-major in shared memory (Q rows, K rows), fp32 accumulate
#define B200AWQ_WGMMA_SS_N128(TY)                                                                                            \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28," \
               "%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,"  \
               "%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}\n"                                       \
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),           \
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),     \
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),   \
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),   \
                 "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),   \
                 "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),   \
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),   \
                 "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])    \
               : "l"(adesc), "l"(bdesc), "r"(accum))

template <typename T>
__device__ __forceinline__ void wgmma_qk(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_SS_N128("f16");
  else B200AWQ_WGMMA_SS_N128("bf16");
}

// O[64 x N] += P[64 x 16] (registers) * V[16 x N] (shared memory, MN-major: the trailing 1 transposes B)
#define B200AWQ_WGMMA_RS_T_N64(TY)                                                                                           \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"                                                                \
               "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                 \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28," \
               "%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n}\n"                                                    \
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),           \
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),     \
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),   \
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])    \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum))

#define B200AWQ_WGMMA_RS_T_N16(TY)                                                                                           \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"                                                                \
               "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " "                                                 \
               "{%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 1;\n}\n"                                          \
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])            \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum))

#define B200AWQ_WGMMA_RS_T_N128(TY)                                                                                          \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"                                                                \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28," \
               "%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,"  \
               "%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1;\n}\n"                            \
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),           \
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),     \
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),   \
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),   \
                 "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),   \
                 "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),   \
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),   \
                 "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])    \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum))

template <typename T, int N>
__device__ __forceinline__ void wgmma_pv(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
  if constexpr (N == 16) {
    if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_RS_T_N16("f16");
    else B200AWQ_WGMMA_RS_T_N16("bf16");
  } else if constexpr (N == 64) {
    if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_RS_T_N64("f16");
    else B200AWQ_WGMMA_RS_T_N64("bf16");
  } else {
    if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_RS_T_N128("f16");
    else B200AWQ_WGMMA_RS_T_N128("bf16");
  }
}

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
