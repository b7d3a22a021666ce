// The RMSNorm row statistic and the normalised value, shared by rmsnorm.cu and the RMSNorm prologues of the W4A16
// decode kernels (w4a16_decode.cu, w4a16_ring.cu).  A prologue is bit-identical to rmsnorm.cu followed by the plain
// launch only if every kernel sums the squares in the same order, so that order is defined here and nowhere else:
//   * 256 threads ("virtual" threads in a kernel that has another CTA shape); thread t owns the 8-element chunks
//     t, t + 256, t + 512, ... of the row and accumulates each chunk with fmaf in element order, starting from 0.f;
//   * each warp of 32 such threads adds its values with an xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same
//     sum: the two operands of each add are the same on both lanes);
//   * the 8 warp totals are added in warp order, starting from 0.f;
//   * r = rsqrtf(total / n + eps), and y_i = rn_T((x_i * r) * gamma_i), fp16 clamped to +-(65504 - 1000).
#pragma once
#include "w4_common.cuh"

namespace b200awq {

constexpr int kNormThreads = 256;               // threads (real or virtual) of the summation order above
constexpr int kNormWarps = kNormThreads / 32;

template <typename T>
__device__ __forceinline__ float2 pair_to_float2(uint32_t v) {
  if constexpr (TypeTraits<T>::kIsBf16) return __bfloat1622float2(u32_as_b2(v));
  else return __half22float2(u32_as_h2(v));
}

// reference reduction.cuh:72-82: finite clamp for fp16 only
template <typename T>
__device__ __forceinline__ T norm_round(float v) {
  if constexpr (TypeTraits<T>::kIsBf16) {
    return __float2bfloat16_rn(v);
  } else {
    constexpr float kLim = 65504.f - 1000.f;
    return v > 0.f ? __float2half_rn(fminf(v, kLim)) : __float2half_rn(fmaxf(v, -kLim));
  }
}

// two normalised elements: x2 / g2 hold two consecutive elements of the row / of gamma
template <typename T>
__device__ __forceinline__ uint32_t norm_pair(uint32_t x2, uint32_t g2, float r) {
  const float2 x = pair_to_float2<T>(x2), g = pair_to_float2<T>(g2);
  const T lo = norm_round<T>((x.x * r) * g.x), hi = norm_round<T>((x.y * r) * g.y);
  return (uint32_t)(*reinterpret_cast<const uint16_t*>(&lo)) | ((uint32_t)(*reinterpret_cast<const uint16_t*>(&hi)) << 16);
}

// one thread's accumulator s after one more 8-element chunk v
template <typename T>
__device__ __forceinline__ float norm_chunk_sumsq(uint4 v, float s) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 p = pair_to_float2<T>(w[e]);
    s = fmaf(p.x, p.x, s);
    s = fmaf(p.y, p.y, s);
  }
  return s;
}

// the warp's total of its 32 accumulators (all lanes get it)
__device__ __forceinline__ float norm_warp_sum(float s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// Thread t's accumulator over a row of n elements (n % 8 == 0, row 16-byte aligned), for a kernel that plays thread t
// itself: its first NF chunks are loaded by norm_first_chunks, so that the kernel can issue other loads behind them
// before the first use, and the rest are loaded here.
template <typename T, int NF>
__device__ __forceinline__ void norm_first_chunks(const T* row, int n, int t, uint4 (&v)[NF]) {
  const uint4* xv = reinterpret_cast<const uint4*>(row);
#pragma unroll
  for (int j = 0; j < NF; ++j) {
    const int c = t + j * kNormThreads;
    v[j] = c < (n >> 3) ? xv[c] : make_uint4(0u, 0u, 0u, 0u);
  }
}
template <typename T, int NF>
__device__ __forceinline__ float norm_thread_sumsq(const uint4 (&v)[NF], const T* row, int n, int t) {
  const uint4* xv = reinterpret_cast<const uint4*>(row);
  const int nchunk = n >> 3;
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NF; ++j)
    if (t + j * kNormThreads < nchunk) s = norm_chunk_sumsq<T>(v[j], s);
  for (int c = t + NF * kNormThreads; c < nchunk; c += kNormThreads) s = norm_chunk_sumsq<T>(xv[c], s);
  return s;
}

// r from the 8 warp totals
__device__ __forceinline__ float norm_rstd(const float* warp_totals, int n, float eps) {
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kNormWarps; ++w) t += warp_totals[w];
  return rsqrtf(t / (float)n + eps);
}

}  // namespace b200awq
