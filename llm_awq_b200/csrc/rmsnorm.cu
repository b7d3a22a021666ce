// RMSNorm ("T5 layer norm": no mean subtraction, no bias) for the decoder layers around the W4A16 linears.
//
// Replaces the reference's generalT5LayerNorm (awq/kernels/csrc/layernorm/layernorm.cu:38-64, host :111-131,
// exported as `layernorm_forward_cuda` at csrc/pybind.cpp:17, called from tinychat/models/llama.py:33-36 and
// tinychat/modules/fused_norm.py:16-21).  Numerical contract of the reference, kept here:
//     var  = sum_i float(x_i)^2            (fp32)
//     r    = rsqrtf(var / n + eps)
//     y_i  = rn_T( (float(x_i) * r) * float(gamma_i) )     fp16 additionally clamped to +-(65504 - 1000)
// (layernorm.cu:50-62, reduction.cuh:72-82).  Only the summation order of `var` differs.
//
// HBM-bound: algorithmic bytes = 2 * m * n * sizeof(T) (+ n * sizeof(T) of gamma, L2-resident).  One CTA per row;
// the row is read ONCE with 16-byte loads and kept in registers between the reduction and the scaling (the
// reference reads it twice with 2-byte loads); all loads of a thread are issued before the first use.  Rows wider
// than the register budget, not a multiple of 8 elements, or on pointers that are not 16-byte aligned take the generic
// two-pass kernel, which sums in the same order.  That order, norm_round and norm_pair live in rmsnorm_stat.cuh: the
// W4A16 decode kernels' RMSNorm prologues use the same ones, which makes them bit-identical to this kernel.
#include "rmsnorm_stat.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

// r of this CTA's row from each thread's accumulator s, in the order of rmsnorm_stat.cuh
__device__ __forceinline__ float block_rstd(float s, float* red, int n, float eps) {
  s = norm_warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  return norm_rstd(red, n, eps);  // every thread, same fixed order: deterministic, no second barrier
}

// NCH 16-byte chunks per thread live in registers.
template <typename T, int NCH>
__global__ void __launch_bounds__(kNormThreads) rmsnorm_rows_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                                    T* __restrict__ y, float eps, int n) {
  __shared__ float red[kNormThreads / 32];
  const int nchunk = n >> 3, tid = threadIdx.x;
  const uint4* gv = reinterpret_cast<const uint4*>(gamma);
  uint4 g[NCH];
#pragma unroll
  for (int j = 0; j < NCH; ++j) {  // gamma is a constant of the model: fetched before the dependency wait
    const int c = tid + j * kNormThreads;
    g[j] = c < nchunk ? __ldg(gv + c) : make_uint4(0, 0, 0, 0);
  }
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const uint4* xv = reinterpret_cast<const uint4*>(x + (size_t)blockIdx.x * n);
  uint4 v[NCH];
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int c = tid + j * kNormThreads;
    v[j] = c < nchunk ? xv[c] : make_uint4(0, 0, 0, 0);
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NCH; ++j) s = norm_chunk_sumsq<T>(v[j], s);
  const float r = block_rstd(s, red, n, eps);
  uint4* yv = reinterpret_cast<uint4*>(y + (size_t)blockIdx.x * n);
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int c = tid + j * kNormThreads;
    if (c < nchunk)
      yv[c] = make_uint4(norm_pair<T>(v[j].x, g[j].x, r), norm_pair<T>(v[j].y, g[j].y, r), norm_pair<T>(v[j].z, g[j].z, r),
                         norm_pair<T>(v[j].w, g[j].w, r));
  }
}

// any n and alignment: two passes over the row (the second one hits L1 / L2).  The sum of squares runs in the order of
// rmsnorm_stat.cuh -- thread t owns the 8-element chunks t, t + 256, ..., each in element order -- so a row that
// either kernel can take gives the same bits on both, whatever the alignment of its pointers.
template <typename T>
__global__ void __launch_bounds__(kNormThreads) rmsnorm_generic_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                                       T* __restrict__ y, float eps, int n) {
  __shared__ float red[kNormThreads / 32];
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const T* xr = x + (size_t)blockIdx.x * n;
  float s = 0.f;
  for (int c = threadIdx.x; c < (n + 7) / 8; c += kNormThreads) {
    const int end = min(8 * c + 8, n);
    for (int i = 8 * c; i < end; ++i) {
      const float f = to_float<T>(xr[i]);
      s = fmaf(f, f, s);
    }
  }
  const float r = block_rstd(s, red, n, eps);
  T* yr = y + (size_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += kNormThreads)
    yr[i] = norm_round<T>((to_float<T>(xr[i]) * r) * to_float<T>(gamma[i]));
}

template <typename T>
int launch_t(const void* x, const void* gamma, void* y, float eps, int m, int n, bool pdl, cudaStream_t stream) {
  const bool vec = n % 8 == 0 && aligned16(x) && aligned16(gamma) && aligned16(y);
  const int per = (n / 8 + kNormThreads - 1) / kNormThreads;
  const dim3 grid((unsigned)m), block(kNormThreads);
  if (vec && per <= 1) return launch_kernel(rmsnorm_rows_kernel<T, 1>, grid, block, 0, stream, pdl, 1, x, gamma, y, eps, n);
  if (vec && per <= 2) return launch_kernel(rmsnorm_rows_kernel<T, 2>, grid, block, 0, stream, pdl, 1, x, gamma, y, eps, n);
  if (vec && per <= 4) return launch_kernel(rmsnorm_rows_kernel<T, 4>, grid, block, 0, stream, pdl, 1, x, gamma, y, eps, n);
  if (vec && per <= 8) return launch_kernel(rmsnorm_rows_kernel<T, 8>, grid, block, 0, stream, pdl, 1, x, gamma, y, eps, n);
  return launch_kernel(rmsnorm_generic_kernel<T>, grid, block, 0, stream, pdl, 1, x, gamma, y, eps, n);
}

}  // namespace

int launch_rmsnorm(const void* x, const void* gamma, void* y, float eps, int m, int n, int dtype, bool pdl, cudaStream_t stream) {
  if (dtype == B200AWQ_DTYPE_F16) return launch_t<__half>(x, gamma, y, eps, m, n, pdl, stream);
  return launch_t<__nv_bfloat16>(x, gamma, y, eps, m, n, pdl, stream);
}

}  // namespace b200awq
