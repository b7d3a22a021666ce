// Row kernels of the W8A8 vision-tower path: per-token int8 quantisation, LayerNorm + quantisation, GELU +
// quantisation.  One CTA per row: the row is read once into registers (16-byte loads when the row and the pointers
// allow, else one element per access), reduced across the block, then written as int8 codes plus a per-row fp16
// scale.  HBM-bound.
//
// Replace, with the reference's roundings (w8a8_math.cuh for the fast-math instructions):
//   quant_per_token   invoke_quant     (w8a8/quantization.cu:54-112)
//   layernorm_quant   rms_norm_general (w8a8/layernorm.cu:55-231) -- a LayerNorm with mean and beta despite its name
//   gelu_quant        gelu_and_quant   (w8a8/act.cu:22-96)
#include <cuda_bf16.h>

#include "w4_common.cuh"
#include "w4a16_kernels.h"
#include "w8a8_math.cuh"

namespace b200awq {
namespace {

constexpr int kMaxThreads = 1024;
// row chunks held in registers per thread: 4 x 8 elements with 16-byte accesses (n <= 32768), 8 single elements
// otherwise (n <= 8192)
template <int VEC>
__host__ __device__ constexpr int chunks_per_thread() { return VEC == 8 ? 4 : 8; }

// VEC consecutive elements (VEC = 8: one 16-byte load)
template <int VEC, typename T>
__device__ __forceinline__ void load_row(const T* p, T (&e)[VEC]) {
  if constexpr (VEC == 8) *reinterpret_cast<uint4*>(e) = *reinterpret_cast<const uint4*>(p);
  else e[0] = p[0];
}
template <int VEC, typename T>
__device__ __forceinline__ void store_row(T* p, const T (&e)[VEC]) {
  if constexpr (VEC == 8) *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(e);
  else p[0] = e[0];
}
template <int VEC>
__device__ __forceinline__ void store_codes(int8_t* p, const int8_t (&c)[VEC]) {
  if constexpr (VEC == 8)
    *reinterpret_cast<uint2*>(p) = make_uint2(pack_s8x4(c[0], c[1], c[2], c[3]), pack_s8x4(c[4], c[5], c[6], c[7]));
  else p[0] = c[0];
}

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < nw ? red[lane] : red[0];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = fadd_ftz(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fadd_ftz(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) red[warp] = a, red[32 + warp] = b;
  __syncthreads();
  a = lane < nw ? red[lane] : 0.f;
  b = lane < nw ? red[32 + lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = fadd_ftz(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fadd_ftz(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
}

// ---------------------------------------------------------------- invoke_quant
// scale = rn_f16(amax / 127); q = cvt.rni.sat(x * (127 / amax)).  A zero row gives 0 * inf = NaN -> code 0.
template <typename T, int VEC>
__global__ void __launch_bounds__(kMaxThreads) quant_per_token_kernel(const T* __restrict__ x, int8_t* __restrict__ q,
                                                                      __half* __restrict__ scales, int n) {
  constexpr int C = chunks_per_thread<VEC>();
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const size_t row = blockIdx.x;
  const int nc = n / VEC;
  T v[C][VEC];
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      load_row<VEC>(x + row * n + ci * VEC, v[j]);
#pragma unroll
      for (int e = 0; e < VEC; ++e) amax = fmaxf(amax, fabsf(to_float(v[j][e])));
    }
  }
  amax = block_max(amax, red);
  if (threadIdx.x == 0) scales[row] = __float2half_rn(fdiv_approx(amax, 127.f));
  const float inv = fdiv_approx(127.f, amax);
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      int8_t c[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) c[e] = f2s8_rni_sat(fmul_ftz(to_float(v[j][e]), inv));
      store_codes<VEC>(q + row * n + ci * VEC, c);
    }
  }
}

// ---------------------------------------------------------------- rms_norm_general
// mean and E[x^2] - mean^2 in fp32, rstd = rsqrt.approx(var + eps), y = (x - mean) rstd gamma (+ beta).
//   per token:  amax over rn_T(y) starting from rn_T(1e-6); q = cvt(y * (127 / amax)) from the UNROUNDED y;
//               scale = rn_f16(amax / 127)
//   per tensor: beta is ignored (the reference passes none); q = cvt(rn_T(y) * scale[0])
template <typename T, int VEC, bool kPerToken>
__global__ void __launch_bounds__(kMaxThreads) layernorm_quant_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                                      const T* __restrict__ beta, int8_t* __restrict__ q,
                                                                      __half* __restrict__ scale, int n, float eps) {
  constexpr int C = chunks_per_thread<VEC>();
  __shared__ float red[64];
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const size_t row = blockIdx.x;
  const int nc = n / VEC;
  float v[C][VEC];
  float sum = 0.f, sq = 0.f;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      T e8[VEC];
      load_row<VEC>(x + row * n + ci * VEC, e8);
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        v[j][e] = to_float(e8[e]);
        sum = fadd_ftz(sum, v[j][e]);
        sq = ffma_ftz(v[j][e], v[j][e], sq);
      }
    }
  }
  block_sum2(sum, sq, red);
  const float mean = fdiv_approx(sum, (float)n);
  const float var = ffma_ftz(-mean, mean, fdiv_approx(sq, (float)n));
  const float rstd = frsqrt_approx(fadd_ftz(var, eps));
  const float tscale = kPerToken ? 0.f : __half2float(scale[0]);
  float amax = to_float(from_float<T>(1e-6f));
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      T g8[VEC], b8[VEC];
      load_row<VEC>(gamma + ci * VEC, g8);
      if (kPerToken && beta) load_row<VEC>(beta + ci * VEC, b8);
      int8_t c[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const float d = fmul_ftz(fsub_ftz(v[j][e], mean), rstd);
        float y;
        if (kPerToken && beta) y = ffma_ftz(d, to_float(g8[e]), to_float(b8[e]));
        else y = fmul_ftz(d, to_float(g8[e]));
        const float yt = to_float(from_float<T>(y));
        if constexpr (kPerToken) {
          amax = fmaxf(amax, fabsf(yt));
          v[j][e] = y;
        } else {
          c[e] = f2s8_rni_sat(fmul_ftz(yt, tscale));
        }
      }
      if constexpr (!kPerToken) store_codes<VEC>(q + row * n + ci * VEC, c);
    }
  }
  if constexpr (kPerToken) {
    __syncthreads();  // `red` is reused
    amax = block_max(amax, red);
    const float inv = fdiv_approx(127.f, amax);
#pragma unroll
    for (int j = 0; j < C; ++j) {
      const int ci = threadIdx.x + j * blockDim.x;
      if (ci < nc) {
        int8_t c[VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) c[e] = f2s8_rni_sat(fmul_ftz(v[j][e], inv));
        store_codes<VEC>(q + row * n + ci * VEC, c);
      }
    }
    if (threadIdx.x == 0) scale[row] = __float2half_rn(fdiv_approx(amax, 127.f));
  }
}

// ---------------------------------------------------------------- gelu_and_quant (fp16 only)
// gelu_fast as the reference's chain of fp16 operations around tanh.approx:
//   t = rn(tanh(rn(x c1) * rn(1 + rn(rn(c2 x) x)))),  gelu = rn(rn(0.5 x) * rn(1 + t))
__device__ __forceinline__ __half gelu_fast_h(__half x) {
  const __half c1 = __float2half_rn(0.79788456f), c2 = __float2half_rn(0.044715f);
  const __half one = __float2half_rn(1.f), half_ = __float2half_rn(0.5f);
  const __half inner = __hmul(__hmul(x, c1), __hadd(one, __hmul(__hmul(c2, x), x)));
  const __half t = __float2half_rn(ftanh_approx(__half2float(inner)));
  return __hmul(__hmul(half_, x), __hadd(one, t));
}

// tmp = gelu(x).  amax over |gelu| except that values in (0, 1e-4] enter negated (so never raise it); scale =
// rn_f16(amax / 127); q = cvt(f32(rn_f16(rn_f16(127 / amax) * tmp))) -- rn_f16(127 / amax) is inf below amax ~ 0.0019.
template <int VEC>
__global__ void __launch_bounds__(kMaxThreads) gelu_quant_kernel(const __half* __restrict__ x, int8_t* __restrict__ q,
                                                                 __half* __restrict__ scales, __half* __restrict__ tmp,
                                                                 int n) {
  constexpr int C = chunks_per_thread<VEC>();
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const size_t row = blockIdx.x;
  const int nc = n / VEC;
  const __half small = __float2half_rn(0.0001f);
  __half g[C][VEC];
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      __half e8[VEC];
      load_row<VEC>(x + row * n + ci * VEC, e8);
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        g[j][e] = gelu_fast_h(e8[e]);
        const __half a = __hgt(g[j][e], small) ? g[j][e] : __hneg(g[j][e]);
        amax = fmaxf(amax, __half2float(a));
      }
      store_row<VEC>(tmp + row * n + ci * VEC, g[j]);
    }
  }
  amax = block_max(amax, red);
  if (threadIdx.x == 0) scales[row] = __float2half_rn(fdiv_approx(amax, 127.f));
  const __half hs = __float2half_rn(fdiv_approx(127.f, amax));
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const int ci = threadIdx.x + j * blockDim.x;
    if (ci < nc) {
      int8_t c[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) c[e] = f2s8_rni_sat(__half2float(__hmul(hs, g[j][e])));
      store_codes<VEC>(q + row * n + ci * VEC, c);
    }
  }
}

// threads for a row of `chunks` accesses: one access per thread where possible, a multiple of 32
unsigned row_threads(int chunks) {
  const int per = (chunks + kMaxThreads - 1) / kMaxThreads;
  const int t = (chunks + per - 1) / per;
  return (unsigned)(((t + 31) / 32) * 32);
}

template <typename... KArgs, typename... Args>
int launch_rows(void (*kern)(KArgs...), int m, int chunks, bool pdl, cudaStream_t stream, Args... args) {
  if (chunks > chunks_per_thread<1>() * kMaxThreads) return B200AWQ_ERR_SHAPE;  // (16-byte rows: 4096 chunks, checked by the caller)
  return launch_kernel(kern, dim3((unsigned)m), dim3(row_threads(chunks)), 0, stream, pdl, 1, args...);
}

template <typename T>
int quant_t(const void* x, void* q, void* scales, int m, int n, bool pdl, cudaStream_t st) {
  if (n % 8 == 0 && aligned16(x) && aligned16(q))
    return launch_rows(quant_per_token_kernel<T, 8>, m, n / 8, pdl, st, x, q, scales, n);
  return launch_rows(quant_per_token_kernel<T, 1>, m, n, pdl, st, x, q, scales, n);
}

template <typename T, bool kPerToken>
int layernorm_t(const void* x, const void* gamma, const void* beta, void* q, void* scale, int m, int n, float eps, bool pdl,
                cudaStream_t st) {
  if (n % 8 == 0 && aligned16(x) && aligned16(gamma) && (!beta || aligned16(beta)) && aligned16(q))
    return launch_rows(layernorm_quant_kernel<T, 8, kPerToken>, m, n / 8, pdl, st, x, gamma, beta, q, scale, n, eps);
  return launch_rows(layernorm_quant_kernel<T, 1, kPerToken>, m, n, pdl, st, x, gamma, beta, q, scale, n, eps);
}

}  // namespace

int w8a8_row_limit() { return 8 * chunks_per_thread<8>() * kMaxThreads; }

int launch_quant_per_token(const void* x, void* q, void* scales, int m, int n, int dtype, bool pdl, cudaStream_t st) {
  if (m == 0) return 0;
  if (dtype == B200AWQ_DTYPE_F16) return quant_t<__half>(x, q, scales, m, n, pdl, st);
  return quant_t<__nv_bfloat16>(x, q, scales, m, n, pdl, st);
}

int launch_layernorm_quant(const void* x, const void* gamma, const void* beta, void* q, void* scale, int m, int n, float eps,
                           bool per_token, int dtype, bool pdl, cudaStream_t st) {
  if (m == 0) return 0;
  const bool h = dtype == B200AWQ_DTYPE_F16;
  if (per_token)
    return h ? layernorm_t<__half, true>(x, gamma, beta, q, scale, m, n, eps, pdl, st)
             : layernorm_t<__nv_bfloat16, true>(x, gamma, beta, q, scale, m, n, eps, pdl, st);
  return h ? layernorm_t<__half, false>(x, gamma, nullptr, q, scale, m, n, eps, pdl, st)
           : layernorm_t<__nv_bfloat16, false>(x, gamma, nullptr, q, scale, m, n, eps, pdl, st);
}

int launch_gelu_quant(const void* x, void* q, void* scales, void* tmp, int m, int n, bool pdl, cudaStream_t st) {
  if (m == 0) return 0;
  if (n % 8 == 0 && aligned16(x) && aligned16(q) && aligned16(tmp))
    return launch_rows(gelu_quant_kernel<8>, m, n / 8, pdl, st, x, q, scales, tmp, n);
  return launch_rows(gelu_quant_kernel<1>, m, n, pdl, st, x, q, scales, tmp, n);
}

}  // namespace b200awq
