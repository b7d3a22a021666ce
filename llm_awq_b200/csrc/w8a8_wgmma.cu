// Tensor-core W8A8 GEMM for sm_90a: TMA -> 128-byte-swizzled shared memory -> s8 x s8 -> s32 wgmma_ss with both
// operands taken from shared-memory descriptors -> exact int32 accumulators -> the reference's fp32 epilogue -> fp16.
//
// Replaces the reference's dense_kernel0 / dense_kernel0_fuse_bias (w8a8/w8a8_gemm_cuda.cu; Ampere cp.async +
// mma.sync.m16n8k32.s8), behind w8a8_gemm_forward_cuda and w8a8_gemm_fuse_bias_forward_cuda.
//
//   y[m, n] = rn_f16(f32(acc) * (ws[n] * as[m]))                  no bias   (w8a8_gemm_cuda.cu:893-899)
//   y[m, n] = rn_f16(fma(as[m], f32(acc) * ws[n], bias[n]))        bias      (w8a8_gemm_cuda.cu:573-577)
// with acc = sum_k x[m, k] w[n, k] exact in int32, every product / FMA flushing denormals like the reference's
// fast-math build.  Behind b200awq_w8a8_linear the store loop also applies the vision encoder layers' layer scale and
// residual to the rounded y (w8a8_store_epilogue), in instantiations of their own.
//
// Tile: 128 tokens x 128 output channels, 128 k per pipeline stage (one 128-byte swizzle row per token / channel).
//   * x [M, K] int8 and w [N, K] int8, both K-major, arrive by TMA; rows past M / N and k past K are zero-filled, so
//     any k % 16 == 0 (the TMA stride rule) is exact.
//   * wgmma M = 64 tokens per consumer warpgroup (A = x rows from shared memory), N = 128 channels (B = w rows),
//     k = 32 per instruction, 4 per stage; 64 int32 accumulators per thread for the whole k range.
// Warp roles (288 threads, one tile per CTA, two CTAs per SM so that one's epilogue hides under the other's loads):
//   warpgroups 0, 1   wgmma for tokens [0, 64) / [64, 128) of the tile, then the epilogue: fp16 results staged in the
//                     (drained) pipeline buffers, written out as coalesced 16-byte stores masked at the M / N tails
//   warp 8, one thread  TMA producer over a full / empty mbarrier ring
#include "tma_wgmma.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"
#include "w8a8_math.cuh"

namespace b200awq {
namespace {

constexpr int kTM = 128;                      // tokens per tile
constexpr int kTN = 128;                      // output channels per tile
constexpr int kTK = 128;                      // k per stage (bytes per operand row)
constexpr int kStages = 3;
constexpr int kThreads = 288;                 // 2 consumer warpgroups + 1 producer warp
constexpr int kXBytes = kTM * kTK;            // 16 KB
constexpr int kWBytes = kTN * kTK;            // 16 KB
constexpr int kStageBytes = kXBytes + kWBytes;
constexpr int kOutRow = kTN * 2 + 16;         // staged fp16 row (+ pad against bank conflicts)
static_assert(kTM * kOutRow <= kStages * kStageBytes, "epilogue staging must fit in the pipeline buffers");
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 64 /*barriers*/;

__device__ __forceinline__ float ldg_h(const __half* p) { return __half2float(__ldg(p)); }

// The layer scale and residual of b200awq_w8a8_linear on the 8 consecutive fp16 values v of one 16-byte store (the
// tile's rn_f16 outputs), given the matching 16 B of the layer scale (l, if has_ls) and of the residual (r, if has_res):
//   v = rn_f16(f32(v) * f32(l)), then v = rn_f16(f32(r) + f32(v))
// one fp32 operation each, rounded once: PyTorch's fp16 `out * ls` and `residual + out` (products and sums of fp16
// values are exact in fp32 and never subnormal there, so no flush can apply).
__device__ __forceinline__ uint4 w8a8_epilogue_x8(uint4 v, bool has_ls, uint4 l, bool has_res, uint4 r) {
  uint32_t vw[4] = {v.x, v.y, v.z, v.w};
  const uint32_t lw[4] = {l.x, l.y, l.z, l.w}, rw[4] = {r.x, r.y, r.z, r.w};
  auto f = [](uint32_t w, int h) { return __half2float(__ushort_as_half((unsigned short)(w >> (16 * h)))); };
  auto bits = [](float x) { return (uint32_t)__half_as_ushort(__float2half_rn(x)); };
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint32_t o = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t e = (vw[q] >> (16 * h)) & 0xffffu;
      if (has_ls) e = bits(__fmul_rn(f(e, 0), f(lw[q], h)));
      if (has_res) e = bits(__fadd_rn(f(rw[q], h), f(e, 0)));
      o |= e << (16 * h);
    }
    vw[q] = o;
  }
  return make_uint4(vw[0], vw[1], vw[2], vw[3]);
}

// b200awq_w8a8_linear's store loop over the staged fp16 tile (after the staging writes, which the barrier here
// completes): thread e stores pieces e + 256 p of the tile, always the same 8 channels (one layer-scale load) and
// kPieces rows 16 apart.  The residual rows are all loaded right after the barrier, before the first store; loaded
// before it they would be live across the staging, which already fills the 96 registers two CTAs of 9 warps allow.
// Rows at or past M and channels at or past N are neither read nor stored.
__device__ __forceinline__ void w8a8_store_epilogue(const uint8_t* stage_out, __half* __restrict__ y, int M, int N, int m0,
                                                    int n0, const __half* layer_scale, const __half* residual) {
  constexpr int kPieces = kTM * (kTN / 8) / 256;
  const int cc = threadIdx.x & 15, n = n0 + cc * 8, r0 = threadIdx.x >> 4;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  const bool n_ok = n < N;
  const uint4 lv = layer_scale && n_ok ? *reinterpret_cast<const uint4*>(layer_scale + n) : zero;
  const __half* rp = residual + (size_t)(m0 + r0) * N + n;
  asm volatile("bar.sync 1, 256;" ::: "memory");
  uint4 rv[kPieces];
#pragma unroll
  for (int p = 0; p < kPieces; ++p)
    rv[p] = residual && n_ok && m0 + r0 + 16 * p < M ? *reinterpret_cast<const uint4*>(rp + (size_t)p * 16 * N) : zero;
  __half* yp = y + (size_t)(m0 + r0) * N + n;
#pragma unroll
  for (int p = 0; p < kPieces; ++p) {
    if (n_ok && m0 + r0 + 16 * p < M) {
      const uint4 v = *reinterpret_cast<const uint4*>(stage_out + (r0 + 16 * p) * kOutRow + cc * 16);
      *reinterpret_cast<uint4*>(yp + (size_t)p * 16 * N) =
          w8a8_epilogue_x8(v, layer_scale != nullptr, lv, residual != nullptr, rv[p]);
    }
  }
}

// Epi: empty for the GEMM entries' kernels, whose parameters are then exactly the reference epilogue's; or the
// (layer_scale, residual) pointers of b200awq_w8a8_linear, applied by w8a8_store_epilogue in place of the plain store
// loop.  The empty pack keeps the plain instantiations' code and (demangled) names what they were before the epilogue.
template <bool kBias, typename... Epi>
__global__ void __launch_bounds__(kThreads, 2)
w8a8_wgmma_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                  const __half* __restrict__ wscales, const __half* __restrict__ ascales, const __half* __restrict__ bias,
                  __half* __restrict__ y, int M, int N, int K, Epi... epi) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);  // [kStages] TMA -> consumers
  uint64_t* empty = full + kStages;  // [kStages] consumers (8 warps) -> TMA: the stage's wgmmas have completed
  // stage s: x tile at smem + s * kStageBytes, w tile kXBytes further (both 1024-aligned)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * kTN, m0 = blockIdx.y * kTM;
  const int num_kb = (K + kTK - 1) / kTK;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp == 8) {
    // =========================================================== TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tm_x);
      tma_prefetch_desc(&tm_w);
      pdl_wait_prior_grid();  // the activation codes come from the previous kernel in the stream
      int s = 0;
      uint32_t ph = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], kStageBytes);
        uint8_t* st = smem + s * kStageBytes;
        tma_load_2d(st, &tm_x, &full[s], kb * kTK, m0);
        tma_load_2d(st + kXBytes, &tm_w, &full[s], kb * kTK, n0);
        if (++s == kStages) s = 0, ph ^= 1;
      }
    }
    return;
  }

  // =========================================================== wgmma (warpgroups 0, 1)
  const int wg = warp >> 2;
  int acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0;
  int s = 0, prev = 0;
  uint32_t ph = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full[s], ph);
    const uint32_t st = smem_u32(smem + s * kStageBytes);
    const uint64_t adesc = make_sw128_desc(st + wg * 64 * kTK);
    const uint64_t bdesc = make_sw128_desc(st + kXBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTK / 32; ++kk)  // +32 B along k per instruction
      wgmma_ss(acc, adesc + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), (kb | kk) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();  // the previous stage's wgmmas have completed: its buffers may be refilled
    acc_fence(acc);
    if (kb > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    prev = s;
    if (++s == kStages) s = 0, ph ^= 1;
  }
  wgmma_wait<0>();
  acc_fence(acc);

  // ------------------------------------------------ epilogue
  pdl_wait_prior_grid();  // scales and bias may come from the previous kernel too (a no-op once the producer waited)
  // every wgmma of both warpgroups has completed and every TMA load has landed: the pipeline buffers are free
  asm volatile("bar.sync 1, 256;" ::: "memory");
  uint8_t* stage_out = smem;  // [kTM][kOutRow] fp16
  // acc[4 j + e]: token 16 (warp & 3) + g + 8 (e >> 1) of this warpgroup's 64, channel 8 j + 2 t + (e & 1)
  const int g = lane >> 2, t = lane & 3;
  const int r_lo = wg * 64 + (warp & 3) * 16 + g;
  float as_lo = 0.f, as_hi = 0.f;
  if (m0 + r_lo < M) as_lo = ldg_h(ascales + m0 + r_lo);
  if (m0 + r_lo + 8 < M) as_hi = ldg_h(ascales + m0 + r_lo + 8);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = 8 * j + 2 * t;
    float ws0 = 0.f, ws1 = 0.f, b0 = 0.f, b1 = 0.f;
    if (n0 + c < N) {  // n % 8 == 0: both channels of the pair are in range or neither is
      ws0 = ldg_h(wscales + n0 + c), ws1 = ldg_h(wscales + n0 + c + 1);
      if constexpr (kBias) b0 = ldg_h(bias + n0 + c), b1 = ldg_h(bias + n0 + c + 1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float as = h ? as_hi : as_lo;
      float v0, v1;
      if constexpr (kBias) {
        v0 = ffma_ftz(fmul_ftz(s32_to_f32(acc[4 * j + 2 * h]), ws0), as, b0);
        v1 = ffma_ftz(fmul_ftz(s32_to_f32(acc[4 * j + 2 * h + 1]), ws1), as, b1);
      } else {
        v0 = fmul_ftz(s32_to_f32(acc[4 * j + 2 * h]), fmul_ftz(ws0, as));
        v1 = fmul_ftz(s32_to_f32(acc[4 * j + 2 * h + 1]), fmul_ftz(ws1, as));
      }
      *reinterpret_cast<__half2*>(stage_out + (r_lo + 8 * h) * kOutRow + c * 2) = __floats2half2_rn(v0, v1);
    }
  }
  if constexpr (sizeof...(Epi) != 0) {
    w8a8_store_epilogue(stage_out, y, M, N, m0, n0, epi...);
  } else {
    asm volatile("bar.sync 1, 256;" ::: "memory");
    for (int e = threadIdx.x; e < kTM * (kTN / 8); e += 256) {
      const int r = e >> 4, cc = e & 15;
      const int m = m0 + r, n = n0 + cc * 8;
      if (m < M && n < N)
        *reinterpret_cast<uint4*>(y + (size_t)m * N + n) = *reinterpret_cast<const uint4*>(stage_out + r * kOutRow + cc * 16);
    }
  }
}

int encode_kmajor_s8(EncodeTiledFn enc, CUtensorMap* tm, const void* p, int rows, int K, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K};
  cuuint32_t box[2] = {(cuuint32_t)kTK, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(p), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : B200AWQ_ERR_DRIVER;
}

}  // namespace

int launch_w8a8_gemm(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias, void* y,
                     int M, int N, int K, bool pdl, cudaStream_t stream, const void* layer_scale, const void* residual) {
  if (M < 1 || N < 8 || N % 8 || K < 16 || K % 16) return B200AWQ_ERR_SHAPE;
  EncodeTiledFn enc = get_encoder();
  if (!enc) return B200AWQ_ERR_DRIVER;
  CUtensorMap tm_x, tm_w;
  if (int e = encode_kmajor_s8(enc, &tm_x, x, M, K, kTM)) return e;
  if (int e = encode_kmajor_s8(enc, &tm_w, w, N, K, kTN)) return e;
  const dim3 grid((unsigned)((N + kTN - 1) / kTN), (unsigned)((M + kTM - 1) / kTM));
  if (layer_scale || residual) {  // b200awq_w8a8_linear's instantiations, only when either operand is given
    using P = const __half*;
    auto kern = bias ? w8a8_wgmma_kernel<true, P, P> : w8a8_wgmma_kernel<false, P, P>;
    const cudaError_t ea = bias ? ensure_dyn_smem<w8a8_wgmma_kernel<true, P, P>>(kSmemBytes)
                                : ensure_dyn_smem<w8a8_wgmma_kernel<false, P, P>>(kSmemBytes);
    if (ea) return (int)ea;
    return launch_kernel(kern, grid, dim3(kThreads), kSmemBytes, stream, pdl, 1, tm_x, tm_w, wscales, ascales, bias, y, M, N,
                         K, static_cast<P>(layer_scale), static_cast<P>(residual));
  }
  auto kern = bias ? w8a8_wgmma_kernel<true> : w8a8_wgmma_kernel<false>;
  const cudaError_t ea = bias ? ensure_dyn_smem<w8a8_wgmma_kernel<true>>(kSmemBytes)
                              : ensure_dyn_smem<w8a8_wgmma_kernel<false>>(kSmemBytes);
  if (ea) return (int)ea;
  return launch_kernel(kern, grid, dim3(kThreads), kSmemBytes, stream, pdl, 1, tm_x, tm_w, wscales, ascales, bias, y, M, N, K);
}

}  // namespace b200awq
