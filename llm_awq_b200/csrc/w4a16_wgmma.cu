// Tensor-core W4A16 kernel for sm_90a: TMA -> shared memory -> register dequantisation straight into the
// wgmma A fragment -> wgmma_rs with the activation tile as the shared-memory B operand.
//
// Replaces the reference's gemm_w4a16_T1 / gemm_w4a16_T2 (quantization_new/gemm/gemm_cuda.cu:312-752, :922-1124;
// Ampere cp.async + ldmatrix + mma.sync) and, for 128-channel-aligned layers, the small-M split-K tiles of its
// GEMV / GEMM (gemv_cuda.cu:74-229, gemm_cuda.cu:1155-1206).
//
// Orientation: the tile is computed TRANSPOSED, D[oc, tok] = W~[oc, k] . X[tok, k]^T.
//   * wgmma M = 64 output channels per consumer warpgroup, two consumer warpgroups = 128 channels per tile.
//     The A operand comes from REGISTERS: in the packed format (w4_common.cuh) word t of a (channel, 32-k block)
//     chunk dequantises to the k pairs 2t, 2t + 8, 2t + 16, 2t + 24, which is exactly what lane (g, t) of an
//     m16n8k16 / wgmma A fragment holds for two k16 steps.  So a thread reads 4 words per 64-k stage (2 channels x
//     2 blocks), applies scale / zero with one exact FMA per pair (operand bits equal the reference's) and hands the
//     registers to wgmma: the dequantised weights never touch shared memory.
//   * wgmma N = TN tokens (16..128).  The activation tile X[tok, 64 k] arrives by TMA with the 128-byte swizzle and
//     is consumed in place as the K-major B operand.
//   * D (64 channels x TN fp32 per warpgroup) stays in registers for the whole k range.
// Warp roles (384 threads, persistent over output tiles):
//   warpgroup 0, one thread   TMA producer (activation tile + packed-weight tile per stage)
//   warpgroups 1, 2           dequantise + wgmma for channels [0, 64) / [64, 128) of the tile (each waits for its
//                             wgmmas before the next stage reuses the A registers; the two warpgroups overlap);
//                             epilogue through a shared-memory transpose into coalesced 16-byte stores
// Small token counts: the k range is split over a thread-block cluster (2..8 CTAs share a tile) and the fp32 partial
// tiles are reduced through distributed shared memory in the epilogue (mbarriers with cluster scope, fixed order).
#include "tma_wgmma.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

constexpr int kBM = 128;        // output channels per tile
constexpr int kBK = 64;         // k per pipeline stage
constexpr int kWgThreads = 384;  // producer warpgroup + 2 consumer warpgroups
constexpr int kWBytes = kBM * kBK / 2;  // 4096: packed weights per stage

// ---------------------------------------------------------------- cluster-scope mbarrier helpers (split-K)
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* local_bar, uint32_t rank) {
  const uint32_t a = map_to_rank(smem_u32(local_bar), rank);
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(a) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}

// add_epilogue over the 8 consecutive elements of one 16-byte store of y, given the matching 16 B of the bias (b, if
// has_bias) and of the residual (r, if has_res).  Works on the 16-bit halves of 32-bit words (no local arrays).
template <typename T>
__device__ __forceinline__ uint4 add_epilogue_x8(uint4 v, bool has_bias, uint4 b, bool has_res, uint4 r) {
  auto f = [](uint32_t w, int h) {  // element h of word w as fp32
    const unsigned short b = (unsigned short)(w >> (16 * h));
    if constexpr (TypeTraits<T>::kIsBf16) return __bfloat162float(__ushort_as_bfloat16(b));
    else return __half2float(__ushort_as_half(b));
  };
  auto bits = [](float x) -> uint32_t {
    if constexpr (TypeTraits<T>::kIsBf16) return __bfloat16_as_ushort(from_float<T>(x));
    else return __half_as_ushort(from_float<T>(x));
  };
  uint32_t vw[4] = {v.x, v.y, v.z, v.w};
  const uint32_t bw[4] = {b.x, b.y, b.z, b.w}, rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint32_t o = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // add_epilogue, element by element
      uint32_t e = (vw[q] >> (16 * h)) & 0xffffu;
      if (has_bias) e = bits(f(e, 0) + f(bw[q], h));
      if (has_res) e = bits(f(rw[q], h) + f(e, 0));
      o |= e << (16 * h);
    }
    vw[q] = o;
  }
  return make_uint4(vw[0], vw[1], vw[2], vw[3]);
}

template <int TN>
struct WgSmem {
  static constexpr int kXBytes = TN * 128;  // TN token rows x 64 k x 2 B (a multiple of 1024: stages stay aligned)
  static constexpr int kStageBytes = kXBytes + kWBytes;
  static constexpr int kStages = (160 * 1024) / kStageBytes >= 8 ? 8 : (160 * 1024) / kStageBytes;
  static constexpr int kOutRow = 256 + 16;             // 128 channels x 2 B (+ pad)
  static constexpr int kOutBytes = TN * kOutRow;       // epilogue transpose (no split)
  static constexpr int kPartBytes = TN * kBM * 4;      // fp32 partial tile (split-K)
  static constexpr int kEpiBytes = kOutBytes > kPartBytes ? kOutBytes : kPartBytes;
  static constexpr int kTotal = kStages * kStageBytes + kEpiBytes + 1024 /*align*/ + 256 /*barriers*/;
};

// EPI: bias / residual (either may be null) are added to each stored value (add_epilogue).  TN stays the last template
// argument: tests read the token tile from the end of the kernel's name.
template <typename T, bool EPI, int TN>
__global__ void __launch_bounds__(kWgThreads, 1)
w4a16_wgmma_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                   const T* __restrict__ scales, const T* __restrict__ szeros, T* __restrict__ y, int M, int N, int K, int S,
                   const T* __restrict__ bias, const T* __restrict__ residual) {
  using L = WgSmem<TN>;
  constexpr int STAGES = L::kStages;
  constexpr int NA = TN / 2;  // accumulator registers per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* xs = smem;                              // [STAGES][TN * 128]   (1024-aligned each)
  uint8_t* ws = xs + STAGES * L::kXBytes;          // [STAGES][4096]
  uint8_t* epi = ws + STAGES * kWBytes;            // [TN][kOutRow] T  or  [TN][128] fp32 partial tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi + L::kEpiBytes);
  uint64_t* full = bars;             // [STAGES]  TMA -> consumers
  uint64_t* empty = full + STAGES;   // [STAGES]  consumers (8 warps) -> TMA: the stage's wgmmas have completed
  uint64_t* pfull = empty + STAGES;  // split-K: every rank's partial tile is written   (8 S remote arrivals)
  uint64_t* pempty = pfull + 1;      // split-K: every rank has finished reading MY tile (8 S remote arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tok_tiles = (M + TN - 1) / TN;
  const int num_tiles = tok_tiles * (N / kBM);
  // split-K over a thread-block cluster: rank r of S owns k blocks [kb0, kb0 + num_kb) of the SAME tile; the cluster
  // walks the tiles together
  const int crank = (S > 1) ? (int)cluster_ctarank() : 0;
  const int num_kb = K / kBK / S;
  const int kb0 = crank * num_kb;
  const int tile0 = (int)(blockIdx.x / S);
  const int tile_step = (int)(gridDim.x / S);
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    mbar_init(pfull, 8 * S);
    mbar_init(pempty, 8 * S);
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
  }
  __syncthreads();
  if (S > 1) cluster_sync_all();  // remote mbarrier arrivals must not race the inits

  pdl_launch_dependents();

  if (warp < 4) {
    // =========================================================== TMA producer
    if (threadIdx.x == 0) {
      pdl_wait_prior_grid();  // activations come from the previous kernel in the stream
      int s = 0;
      uint32_t ph = 0;
      for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        const int oc_tile = tile / tok_tiles, tok_tile = tile % tok_tiles;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          mbar_expect_tx(&full[s], L::kXBytes + kWBytes);
          tma_load_2d(xs + s * L::kXBytes, &tm_x, &full[s], (kb0 + kb) * kBK, tok_tile * TN);
          tma_load_2d(ws + s * kWBytes, &tm_w, &full[s], (kb0 + kb) * kBK, oc_tile * (kBM / 4));
          if (++s == STAGES) s = 0, ph ^= 1;
        }
      }
    }
  } else {
    // =========================================================== dequant + wgmma + epilogue (warpgroups 1, 2)
    const int ct = threadIdx.x - 128;            // 0..255 among the consumers
    const int wg = ct >> 7;                      // channel half of the tile
    const int g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;  // this thread's two channels inside the tile: r0, r0 + 8
    // byte offset of word t of (channel r, 32-k block 0) in a stage's weight tile (4 channels x 2 blocks per 128 B)
    const int wo0 = (r0 >> 2) * 128 + (r0 & 3) * 32 + t * 4;
    const int wo1 = ((r0 + 8) >> 2) * 128 + ((r0 + 8) & 3) * 32 + t * 4;
    const int ngk = num_kb / 2;  // 128-k groups of this rank's k range (num_kb is even)
    int s = 0;
    uint32_t ph = 0, pph = 0;
    float acc[NA];
#pragma unroll
    for (int i = 0; i < NA; ++i) acc[i] = 0.f;
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const int oc_tile = tile / tok_tiles, tok_tile = tile % tok_tiles;
      const int n0 = oc_tile * kBM + r0;
      const uint16_t* sp = reinterpret_cast<const uint16_t*>(scales) + (size_t)(kb0 / 2) * N + n0;
      const uint16_t* zp = reinterpret_cast<const uint16_t*>(szeros) + (size_t)(kb0 / 2) * N + n0;
      // scale / zero of both channels, one 128-k group ahead
      uint16_t ns0 = __ldg(sp), ns1 = __ldg(sp + 8), nz0 = __ldg(zp), nz1 = __ldg(zp + 8);
      uint32_t s0 = 0, s1 = 0, z0 = 0, z1 = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        if ((kb & 1) == 0) {
          s0 = splat16(ns0), s1 = splat16(ns1), z0 = splat16(nz0), z1 = splat16(nz1);
          const int gn = kb / 2 + 1;
          if (gn < ngk) {
            ns0 = __ldg(sp + (size_t)gn * N), ns1 = __ldg(sp + (size_t)gn * N + 8);
            nz0 = __ldg(zp + (size_t)gn * N), nz1 = __ldg(zp + (size_t)gn * N + 8);
          }
        }
        mbar_wait(&full[s], ph);
        const uint8_t* wst = ws + s * kWBytes;
        uint32_t q0[2][4], q1[2][4];  // [32-k block][pair j]: channel r0 / r0 + 8
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          dequant_word<T>(*reinterpret_cast<const uint32_t*>(wst + wo0 + b * 16), s0, z0, q0[b]);
          dequant_word<T>(*reinterpret_cast<const uint32_t*>(wst + wo1 + b * 16), s1, z1, q1[b]);
        }
        const uint64_t bdesc = make_sw128_desc(smem_u32(xs + s * L::kXBytes));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          // k16 step kk = block kk / 2, pairs j = 2 (kk & 1) (k 2t) and j + 1 (k 2t + 8)
          const int b = kk >> 1, j = 2 * (kk & 1);
          const uint32_t a[4] = {q0[b][j], q1[b][j], q0[b][j + 1], q1[b][j + 1]};
          wgmma_rs<T, TN, false>(acc, a, bdesc + (uint64_t)(kk * 2) /* +32 B */, (kb | kk) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        // The A fragments live in registers that the next stage's dequantisation overwrites (ptxas reuses them), so
        // this stage's wgmmas must have completed first; the other consumer warpgroup keeps the tensor core busy.
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);  // the stage's shared memory may be refilled
        if (++s == STAGES) s = 0, ph ^= 1;
      }
      acc_fence(acc);

      // ------------------------------------------------ epilogue for this tile
      // acc[4 i + e]: channel r0 + 8 (e >> 1), token 8 i + 2 t + (e & 1)
      // The consumers already follow the producer's griddepcontrol.wait (through the full barriers); their own wait
      // makes the stream order of bias / residual explicit and returns at once.
      if (EPI) pdl_wait_prior_grid();
      if (S > 1) {
        // split-K: fp32 partial tile -> own shared memory; every rank then reduces TN / S tokens of the tile over
        // distributed shared memory and stores them (no atomics, fixed summation order)
        float* pbuf = reinterpret_cast<float*>(epi);  // [TN][128]
        mbar_wait_cluster(pempty, pph ^ 1);            // all ranks have finished reading my previous partial tile
#pragma unroll
        for (int i = 0; i < NA; ++i) pbuf[(8 * (i >> 2) + 2 * t + (i & 1)) * kBM + r0 + 8 * ((i >> 1) & 1)] = acc[i];
        __syncwarp();
        if (lane == 0)
          for (int r = 0; r < S; ++r) mbar_arrive_remote(pfull, (uint32_t)r);
        mbar_wait_cluster(pfull, pph);  // every rank's partial tile is in its shared memory
        const int tpr = (TN + S - 1) / S;  // S need not divide TN (any S <= 8 dividing the group count)
        const uint32_t base = smem_u32(pbuf);
        for (int e = ct; e < tpr * kBM; e += 256) {
          const int tt = crank * tpr + e / kBM, ch = e % kBM;
          const int tok = tok_tile * TN + tt;
          if (tt < TN && tok < M) {
            float v = 0.f;
            for (int r = 0; r < S; ++r) v += ld_cluster_f32(map_to_rank(base + (uint32_t)(tt * kBM + ch) * 4u, (uint32_t)r));
            const size_t i = (size_t)tok * N + oc_tile * kBM + ch;
            y[i] = EPI ? add_epilogue<T>(from_float<T>(v), bias, residual, (size_t)(oc_tile * kBM + ch), i) : from_float<T>(v);
          }
        }
        __syncwarp();
        if (lane == 0)
          for (int r = 0; r < S; ++r) mbar_arrive_remote(pempty, (uint32_t)r);
        pph ^= 1;
      } else {
#pragma unroll
        for (int i = 0; i < NA; ++i) {
          const int tok = 8 * (i >> 2) + 2 * t + (i & 1), ch = r0 + 8 * ((i >> 1) & 1);
          *reinterpret_cast<T*>(epi + tok * L::kOutRow + ch * 2) = from_float<T>(acc[i]);
        }
        if constexpr (EPI) {
          // the 16-byte stores below, thread ct taking pieces ct + 256 p: always the same 8 channels (one bias load),
          // TN / 16 token rows.  Bias and residual are loaded BEFORE the barrier, so that their latency overlaps the
          // wait for the other warps' staging.
          constexpr int kPieces = TN / 16;
          const int cc = ct & 15;
          const size_t n = (size_t)oc_tile * kBM + cc * 8;
          const uint4 zero = make_uint4(0, 0, 0, 0);
          const uint4 bv = bias ? *reinterpret_cast<const uint4*>(bias + n) : zero;
          uint4 rv[kPieces];
#pragma unroll
          for (int p = 0; p < kPieces; ++p) {
            const int tok = tok_tile * TN + (ct >> 4) + 16 * p;
            rv[p] = residual && tok < M ? *reinterpret_cast<const uint4*>(residual + (size_t)tok * N + n) : zero;
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
          for (int p = 0; p < kPieces; ++p) {
            const int rr = (ct >> 4) + 16 * p, tok = tok_tile * TN + rr;
            if (tok < M) {
              const uint4 v = *reinterpret_cast<const uint4*>(epi + rr * L::kOutRow + cc * 16);
              *reinterpret_cast<uint4*>(y + (size_t)tok * N + n) = add_epilogue_x8<T>(v, bias, bv, residual, rv[p]);
            }
          }
        } else {
          asm volatile("bar.sync 1, 256;" ::: "memory");
          for (int e = ct; e < TN * 16; e += 256) {
            const int rr = e >> 4, cc = e & 15;
            const int tok = tok_tile * TN + rr;
            if (tok < M)
              *reinterpret_cast<uint4*>(y + (size_t)tok * N + oc_tile * kBM + cc * 8) =
                  *reinterpret_cast<const uint4*>(epi + rr * L::kOutRow + cc * 16);
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");  // staging buffer free for the next tile
      }
    }
    if (S > 1) mbar_wait_cluster(pempty, pph ^ 1);  // nobody is still reading my last partial tile
  }

  __syncwarp();
  if (S > 1) cluster_sync_all();  // no CTA of the cluster exits while a peer may still touch its shared memory
}

// ------------------------------------------------------------------------------------ host
// max_clusters <= 0: one cluster per tile (all resident at once when they fit); else a persistent grid of that many
template <typename T, int TN, bool EPI>
static int launch_wgmma_t(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K,
                          bool pdl, int max_clusters, int S, const Epilogue& epi, cudaStream_t stream) {
  using L = WgSmem<TN>;
  EncodeTiledFn enc = get_encoder();
  if (!enc) return B200AWQ_ERR_DRIVER;
  CUtensorMap tm_x, tm_w;
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)TN};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tm_x, TypeTraits<T>::kIsBf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                     const_cast<void*>(x), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return B200AWQ_ERR_DRIVER;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)(N / 4)};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)(kBM / 4)};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(qw), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return B200AWQ_ERR_DRIVER;
  }
  if (cudaError_t ea = ensure_dyn_smem<w4a16_wgmma_kernel<T, EPI, TN>>(L::kTotal)) return (int)ea;
  const int tiles = ((M + TN - 1) / TN) * (N / kBM);
  int clusters = tiles;
  if (max_clusters > 0 && max_clusters < clusters) clusters = max_clusters;
  return launch_kernel(w4a16_wgmma_kernel<T, EPI, TN>, dim3((unsigned)(clusters * S)), dim3(kWgThreads), (size_t)L::kTotal,
                       stream, pdl, (unsigned)S, tm_x, tm_w, sc, sz, y, M, N, K, S, epi.bias, epi.residual);
}

template <typename T, bool EPI>
static int launch_wgmma_tn(int tn, const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N,
                           int K, bool pdl, int max_clusters, int S, const Epilogue& epi, cudaStream_t stream) {
  switch (tn) {
    case 16: return launch_wgmma_t<T, 16, EPI>(x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
    case 32: return launch_wgmma_t<T, 32, EPI>(x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
    case 64: return launch_wgmma_t<T, 64, EPI>(x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
    default: return launch_wgmma_t<T, 128, EPI>(x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
  }
}

static int launch_wgmma(int tn, const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K,
                        int dtype, bool pdl, int max_clusters, int S, const Epilogue& epi, cudaStream_t stream) {
  const bool f16 = dtype == B200AWQ_DTYPE_F16;
  if (epi.on())
    return f16 ? launch_wgmma_tn<__half, true>(tn, x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream)
               : launch_wgmma_tn<__nv_bfloat16, true>(tn, x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
  return f16 ? launch_wgmma_tn<__half, false>(tn, x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream)
             : launch_wgmma_tn<__nv_bfloat16, false>(tn, x, qw, sc, sz, y, M, N, K, pdl, max_clusters, S, epi, stream);
}

int launch_umma(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi) {
  if (M < 1 || N % kBM || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int sms = sm_count();
  if (sms == 0) return B200AWQ_ERR_DEVICE;
  // joint choice of the token tile and the k split by a small cost model (cycles per CTA, estimated): a 64-k stage
  // costs max(dequantisation ~400, wgmma 4 * tn + 100), a tile's epilogue ~10 tn (+6000 when the partial tiles of
  // a split are reduced over the cluster), a launch ~12000; makespan = waves x that.  A split (cluster of S CTAs on
  // one tile) needs tn <= 64, S dividing the group count and >= 512 k per CTA.
  int tn = 16, S = 1;
  long best = -1;
  for (int c = 128; c >= 16; c >>= 1) {
    if (c > 16 && c / 2 >= M) continue;
    const int tiles = ((M + c - 1) / c) * (N / kBM);
    for (int sp = 1; sp <= 8; sp *= 2) {
      if (sp > 1 && (c > 64 || (K / kGroup) % sp || K / sp < 512)) continue;
      const long per_tile = (long)(K / kBK / sp) * (4 * c + 100 > 400 ? 4 * c + 100 : 400) + 10 * c + (sp > 1 ? 6000 : 0);
      const long slots = sms / sp;  // clusters that run at once
      const long cost = 12000 + ((tiles + slots - 1) / slots) * per_tile;
      if (best < 0 || cost < best) best = cost, tn = c, S = sp;
    }
  }
  // a persistent grid of one CTA per SM
  return launch_wgmma(tn, x, qw, sc, sz, y, M, N, K, dtype, pdl, sms / S > 0 ? sms / S : 1, S, epi, stream);
}

// Skinny batches (HBM-bound): one 16-token tile, one CTA per 128 output channels and k slice, every CTA resident at
// once so that several stream their weights per SM.  The k split is the smallest (<= 8, dividing the group count)
// whose slice is <= 512 k, or <= 1024 k once there are at least two CTAs per SM.
int launch_flat(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi) {
  if (M < 1 || M > 16 || N % kBM || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int groups = K / kGroup;
  const int sms = sm_count();
  if (sms == 0) return B200AWQ_ERR_DEVICE;
  int S = 1;
  for (int s = 1; s <= 8; ++s) {
    if (groups % s) continue;
    S = s;
    const int kc = K / s;
    if (kc <= 512) break;
    if (kc <= 1024 && (N / kBM) * s >= 2 * sms) break;
  }
  return launch_wgmma(16, x, qw, sc, sz, y, M, N, K, dtype, pdl, 0, S, epi, stream);
}

}  // namespace b200awq
