// The LM head: logits[i, v] = (float) rn_T( sum_k x^[i, k] W[v, k] ) for 1 <= m <= 8 rows, with x^ = x or, with gamma,
// x^ = RMSNorm(x, gamma, eps) bit for bit as rmsnorm.cu writes it (DESIGN §3.13).  One launch, no workspace, no atomics.
//
// HBM-bound: the dense [vocab, k] weight is read once.  One persistent CTA per SM owns a contiguous block of vocabulary
// rows, i.e. one contiguous byte range of W whatever k is.  A producer warp streams that range into a ring of
// shared-memory slots of whole rows with bulk copies (its first lap before griddepcontrol.wait: W does not depend on the
// previous grid); eight consumer warps read x (after the wait) into shared memory once, normalise it with the NORM
// prologue, and then take the block's rows round robin, row r on warp r % 8.
//
// Summation order of a logit, a function of k alone: lane l of the row's warp owns the 8-element chunks l, l + 32, ...
// of the row and accumulates them in increasing order with fmaf in element order, starting from 0.f; the 32 lane sums
// meet in an xor butterfly 16, 8, 4, 2, 1.  Neither the row's index, vocab, m, the other rows of x, the grid nor the SM
// count changes it.
#include <algorithm>

#include "rmsnorm_stat.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

constexpr int kHeadConsumerWarps = 8;  // = kNormWarps: the consumers are the norm's 256 threads
constexpr int kHeadThreads = (kHeadConsumerWarps + 1) * 32;  // + one producer warp
constexpr int kHeadSlotBytes = 16384;  // target bytes of one ring slot (whole rows; one row when a row is larger)
constexpr int kHeadMaxSlots = 16;
constexpr int kHeadSmemBudget = 227 * 1024;  // the opt-in dynamic shared memory of one sm_90 CTA
constexpr int kHeadHeader = 2 * kHeadMaxSlots * 8 + kNormWarps * kLmHeadMaxM * 4;  // barriers, warp totals of the norm

struct HeadPlan {
  int rows_per_cta, grid, slot_rows, slots;
  size_t smem;
};

// The plan from the shape and the SM count alone.
HeadPlan head_plan(int m, int vocab, int k, int sms) {
  HeadPlan p{};
  p.rows_per_cta = (vocab + sms - 1) / sms;
  p.grid = (vocab + p.rows_per_cta - 1) / p.rows_per_cta;
  const int row_bytes = k * 2;
  p.slot_rows = std::max(1, kHeadSlotBytes / row_bytes);
  const size_t x_bytes = (size_t)m * k * 2;
  const size_t slot_bytes = (size_t)p.slot_rows * row_bytes;
  p.slots = (int)std::min<size_t>(kHeadMaxSlots, (kHeadSmemBudget - kHeadHeader - x_bytes) / slot_bytes);
  p.smem = kHeadHeader + x_bytes + (size_t)p.slots * slot_bytes;
  return p;
}

struct HeadArgs {
  const void* x;
  long long x_stride;  // elements between rows of x
  const void* gamma;
  float eps;
  const void* w;
  float* logits;
  int vocab, k, rows_per_cta, slot_rows, slots;
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// acc[i] += the 8 products of the chunk (w, x_i) in element order
template <typename T, int M>
__device__ __forceinline__ void chunk_fma(uint4 w, const uint4 (&xv)[M], float (&acc)[M]) {
  const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 wf = pair_to_float2<T>(ww[e]);
#pragma unroll
    for (int i = 0; i < M; ++i) {
      const uint32_t xw = e == 0 ? xv[i].x : e == 1 ? xv[i].y : e == 2 ? xv[i].z : xv[i].w;
      const float2 xf = pair_to_float2<T>(xw);
      acc[i] = fmaf(xf.x, wf.x, acc[i]);
      acc[i] = fmaf(xf.y, wf.y, acc[i]);
    }
  }
}

template <typename T, int M, bool NORM>
__device__ __forceinline__ void lm_head_body(const HeadArgs& a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + kHeadMaxSlots;
  float* red = reinterpret_cast<float*>(empty + kHeadMaxSlots);  // [M][kNormWarps]
  T* xs = reinterpret_cast<T*>(smem + kHeadHeader);               // [M][k]
  unsigned char* ring = smem + kHeadHeader + (size_t)M * a.k * 2;

  const int k = a.k, nchunk = k >> 3, row_bytes = k * 2;
  const int r0 = blockIdx.x * a.rows_per_cta;
  const int nrows = min(a.rows_per_cta, a.vocab - r0);
  const int nslots = (nrows + a.slot_rows - 1) / a.slot_rows;
  const size_t slot_bytes = (size_t)a.slot_rows * row_bytes;
  const unsigned char* wblock = static_cast<const unsigned char*>(a.w) + (size_t)r0 * row_bytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.slots; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kHeadConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp == kHeadConsumerWarps) {  // producer: slot s holds rows [s * slot_rows, ...) of the block
    if (lane != 0) return;
    for (int s = 0; s < nslots; ++s) {
      const int q = s % a.slots;
      if (s >= a.slots) mbar_wait(&empty[q], ((s / a.slots) - 1) & 1);
      const uint32_t bytes = (uint32_t)(min(a.slot_rows, nrows - s * a.slot_rows) * row_bytes);
      mbar_expect_tx(&full[q], bytes);
      bulk_g2s(ring + (size_t)q * slot_bytes, wblock + (size_t)s * slot_bytes, bytes, &full[q]);
    }
    return;
  }

  // consumers: x (and its statistic) after the dependency wait
  pdl_wait_prior_grid();
  const int t = threadIdx.x;  // 0..255: thread t of the norm's summation order
  float ss[M];
#pragma unroll
  for (int i = 0; i < M; ++i) {
    const uint4* xr = reinterpret_cast<const uint4*>(static_cast<const T*>(a.x) + (long long)i * a.x_stride);
    uint4* xd = reinterpret_cast<uint4*>(xs + (size_t)i * k);
    ss[i] = 0.f;
    for (int c = t; c < nchunk; c += kNormThreads) {
      const uint4 v = xr[c];
      if constexpr (NORM) ss[i] = norm_chunk_sumsq<T>(v, ss[i]);
      xd[c] = v;
    }
  }
  if constexpr (NORM) {
#pragma unroll
    for (int i = 0; i < M; ++i) {
      const float s = norm_warp_sum(ss[i]);
      if (lane == 0) red[i * kNormWarps + warp] = s;
    }
    consumer_sync();
    const uint4* gv = reinterpret_cast<const uint4*>(a.gamma);
#pragma unroll
    for (int i = 0; i < M; ++i) {
      const float r = norm_rstd(red + i * kNormWarps, k, a.eps);
      uint4* xd = reinterpret_cast<uint4*>(xs + (size_t)i * k);
      for (int c = t; c < nchunk; c += kNormThreads) {  // the chunks this thread stored above
        const uint4 v = xd[c], g = __ldg(gv + c);
        xd[c] = make_uint4(norm_pair<T>(v.x, g.x, r), norm_pair<T>(v.y, g.y, r), norm_pair<T>(v.z, g.z, r),
                           norm_pair<T>(v.w, g.w, r));
      }
    }
  }
  consumer_sync();

  const uint32_t xs_u32 = smem_u32(xs), ring_u32 = smem_u32(ring);
  float* out = a.logits + r0;
  for (int s = 0; s < nslots; ++s) {
    const int q = s % a.slots;
    mbar_wait(&full[q], (s / a.slots) & 1);
    const int first = s * a.slot_rows, last = min(nrows, first + a.slot_rows);
    for (int r = first + (warp - first % kHeadConsumerWarps + kHeadConsumerWarps) % kHeadConsumerWarps; r < last;
         r += kHeadConsumerWarps) {
      const uint32_t wrow = ring_u32 + (uint32_t)(q * slot_bytes + (size_t)(r - first) * row_bytes);
      float acc[M];
#pragma unroll
      for (int i = 0; i < M; ++i) acc[i] = 0.f;
#pragma unroll 2
      for (int c = lane; c < nchunk; c += 32) {
        const uint4 w = lds128(wrow + c * 16);
        uint4 xv[M];
#pragma unroll
        for (int i = 0; i < M; ++i) xv[i] = lds128(xs_u32 + (uint32_t)(i * row_bytes + c * 16));
        chunk_fma<T, M>(w, xv, acc);
      }
      float mine = 0.f;
#pragma unroll
      for (int i = 0; i < M; ++i) {
        const float v = to_float<T>(from_float<T>(norm_warp_sum(acc[i])));
        if (lane == i) mine = v;
      }
      if (lane < M) out[(size_t)lane * a.vocab + r] = mine;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[q]);
  }
}

}  // namespace

// Named kernels (the plain and the normed head launch under these names in a profile).
template <typename T, int M>
__global__ void __launch_bounds__(kHeadThreads, 1) lm_head_kernel(const HeadArgs a) {
  lm_head_body<T, M, false>(a);
}
template <typename T, int M>
__global__ void __launch_bounds__(kHeadThreads, 1) lm_head_norm_kernel(const HeadArgs a) {
  lm_head_body<T, M, true>(a);
}

namespace {

template <typename T, int M>
int launch_m(const HeadArgs& a0, const HeadPlan& p, bool norm, bool pdl, cudaStream_t stream) {
  constexpr auto plain = lm_head_kernel<T, M>;
  constexpr auto normed = lm_head_norm_kernel<T, M>;
  if (cudaError_t e = norm ? ensure_dyn_smem<normed>(kHeadSmemBudget) : ensure_dyn_smem<plain>(kHeadSmemBudget))
    return (int)e;
  HeadArgs a = a0;
  a.rows_per_cta = p.rows_per_cta, a.slot_rows = p.slot_rows, a.slots = p.slots;
  return launch_kernel(norm ? normed : plain, dim3((unsigned)p.grid), dim3(kHeadThreads), p.smem, stream, pdl, 1, a);
}

template <typename T>
int launch_t(const HeadArgs& a, const HeadPlan& p, int m, bool norm, bool pdl, cudaStream_t stream) {
  switch (m) {
    case 1: return launch_m<T, 1>(a, p, norm, pdl, stream);
    case 2: return launch_m<T, 2>(a, p, norm, pdl, stream);
    case 3: return launch_m<T, 3>(a, p, norm, pdl, stream);
    case 4: return launch_m<T, 4>(a, p, norm, pdl, stream);
    case 5: return launch_m<T, 5>(a, p, norm, pdl, stream);
    case 6: return launch_m<T, 6>(a, p, norm, pdl, stream);
    case 7: return launch_m<T, 7>(a, p, norm, pdl, stream);
    default: return launch_m<T, 8>(a, p, norm, pdl, stream);
  }
}

}  // namespace

int launch_lm_head(const void* x, long long x_row_stride, const void* gamma, float eps, const void* weight, float* logits,
                   int m, int vocab, int k, int dtype, bool pdl, cudaStream_t stream) {
  const int sms = sm_count();
  if (sms < 1) return (int)cudaErrorInvalidDevice;
  const HeadPlan p = head_plan(m, vocab, k, sms);
  const HeadArgs a{x, x_row_stride, gamma, eps, weight, logits, vocab, k, 0, 0, 0};
  const bool norm = gamma != nullptr;
  if (dtype == B200AWQ_DTYPE_F16) return launch_t<__half>(a, p, m, norm, pdl, stream);
  return launch_t<__nv_bfloat16>(a, p, m, norm, pdl, stream);
}

}  // namespace b200awq
