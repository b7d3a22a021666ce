// Persistent, warp-specialised W4A16 decode kernel for SEVERAL tokens (2 <= M <= 4 by dispatch, up to 8) and for bf16:
// fp16 / bf16 tensor-core MACs with the tokens in the MMA columns.  (One fp16 token is served by w4a16_decode.cu, the
// third generation of this structure: 8 KB copies instead of the 4 KB ones below, int8-digit MACs.)
//
// Replaces the reference's gemv_kernel (quantization_new/gemv/gemv_cuda.cu:74-229).  Design:
//   * ONE CTA per SM per launch (grid = #SMs), ~95 KB of shared memory and <= 102 registers per thread, so the
//     CTAs of TWO consecutive launches co-reside on every SM: with programmatic dependent launch the next
//     layer's CTA fills its whole ring with weights while this layer is still computing.  No CTA churn: the
//     per-CTA prologue (barrier init, activation staging, group sums) is paid once per SM per launch.
//   * the weight stream is a 5-slot ring in shared memory.  A slot is 16 output channels x 2048 input channels
//     (16 KB packed + 1 KB of scales / zeros).  One PRODUCER warp fills it: lane 0 issues four 4 KB bulk-async
//     copies (cp.async.bulk -> UBLKCP; a 4-row "quad" of the packed layout is contiguous over k), all lanes
//     fetch the slot's scales / zeros with 16-byte cp.async; everything completes on the slot's `full` mbarrier.
//     The producer never waits for the activations, so it runs ahead of griddepcontrol.wait.
//   * 8 CONSUMER warps split the slot's 16 groups of 128 input channels.  Quad rows are placed 4 KB + 16 B
//     apart, which makes the eight 16-byte rows of every ldmatrix phase hit eight different bank groups: the
//     packed words go shared -> registers with ldmatrix.x4 at full shared-memory bandwidth (a plain layout
//     has 2-way conflicts on every weight read).  ldmatrix hands lane (g, tig) word `tig` of the chunk
//     (channel g, 32-k block m) for m = 0..3; one LOP3 per nibble pair turns it into the A operand of
//     m16n8k16 tensor-core MACs (rows = 16 channels, columns = tokens, fp32 accumulate).  The activations are
//     staged ONCE per CTA in the matching order, so every B fragment is an aligned register pair.
//   * fp16 (MODE 2): operands are the raw biased LOP3 outputs (1024+q | 64+q); scale, zero and bias are applied
//     per 128-k group in fp32, y += s*(acc - C) + z*X with X = sum x, C = 1024 X_lo + 64 X_hi computed once per
//     CTA.  bf16 (MODE 0): operands rn_bf16(q*s + z), bit-identical to the reference's.
//   * work split: the N/8 channel octets are dealt evenly to clusters of two CTAs; inside a cluster rank r
//     takes half of k for all of the cluster's channels (balance 98.8 % on 4096 x 4096 where whole-row-block
//     granularity gives 86 %).  A FINISHER warp sums the 8 consumer warps' partials of a row block in a fixed
//     order; rank 1 pushes its sums into rank 0's shared memory with st.async (completing bytes on an mbarrier:
//     no cluster barrier or fence after the math), rank 0 adds and stores y.  Deterministic, no atomics, no
//     workspace.
//
// Contract notes: the packed weights / scales / zeros are read BEFORE griddepcontrol.wait, i.e. they must not be
// produced by the kernel that immediately precedes this launch in the stream (weights are constants in inference);
// x and y are only touched after the wait.
#include <algorithm>

#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

#ifdef B200AWQ_TRACE
extern __device__ unsigned long long g_trace_buf[1024 * 2 * 8];  // defined in w4a16_stream.cu (trace build, -rdc)
__device__ __forceinline__ unsigned long long ring_globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define RING_STAMP(ev)                                                       \
  if (lane == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1))       \
  g_trace_buf[(((unsigned)a.seq & 1023u) * 2 + (blockIdx.x != 0)) * 8 + (ev)] = ring_globaltimer_ns()
// per-warp cycle accounting of CTA 0 (last launch wins): [warp 0..10][0..3] = cycles waiting / working / hand-off / count
__device__ long long g_ring_dbg[20 * 4];
__device__ int g_ring_dbg_flags;  // bit 0: consumers skip the math (streaming limit of the ring), bit 1: skip x staging
#define RING_CLK(var) const long long var = clock64()
#define RING_ACC(slot, expr) dbg_acc[slot] += (expr)
#define RING_DBG_DECL long long dbg_acc[4] = {0, 0, 0, 0}; const int dbg_flags = g_ring_dbg_flags
#define RING_DBG_FLUSH(w)                                        \
  if (lane == 0 && blockIdx.x == 0)                              \
    for (int i_ = 0; i_ < 4; ++i_) g_ring_dbg[(w) * 4 + i_] = dbg_acc[i_]
#define RING_DRY (dbg_flags & 1)
#else
#define RING_STAMP(ev)
#define RING_CLK(var)
#define RING_ACC(slot, expr)
#define RING_DBG_DECL
#define RING_DBG_FLUSH(w)
#define RING_DRY 0
#endif

constexpr int kRingCons = 8;                          // consumer warps
constexpr int kRingProd = 2;                          // producer warps (one thread's bulk-copy issue rate is ~45 B/clk)
constexpr int kRingThreads = (kRingCons + kRingProd + 1) * 32;  // + finisher warp
constexpr int kSlotGroups = 16;                       // 128-k groups per ring slot
constexpr int kQS = kSlotGroups * 256 + 16;           // bytes between the 4 quad rows of a slot (bank skew)
constexpr int kSlotW = 4 * kQS;                       // packed weights of a slot; then scales [16][16], zeros [16][16]
constexpr int kSlotBytes = ((kSlotW + 1024 + 127) / 128) * 128;
constexpr int kRingMaxRb = 128;                       // row blocks per CTA the exchange buffers are sized for

struct RingLayout {
  int bars, x, xsum, red, xchg, ring, total;
  int xrow;  // bytes per staged token
  int ngr;   // groups per rank (upper bound, xsum row length)
};

struct RingArgs {
  const void* x;
  const uint16_t* qw;
  const void* sc;
  const void* sz;
  void* y;
  int M, N, K;
  int S;      // CTAs per cluster = k split (1 or 2)
  int units;  // clusters
  int NS;     // ring slots
  int Mp;     // power of two >= M
  int nrb_max;  // most row blocks any CTA owns
  int seq;
  RingLayout L;
};

__device__ __forceinline__ void ring_cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void ring_cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint16_t lds16(uint32_t addr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kRingCons * 32) : "memory"); }

// One 128-k group of one row block, one warp: 16 (TWO) or 8 channels x 128 input channels.
//   wsrc  this lane's ldmatrix row address (channel lane & 7, 32-k block lane >> 3) of the first octet
//   xsrc  this lane's 64 bytes of staged activations (token g, word slot tig) of the group
//   ssrc  &scales[group][channel g] in the slot (zeros 512 B further, channel 8 + g 16 B further)
//   csrc  &xsum[token 2 tig][group] (MODE 2)
template <typename T, int MODE, bool M1, bool TWO>
__device__ __forceinline__ void group_step(uint32_t wsrc, uint32_t xsrc, uint32_t ssrc, const float2* csrc, int cstride,
                                           bool live, uint32_t (&xq)[16], float (&yacc)[4], float (&yacc2)[4]) {
  constexpr bool kBf16 = TypeTraits<T>::kIsBf16;
  uint32_t wa[4], wb[4] = {0u, 0u, 0u, 0u};
  ldsm4(wa, wsrc);
  if (TWO) ldsm4(wb, wsrc + 2 * kQS);
  if (live) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint4 v = lds128(xsrc + q * 16);
      xq[4 * q] = v.x, xq[4 * q + 1] = v.y, xq[4 * q + 2] = v.z, xq[4 * q + 3] = v.w;
    }
  }
  const uint16_t s_a = lds16(ssrc), z_a = lds16(ssrc + 512);
  const uint16_t s_b = TWO ? lds16(ssrc + 16) : (uint16_t)0, z_b = TWO ? lds16(ssrc + 528) : (uint16_t)0;
  if (MODE == 0) {
    const uint32_t sa2 = splat16(s_a), za2 = splat16(z_a), sb2 = splat16(s_b), zb2 = splat16(z_b);
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      uint32_t oa[4], ob[4] = {0u, 0u, 0u, 0u};
      dequant_word<T>(wa[m], sa2, za2, oa);
      if (TWO) dequant_word<T>(wb[m], sb2, zb2, ob);
      float(&acc)[4] = (m & 1) ? yacc2 : yacc;
      mma_16816<T>(acc, oa[0], ob[0], oa[1], ob[1], xq[4 * m], xq[4 * m + 1], acc);
      mma_16816<T>(acc, oa[2], ob[2], oa[3], ob[3], xq[4 * m + 2], xq[4 * m + 3], acc);
    }
  } else {
    const float zero4[4] = {0.f, 0.f, 0.f, 0.f};
    float part[4][4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      uint32_t oa[4], ob[4] = {0u, 0u, 0u, 0u};
      unpack_word_biased<T>(wa[m], oa);
      if (TWO) unpack_word_biased<T>(wb[m], ob);
      mma_16816<T>(part[m], oa[0], ob[0], oa[1], ob[1], xq[4 * m], xq[4 * m + 1], zero4);
      mma_16816<T>(part[m], oa[2], ob[2], oa[3], ob[3], xq[4 * m + 2], xq[4 * m + 3], part[m]);
    }
    // part[.][0..1]: (channel g, tokens 2 tig, + 1); part[.][2..3]: channel 8 + g
    const float sa = bits16_to_float(s_a, kBf16), za = bits16_to_float(z_a, kBf16);
    const float2 c0 = csrc[0];
    const float p0 = (part[0][0] + part[1][0]) + (part[2][0] + part[3][0]);
    yacc[0] = fmaf(za, c0.x, fmaf(sa, p0 - c0.y, yacc[0]));
    if (TWO) {
      const float sbf = bits16_to_float(s_b, kBf16), zb = bits16_to_float(z_b, kBf16);
      const float p2 = (part[0][2] + part[1][2]) + (part[2][2] + part[3][2]);
      yacc[2] = fmaf(zb, c0.x, fmaf(sbf, p2 - c0.y, yacc[2]));
    }
    if (!M1) {
      const float2 c1 = csrc[cstride];
      const float p1 = (part[0][1] + part[1][1]) + (part[2][1] + part[3][1]);
      yacc[1] = fmaf(za, c1.x, fmaf(sa, p1 - c1.y, yacc[1]));
      if (TWO) {
        const float sbf = bits16_to_float(s_b, kBf16), zb = bits16_to_float(z_b, kBf16);
        const float p3 = (part[0][3] + part[1][3]) + (part[2][3] + part[3][3]);
        yacc[3] = fmaf(zb, c1.x, fmaf(sbf, p3 - c1.y, yacc[3]));
      }
    }
  }
}

template <typename T, int MODE, bool M1>
__global__ void __launch_bounds__(kRingThreads, 2) w4a16_ring_kernel(const __grid_constant__ RingArgs a) {
  constexpr bool kBf16 = TypeTraits<T>::kIsBf16;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  RING_STAMP(0);
  const RingLayout& L = a.L;
  const int S = a.S, NS = a.NS, N = a.N, K = a.K, M = a.M;
  const int rank = (S > 1) ? (int)cluster_ctarank() : 0;
  const int unit = (S > 1) ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int O = N >> 3, G = K >> 7;
  const int o_lo = (int)(((long long)unit * O) / a.units), o_hi = (int)(((long long)(unit + 1) * O) / a.units);
  const int nrb = (o_hi - o_lo + 1) >> 1;  // row blocks of 16 channels (the last one may hold 8)
  const int kg_lo = (rank * G) / S, kg_hi = ((rank + 1) * G) / S;
  const int ngr = kg_hi - kg_lo;           // this rank's groups
  const int nsl = (ngr + kSlotGroups - 1) / kSlotGroups;
  const int items = nrb * nsl;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);
  uint64_t* full = bars;
  uint64_t* empty = bars + NS;
  uint64_t* rbfull = bars + 2 * NS;
  uint64_t* rbfree = rbfull + 2;
  uint64_t* xch = rbfree + 2;  // [row block] (rank 0 of a 2-CTA cluster)
  uint8_t* ring = smem + L.ring;
  float* red = reinterpret_cast<float*>(smem + L.red);    // [2][warp][16 ch][8 tok]
  float* xchg = reinterpret_cast<float*>(smem + L.xchg);  // [row block][16 ch][Mp]  rank 1's sums land here
  const int Mp = a.Mp;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], kRingProd * 33);  // per producer warp: lane 0's expect_tx arrive + 32 cp.async arrives
      mbar_init(&empty[s], kRingCons);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&rbfull[i], kRingCons);
      mbar_init(&rbfree[i], 1);
    }
    if (S > 1 && rank == 0) {
      for (int rb = 0; rb < nrb; ++rb) {
        const int nch = min(16, (o_hi - o_lo - 2 * rb) * 8);
        mbar_init(&xch[rb], 1);
        mbar_expect_tx(&xch[rb], (uint32_t)(nch * M * 4));
      }
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  pdl_launch_dependents();
  __syncthreads();
  if (S > 1) cluster_arrive();  // publishes the barrier inits to the peer CTA; waited for below, off the producer's path

  if (warp >= kRingCons && warp < kRingCons + kRingProd) {
    // ------------------------------------------------------------------ producers: weights + scales into the ring
    // producer p copies quad rows p and p + 2 of every slot, and the scales (p = 0) / zeros (p = 1)
    const int pw = warp - kRingCons;
    const uint8_t* scb = reinterpret_cast<const uint8_t*>(a.sc);
    const uint8_t* szb = reinterpret_cast<const uint8_t*>(a.sz);
    int slot = 0, use = 0, rb = 0, j = 0;
    bool waited = (S == 1);
    RING_DBG_DECL;
    for (int it = 0; it < items; ++it) {
      RING_CLK(t0);
      if (use > 0) {
        if (!waited) cluster_wait(), waited = true;
        mbar_wait(&empty[slot], (uint32_t)((use - 1) & 1));
      }
      RING_CLK(t1);
      RING_ACC(0, t1 - t0);
      const int g0 = kg_lo + j * kSlotGroups, ng = min(kSlotGroups, kg_hi - g0);
      const int n0 = (o_lo + 2 * rb) * 8, nch = min(16, o_hi * 8 - n0);
      uint8_t* sw = ring + slot * kSlotBytes;
      if (lane == 0) {
        const uint32_t len = (uint32_t)ng * 256u;
        const int nq = nch >> 2;  // 4 quad rows, or 2 for a trailing octet
        mbar_expect_tx(&full[slot], (uint32_t)((nq - pw + 1) >> 1) * len);
        for (int q = pw; q < nq; q += kRingProd)
          bulk_g2s(sw + q * kQS, a.qw + (size_t)((n0 >> 2) + q) * K + (size_t)g0 * kGroup, len, &full[slot]);
      }
      {  // 32 pieces of 16 B: 16 groups x 2 halves of 8 channels
        const int grp = lane >> 1, half = lane & 1;
        if (grp < ng && half * 8 < nch)
          ring_cp_async16(smem_u32(sw) + kSlotW + pw * 512 + grp * 32 + half * 16,
                          (pw ? szb : scb) + ((size_t)(g0 + grp) * N + n0 + half * 8) * 2);
      }
      ring_cp_async_arrive(&full[slot]);
      RING_CLK(t2);
      RING_ACC(1, t2 - t1);
      RING_ACC(3, 1);
      if (++j == nsl) j = 0, ++rb;
      if (++slot == NS) slot = 0, ++use;
    }
    if (!waited) cluster_wait();
    if (pw == 0) {
      RING_STAMP(1);
    }
    RING_DBG_FLUSH(warp);
    return;
  }

  if (S > 1) cluster_wait();
  RING_STAMP(2);
  pdl_wait_prior_grid();  // activations (and y) belong to the stream order from here on
  RING_STAMP(3);

  if (warp == kRingCons + kRingProd) {
    // ------------------------------------------------------------------ finisher: cross-warp sum, k-split exchange, y
    T* y = reinterpret_cast<T*>(a.y);
    const int ch = lane >> 1, tok0 = (lane & 1) * 4;
    for (int rb = 0; rb < nrb; ++rb) {
      const int rs = rb & 1;
      mbar_wait(&rbfull[rs], (uint32_t)((rb >> 1) & 1));
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < kRingCons; ++w) {  // fixed order: deterministic
        const float4 p = *reinterpret_cast<const float4*>(red + (rs * kRingCons + w) * 128 + lane * 4);
        v.x += p.x, v.y += p.y, v.z += p.z, v.w += p.w;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&rbfree[rs]);
      const int n0 = (o_lo + 2 * rb) * 8, nch = min(16, o_hi * 8 - n0);
      float vv[4] = {v.x, v.y, v.z, v.w};
      if (S > 1 && rank == 1) {
        const uint32_t dbar = map_to_rank(smem_u32(&xch[rb]), 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int tok = tok0 + i;
          if (tok < M && ch < nch) {
            const uint32_t dst = map_to_rank(smem_u32(&xchg[(rb * 16 + ch) * Mp + tok]), 0);
            asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(dst),
                         "r"(__float_as_uint(vv[i])), "r"(dbar)
                         : "memory");
          }
        }
      } else {
        if (S > 1) mbar_wait(&xch[rb], 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int tok = tok0 + i;
          if (tok < M && ch < nch) {
            float r = vv[i];
            if (S > 1) r += xchg[(rb * 16 + ch) * Mp + tok];
            y[(size_t)tok * N + n0 + ch] = from_float<T>(r);
          }
        }
      }
    }
    RING_STAMP(6);
    return;
  }

  // -------------------------------------------------------------------- consumers
  const int g = lane >> 2, tig = lane & 3;
  const int xrow = L.xrow;
  uint8_t* xbuf = smem + L.x;                                 // [token][group][tig][m][j] pairs (see header)
  float2* xsum = reinterpret_cast<float2*>(smem + L.xsum);    // [8 tokens][L.ngr] {X, C}
  {
    // stage the activations of this rank's k range in fragment order, and the per-group sums (MODE 2)
    const T* xg = reinterpret_cast<const T*>(a.x) + (size_t)kg_lo * kGroup;
    const int nchunk = ngr * 16;  // 16-byte chunks per token
    for (int tok = 0; tok < M; ++tok) {
      for (int c0 = 0; c0 < nchunk; c0 += kRingCons * 32) {
        const int c = c0 + tid;
        const bool ok = c < nchunk;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (ok) v = *reinterpret_cast<const uint4*>(xg + (size_t)tok * K + (size_t)c * 8);
        // chunk c holds k = 8c .. 8c+7 = the four word-pairs u = 0..3 of (32-k block m = (c & 15) >> 2, nibble pair
        // j = c & 3): lane tig = u reads it at [tig][m * 4 + j]
        if (ok) {
          uint8_t* d = xbuf + tok * xrow + (c >> 4) * 256 + (c & 15) * 4;
          *reinterpret_cast<uint32_t*>(d) = v.x;
          *reinterpret_cast<uint32_t*>(d + 64) = v.y;
          *reinterpret_cast<uint32_t*>(d + 128) = v.z;
          *reinterpret_cast<uint32_t*>(d + 192) = v.w;
        }
        if (MODE == 2) {
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
          float f = 0.f;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float2 p;
            if constexpr (kBf16) p = __bfloat1622float2(u32_as_b2(w[e]));
            else p = __half22float2(u32_as_h2(w[e]));
            f += p.x + p.y;
          }
          // 16 consecutive lanes = one group; even chunks sit on low-nibble positions (pairs j = 0, 2), odd on high
          f += __shfl_xor_sync(0xffffffffu, f, 2);
          f += __shfl_xor_sync(0xffffffffu, f, 4);
          f += __shfl_xor_sync(0xffffffffu, f, 8);
          const float o = __shfl_xor_sync(0xffffffffu, f, 1);
          if (ok && (c & 15) == 0) {
            const float lo = f, hi = o, X = lo + hi;
            xsum[tok * L.ngr + (c >> 4)] = make_float2(X, kBf16 ? 128.f * X : 1024.f * lo + 64.f * hi);
          }
        }
      }
    }
    if (MODE == 2)  // tokens that do not exist must contribute exactly zero
      for (int i = tid + M * L.ngr; i < 8 * L.ngr; i += kRingCons * 32) xsum[i] = make_float2(0.f, 0.f);
  }
  consumer_bar();
  RING_STAMP(4);

  // ldmatrix row address of this lane: matrix m = lane >> 3 is the 32-k block, row = channel (lane & 7) of the octet
  const int lm = lane >> 3, lg = lane & 7;
  const uint32_t ldsm_off = (uint32_t)((lg >> 2) * kQS + (lm >> 1) * 128 + (lg & 3) * 32 + (lm & 1) * 16 + warp * 256);
  const uint32_t ring_u32 = smem_u32(ring);
  const bool live = g < M;
  const uint32_t x_u32 = smem_u32(xbuf) + (uint32_t)((live ? g : 0) * xrow + tig * 64);
  uint32_t xq[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) xq[i] = 0u;

  int slot = 0, use = 0;
  RING_DBG_DECL;
  for (int rb = 0; rb < nrb; ++rb) {
    const int n0 = (o_lo + 2 * rb) * 8;
    const bool two = (o_hi * 8 - n0) >= 16;  // second octet present
    float yacc[4] = {0.f, 0.f, 0.f, 0.f}, yacc2[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < nsl; ++j) {
      RING_CLK(t0);
      mbar_wait(&full[slot], (uint32_t)(use & 1));
      RING_CLK(t1);
      RING_ACC(0, t1 - t0);
      const int ng = min(kSlotGroups, ngr - j * kSlotGroups);
      const uint32_t sb = ring_u32 + (uint32_t)slot * kSlotBytes;
#pragma unroll
      for (int step = 0; step < 2; ++step) {
        const int gi = warp + kRingCons * step;
        if (gi < ng && !RING_DRY) {
          const int Gl = j * kSlotGroups + gi;
          const uint32_t wsrc = sb + ldsm_off + step * (kRingCons * 256);
          const uint32_t xsrc = x_u32 + (uint32_t)Gl * 256u;
          const uint32_t ssrc = sb + kSlotW + (uint32_t)(gi * 32 + g * 2);
          const float2* csrc = xsum + (2 * tig) * L.ngr + Gl;
          if (two) group_step<T, MODE, M1, true>(wsrc, xsrc, ssrc, csrc, L.ngr, live, xq, yacc, yacc2);
          else group_step<T, MODE, M1, false>(wsrc, xsrc, ssrc, csrc, L.ngr, live, xq, yacc, yacc2);
        }
      }
      RING_CLK(t2);
      RING_ACC(1, t2 - t1);
      RING_ACC(3, 1);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);  // the slot's words are in registers / consumed
      if (++slot == NS) slot = 0, ++use;
    }
    // this warp's partial sums of the row block -> red[rb & 1][warp]; the finisher adds the 8 warps
    const int rs = rb & 1;
    RING_CLK(t3);
    if (rb >= 2) mbar_wait(&rbfree[rs], (uint32_t)(((rb >> 1) - 1) & 1));
    if (MODE == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) yacc[i] += yacc2[i];
    }
    float* r = red + (rs * kRingCons + warp) * 128;
    *reinterpret_cast<float2*>(r + g * 8 + 2 * tig) = make_float2(yacc[0], yacc[1]);
    *reinterpret_cast<float2*>(r + (g + 8) * 8 + 2 * tig) = make_float2(yacc[2], yacc[3]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&rbfull[rs]);
    RING_CLK(t4);
    RING_ACC(2, t4 - t3);
  }
  RING_STAMP(5);
  RING_DBG_FLUSH(warp);
}


#ifdef B200AWQ_TRACE
extern "C" int b200awq_debug_ring_stats(long long* host) {
  return (int)cudaMemcpyFromSymbol(host, g_ring_dbg, sizeof(long long) * 80);
}
extern "C" int b200awq_debug_ring_flags(int flags) {
  return (int)cudaMemcpyToSymbol(g_ring_dbg_flags, &flags, sizeof(int));
}
#endif

// ------------------------------------------------------------------------------------ host
namespace {

int sm_count() {
  static int cnt[32] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  dev &= 31;
  if (cnt[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    cnt[dev] = v;
  }
  return cnt[dev];
}

int next_ring_seq() {
  static int seq = 0;
  return seq++;
}

constexpr int kRingSmemBudget = 113 * 1024;  // two CTAs (+ 1 KB reserved each) per 228 KB SM

template <typename T, int MODE, bool M1>
int launch_ring_t(const RingArgs& a, bool pdl, cudaStream_t stream) {
  auto kern = w4a16_ring_kernel<T, MODE, M1>;
  static bool attr_set[32] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200AWQ_ERR_DEVICE;
  if (!attr_set[dev & 31]) {
    if (cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kRingSmemBudget)) return (int)e;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    attr_set[dev & 31] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(a.units * a.S));
  cfg.blockDim = dim3(kRingThreads);
  cfg.dynamicSmemBytes = (size_t)a.L.total;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  if (a.S > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = (unsigned)a.S;
    attrs[na].val.clusterDim.y = 1;
    attrs[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl) {
    attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, a);
  return e == cudaSuccess ? 0 : (int)e;
}

}  // namespace

int launch_ring(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, const RingTuning& tune, cudaStream_t stream) {
  if (M < 1 || M > 8 || N % 8 || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int nsm = sm_count();
  if (nsm < 2) return B200AWQ_ERR_SHAPE;
  const int G = K / kGroup, O = N / 8;
  RingArgs a{};
  a.x = x, a.qw = static_cast<const uint16_t*>(qw), a.sc = sc, a.sz = sz, a.y = y;
  a.M = M, a.N = N, a.K = K;
  a.S = (tune.split == 1 || tune.split == 2) ? tune.split : ((G >= 2 * kRingCons && nsm % 2 == 0) ? 2 : 1);
  if (a.S == 2 && (G < 2 || nsm % 2)) a.S = 1;
  a.units = nsm / a.S;
  a.Mp = M <= 1 ? 1 : (M <= 2 ? 2 : (M <= 4 ? 4 : 8));
  a.seq = next_ring_seq();
  const int oct_max = (O + a.units - 1) / a.units;
  const int nrb_max = (oct_max + 1) / 2;
  if (nrb_max > kRingMaxRb) return B200AWQ_ERR_SHAPE;
  a.nrb_max = nrb_max;
  const int ngr = (G + a.S - 1) / a.S;
  // arithmetic: fp16 -> group-factored fp16 MACs (MODE 2); bf16 -> operand-exact (MODE 0).  (One fp16 token normally
  // never gets here: w4a16_decode.cu serves it.)
  const int mode = (tune.mode == 0 || tune.mode == 2) ? tune.mode : (dtype == B200AWQ_DTYPE_F16 ? 2 : 0);
  RingLayout& L = a.L;
  L.ngr = ngr;
  L.xrow = ngr * 256;
  int off = 0;
  L.bars = off, off += 8 * (2 * 8 + 4 + kRingMaxRb);
  off = (off + 127) & ~127;
  L.x = off, off += M * L.xrow;
  L.xsum = off, off += 8 * ngr * 8;
  L.red = off, off += 2 * kRingCons * 128 * 4;
  L.xchg = off, off += nrb_max * 16 * a.Mp * 4;
  off = (off + 127) & ~127;
  L.ring = off;
  int ns = (kRingSmemBudget - off) / kSlotBytes;
  if (tune.slots > 0) ns = std::min(ns, tune.slots);
  ns = std::min(ns, 8);
  if (ns < 3) return B200AWQ_ERR_SHAPE;  // activations too large next to a useful ring: the caller falls back
  a.NS = ns;
  L.total = off + ns * kSlotBytes;
  const bool m1 = (M == 1);
  if (dtype == B200AWQ_DTYPE_F16) {
    if (mode == 0) return m1 ? launch_ring_t<__half, 0, true>(a, pdl, stream) : launch_ring_t<__half, 0, false>(a, pdl, stream);
    return m1 ? launch_ring_t<__half, 2, true>(a, pdl, stream) : launch_ring_t<__half, 2, false>(a, pdl, stream);
  }
  if (mode == 0)
    return m1 ? launch_ring_t<__nv_bfloat16, 0, true>(a, pdl, stream) : launch_ring_t<__nv_bfloat16, 0, false>(a, pdl, stream);
  return m1 ? launch_ring_t<__nv_bfloat16, 2, true>(a, pdl, stream) : launch_ring_t<__nv_bfloat16, 2, false>(a, pdl, stream);
}

}  // namespace b200awq
