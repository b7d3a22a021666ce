// Persistent, warp-specialised W4A16 decode kernel for SEVERAL tokens (2 <= M <= 4) and for bf16:
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

#include "rmsnorm_stat.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

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
  RingLayout L;
  const void* bias;      // EPI: [N] or null
  const void* residual;  // EPI: [M, N] or null
  const void* gamma;     // NORM: [K], the RMSNorm weight applied to every token row of x before the product
  float eps;             // NORM
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kRingCons * 32) : "memory"); }

// One 128-k group of one row block, one warp: 16 (TWO) or 8 channels x 128 input channels.
//   wsrc  this lane's ldmatrix row address (channel lane & 7, 32-k block lane >> 3) of the first octet
//   xsrc  this lane's 64 bytes of staged activations (token g, word slot tig) of the group
//   ssrc  &scales[group][channel g] in the slot (zeros 512 B further, channel 8 + g 16 B further)
//   csrc  &xsum[token 2 tig][group] (MODE 2)
template <typename T, bool M1, bool TWO>
__device__ __forceinline__ void group_step(uint32_t wsrc, uint32_t xsrc, uint32_t ssrc, const float2* csrc, int cstride,
                                           bool live, uint32_t (&xq)[16], float (&yacc)[4], float (&yacc2)[4]) {
  constexpr int MODE = TypeTraits<T>::kIsBf16 ? 0 : 2;
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
  if constexpr (MODE == 0) {
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
      unpack_word_biased(wa[m], oa);
      if (TWO) unpack_word_biased(wb[m], ob);
      mma_16816<T>(part[m], oa[0], ob[0], oa[1], ob[1], xq[4 * m], xq[4 * m + 1], zero4);
      mma_16816<T>(part[m], oa[2], ob[2], oa[3], ob[3], xq[4 * m + 2], xq[4 * m + 3], part[m]);
    }
    // part[.][0..1]: (channel g, tokens 2 tig, + 1); part[.][2..3]: channel 8 + g
    const float sa = half_bits_to_float(s_a), za = half_bits_to_float(z_a);
    const float2 c0 = csrc[0];
    const float p0 = (part[0][0] + part[1][0]) + (part[2][0] + part[3][0]);
    yacc[0] = fmaf(za, c0.x, fmaf(sa, p0 - c0.y, yacc[0]));
    if (TWO) {
      const float sbf = half_bits_to_float(s_b), zb = half_bits_to_float(z_b);
      const float p2 = (part[0][2] + part[1][2]) + (part[2][2] + part[3][2]);
      yacc[2] = fmaf(zb, c0.x, fmaf(sbf, p2 - c0.y, yacc[2]));
    }
    if (!M1) {
      const float2 c1 = csrc[cstride];
      const float p1 = (part[0][1] + part[1][1]) + (part[2][1] + part[3][1]);
      yacc[1] = fmaf(za, c1.x, fmaf(sa, p1 - c1.y, yacc[1]));
      if (TWO) {
        const float sbf = half_bits_to_float(s_b), zb = half_bits_to_float(z_b);
        const float p3 = (part[0][3] + part[1][3]) + (part[2][3] + part[3][3]);
        yacc[3] = fmaf(zb, c1.x, fmaf(sbf, p3 - c1.y, yacc[3]));
      }
    }
  }
}

// EPI: the finisher adds a.bias / a.residual to each stored value (add_epilogue)
// NORM: the product reads x^ = RMSNorm(x, a.gamma, a.eps) instead of x, bit-identical to rmsnorm.cu's output (DESIGN
// §3.5c).  The 256 consumer threads ARE the 256 threads of rmsnorm_stat.cuh's summation order: each token row's 8 warp
// totals go through `red` (first written after the staging barrier), and the staging normalises every chunk it copies.
// The body is shared by two kernel names: w4a16_ring_kernel<T, M1, EPI> (NORM = false, the names the plain entries have
// always launched) and w4a16_ring_norm_kernel<T, M1, EPI> (NORM = true).
template <typename T, bool M1, bool EPI, bool NORM>
__device__ __forceinline__ void ring_body(const RingArgs& a) {
  constexpr int MODE = TypeTraits<T>::kIsBf16 ? 0 : 2;  // see the header comment
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
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
    for (int it = 0; it < items; ++it) {
      if (use > 0) {
        if (!waited) cluster_wait(), waited = true;
        mbar_wait(&empty[slot], (uint32_t)((use - 1) & 1));
      }
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
          cp_async<16>(smem_u32(sw) + kSlotW + pw * 512 + grp * 32 + half * 16,
                       (pw ? szb : scb) + ((size_t)(g0 + grp) * N + n0 + half * 8) * 2);
      }
      cp_async_mbar_arrive(&full[slot]);
      if (++j == nsl) j = 0, ++rb;
      if (++slot == NS) slot = 0, ++use;
    }
    if (!waited) cluster_wait();
    return;
  }

  if (S > 1) cluster_wait();
  // NORM: gamma of this thread's first staging chunk, a model constant: loaded before the wait
  const uint4* gam = reinterpret_cast<const uint4*>(static_cast<const T*>(a.gamma) + (size_t)kg_lo * kGroup);
  const uint4 g_first = NORM && warp < kRingCons && tid < ngr * 16 ? __ldg(gam + tid) : make_uint4(0u, 0u, 0u, 0u);
  pdl_wait_prior_grid();  // activations (and y) belong to the stream order from here on

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
          if (tok < M && ch < nch) st_async_f32(map_to_rank(smem_u32(&xchg[(rb * 16 + ch) * Mp + tok]), 0), vv[i], dbar);
        }
      } else {
        if (S > 1) mbar_wait(&xch[rb], 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int tok = tok0 + i;
          if (tok < M && ch < nch) {
            float r = vv[i];
            if (S > 1) r += xchg[(rb * 16 + ch) * Mp + tok];
            const size_t i = (size_t)tok * N + n0 + ch;
            if (EPI)  // after griddepcontrol.wait (above): bias / residual are in stream order
              y[i] = add_epilogue<T>(from_float<T>(r), static_cast<const T*>(a.bias), static_cast<const T*>(a.residual),
                                     (size_t)(n0 + ch), i);
            else
              y[i] = from_float<T>(r);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  const int g = lane >> 2, tig = lane & 3;
  const int xrow = L.xrow;
  uint8_t* xbuf = smem + L.x;                                 // [token][group][tig][m][j] pairs (see header)
  float2* xsum = reinterpret_cast<float2*>(smem + L.xsum);    // [8 tokens][L.ngr] {X, C}
  float rstd[4] = {0.f, 0.f, 0.f, 0.f};                        // NORM: r of each token row
  if constexpr (NORM) {
    constexpr int kNormFirst = 2;  // chunks per token and thread loaded before the first use: all of them up to k = 4096
    constexpr int kTok = M1 ? 1 : 4;
    const T* x0 = static_cast<const T*>(a.x);
    uint4 nv[kTok][kNormFirst];
#pragma unroll
    for (int tok = 0; tok < kTok; ++tok)
      if (tok < M) norm_first_chunks<T, kNormFirst>(x0 + (size_t)tok * K, K, tid, nv[tok]);
#pragma unroll
    for (int tok = 0; tok < kTok; ++tok) {
      if (tok < M) {
        const float s = norm_warp_sum(norm_thread_sumsq<T, kNormFirst>(nv[tok], x0 + (size_t)tok * K, K, tid));
        if (lane == 0) red[tok * kNormWarps + warp] = s;
      }
    }
    consumer_bar();
#pragma unroll
    for (int tok = 0; tok < kTok; ++tok)
      if (tok < M) rstd[tok] = norm_rstd(red + tok * kNormWarps, K, a.eps);
  }
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
        if (NORM && ok) {
          const uint4 gv = c0 == 0 ? g_first : __ldg(gam + c);
          float r = rstd[0];
#pragma unroll
          for (int i = 1; i < 4; ++i)
            if (!M1 && tok == i) r = rstd[i];
          v = make_uint4(norm_pair<T>(v.x, gv.x, r), norm_pair<T>(v.y, gv.y, r), norm_pair<T>(v.z, gv.z, r),
                         norm_pair<T>(v.w, gv.w, r));
        }
        // chunk c holds k = 8c .. 8c+7 = the four word-pairs u = 0..3 of (32-k block m = (c & 15) >> 2, nibble pair
        // j = c & 3): lane tig = u reads it at [tig][m * 4 + j]
        if (ok) {
          uint8_t* d = xbuf + tok * xrow + (c >> 4) * 256 + (c & 15) * 4;
          *reinterpret_cast<uint32_t*>(d) = v.x;
          *reinterpret_cast<uint32_t*>(d + 64) = v.y;
          *reinterpret_cast<uint32_t*>(d + 128) = v.z;
          *reinterpret_cast<uint32_t*>(d + 192) = v.w;
        }
        if constexpr (MODE == 2) {
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
          float f = 0.f;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 p = __half22float2(u32_as_h2(w[e]));
            f += p.x + p.y;
          }
          // 16 consecutive lanes = one group; even chunks sit on low-nibble positions (pairs j = 0, 2), odd on high
          f += __shfl_xor_sync(0xffffffffu, f, 2);
          f += __shfl_xor_sync(0xffffffffu, f, 4);
          f += __shfl_xor_sync(0xffffffffu, f, 8);
          const float o = __shfl_xor_sync(0xffffffffu, f, 1);
          if (ok && (c & 15) == 0) {
            const float lo = f, hi = o, X = lo + hi;
            xsum[tok * L.ngr + (c >> 4)] = make_float2(X, 1024.f * lo + 64.f * hi);
          }
        }
      }
    }
    if (MODE == 2)  // tokens that do not exist must contribute exactly zero
      for (int i = tid + M * L.ngr; i < 8 * L.ngr; i += kRingCons * 32) xsum[i] = make_float2(0.f, 0.f);
  }
  consumer_bar();

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
  for (int rb = 0; rb < nrb; ++rb) {
    const int n0 = (o_lo + 2 * rb) * 8;
    const bool two = (o_hi * 8 - n0) >= 16;  // second octet present
    float yacc[4] = {0.f, 0.f, 0.f, 0.f}, yacc2[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < nsl; ++j) {
      mbar_wait(&full[slot], (uint32_t)(use & 1));
      const int ng = min(kSlotGroups, ngr - j * kSlotGroups);
      const uint32_t sb = ring_u32 + (uint32_t)slot * kSlotBytes;
#pragma unroll
      for (int step = 0; step < 2; ++step) {
        const int gi = warp + kRingCons * step;
        if (gi < ng) {
          const int Gl = j * kSlotGroups + gi;
          const uint32_t wsrc = sb + ldsm_off + step * (kRingCons * 256);
          const uint32_t xsrc = x_u32 + (uint32_t)Gl * 256u;
          const uint32_t ssrc = sb + kSlotW + (uint32_t)(gi * 32 + g * 2);
          const float2* csrc = xsum + (2 * tig) * L.ngr + Gl;
          if (two) group_step<T, M1, true>(wsrc, xsrc, ssrc, csrc, L.ngr, live, xq, yacc, yacc2);
          else group_step<T, M1, false>(wsrc, xsrc, ssrc, csrc, L.ngr, live, xq, yacc, yacc2);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);  // the slot's words are in registers / consumed
      if (++slot == NS) slot = 0, ++use;
    }
    // this warp's partial sums of the row block -> red[rb & 1][warp]; the finisher adds the 8 warps
    const int rs = rb & 1;
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
  }
}

template <typename T, bool M1, bool EPI>
__global__ void __launch_bounds__(kRingThreads, 2) w4a16_ring_kernel(const __grid_constant__ RingArgs a) {
  ring_body<T, M1, EPI, false>(a);
}

template <typename T, bool M1, bool EPI>
__global__ void __launch_bounds__(kRingThreads, 2) w4a16_ring_norm_kernel(const __grid_constant__ RingArgs a) {
  ring_body<T, M1, EPI, true>(a);
}

// ------------------------------------------------------------------------------------ host
namespace {

constexpr int kRingSmemBudget = 113 * 1024;  // two CTAs (+ 1 KB reserved each) per 228 KB SM

template <typename T, bool M1, bool EPI, bool NORM>
int launch_ring_t(const RingArgs& a, bool pdl, cudaStream_t stream) {
  constexpr auto kern = NORM ? w4a16_ring_norm_kernel<T, M1, EPI> : w4a16_ring_kernel<T, M1, EPI>;
  if (cudaError_t e = ensure_dyn_smem<kern>(kRingSmemBudget, true)) return (int)e;
  return launch_kernel(kern, dim3((unsigned)(a.units * a.S)), dim3(kRingThreads),
                       (size_t)a.L.total, stream, pdl, (unsigned)a.S, a);
}

template <typename T, bool EPI, bool NORM>
int launch_ring_m(const RingArgs& a, bool pdl, cudaStream_t stream) {
  return a.M == 1 ? launch_ring_t<T, true, EPI, NORM>(a, pdl, stream) : launch_ring_t<T, false, EPI, NORM>(a, pdl, stream);
}

template <typename T>
int launch_ring_dt(const RingArgs& a, bool epi, bool norm, bool pdl, cudaStream_t stream) {
  if (norm) return epi ? launch_ring_m<T, true, true>(a, pdl, stream) : launch_ring_m<T, false, true>(a, pdl, stream);
  return epi ? launch_ring_m<T, true, false>(a, pdl, stream) : launch_ring_m<T, false, false>(a, pdl, stream);
}

}  // namespace

int launch_ring(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi, const NormPrologue& norm) {
  if (M < 1 || M > 4 || N % 8 || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int nsm = sm_count();
  if (nsm == 0) return B200AWQ_ERR_DEVICE;
  if (nsm < 2) return B200AWQ_ERR_SHAPE;
  const int G = K / kGroup, O = N / 8;
  RingArgs a{};
  a.x = x, a.qw = static_cast<const uint16_t*>(qw), a.sc = sc, a.sz = sz, a.y = y;
  a.bias = epi.bias, a.residual = epi.residual;
  a.gamma = norm.gamma, a.eps = norm.eps;
  a.M = M, a.N = N, a.K = K;
  a.S = (G >= 2 * kRingCons && nsm % 2 == 0) ? 2 : 1;
  a.units = nsm / a.S;
  a.Mp = M <= 1 ? 1 : (M <= 2 ? 2 : 4);
  const int oct_max = (O + a.units - 1) / a.units;
  const int nrb_max = (oct_max + 1) / 2;
  if (nrb_max > kRingMaxRb) return B200AWQ_ERR_SHAPE;
  const int ngr = (G + a.S - 1) / a.S;
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
  const int ns = std::min((kRingSmemBudget - off) / kSlotBytes, 8);
  if (ns < 3) return B200AWQ_ERR_SHAPE;  // activations too large next to a useful ring: the caller falls back
  a.NS = ns;
  L.total = off + ns * kSlotBytes;
  if (dtype == B200AWQ_DTYPE_F16) return launch_ring_dt<__half>(a, epi.on(), norm.on(), pdl, stream);
  return launch_ring_dt<__nv_bfloat16>(a, epi.on(), norm.on(), pdl, stream);
}

}  // namespace b200awq
