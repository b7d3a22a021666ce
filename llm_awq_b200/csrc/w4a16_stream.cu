// HBM-bound W4A16 streaming kernel for small token counts (decode GEMV, M <= 16).
//
// Replaces the reference's gemv_kernel (quantization_new/gemv/gemv_cuda.cu:74-229) and,
// for 8 <= M <= 16, its split-K GEMM tile (gemm_cuda.cu:1155-1168).  Design:
//   * one CTA owns 8*RO output channels x Kc input channels.  Its slice of `qweight`
//     is 2*RO contiguous byte ranges (the packing interleaves 4 rows, so a 4-row "quad"
//     is contiguous over k); they are pulled into shared memory with bulk async copies
//     (cp.async.bulk -> SASS UBLKCP) issued by ONE thread at the very top of the kernel,
//     in k order and in pieces that each complete on their own mbarrier, so all of the
//     CTA's HBM traffic is in flight at once, no registers are pinned by outstanding
//     loads, and the math starts as soon as the first piece has landed.  Several CTAs
//     co-reside per SM -> 100+ KB in flight per SM.
//   * everything that does not depend on the activations -- the weight prefetch and the
//     staging of this CTA's scales / zeros into shared memory -- happens BEFORE
//     griddepcontrol.wait: with programmatic dependent launch the next linear layer
//     streams its weights while the previous one is still computing / draining.  Only
//     the part after the wait is serialised between consecutive layers, so it is kept
//     short: one round trip to L2 for the activations, then math out of shared memory.
//   * each lane dequantises its own 16-byte chunks (32 weights of ONE output channel,
//     for two channels 8 apart) in registers and feeds them as the A operand of
//     m16n8k16 tensor-core MACs (rows = 16 output channels, columns = 8 tokens).  The k
//     order inside a fragment is simply "whatever the lane holds": A and B use the same
//     lane-local k slots, so the reference's register-oriented packing needs no shuffles;
//     the activations are re-ordered once while they are staged into shared memory so
//     that every B fragment is one aligned register pair.  Accumulation is fp32.
//   * the 8 warps of a CTA split the k groups; partials are reduced through shared
//     memory, and across the CTAs of a thread-block cluster (split-K for large k)
//     through distributed shared memory.  No global atomics, no workspace.
//
// MODE 0: operands w~ = rn_T(q*s + z) bit-identical to the reference's (13 ALU ops per 8
//         weights).  Default for bf16, where operand rounding (2^-9) is part of the 1e-3 contract.
// MODE 2: raw biased operands straight out of the LOP3 (1024+q for low nibbles | 64+q for high
//         nibbles in fp16, 128+q for bf16; 5 ALU ops per 8 weights); scale, zero and the bias are
//         applied per 128-k group in fp32:
//             y += s*(acc - C) + z*X,   X = sum_k x_k,  C = 1024*X_lo + 64*X_hi  (bf16: 128*X).
//         Exact in the integer q; differs from MODE 0 only by not rounding q*s+z to T.
//         Default for fp16 (that rounding is 2^-12 relative: ~2e-4 normwise, inside 1e-3).
#include <algorithm>
#include <atomic>

#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {


__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Watchdog of the fused exchange (below): a rank whose peer never delivers (peer died, mismatched launch sequence)
// gives up after kExchangeTimeoutNs, poisons its outputs with NaN and marks the exchange dead for the rest of the
// process, so that a broken job produces visibly wrong numbers quickly instead of spinning on the GPU for ever.
constexpr unsigned long long kExchangeTimeoutNs = 10ull * 1000 * 1000 * 1000;
__device__ unsigned int g_exchange_dead = 0;

#ifdef B200AWQ_TRACE
// Debug build only (-DB200AWQ_TRACE): wall-clock stamps of the first and last CTA of each launch.
__device__ unsigned long long g_trace_buf[1024 * 2 * 8];
#define B200AWQ_STAMP(ev)                                                     \
  if (threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) \
  g_trace_buf[(((unsigned)seq & 1023u) * 2 + (blockIdx.x != 0)) * 8 + (ev)] = globaltimer_ns()
#else
#define B200AWQ_STAMP(ev)
#endif

struct StreamSmem {
  int w, s, z, x, red, cpart, rbuf, xsum, bars, total;
  int ngroups, nrounds, nbar;  // derived on the host so the kernel prologue has no integer divisions
  int rbs;                     // row blocks (of 8*RO channels) this CTA processes one after the other
};

__host__ __device__ inline StreamSmem stream_smem_layout(int RO, int TT, int MODE, int M, int Kc, int rpb, int rbs, int kStreamWarps,
                                                         bool split) {
  StreamSmem L;
  const int ng = Kc / kGroup;
  const int nbar = ((ng + kStreamWarps - 1) / kStreamWarps + rpb - 1) / rpb;
  int off = 0;
  L.w = off, off += rbs * 2 * RO * Kc * 2;
  L.s = off, off += rbs * ng * 8 * RO * 2;
  L.z = off, off += rbs * ng * 8 * RO * 2;
  off = (off + 15) & ~15;
  L.x = off, off += M * (Kc * 2 + 16);
  L.red = off, off += kStreamWarps * TT * 128 * 4;
  L.cpart = off, off += TT * 128 * 4;
  L.rbuf = off, off += (split ? 8 * TT * 128 * 4 : 0);  // split-k: partial sums pushed by the other CTAs of the cluster
  L.xsum = off, off += (MODE ? 8 * TT * ng * 8 : 0);
  L.bars = off, off += (rbs * nbar + 2) * 8;
  L.total = off;
  L.ngroups = ng;
  L.nrounds = (ng + kStreamWarps - 1) / kStreamWarps;
  L.nbar = nbar;
  L.rbs = rbs;
  return L;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <typename T, int RO, int TT, int MODE, int kStreamWarps>
__global__ void __launch_bounds__(kStreamWarps * 32, TT == 1 ? (kStreamWarps == 16 ? 2 : 4) : (kStreamWarps == 16 ? 1 : 2))
w4a16_stream_kernel(const T* __restrict__ x, const uint16_t* __restrict__ qw, const T* __restrict__ scales,
                    const T* __restrict__ szeros, T* __restrict__ y, int M, int N, int K, int Kc, int S, int rpb, int seq,
                    const __grid_constant__ StreamSmem L, const __grid_constant__ PeerArgs pa) {
  B200AWQ_STAMP(0);
  constexpr bool kBf16 = TypeTraits<T>::kIsBf16;
  constexpr int R = 8 * RO;  // output channels per CTA
  constexpr int kStreamThreads = kStreamWarps * 32;
  constexpr int kRoundK = kStreamWarps * kGroup;  // input channels consumed per round of the warps
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, tig = lane & 3;
  const int rank = (S > 1) ? (int)cluster_ctarank() : 0;
  const int rb0 = ((S > 1) ? (int)(blockIdx.x / S) : (int)blockIdx.x) * L.rbs;  // first row block of this CTA
  const int rbs = min(L.rbs, N / R - rb0);                                      // (the last CTA may own fewer)
  const int kbase = rank * Kc;
  const int ngroups = L.ngroups, nrounds = L.nrounds, nbar = L.nbar;
  const int wrow = Kc * 2;       // bytes of one 4-row quad over this CTA's k range
  const int xrow = Kc * 2 + 16;  // padded activation row (bank spread between tokens)

  uint8_t* wbuf = smem + L.w;
  uint16_t* sbuf = reinterpret_cast<uint16_t*>(smem + L.s);  // [group][R]
  uint16_t* zbuf = reinterpret_cast<uint16_t*>(smem + L.z);
  uint8_t* xbuf = smem + L.x;                                // [token][Kc] natural order (+16 B pad per row)
  float* red = reinterpret_cast<float*>(smem + L.red);      // [warp][tt][16 rows][8 tok]
  float* cpart = reinterpret_cast<float*>(smem + L.cpart);  // [tt][16][8]
  float2* xsum = reinterpret_cast<float2*>(smem + L.xsum);  // [8 TT tok][group] {X, C}   (MODE 2)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);
  uint64_t* xbar = bars + L.rbs * nbar;
  uint64_t* rbar = xbar + 1;                                 // split-k: counts the bytes pushed into rbuf
  float* rbuf = reinterpret_cast<float*>(smem + L.rbuf);    // [cluster rank][tt][16][8]

  if (tid == 0) {
    for (int b = 0; b <= L.rbs * nbar + 1; ++b) mbar_init(&bars[b], 1);
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    B200AWQ_STAMP(7);
  }
  pdl_launch_dependents();
  // ---- scales / zeros of this CTA's rows and groups -> shared memory, asynchronously (16-byte pieces)
  {
    constexpr int PPG = R / 8;  // 16-byte pieces per group per tensor
    const int pieces = ngroups * PPG;
    for (int rbi = 0; rbi < rbs; ++rbi) {
      const size_t goff = ((size_t)(kbase / kGroup) * N + (size_t)(rb0 + rbi) * R) * 2;
      const uint8_t* sg = reinterpret_cast<const uint8_t*>(scales) + goff;
      const uint8_t* zg = reinterpret_cast<const uint8_t*>(szeros) + goff;
      for (int i = tid; i < 2 * pieces; i += kStreamThreads) {
        const int which = i >= pieces;
        const int j = which ? i - pieces : i;
        const int grp = j / PPG, pc = j - grp * PPG;
        cp_async16(reinterpret_cast<uint8_t*>(which ? zbuf : sbuf) + ((rbi * ngroups + grp) * PPG + pc) * 16,
                   (which ? zg : sg) + (size_t)grp * N * 2 + pc * 16);
      }
    }
    if (MODE) {  // tokens M .. 8*TT-1 do not exist: their correction terms must read as zero
      for (int i = tid + M * ngroups; i < 8 * TT * ngroups; i += kStreamThreads) xsum[i] = make_float2(0.f, 0.f);
    }
  }
  __syncthreads();  // barrier inits and the zeroed correction terms visible to everyone
  // ---- weight prefetch: 2*RO quad rows (x rbs row blocks) x nbar pieces of (rpb * 1024 k) each, one bulk copy per
  // (quad row, piece); the copies of different quad rows are issued by different warps (a single thread needs
  // ~0.15 us per cp.async.bulk: measured 0.64 us for four of them)
  if (lane == 0 && warp < 2 * RO) {
    const int piece = rpb * kRoundK * 2;  // bytes per quad row per barrier
    for (int rbi = 0; rbi < rbs; ++rbi)
      for (int b = 0; b < nbar; ++b) {
        const int off = b * piece;
        const int len = min(piece, wrow - off);
        if (warp == 0) mbar_expect_tx(&bars[rbi * nbar + b], 2 * RO * len);
        bulk_g2s(wbuf + (rbi * 2 * RO + warp) * wrow + off,
                 reinterpret_cast<const uint8_t*>(qw + (size_t)((rb0 + rbi) * 2 * RO + warp) * K + kbase) + off, len,
                 &bars[rbi * nbar + b]);
      }
  }
  B200AWQ_STAMP(1);
  if (S > 1) cluster_sync_all();  // ... and to the other CTAs of the cluster, BEFORE the wait (overlaps the previous kernel)
  B200AWQ_STAMP(2);
  pdl_wait_prior_grid();  // activations (and y) belong to the stream order from here on
  B200AWQ_STAMP(3);

  // ---- activations: M bulk copies x[m, kbase .. kbase + Kc) -> xbuf (natural order)
  if (tid == 0) {
    mbar_expect_tx(xbar, (uint32_t)M * Kc * 2);
    for (int m = 0; m < M; ++m) bulk_g2s(xbuf + m * xrow, x + (size_t)m * K + kbase, Kc * 2, xbar);
  }
  mbar_wait(xbar, 0);
  if (MODE) {
    // {X, C} of (token, group) for THIS warp's groups only (nobody else reads them): lane = (group
    // slot, 16-element chunk); the first 16 B of a chunk sit on low-nibble positions, the second on
    // high-nibble ones (pairs 0-3 | 4-7 of each half of the 32-k block).
    const int gslot = lane >> 3, chunk = lane & 7;
    for (int g0 = warp; g0 < ngroups; g0 += 4 * kStreamWarps) {  // 4 of this warp's groups per pass
      const int G = g0 + gslot * kStreamWarps;
      for (int m = 0; m < M; ++m) {
        float lo = 0.f, hi = 0.f;
        if (G < ngroups) {
          const uint4* src = reinterpret_cast<const uint4*>(xbuf + m * xrow + G * 256 + chunk * 32);
          const uint4 va = src[0], vb = src[1];
          const uint32_t av[4] = {va.x, va.y, va.z, va.w}, bv[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float2 fa, fb;
            if constexpr (kBf16) {
              fa = __bfloat1622float2(u32_as_b2(av[e]));
              fb = __bfloat1622float2(u32_as_b2(bv[e]));
            } else {
              fa = __half22float2(u32_as_h2(av[e]));
              fb = __half22float2(u32_as_h2(bv[e]));
            }
            lo += fa.x + fa.y;
            hi += fb.x + fb.y;
          }
        }
#pragma unroll
        for (int d = 1; d < 8; d <<= 1) {
          lo += __shfl_xor_sync(0xffffffffu, lo, d);
          hi += __shfl_xor_sync(0xffffffffu, hi, d);
        }
        if (chunk == 0 && G < ngroups) {
          const float X = lo + hi;
          xsum[m * ngroups + G] = make_float2(X, kBf16 ? 128.f * X : 1024.f * lo + 64.f * hi);
        }
      }
    }
    __syncwarp();
  }
  cp_async_wait_all();  // scales / zeros (issued before the wait; their latency overlapped everything above)
  __syncthreads();
  B200AWQ_STAMP(4);

  const float zero4[4] = {0.f, 0.f, 0.f, 0.f};
  for (int rbi = 0; rbi < rbs; ++rbi) {  // row blocks of this CTA: weights of all of them were prefetched above
  const int n0 = (rb0 + rbi) * R;
  float acc[TT][4];
#pragma unroll
  for (int t = 0; t < TT; ++t)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[t][i] = 0.f;

  // per-lane walking pointers; lanes whose token does not exist feed zeros
  const uint8_t* xp[TT];
  bool live[TT];
#pragma unroll
  for (int t = 0; t < TT; ++t) {
    const int tok = g + 8 * t;
    live[t] = tok < M;
    xp[t] = xbuf + (live[t] ? tok : 0) * xrow + (warp * kGroup + tig * 32) * 2;
  }
  const uint8_t* wp = wbuf + (rbi * 2 * RO + (g >> 2)) * wrow + (warp * 2 + (tig >> 1)) * 128 + (g & 3) * 32 + (tig & 1) * 16;
  const uint16_t* sq = sbuf + (rbi * ngroups + warp) * R + g;
  const uint16_t* zq = zbuf + (rbi * ngroups + warp) * R + g;
  const float2* sump = xsum + (2 * tig) * ngroups + warp;  // token 2 tig (+ 8 t), this warp's first group
  uint4 xq[TT][4];
#pragma unroll
  for (int t = 0; t < TT; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) xq[t][j] = make_uint4(0, 0, 0, 0);

  for (int rnd = 0, G = warp, left = 0, bar = rbi * nbar; rnd < nrounds; ++rnd, G += kStreamWarps) {
    if (left == 0) {
      mbar_wait(&bars[bar++], 0);
      left = rpb;
    }
    --left;
    if (G >= ngroups) break;  // only in the last round, when ngroups % 8 != 0
    // B fragments: token g (+ 8 t) of this lane, the 32 k of block (G, tig) in natural order: xq[j]
    // holds the k pairs 4j .. 4j+3 = what nibble pair j of words 0..3 multiplies (dead lanes keep 0)
#pragma unroll
    for (int t = 0; t < TT; ++t) {
      if (live[t]) {
#pragma unroll
        for (int j = 0; j < 4; ++j) xq[t][j] = reinterpret_cast<const uint4*>(xp[t])[j];
      }
      xp[t] += kRoundK * 2;
    }
    // A: the 16-byte chunk of (row n0 + 8 ro + g, 32-k block 4G + tig) for ro = 0 (rows 0-7 of
    // the MMA) and ro = 1 (rows 8-15)
    uint32_t wa[4], wb[4] = {0, 0, 0, 0};
    {
      const uint4 v = *reinterpret_cast<const uint4*>(wp);
      wa[0] = v.x, wa[1] = v.y, wa[2] = v.z, wa[3] = v.w;
      if (RO == 2) {
        const uint4 v2 = *reinterpret_cast<const uint4*>(wp + 2 * wrow);
        wb[0] = v2.x, wb[1] = v2.y, wb[2] = v2.z, wb[3] = v2.w;
      }
      wp += kStreamWarps * 256;
    }
    const uint16_t s_a = sq[0], z_a = zq[0], s_b = sq[8 * (RO - 1)], z_b = zq[8 * (RO - 1)];
    sq += kStreamWarps * R;
    zq += kStreamWarps * R;
    const uint32_t sa2 = splat16(s_a), za2 = splat16(z_a), sb2 = splat16(s_b), zb2 = splat16(z_b);

    float part[TT][4], part2[TT][4];
#pragma unroll
    for (int uu = 0; uu < 4; uu += 2) {
      // words uu, uu+1 of both octets; the MMA of nibble pair j takes (word uu, word uu+1) as its two
      // k slots, so its B operand is the ADJACENT register pair (4j + uu, 4j + uu + 1) of xq[j]
      uint32_t oa0[4], oa1[4], ob0[4] = {0, 0, 0, 0}, ob1[4] = {0, 0, 0, 0};
      if (MODE == 0) {
        dequant_word<T>(wa[uu], sa2, za2, oa0);
        dequant_word<T>(wa[uu + 1], sa2, za2, oa1);
        if (RO == 2) {
          dequant_word<T>(wb[uu], sb2, zb2, ob0);
          dequant_word<T>(wb[uu + 1], sb2, zb2, ob1);
        }
      } else {
        unpack_word_biased<T>(wa[uu], oa0);
        unpack_word_biased<T>(wa[uu + 1], oa1);
        if (RO == 2) {
          unpack_word_biased<T>(wb[uu], ob0);
          unpack_word_biased<T>(wb[uu + 1], ob1);
        }
      }
#pragma unroll
      for (int t = 0; t < TT; ++t) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t b0 = uu ? xq[t][j].z : xq[t][j].x, b1 = uu ? xq[t][j].w : xq[t][j].y;
          if (MODE == 0) {
            mma_16816<T>(acc[t], oa0[j], ob0[j], oa1[j], ob1[j], b0, b1, acc[t]);
          } else {
            // two independent accumulation chains (even / odd j); low-nibble pairs are j = 0, 2
            float(&dst)[4] = (j & 1) ? part2[t] : part[t];
            if (uu == 0 && j < 2)
              mma_16816<T>(dst, oa0[j], ob0[j], oa1[j], ob1[j], b0, b1, zero4);
            else
              mma_16816<T>(dst, oa0[j], ob0[j], oa1[j], ob1[j], b0, b1, dst);
          }
        }
      }
    }
    if (MODE) {
      // part[t][0..1]: (row g of octet 0, tokens 8t + 2tig, + 1); part[t][2..3]: row g of octet 1
      const float sa = bits16_to_float(s_a, kBf16), za = bits16_to_float(z_a, kBf16);
      const float sb = bits16_to_float(s_b, kBf16), zb = bits16_to_float(z_b, kBf16);
#pragma unroll
      for (int t = 0; t < TT; ++t) {
        const float2 c0 = sump[(8 * t) * ngroups], c1 = sump[(8 * t + 1) * ngroups];  // {X, C}, zeros if absent
        acc[t][0] = fmaf(za, c0.x, fmaf(sa, (part[t][0] - c0.y) + part2[t][0], acc[t][0]));
        acc[t][1] = fmaf(za, c1.x, fmaf(sa, (part[t][1] - c1.y) + part2[t][1], acc[t][1]));
        acc[t][2] = fmaf(zb, c0.x, fmaf(sb, (part[t][2] - c0.y) + part2[t][2], acc[t][2]));
        acc[t][3] = fmaf(zb, c1.x, fmaf(sb, (part[t][3] - c1.y) + part2[t][3], acc[t][3]));
      }
      sump += kStreamWarps;
    }
  }

  B200AWQ_STAMP(5);
  // acc[t][0..1]: (channel g, tokens 8t + 2tig, +1); acc[t][2..3]: channel 8 + g
#pragma unroll
  for (int t = 0; t < TT; ++t) {
    float* r = red + (warp * TT + t) * 128;
    *reinterpret_cast<float2*>(r + g * 8 + 2 * tig) = make_float2(acc[t][0], acc[t][1]);
    *reinterpret_cast<float2*>(r + (g + 8) * 8 + 2 * tig) = make_float2(acc[t][2], acc[t][3]);
  }
  __syncthreads();
  for (int e = tid; e < TT * 128; e += kStreamThreads) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kStreamWarps; ++w) v += red[w * TT * 128 + e];
    if (S == 1) {
      const int t = e >> 7, row = (e >> 3) & 15, tok = 8 * t + (e & 7);
      if (tok < M && row < R) {
        if (pa.world > 1) cpart[e] = v;  // exchanged with the peer GPUs below
        else y[(size_t)tok * N + n0 + row] = from_float<T>(v);
      }
    } else {
      cpart[e] = v;
    }
  }
  if (S > 1) {
    // split-k reduce WITHOUT cluster barriers or fences at the end of the kernel (each of them is lowered to a
    // GPU-scope MEMBAR): the other CTAs PUSH their partial sums into the leader's shared memory with st.async,
    // every store completing 4 bytes on the leader's mbarrier; they can exit right away.
    const int nvalid = M * R;  // live (token, channel) sums per CTA
    if (rank != 0) {
      const uint32_t dst_bar = map_to_rank(smem_u32(rbar), 0);
      for (int e = tid; e < TT * 128; e += kStreamThreads) {
        const int t = e >> 7, row = (e >> 3) & 15, tok = 8 * t + (e & 7);
        if (tok < M && row < R) {
          const uint32_t dst = map_to_rank(smem_u32(&rbuf[rank * TT * 128 + e]), 0);
          asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(dst),
                       "r"(__float_as_uint(cpart[e])), "r"(dst_bar)
                       : "memory");
        }
      }
    } else {
      if (tid == 0) mbar_expect_tx(rbar, (uint32_t)((S - 1) * nvalid * 4));
      mbar_wait(rbar, (uint32_t)(rbi & 1));
      for (int e = tid; e < TT * 128; e += kStreamThreads) {
        const int t = e >> 7, row = (e >> 3) & 15, tok = 8 * t + (e & 7);
        if (tok < M && row < R) {
          float v = cpart[e];
          for (int r = 1; r < S; ++r) v += rbuf[r * TT * 128 + e];  // fixed order
          if (pa.world > 1) cpart[e] = v;  // only this thread reads / writes the leader's own cpart[e]
          else y[(size_t)tok * N + n0 + row] = from_float<T>(v);
        }
      }
    }
  }
  if (pa.world > 1 && rank == 0) {  // the CTA that holds the final sums of this row block (cluster leader if k is split)
    // ---- row-parallel all-reduce fused into the epilogue (one-shot over NVLink peer memory):
    // every rank writes its fp32 partials of this row block into EVERY rank's exchange buffer, then polls the
    // words of all sources and sums them in rank order.  Epochs are per channel OCTET and live in device memory,
    // which keeps the protocol valid under CUDA-graph replay; regions alternate with the epoch parity, and a
    // rank can never run two epochs ahead of a peer because it needs that peer's words to finish an epoch.
    __shared__ unsigned int s_ep[2];
    const int idx = n0 >> 3;
    if (tid < R / 8) s_ep[tid] = pa.epoch[idx + tid] + 1u;
    __syncthreads();
    const int W = pa.world;
    // Every exchanged element is ONE 8-byte word {fp32 partial, epoch}: the epoch travels with the value, so a
    // reader that sees the epoch has the value (ONE scalar 8-byte access: aligned 64-bit accesses are single-copy
    // atomic, a .v2.u32 pair is not guaranteed to be) and no system-scope fence or separate flag is needed (a
    // st.release.sys / ld.acquire.sys pair was measured at ~8 us per kernel).
    // A word's slot is keyed by (channel, token) and its epoch counter by the channel's octet, i.e. by the SAME
    // key whatever the layer's n (and this kernel's row-block height) is: layers of different widths can share
    // one exchange.
    for (int e = tid; e < TT * 128; e += kStreamThreads) {
      const int t = e >> 7, row = (e >> 3) & 15, tok = 8 * t + (e & 7);
      if (tok < M && row < R) {
        const unsigned int ep = s_ep[row >> 3];
        const unsigned long long word = ((unsigned long long)ep << 32) | (unsigned long long)__float_as_uint(cpart[e]);
        const size_t off = (size_t)((ep & 1u) * W + pa.rank) * pa.cap + (size_t)(n0 + row) * pa.tok_cap + tok;
        for (int r = 0; r < W; ++r)
          asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(pa.data[r] + off), "l"(word) : "memory");
      }
    }
    const unsigned long long t_exchange = globaltimer_ns();
    bool dead = *(volatile unsigned int*)&g_exchange_dead != 0u;
    for (int e = tid; e < TT * 128; e += kStreamThreads) {
      const int t = e >> 7, row = (e >> 3) & 15, tok = 8 * t + (e & 7);
      if (tok < M && row < R) {
        const unsigned int ep = s_ep[row >> 3];
        float v = 0.f;
        for (int r = 0; r < W; ++r) {  // fixed rank order: bit-identical results on every rank
          const unsigned long long* srcp =
              pa.data[pa.rank] + (size_t)((ep & 1u) * W + r) * pa.cap + (size_t)(n0 + row) * pa.tok_cap + tok;
          unsigned long long word = 0;
          unsigned int polls = 0;
          while (!dead) {
            asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(word) : "l"(srcp) : "memory");
            if ((unsigned int)(word >> 32) == ep) break;
            if ((++polls & 0xfffu) == 0u &&
                (globaltimer_ns() - t_exchange > kExchangeTimeoutNs || *(volatile unsigned int*)&g_exchange_dead != 0u)) {
              dead = true;
              atomicExch(&g_exchange_dead, 1u);
            }
          }
          v += dead ? __uint_as_float(0x7fc00000u) : __uint_as_float((unsigned int)word);
        }
        y[(size_t)tok * N + n0 + row] = from_float<T>(v);
      }
    }
    __syncthreads();
    if (tid < R / 8) pa.epoch[idx + tid] = s_ep[tid];
  }
  if (rbi + 1 < rbs) __syncthreads();  // `red` / `cpart` are reused by the next row block
  }  // rbi
  B200AWQ_STAMP(6);
}

#ifdef B200AWQ_TRACE
extern "C" int b200awq_debug_read_trace(unsigned long long* host, int count) {
  return (int)cudaMemcpyFromSymbol(host, g_trace_buf, sizeof(unsigned long long) * (size_t)count);
}
#endif

// ------------------------------------------------------------------------------------ host
constexpr int kStreamSmemCap = 200 * 1024;

static int next_seq() {  // launch counter for the trace build's stamps only
  static std::atomic<int> seq{0};
  return seq.fetch_add(1, std::memory_order_relaxed);
}

static int pick_splits(int K, int kc_target, int kc_env) {
  const int groups = K / kGroup;
  if (kc_env > 0 && kc_env % kGroup == 0 && K % kc_env == 0) {
    const int s = K / kc_env;
    if (s == 1 || s == 2 || s == 4 || s == 8) return s;
  }
  int best = 1;
  for (int s = 1; s <= 8; s *= 2) {  // cluster sizes: powers of two, <= 8 (portable limit)
    if (groups % s) continue;
    best = s;
    if (K / s <= kc_target) break;
  }
  return best;
}

template <typename T, int RO, int TT, int MODE, int kStreamWarps>
static int launch_stream_w(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K,
                           int S, int rpb, bool pdl, const StreamTuning& tune, cudaStream_t stream, const PeerArgs* peers) {
  const int Kc = K / S;
  PeerArgs pa{};
  if (peers) pa = *peers;
  if (pa.world > 1 && TT != 1) return B200AWQ_ERR_SHAPE;
  // several row blocks per CTA (all weight slices prefetched up front, activations / group sums staged once) is a
  // tuning knob only: fat long-lived CTAs keep the NEXT launch's CTAs from becoming resident, which costs more
  // than the saved prologues
  const int nblk = N / (8 * RO);
  int rbs = (tune.rbs > 0) ? tune.rbs : 1;
  if (S != 1 || rbs > nblk) rbs = 1;
  StreamSmem L = stream_smem_layout(RO, TT, MODE, M, Kc, rpb, rbs, kStreamWarps, S > 1);
  if (L.total > kStreamSmemCap && rbs > 1) rbs = 1, L = stream_smem_layout(RO, TT, MODE, M, Kc, rpb, 1, kStreamWarps, S > 1);
  if (L.total > kStreamSmemCap) return B200AWQ_ERR_SHAPE;
  constexpr int kStreamThreads = kStreamWarps * 32;
  auto kern = w4a16_stream_kernel<T, RO, TT, MODE, kStreamWarps>;
  static bool attr_set[32] = {};  // per kernel instantiation and device
  if (cudaError_t ea = ensure_dyn_smem(kern, kStreamSmemCap, attr_set)) return (int)ea;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)((nblk + rbs - 1) / rbs) * S);
  cfg.blockDim = dim3(kStreamThreads);
  // Co-residency: a launch that fits in one wave runs fastest with FEW CTAs per SM (the next launch's
  // CTAs only need enough room to prefetch); multi-wave launches want as many as fit (measured, DESIGN.md).
  size_t dyn = L.total;
  const int ctas = ((nblk + rbs - 1) / rbs) * S;
  int dev = 0, nsm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  if (nsm <= 0) nsm = 132;
  const int per_sm = ctas <= 2 * nsm ? 2 : (ctas <= 3 * nsm ? 3 : 0);
  if (tune.pad > 0)  // > 0: explicit extra bytes (limits co-residency), 0: heuristic, < 0: none
    dyn += (size_t)tune.pad;
  else if (tune.pad == 0 && per_sm > 0 && S == 1)
    dyn = std::max(dyn, (size_t)(233472 / (per_sm + 1) - 512));
  if (dyn > (size_t)kStreamSmemCap) dyn = L.total;
  cfg.dynamicSmemBytes = dyn;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  if (S > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = S;
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
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, (const T*)x, (const uint16_t*)qw, (const T*)sc, (const T*)sz, (T*)y, M, N,
                                     K, Kc, S, rpb, next_seq(), L, pa);
  return e == cudaSuccess ? 0 : (int)e;
}

template <typename T, int RO, int TT, int MODE>
static int launch_stream_t(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K,
                           int S, int rpb, bool pdl, const StreamTuning& tune, cudaStream_t stream, const PeerArgs* peers) {
  // 8 warps per CTA by default; 16 (shorter serial chain after griddepcontrol.wait, half the co-residency) is a knob
  if (tune.warps == 16)  // 16 warps or several row blocks per CTA do not pay
    return launch_stream_w<T, RO, TT, MODE, 16>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
  return launch_stream_w<T, RO, TT, MODE, 8>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
}

template <typename T, int MODE>
static int launch_stream_m(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K,
                           int S, int ro, int rpb, bool pdl, const StreamTuning& tune, cudaStream_t stream,
                           const PeerArgs* peers) {
  if (M <= 8) {
    if (ro == 2) return launch_stream_t<T, 2, 1, MODE>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
    return launch_stream_t<T, 1, 1, MODE>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
  }
  if (ro == 2) return launch_stream_t<T, 2, 2, MODE>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
  return launch_stream_t<T, 1, 2, MODE>(x, qw, sc, sz, y, M, N, K, S, rpb, pdl, tune, stream, peers);
}

int launch_stream(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                  bool pdl, const StreamTuning& tune, cudaStream_t stream, const PeerArgs* peers) {
  if (M < 1 || M > 16 || N % 8 || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int ro = (N % 16 == 0) ? 2 : 1;
  // k per CTA: splitting k over a cluster doubles the CTAs and adds the cluster reduction; up to 4 tokens the unsplit
  // 4096 rather than 2048, above that shared memory for x decides
  const int kc_target = M <= 4 ? 4096 : (M <= 8 ? 2048 : 1024);
  const int S = pick_splits(K, kc_target, tune.kc);
  const int rpb = tune.rpb > 0 ? tune.rpb : 64;  // default: one barrier (4 large copies) per CTA
  // default arithmetic: fp16 -> group-factored (MODE 2), bf16 -> operand-exact (MODE 0); see the header comment
  const int mode = (tune.mode == 0 || tune.mode == 2) ? tune.mode : (dtype == B200AWQ_DTYPE_F16 ? 2 : 0);
  if (dtype == B200AWQ_DTYPE_F16) {
    if (mode == 0) return launch_stream_m<__half, 0>(x, qw, sc, sz, y, M, N, K, S, ro, rpb, pdl, tune, stream, peers);
    return launch_stream_m<__half, 2>(x, qw, sc, sz, y, M, N, K, S, ro, rpb, pdl, tune, stream, peers);
  }
  if (mode == 0) return launch_stream_m<__nv_bfloat16, 0>(x, qw, sc, sz, y, M, N, K, S, ro, rpb, pdl, tune, stream, peers);
  return launch_stream_m<__nv_bfloat16, 2>(x, qw, sc, sz, y, M, N, K, S, ro, rpb, pdl, tune, stream, peers);
}

}  // namespace b200awq
