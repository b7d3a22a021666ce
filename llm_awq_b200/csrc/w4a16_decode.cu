// One-token W4A16 decode kernel (GEMV, M = 1): the HBM-bound hot path of BASELINE configs[1].
//
// Replaces the reference's gemv_kernel (quantization_new/gemv/gemv_cuda.cu:74-229).  Third generation of the decode
// path:
//   * HBM streams a read-only buffer at full rate only with tens of KB in flight per SM, and a bulk-async copy
//     (UBLKCP) carries a fixed latency whatever its size, so small copies cap the rate.  Here every copy is one QUAD
//     ROW (4 output channels, contiguous over k in the packed layout) x up to 4096 input channels = 8 KB, and
//     70..88 KB of copies are in flight per CTA.
//   * a launch boundary costs microseconds in which nothing can be computed (the previous layer's tail,
//     griddepcontrol.wait, the staging of the activations).  Two CTAs of consecutive launches co-reside on
//     every SM (<= 113 KB and <= 102 registers x 320 threads each), the PRODUCER warp never waits for the activations,
//     so HBM keeps streaming into the next launch's ring through the bubble; the consumers then have to drain the ring
//     faster than HBM fills it: int8 tensor-core MACs on the packed bytes AS THEY ARE (no dequantisation).
//
// Work split: the N / 4 quad rows are dealt evenly and contiguously to the clusters (S CTAs each, S = 1 unless the
// layer has too few rows to balance the SMs, then k is split S ways inside the cluster and rank 0 adds the partial
// sums it receives through distributed shared memory).  A CTA walks its quad rows in ROW BLOCKS of 16 channels (4
// quad rows; the last block may hold fewer) and, for long k, in PIECES of <= 32 groups of 128 input channels.
//
// Ring slot = one octet (two quad rows) x one piece: 2 bulk copies of <= 8 KB + the octet's scales / zeros (8-byte
// cp.async per group and quad row), one `full` mbarrier.  The second quad row sits 8 KB + 16 B after the first: the
// eight 16-byte rows of every ldmatrix phase then hit eight different bank groups.
//
// Arithmetic (exact int32 partial sums, fp32 scale application):
//   a packed byte b = 16 h + l holds two weights of one channel.  With the activation vector split, per 128-k group,
//   into three signed 7-bit digits of a block-fixed-point number  x_k = e_g (d0 + d1 / 128 + d2 / 16384)  (e_g a power
//   of two, |d| <= 64: every fp16 / bf16 activation is represented to 2^-21 of the group's largest magnitude),
//       raw  = sum_k b_k LO_k,   high = sum_k (b_k & 0xf0) [LO_k | HI_k]      (u8 x s8 IMMA.16832, one LOP3 per word)
//       sum_k l_k x_lo + h_k x_hi = raw - high.LO + high.HI / 16
//   the three digits and their LO / HI variants occupy six of the eight "token" columns of the MMA, which one token
//   leaves free.  y += s_g (e_g sum_d 2^-7d T_d) + z_g X_g with X_g = sum_k x_k.  The dequantised weight
//   q s + z is therefore used UNROUNDED (the reference rounds it to fp16 first, gemv_cuda.cu:161): results agree
//   with the reference kernel to ~3e-4 normwise, inside the 1e-3 contract (tests/test_gpu_parity*.py).
//
// Contract notes: packed weights / scales / zeros are read BEFORE griddepcontrol.wait, i.e. they must not be produced
// by the kernel immediately preceding this launch in the stream (weights are constants in inference); x and y are only
// touched after the wait.
#include <algorithm>

#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

#ifdef B200AWQ_TRACE
extern __device__ unsigned long long g_trace_buf[1024 * 2 * 8];  // defined in w4a16_stream.cu (trace build, -rdc)
extern __device__ long long g_ring_dbg[20 * 4];                    // w4a16_ring.cu
extern __device__ int g_ring_dbg_flags;
__device__ __forceinline__ unsigned long long dec_globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define DEC_STAMP(ev)                                                  \
  if (lane == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) \
  g_trace_buf[(((unsigned)a.seq & 1023u) * 2 + (blockIdx.x != 0)) * 8 + (ev)] = dec_globaltimer_ns()
#define DEC_CLK(var) const long long var = clock64()
#define DEC_ACC(slot, expr) dbg_acc[slot] += (expr)
#define DEC_DBG_DECL long long dbg_acc[4] = {0, 0, 0, 0}; const int dbg_flags = g_ring_dbg_flags
#define DEC_DBG_FLUSH(w)            \
  if (lane == 0 && blockIdx.x == 0) \
    for (int i_ = 0; i_ < 4; ++i_) g_ring_dbg[(w) * 4 + i_] = dbg_acc[i_]
#define DEC_DRY (dbg_flags & 1)
#else
#define DEC_STAMP(ev)
#define DEC_CLK(var)
#define DEC_ACC(slot, expr)
#define DEC_DBG_DECL
#define DEC_DBG_FLUSH(w)
#define DEC_DRY 0
#endif

// consumer warps per CTA: 16 (default, <= 56 registers) or 8 (<= 102 registers); warp w owns the groups g % CONS == w of every
// piece.  + producer warp + finisher warp.
constexpr int kDecPiece = 32;                          // groups of 128 input channels per bulk copy (8 KB of one quad row)
constexpr int kDecQuadBytes = kDecPiece * 256;         // 4 channels x 4096 k, packed
constexpr int kDecQuadB = kDecQuadBytes + 16;          // offset of a slot's second quad row (bank skew)
constexpr int kDecScaleOff = kDecQuadB + kDecQuadBytes + 16;  // [quad 2][scales, zeros][group 32][4 ch] x 16 bit
constexpr int kDecSlotBytes = ((kDecScaleOff + 2 * 2 * kDecPiece * 8 + 127) / 128) * 128;
constexpr int kDecGroupBytes = 6 * 4 * 16;             // digits of one group: [column 0..5][tig][32-k block m] words
constexpr int kDecRed = 8;                             // row blocks whose partial sums may wait for the finisher
constexpr int kDecMaxSlots = 8;
constexpr int kDecMaxRb = 128;                         // row blocks per CTA the exchange buffers are sized for
constexpr int kDecSmemBudget = 113 * 1024;             // two CTAs (+ 1 KB reserved each) per 228 KB SM

struct DecLayout {
  int bars, x, gx, red, xchg, ring, total;
};

struct DecArgs {
  const void* x;
  const uint16_t* qw;
  const void* sc;
  const void* sz;
  const uint16_t* qw2;  // FUSED (gate + up + SiLU * mul): the second weight set (up projection); the first one is the gate
  const void* sc2;
  const void* sz2;
  void* y;
  int N, K;
  int S;        // CTAs per cluster = k split
  int units;    // clusters
  int NS;       // ring slots
  int nrb_max;  // most row blocks any CTA owns
  int seq;
  DecLayout L;
};

__device__ __forceinline__ void dec_cp_async8(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void dec_cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void dec_ldsm4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ uint4 dec_lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint16_t dec_lds16(uint32_t addr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void dec_sts8(uint32_t addr, int v) {
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void dec_cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void dec_cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void dec_imma(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1,
                                         const int (&c)[4]) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]));
}

// silu(g) * u with the reference's roundings (tinychat/modules/fused_mlp.py:40-60,80: gate and up outputs are tensors
// of T, F.silu rounds to T, the product rounds to T)
template <typename T>
__device__ __forceinline__ T silu_mul_rounded(float gate_acc, float up_acc) {
  const float g = (float)from_float<T>(gate_acc), u = (float)from_float<T>(up_acc);
  const float s = (float)from_float<T>(g / (1.f + expf(-g)));
  return from_float<T>(s * u);
}

// FUSED = false: y = x W~^T.   FUSED = true: y = silu(x Wgate~^T) * (x Wup~^T), both weight sets walked row block by row
// block through the same ring (SURVEY.md §8f-1: one read of x, two weight streams, one [1, n] write).
template <typename T, int CONS, bool FUSED>
__global__ void __launch_bounds__((CONS + 2) * 32, 2) w4a16_decode_kernel(const __grid_constant__ DecArgs a) {
  constexpr bool kBf16 = TypeTraits<T>::kIsBf16;
  constexpr int kDecCons = CONS;
  constexpr int NT = FUSED ? 2 : 1;   // weight sets
  constexpr int RW = 16 * NT;         // partial sums per row block and warp
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  DEC_STAMP(0);
  const DecLayout& L = a.L;
  const int S = a.S, NS = a.NS, N = a.N, K = a.K;
  const int rank = (S > 1) ? (int)cluster_ctarank() : 0;
  const int unit = (S > 1) ? (int)(blockIdx.x / (unsigned)S) : (int)blockIdx.x;
  const int Q = N >> 2, G = K >> 7;
  const int q_lo = (int)(((unsigned)unit * (unsigned)Q) / (unsigned)a.units);  // Q * units < 2^31 (checked by the launcher)
  const int q_hi = (int)(((unsigned)(unit + 1) * (unsigned)Q) / (unsigned)a.units);
  const int nq = q_hi - q_lo;
  const int nrb = (nq + 3) >> 2;           // row blocks of 16 channels (the last one may hold 4, 8 or 12)
  const int kg_lo = (rank * G) / S, kg_hi = ((rank + 1) * G) / S;
  const int ngr = kg_hi - kg_lo;           // this rank's groups
  const int npc = (ngr + kDecPiece - 1) / kDecPiece;  // pieces

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bars);
  uint64_t* full = bars;
  uint64_t* empty = bars + kDecMaxSlots;
  uint64_t* rbfull = bars + 2 * kDecMaxSlots;
  uint64_t* rbfree = rbfull + kDecRed;
  uint64_t* xch = rbfree + kDecRed;  // [row block] (rank 0 of a cluster)
  uint8_t* ring = smem + L.ring;
  float* red = reinterpret_cast<float*>(smem + L.red);    // [kDecRed][warp][16 ch]
  float* xchg = reinterpret_cast<float*>(smem + L.xchg);  // [peer 1..S-1][row block][16 ch]: the peers' sums land here (rank 0)

  // Prologue, kept off the ring's critical path: the PRODUCER warp initialises the ring barriers itself (one barrier
  // per lane) and issues the whole first lap of copies before it joins the CTA barrier -- the weights of a small layer
  // have to land inside the launch bubble of its predecessor; another warp initialises the row-block barriers.
  pdl_launch_dependents();
  if (warp == kDecCons) {
    if (lane < NS) {
      mbar_init(&full[lane], 33);  // lane 0's expect_tx arrive + 32 cp.async arrives
      mbar_init(&empty[lane], kDecCons);
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
  } else if (warp == 0) {
    if (lane < kDecRed) {
      mbar_init(&rbfull[lane], kDecCons);
      mbar_init(&rbfree[lane], 1);
    }
    if (S > 1 && rank == 0) {
      for (int rb = lane; rb < nrb; rb += 32) {
        const int nch = min(16, (nq - 4 * rb) * 4);
        mbar_init(&xch[rb], 1);
        mbar_expect_tx(&xch[rb], (uint32_t)(nch * 4 * NT * (S - 1)));
      }
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }

  if (warp == kDecCons) {
    // ------------------------------------------------------------------ producer: weights + scales into the ring
    const uint8_t* scb = reinterpret_cast<const uint8_t*>(a.sc);
    const uint8_t* szb = reinterpret_cast<const uint8_t*>(a.sz);
    int slot = 0, use = 0;
    bool joined = false;  // the CTA barrier is joined once, after the first lap (or at the end of a short walk)
    DEC_DBG_DECL;
#ifdef B200AWQ_TRACE
    const long long clk_begin = clock64();
    const unsigned long long ns_begin = dec_globaltimer_ns();
#endif
    for (int rb = 0; rb < nrb; ++rb) {
      const int qb = q_lo + 4 * rb, nqb = min(4, q_hi - qb);  // quad rows of this row block
      for (int pt = 0; pt < npc * NT; ++pt) {
        const int p = FUSED ? (pt >= npc ? pt - npc : pt) : pt;
        const bool second = FUSED && pt >= npc;
        const uint16_t* qwt = second ? a.qw2 : a.qw;
        const uint8_t* sct = second ? reinterpret_cast<const uint8_t*>(a.sc2) : scb;
        const uint8_t* szt = second ? reinterpret_cast<const uint8_t*>(a.sz2) : szb;
        const int g0 = kg_lo + p * kDecPiece, ng = min(kDecPiece, kg_hi - g0);
        for (int h = 0; h < nqb; h += 2) {  // one slot per octet
          DEC_CLK(t0);
          if (use > 0) {
            if (!joined) {
              asm volatile("bar.sync 0;" ::: "memory");  // the CTA barrier the other warps wait at (below)
              if (S > 1) dec_cluster_arrive();
              joined = true;
            }
            mbar_wait(&empty[slot], (uint32_t)((use - 1) & 1));
          }
          DEC_CLK(t1);
          DEC_ACC(0, t1 - t0);
          const int q0 = qb + h, nqs = min(2, nqb - h);
          uint8_t* sw = ring + slot * kDecSlotBytes;
          const uint32_t len = (uint32_t)ng * 256u;
          if (lane == 0) {
            mbar_expect_tx(&full[slot], (uint32_t)nqs * len);
            bulk_g2s(sw, qwt + (size_t)q0 * K + (size_t)g0 * kGroup, len, &full[slot]);
            if (nqs > 1) bulk_g2s(sw + kDecQuadB, qwt + (size_t)(q0 + 1) * K + (size_t)g0 * kGroup, len, &full[slot]);
          }
          if (lane < ng) {  // lane = group: 8 bytes (4 channels) of scales and of zeros per quad row
            const size_t off = ((size_t)(g0 + lane) * N + (size_t)q0 * 4) * 2;
            const uint32_t dst = smem_u32(sw) + kDecScaleOff + lane * 8;
            dec_cp_async8(dst, sct + off);
            dec_cp_async8(dst + kDecPiece * 8, szt + off);
            if (nqs > 1) {
              dec_cp_async8(dst + 2 * kDecPiece * 8, sct + off + 8);
              dec_cp_async8(dst + 3 * kDecPiece * 8, szt + off + 8);
            }
          }
          dec_cp_async_arrive(&full[slot]);
          DEC_CLK(t2);
          DEC_ACC(1, t2 - t1);
          DEC_ACC(3, 1);
          if (++slot == NS) slot = 0, ++use;
        }
      }
    }
    if (!joined) {
      asm volatile("bar.sync 0;" ::: "memory");
      if (S > 1) dec_cluster_arrive();
    }
    if (S > 1) dec_cluster_wait();
    DEC_STAMP(1);
    DEC_DBG_FLUSH(18);  // the probe prints slot 18 as the producer
#ifdef B200AWQ_TRACE
    if (lane == 0 && blockIdx.x == 0) {  // SM clock actually delivered over the producer's lifetime: cycles and ns
      g_ring_dbg[19 * 4 + 0] = clock64() - clk_begin;
      g_ring_dbg[19 * 4 + 1] = (long long)(dec_globaltimer_ns() - ns_begin);
    }
#endif
    return;
  }

  asm volatile("bar.sync 0;" ::: "memory");  // barrier inits of both initialising warps are visible (the producer joins after its first lap)
  if (S > 1) dec_cluster_arrive();  // publishes rank 0's exchange barriers to the peers
  if (S > 1) dec_cluster_wait();
  DEC_STAMP(2);
  // Consumers: everything the first activation loads need is computed BEFORE the dependency wait, and the loads are the
  // first instructions after it (measured: ~470 cycles passed between the wait returning and the loads issuing when the
  // address arithmetic -- kernel parameters from the constant bank, cold instructions -- came after the wait).
  constexpr int kMaxOwn = 32 / kDecCons;  // groups a warp converts together (k = 4096: all of its groups)
  const int x_eoff = (lane >> 3) * 32 + ((lane >> 2) & 1) * 8 + 2 * (lane & 3);  // see the digit staging below
  const uint32_t* xfirst[kMaxOwn];
#pragma unroll
  for (int i = 0; i < kMaxOwn; ++i) {
    const int Gl = min(warp + i * kDecCons, max(ngr - 1, 0));
    xfirst[i] = reinterpret_cast<const uint32_t*>(reinterpret_cast<const T*>(a.x) + (size_t)(kg_lo + Gl) * kGroup + x_eoff);
  }
  pdl_wait_prior_grid();  // activations (and y) belong to the stream order from here on
  uint32_t xa0[kMaxOwn], xb0[kMaxOwn];
  if (warp < kDecCons) {
#pragma unroll
    for (int i = 0; i < kMaxOwn; ++i) {
      asm volatile("ld.global.u32 %0, [%1];" : "=r"(xa0[i]) : "l"(xfirst[i]) : "memory");
      asm volatile("ld.global.u32 %0, [%1 + 32];" : "=r"(xb0[i]) : "l"(xfirst[i]) : "memory");
    }
  }
#ifdef B200AWQ_TRACE
  const long long clk_wait = clock64();
#endif
  DEC_STAMP(3);

  if (warp == kDecCons + 1) {
    // ------------------------------------------------------------------ finisher
    // Sums the consumer warps' partials of a row block (fixed order) and frees the red slot at once.  With k split over the
    // cluster, ranks > 0 push their sums into rank 0's shared memory (st.async completing bytes on rank 0's mbarrier);
    // rank 0 parks its own sums and completes row blocks (add the peers', round, store) as their words arrive.
    T* y = reinterpret_cast<T*>(a.y);
    float* hold = xchg + (S - 1) * a.nrb_max * RW;  // [row block][RW]: rank 0's own sums until the peers' arrive
    const int ch = lane & 15;
    const bool mine = lane < RW;  // lanes 0-15: channels of the (gate) product, lanes 16-31: of the up product (FUSED)
    // final value of channel `ch` from the summed accumulators of this lane (FUSED: lane ch holds the gate sum, lane
    // 16 + ch the up sum) and its store
    auto finish = [&](float v, int n0, int nch) {
      if (FUSED) {
        const float up = __shfl_down_sync(0xffffffffu, v, 16);
        if (lane < nch) y[n0 + ch] = silu_mul_rounded<T>(v, up);
      } else {
        if (lane < nch) y[n0 + ch] = from_float<T>(v);
      }
    };
    int fl = 0;  // rank 0, k split: next row block to complete
    for (int rb = 0; rb < nrb; ++rb) {
      const int rs = rb % kDecRed;
      mbar_wait(&rbfull[rs], (uint32_t)((rb / kDecRed) & 1));
      float v = 0.f;
      if (mine) {
#pragma unroll
        for (int w = 0; w < kDecCons; ++w) v += red[(rs * kDecCons + w) * RW + lane];  // fixed order: deterministic
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&rbfree[rs]);
      const int n0 = (q_lo + 4 * rb) * 4, nch = min(16, (nq - 4 * rb) * 4);
      if (S == 1) {
        finish(v, n0, nch);
      } else if (rank > 0) {
        if (mine && ch < nch) {
          const uint32_t dbar = map_to_rank(smem_u32(&xch[rb]), 0);
          const uint32_t dst = map_to_rank(smem_u32(&xchg[((rank - 1) * a.nrb_max + rb) * RW + lane]), 0);
          asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(dst),
                       "r"(__float_as_uint(v)), "r"(dbar)
                       : "memory");
        }
      } else {
        if (mine) hold[rb * RW + lane] = v;  // read back by the same lane only
        while (fl <= rb) {
          const bool ok = __all_sync(0xffffffffu, mbar_try_wait(&xch[fl], 0));
          if (!ok) break;
          const int f0 = (q_lo + 4 * fl) * 4, fch = min(16, (nq - 4 * fl) * 4);
          float r = 0.f;
          if (mine && ch < fch) {
            r = hold[fl * RW + lane];
            for (int pr = 0; pr < S - 1; ++pr) r += xchg[(pr * a.nrb_max + fl) * RW + lane];  // fixed order
          }
          finish(r, f0, fch);
          ++fl;
        }
      }
    }
    if (S > 1 && rank == 0) {
      for (; fl < nrb; ++fl) {
        mbar_wait(&xch[fl], 0);
        const int f0 = (q_lo + 4 * fl) * 4, fch = min(16, (nq - 4 * fl) * 4);
        float r = 0.f;
        if (mine && ch < fch) {
          r = hold[fl * RW + lane];
          for (int pr = 0; pr < S - 1; ++pr) r += xchg[(pr * a.nrb_max + fl) * RW + lane];
        }
        finish(r, f0, fch);
      }
    }
    DEC_STAMP(6);
    return;
  }

  // -------------------------------------------------------------------- consumers
  // warp w owns the local groups g with g % 8 == w of every piece: it converts exactly the activations it multiplies,
  // so no CTA-wide barrier stands between the dependency wait and the first MAC.
  const int c = lane >> 2, tig = lane & 3;
  const uint32_t xd_u32 = smem_u32(smem + L.x);
  float* gx = reinterpret_cast<float*>(smem + L.gx);  // [group][tig]: e_g 2^-7 tig / 16 for the digit lanes tig < 3, X_g = sum_k x_k for tig 3
  {
    // Digits.  A digit word [column 2 d + par][u][m] (par 0: low-nibble channels, 1: high-nibble channels) holds the
    // four input channels m * 32 + par * 8 + {0, 16} + 2 u + {0, 1} of the group (see the packed layout in
    // w4_common.cuh): lane (m, par, u) loads those two pairs, converts four values and stores three whole words.
    // Every load is issued before the first use; the group's largest magnitude and the digit sums come from one REDUX
    // each (integer warp reductions), the digits from the 1.5 * 2^23 rounding trick (no F2I on the path).
    const T* xg = reinterpret_cast<const T*>(a.x) + (size_t)kg_lo * kGroup;
    const int m = lane >> 3, par = (lane >> 2) & 1, u = lane & 3;
    const int eoff = m * 32 + par * 8 + 2 * u;                      // first pair; the second one is 16 channels further
    const uint32_t woff = (uint32_t)(par * 64 + u * 16 + m * 4);    // + digit * 128
    uint8_t* xd = smem + L.x;
    for (int G0 = warp; G0 < ngr; G0 += kMaxOwn * kDecCons) {
      uint32_t xa[kMaxOwn], xb[kMaxOwn];
#ifdef B200AWQ_TRACE
      const long long ld_t0 = clock64();
#endif
#pragma unroll
      for (int i = 0; i < kMaxOwn; ++i) {
        if (G0 == warp) {  // the first batch was loaded right behind the dependency wait
          xa[i] = xa0[i], xb[i] = xb0[i];
        } else {
          const int Gl = min(G0 + i * kDecCons, ngr - 1);  // clamped: the extra conversions are not stored
          const uint32_t* src = reinterpret_cast<const uint32_t*>(xg + (size_t)Gl * kGroup + eoff);
          xa[i] = src[0], xb[i] = src[8];
        }
      }
#ifdef B200AWQ_TRACE
      if (G0 == warp && warp == 0 && blockIdx.x == 0) {  // latency of the first activation loads of warp 0 (cycles)
        const uint32_t dep = xa[0] ^ xb[0] ^ xa[kMaxOwn - 1] ^ xb[kMaxOwn - 1];
        long long ld_t1 = dep == 0x9e3779b9u ? 1 : 0;  // a real dependency: the clock below is read after the data arrived
        asm volatile("" ::"l"(ld_t1) : "memory");
        ld_t1 += clock64();
        if (lane == 0) g_ring_dbg[19 * 4 + 2] = ld_t1 - ld_t0, g_ring_dbg[19 * 4 + 3] = ld_t0 - clk_wait;
      }
#endif
#pragma unroll
      for (int i = 0; i < kMaxOwn; ++i) {
        const int Gl = G0 + i * kDecCons;
        const bool valid = Gl < ngr;  // warp-uniform
        float f[4];  // byte order of the word: pair A element 0, pair B element 0, pair A element 1, pair B element 1
        {
          float2 pa, pb;
          if constexpr (kBf16) pa = __bfloat1622float2(u32_as_b2(xa[i])), pb = __bfloat1622float2(u32_as_b2(xb[i]));
          else pa = __half22float2(u32_as_h2(xa[i])), pb = __half22float2(u32_as_h2(xb[i]));
          f[0] = pa.x, f[1] = pb.x, f[2] = pa.y, f[3] = pb.y;
        }
        // non-negative floats order like their bit patterns: the group's largest magnitude with one integer REDUX
        const uint32_t am = max(max(__float_as_uint(fabsf(f[0])), __float_as_uint(fabsf(f[1]))),
                                max(__float_as_uint(fabsf(f[2])), __float_as_uint(fabsf(f[3]))));
        const int ex = (int)(__reduce_max_sync(0xffffffffu, am) >> 23);
#ifdef B200AWQ_TRACE
        if (i == 0 && G0 == warp) { DEC_STAMP(7); }  // the activation loads have returned
#endif
        // e = 2^(floor(log2 amax) - 5): |x| / e < 64.  Groups whose largest magnitude is below 2^-121 (bf16 only)
        // count as zero.
        const bool nz = ex >= 6;
        const float inv_e = nz ? __uint_as_float((uint32_t)(259 - ex) << 23) : 0.f;
        const float e = nz ? __uint_as_float((uint32_t)(ex - 5) << 23) : 0.f;
        constexpr float kMagic = 12582912.f;  // 1.5 * 2^23: (t + kMagic) holds rint(t) in its low mantissa bits
        uint32_t d0[4], d1[4], d2[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float t = f[q] * inv_e;
          const float a0 = t + kMagic;
          const float r1 = (t - (a0 - kMagic)) * 128.f;
          const float a1 = r1 + kMagic;
          const float r2 = (r1 - (a1 - kMagic)) * 128.f;
          const float a2 = r2 + kMagic;
          d0[q] = __float_as_uint(a0), d1[q] = __float_as_uint(a1), d2[q] = __float_as_uint(a2);  // digit = low byte
        }
        const uint32_t w0 = __byte_perm(__byte_perm(d0[0], d0[1], 0x0040), __byte_perm(d0[2], d0[3], 0x0040), 0x5410);
        const uint32_t w1 = __byte_perm(__byte_perm(d1[0], d1[1], 0x0040), __byte_perm(d1[2], d1[3], 0x0040), 0x5410);
        const uint32_t w2 = __byte_perm(__byte_perm(d2[0], d2[1], 0x0040), __byte_perm(d2[2], d2[3], 0x0040), 0x5410);
        // X_g = sum_k x_k from the digit sums (the digits ARE x to 2^-21 of the group's largest magnitude)
        const int s0 = __reduce_add_sync(0xffffffffu, __dp4a((int)w0, 0x01010101, 0));
        const int s1 = __reduce_add_sync(0xffffffffu, __dp4a((int)w1, 0x01010101, 0));
        const int s2 = __reduce_add_sync(0xffffffffu, __dp4a((int)w2, 0x01010101, 0));
        if (valid) {
          uint32_t* dst = reinterpret_cast<uint32_t*>(xd + (size_t)Gl * kDecGroupBytes + woff);
          dst[0] = w0, dst[32] = w1, dst[64] = w2;
          if (lane < 4) {
            const float X = e * fmaf((float)s2, 6.103515625e-05f, fmaf((float)s1, 0.0078125f, (float)s0));
            // the consumers form 16 * (low-nibble sum) + (high-nibble sum): the 1 / 16 lives here
            const float sc16 = lane == 0 ? 0.0625f : (lane == 1 ? 0.0625f * 0.0078125f : 0.0625f * 6.103515625e-05f);
            gx[Gl * 4 + lane] = lane == 3 ? X : e * sc16;
          }
        }
      }
    }
    __syncwarp();
  }
  DEC_STAMP(4);

  // ldmatrix.x4 addresses of this lane: matrix i = lane >> 3 is (octet i & 1, 32-k block i >> 1 [+ 2 for the second
  // instruction]), row = channel lane & 7 of that octet (quad row (lane & 7) >> 2, row (lane & 3) of the 128-byte
  // tile).  The four result registers ARE the A fragment (rows 0-7 = first octet, rows 8-15 = second octet) of one
  // m16n8k32 MAC over 64 input channels: no register shuffling between the load and the MAC.
  const int li = lane >> 3, lr = lane & 7;
  const uint32_t ldsm_off = (uint32_t)((lr >> 2) * kDecQuadB + (lr & 3) * 32 + (li >> 1) * 16);
  const bool ldsm_b = li & 1;  // this lane addresses the second octet's slot
  const uint32_t sc_off = (uint32_t)(kDecScaleOff + (c >> 2) * (2 * kDecPiece * 8) + (c & 3) * 2);  // + group * 8; zeros + 256
  const uint32_t ring_u32 = smem_u32(ring);
  const uint32_t xd_lane = xd_u32 + (uint32_t)(c * 64 + tig * 16);  // columns 6, 7 read the neighbouring words: ignored
  const uint32_t gx_lane = smem_u32(gx) + (uint32_t)tig * 4u;
  // the lanes tig < 3 carry one digit each and apply the SCALE; the lanes tig == 3 (whose MMA columns carry no digit) apply
  // the ZERO term z_g X_g: one 16-bit load, one conversion and one FMA per octet for every lane
  const uint32_t coef_sel = tig == 3 ? (uint32_t)(kDecPiece * 8) : 0u;  // zeros sit 256 B after the scales
  const int zero4[4] = {0, 0, 0, 0};

  int slot = 0, use = 0;
  DEC_DBG_DECL;
  for (int rb = 0; rb < nrb; ++rb) {
    const int nqb = min(4, nq - 4 * rb);
    const bool two = nqb > 2;  // second octet present
    float y0 = 0.f, y1 = 0.f, yg0 = 0.f, yg1 = 0.f;  // FUSED: yg* park the gate sums while the up weights stream
    for (int pt = 0; pt < npc * NT; ++pt) {
      const int p = FUSED ? (pt >= npc ? pt - npc : pt) : pt;
      if (FUSED && pt == npc) yg0 = y0, yg1 = y1, y0 = 0.f, y1 = 0.f;
      const int ng = min(kDecPiece, ngr - p * kDecPiece);
      int slotB = slot, useB = use;
      if (two && ++slotB == NS) slotB = 0, ++useB;
      DEC_CLK(t0);
      mbar_wait(&full[slot], (uint32_t)(use & 1));
      if (two) mbar_wait(&full[slotB], (uint32_t)(useB & 1));
      DEC_CLK(t1);
      DEC_ACC(0, t1 - t0);
      const uint32_t sa_u32 = ring_u32 + (uint32_t)slot * kDecSlotBytes;
      const uint32_t sb_u32 = ring_u32 + (uint32_t)slotB * kDecSlotBytes;  // == sa_u32 without a second octet
      const uint32_t w_lane = (ldsm_b ? sb_u32 : sa_u32) + ldsm_off;
      if (!DEC_DRY) {
        // per-item bases; a group adds its index times a constant (folded into the instructions for the two groups of
        // a full piece)
        const uint32_t xd_item = xd_lane + (uint32_t)(p * kDecPiece) * kDecGroupBytes;
        const uint32_t gx_item = gx_lane + (uint32_t)(p * kDecPiece) * 16u;
        const uint32_t cA_item = sa_u32 + sc_off + coef_sel, cB_item = sb_u32 + sc_off + coef_sel;
        auto mac_group = [&](const uint32_t gi) {
          uint32_t w0[4], w1[4];
          dec_ldsm4(w0, w_lane + gi * 256u);
          dec_ldsm4(w1, w_lane + gi * 256u + 128u);
          const uint4 bv = dec_lds128(xd_item + gi * (uint32_t)kDecGroupBytes);
          float gv;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(gv) : "r"(gx_item + gi * 16u));
          const uint16_t cA = dec_lds16(cA_item + gi * 8u), cB = dec_lds16(cB_item + gi * 8u);
          int accR[4], accH[4];
          dec_imma(accR, w0[0], w0[1], w0[2], w0[3], bv.x, bv.y, zero4);
          dec_imma(accH, w0[0] & 0xf0f0f0f0u, w0[1] & 0xf0f0f0f0u, w0[2] & 0xf0f0f0f0u, w0[3] & 0xf0f0f0f0u, bv.x, bv.y, zero4);
          dec_imma(accR, w1[0], w1[1], w1[2], w1[3], bv.z, bv.w, accR);
          dec_imma(accH, w1[0] & 0xf0f0f0f0u, w1[1] & 0xf0f0f0f0u, w1[2] & 0xf0f0f0f0u, w1[3] & 0xf0f0f0f0u, bv.z, bv.w, accH);
          // digit lanes: columns 2 tig, 2 tig + 1 = digit tig: low-nibble sum accR[0] - accH[0], high-nibble sum accH[1] / 16
          // -> T16 = 16 (accR[0] - accH[0]) + accH[1] (the 1 / 16 is folded into gv); zero-term lanes: T = 1, gv = X_g
          const float t0f = tig == 3 ? 1.f : (float)(((accR[0] - accH[0]) << 4) + accH[1]);
          const float t1f = tig == 3 ? 1.f : (float)(((accR[2] - accH[2]) << 4) + accH[3]);
          y0 = fmaf(bits16_to_float(cA, kBf16) * gv, t0f, y0);
          y1 = fmaf(bits16_to_float(cB, kBf16) * gv, t1f, y1);  // second octet absent: a copy of the first, never stored
        };
        if (ng == kDecPiece && kDecCons == 16) {
          mac_group((uint32_t)warp);
          mac_group((uint32_t)warp + 16u);
        } else {
          for (int gi = warp; gi < ng; gi += kDecCons) mac_group((uint32_t)gi);
        }
      }
      DEC_CLK(t2);
      DEC_ACC(1, t2 - t1);
      DEC_ACC(3, 1);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty[slot]);  // the slots' words are in registers / consumed
        if (two) mbar_arrive(&empty[slotB]);
      }
      slot = slotB, use = useB;
      if (++slot == NS) slot = 0, ++use;
    }
    // digits live in different lanes (tig): add them, then this warp's 16 partial sums -> red[rb % kDecRed][warp]
    DEC_CLK(t3);
    y0 += __shfl_xor_sync(0xffffffffu, y0, 1);
    y1 += __shfl_xor_sync(0xffffffffu, y1, 1);
    y0 += __shfl_xor_sync(0xffffffffu, y0, 2);
    y1 += __shfl_xor_sync(0xffffffffu, y1, 2);
    if (FUSED) {
      yg0 += __shfl_xor_sync(0xffffffffu, yg0, 1);
      yg1 += __shfl_xor_sync(0xffffffffu, yg1, 1);
      yg0 += __shfl_xor_sync(0xffffffffu, yg0, 2);
      yg1 += __shfl_xor_sync(0xffffffffu, yg1, 2);
    }
    const int rs = rb % kDecRed;
    if (rb >= kDecRed) mbar_wait(&rbfree[rs], (uint32_t)((rb / kDecRed - 1) & 1));
    if (tig == 0) {
      float* r = red + (rs * kDecCons + warp) * RW;
      if (FUSED) {
        r[c] = yg0, r[c + 8] = yg1;   // gate
        r[16 + c] = y0, r[24 + c] = y1;  // up
      } else {
        r[c] = y0;
        r[c + 8] = y1;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&rbfull[rs]);
    DEC_CLK(t4);
    DEC_ACC(2, t4 - t3);
  }
  DEC_STAMP(5);
  DEC_DBG_FLUSH(warp);
}

// ------------------------------------------------------------------------------------ host
namespace {

int dec_sm_count() {
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

int next_dec_seq() {
  static int seq = 0;
  return seq++;
}

}  // namespace

namespace {
int launch_decode_impl(const void* x, const void* qw, const void* sc, const void* sz, const void* qw2, const void* sc2,
                       const void* sz2, void* y, int N, int K, int dtype, bool pdl, const DecodeTuning& tune, cudaStream_t stream) {
  const bool fused = qw2 != nullptr;
  const int nt = fused ? 2 : 1;
  if (N % 8 || K % kGroup) return B200AWQ_ERR_SHAPE;
  const int nsm = dec_sm_count();
  if (nsm < 1) return B200AWQ_ERR_SHAPE;
  const int G = K / kGroup, Q = N / 4;
  DecArgs a{};
  a.x = x, a.qw = static_cast<const uint16_t*>(qw), a.sc = sc, a.sz = sz, a.y = y;
  a.qw2 = static_cast<const uint16_t*>(qw2), a.sc2 = sc2, a.sz2 = sz2;
  a.N = N, a.K = K;
  // k split: only when the rows alone cannot balance the SMs (efficiency of dealing Q quad rows to nsm CTAs below
  // ~0.9) and the halves still make copies of >= 4 KB; or when the digits of the whole k range would crowd out the ring
  auto eff = [&](int s) {
    const int units = nsm / s;
    return (double)Q / units / (double)((Q + units - 1) / units);
  };
  int S = 1;
  if (tune.split >= 1 && tune.split <= 8) {
    S = tune.split;
  } else {
    for (int s = 2; s <= 4 && eff(S) < 0.9; s *= 2)
      if (nsm % s == 0 && G / s >= 16 && eff(s) > eff(S) + 0.03) S = s;
    while (G / S > 64 && S < 8 && nsm % (2 * S) == 0) S *= 2;  // digits: 384 B per group, next to a >= 4-slot ring
  }
  if (S > 1 && (nsm % S || G < S)) S = 1;
  a.S = S;
  a.units = nsm / S;
  a.seq = next_dec_seq();
  const int nq_max = (Q + a.units - 1) / a.units;
  const int nrb_max = (nq_max + 3) / 4;
  if (nrb_max > kDecMaxRb || (long long)Q * (a.units + 1) >= (1ll << 31)) return B200AWQ_ERR_SHAPE;
  a.nrb_max = nrb_max;
  const int ngr = (G + S - 1) / S;
  DecLayout& L = a.L;
  int off = 0;
  L.bars = off, off += 8 * (2 * kDecMaxSlots + 2 * kDecRed + kDecMaxRb);
  off = (off + 127) & ~127;
  const int cons = tune.warps == 8 ? 8 : 16;
  L.x = off, off += ngr * kDecGroupBytes;
  L.gx = off, off += ngr * 4 * 4;
  L.red = off, off += kDecRed * cons * 16 * nt * 4;
  L.xchg = off, off += S * nrb_max * 16 * nt * 4;  // the peers' sums (S - 1 regions) + rank 0's own parked sums
  off = (off + 127) & ~127;
  L.ring = off;
  int ns = (kDecSmemBudget - off) / kDecSlotBytes;
  if (tune.slots > 0) ns = std::min(ns, tune.slots);
  ns = std::min(ns, kDecMaxSlots);
  if (ns < 3) return B200AWQ_ERR_SHAPE;  // activations too large next to a useful ring: the caller falls back
  a.NS = ns;
  L.total = off + ns * kDecSlotBytes;

  static bool attr_set[2][2][2][32] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200AWQ_ERR_DEVICE;
  const int ti = dtype == B200AWQ_DTYPE_F16 ? 0 : 1;
  const int ci = cons == 8 ? 0 : 1;
  const int fi = fused ? 1 : 0;
  const void* kerns[2][2][2] = {
      {{(const void*)w4a16_decode_kernel<__half, 8, false>, (const void*)w4a16_decode_kernel<__half, 8, true>},
       {(const void*)w4a16_decode_kernel<__half, 16, false>, (const void*)w4a16_decode_kernel<__half, 16, true>}},
      {{(const void*)w4a16_decode_kernel<__nv_bfloat16, 8, false>, (const void*)w4a16_decode_kernel<__nv_bfloat16, 8, true>},
       {(const void*)w4a16_decode_kernel<__nv_bfloat16, 16, false>, (const void*)w4a16_decode_kernel<__nv_bfloat16, 16, true>}}};
  const void* kern = kerns[ti][ci][fi];
  if (!attr_set[ti][ci][fi][dev & 31]) {
    if (cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemBudget)) return (int)e;
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    attr_set[ti][ci][fi][dev & 31] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(a.units * a.S));
  cfg.blockDim = dim3((unsigned)((cons + 2) * 32));
  cfg.dynamicSmemBytes = (size_t)L.total;
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
  void* args[] = {const_cast<DecArgs*>(&a)};
  cudaError_t e = cudaLaunchKernelExC(&cfg, kern, args);
  return e == cudaSuccess ? 0 : (int)e;
}
}  // namespace

int launch_decode(const void* x, const void* qw, const void* sc, const void* sz, void* y, int N, int K, int dtype, bool pdl,
                  const DecodeTuning& tune, cudaStream_t stream) {
  return launch_decode_impl(x, qw, sc, sz, nullptr, nullptr, nullptr, y, N, K, dtype, pdl, tune, stream);
}

int launch_decode_mlp_front(const void* x, const void* gqw, const void* gsc, const void* gsz, const void* uqw, const void* usc,
                            const void* usz, void* y, int N, int K, int dtype, bool pdl, const DecodeTuning& tune,
                            cudaStream_t stream) {
  if (!uqw || !usc || !usz) return B200AWQ_ERR_ALIGN;
  return launch_decode_impl(x, gqw, gsc, gsz, uqw, usc, usz, y, N, K, dtype, pdl, tune, stream);
}

}  // namespace b200awq
