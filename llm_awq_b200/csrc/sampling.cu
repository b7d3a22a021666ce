// sample_next_token: tinychat's per-token logits chain (temperature, repetition penalty, top-p, top-k) and the choice of
// the token (greedy or the inverse CDF of a caller-given uniform), one launch (DESIGN §3.12).
//
// One cluster of kSampleCtas CTAs per row.  Each CTA holds a contiguous slice of the row in shared memory as the
// order-preserving uint32 image of the processed fp32 logits (`order_key`), so the selection never sorts: the top-p
// boundary and the top-k threshold are each found by four 8-bit radix passes over those keys, MSB first.  A pass builds
// the CTA's histogram of the keys that match the digits decided so far (counts, and for top-p fixed-point softmax
// mass), every CTA then reads all the cluster's histograms over distributed shared memory and takes the same decision.
// The mass of a key is exp(x - max) in fixed point (kMassOne = 1.0): integer sums are exact and do not depend on the
// order of the shared-memory atomics, so the call is deterministic and the passes agree with each other bit for bit.
// The draw is a prefix of kept mass over the cluster's CTAs, then a block scan inside the CTA that holds the target.
#include <math.h>

#include <algorithm>

#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

constexpr int kSampleCtas = 8;  // CTAs per row: one portable cluster
constexpr int kSampleThreads = 512;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kBins = 256;  // 8-bit radix digits
constexpr unsigned long long kMassOne = 1ull << 44;  // fixed point of a probability ratio; vocab * kMassOne < 2^63
constexpr uint32_t kNoBin = 0xffffffffu;

struct SampleArgs {
  const float* logits;
  long long logits_stride;
  const long long* prev;
  long long prev_stride;
  const float* uniforms;
  long long* tokens;
  int batch, vocab, slice, n_prev;  // slice: keys per CTA, a multiple of 32
  float temperature, penalty, thr;  // thr = fp32(1 - top_p)
  int top_p_on, top_k, greedy;
};

// fp32 -> uint32 with the same order (after NaN -> -inf and -0 -> +0, equal keys are equal values)
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// exp(x - max) in units of kMassOne.  The maxima weigh exactly kMassOne, also when the maximum is infinite (an all -inf
// row then draws among its kept entries); -inf entries of a row with a finite maximum weigh 0.
__device__ __forceinline__ unsigned long long fixed_mass(uint32_t k, float mx) {
  const float x = key_value(k);
  if (x == mx) return kMassOne;
  const float p = expf(x - mx);
  return p > 0.f ? __float2ull_rn(p * (float)kMassOne) : 0ull;
}

__device__ __forceinline__ uint32_t ld_cluster_u32(uint32_t cluster_addr) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(cluster_addr) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_cluster_u64(uint32_t cluster_addr) {
  unsigned long long v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(cluster_addr) : "memory");
  return v;
}

template <typename V>
__device__ __forceinline__ V warp_inclusive_scan(V v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const V y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  return v;
}

// Exclusive prefix of `v` over the CTA's threads in thread order; `total` receives the CTA's sum.
__device__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* warp_sums,
                                                   unsigned long long& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long inc = warp_inclusive_scan(v, lane);
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  unsigned long long before = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kSampleWarps; ++w) {
    const unsigned long long s = warp_sums[w];
    if (w < warp) before += s;
    tot += s;
  }
  __syncthreads();  // warp_sums may be reused
  total = tot;
  return before + inc - v;
}

// The radix decisions of one row, written by warp 0 between passes.
struct RowState {
  unsigned long long rem;  // top-p: fixed-point mass still to remove; top-k: keys still to take from the top
  uint32_t prefix;         // key bits decided so far
  uint32_t above;          // top-p: keys above the decided prefix range
  uint32_t digit;          // the last pass's digit
  int keep_last;           // top-p: nothing reaches the threshold (thr rounds to 1): keep the last key only
};

__global__ void __launch_bounds__(kSampleThreads, 1) sample_next_token_kernel(const SampleArgs a) {
  extern __shared__ __align__(16) uint32_t keys[];  // a.slice keys, then a.slice / 32 words of penalty flags
  uint32_t* flags = keys + a.slice;
  // read by the other CTAs of the cluster: double-buffered by pass parity, so one cluster barrier per pass suffices
  __shared__ unsigned long long h_mass[2][kBins];
  __shared__ uint32_t h_cnt[2][kBins];
  __shared__ float cta_max;
  __shared__ unsigned long long cta_total;
  // local
  __shared__ unsigned long long g_mass[kBins];
  __shared__ uint32_t g_cnt[kBins];
  __shared__ unsigned long long warp_sums[kSampleWarps];
  __shared__ RowState st;
  __shared__ float row_max;
  __shared__ unsigned long long draw_lo, draw_target;  // this CTA's first cluster-wide weight, the target weight
  __shared__ uint32_t ties_before;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank();
  const int base = (int)rank * a.slice;
  const int n = max(0, min(a.slice, a.vocab - base));
  const int chunk = (n + kSampleThreads - 1) / kSampleThreads;  // the scans' contiguous per-thread ranges
  const int c0 = min(n, tid * chunk), c1 = min(n, c0 + chunk);
  const int clusters = gridDim.x / kSampleCtas;

  pdl_launch_dependents();
  pdl_wait_prior_grid();  // the logits are normally the previous launch's output

  int pass = 0;  // histogram buffer parity, continued over rows
  for (int b = blockIdx.x / kSampleCtas; b < a.batch; b += clusters) {
    // ---- repetition penalty: mark this slice's ids (each once, however often it occurs)
    const bool penalise = a.penalty > 1.f && a.n_prev > 0;
    if (penalise) {
      for (int i = tid; i < a.slice / 32; i += kSampleThreads) flags[i] = 0;
      __syncthreads();
      const long long* ids = a.prev + (long long)b * a.prev_stride;
      for (int i = tid; i < a.n_prev; i += kSampleThreads) {
        const long long id = ids[i] - base;
        if (id >= 0 && id < n) atomicOr(&flags[id >> 5], 1u << (id & 31));
      }
      __syncthreads();
    }
    // ---- temperature and penalty, keys, the row's maximum
    const float* row = a.logits + (long long)b * a.logits_stride + base;
    float lmax = -INFINITY;
    for (int j = tid; j < n; j += kSampleThreads) {
      float x = row[j];
      if (a.temperature != 1.f) x = __fdiv_rn(x, a.temperature);
      if (penalise && (flags[j >> 5] >> (j & 31) & 1u)) x = x < 0.f ? __fmul_rn(x, a.penalty) : __fdiv_rn(x, a.penalty);
      if (x != x) x = -INFINITY;
      if (x == 0.f) x = 0.f;
      keys[j] = order_key(x);
      lmax = fmaxf(lmax, x);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    if (lane == 0) g_mass[warp] = __float_as_uint(lmax);  // g_mass as scratch
    __syncthreads();
    if (tid == 0) {
      float m = -INFINITY;
      for (int w = 0; w < kSampleWarps; ++w) m = fmaxf(m, __uint_as_float((uint32_t)g_mass[w]));
      cta_max = m;
    }
    cluster_sync_all();
    if (warp == 0) {
      float m = lane < kSampleCtas ? ld_cluster_f32(map_to_rank(smem_u32(&cta_max), lane)) : -INFINITY;
#pragma unroll
      for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) {
        row_max = m;
        st = RowState{0, 0, 0, 0, 0};
        ties_before = 0;
      }
    }
    __syncthreads();
    const float mx = row_max;
    const uint32_t kmax = order_key(mx);

    // One radix pass at bit `shift` over the keys that match st.prefix above it (and lie above `floor_key`):
    // this CTA's histograms, then the cluster's in g_cnt / g_mass.
    auto radix_pass = [&](int shift, bool with_mass, uint32_t floor_key) {
      const int buf = pass++ & 1;
      const uint32_t mask = shift == 24 ? 0u : ~0u << (shift + 8);
      const uint32_t prefix = st.prefix;
      for (int i = tid; i < kBins; i += kSampleThreads) h_cnt[buf][i] = 0, h_mass[buf][i] = 0;
      __syncthreads();
      for (int j0 = warp * 32; j0 < n; j0 += kSampleThreads) {  // warp-uniform trip count
        const int j = j0 + lane;
        uint32_t bin = kNoBin, k = 0;
        if (j < n) {
          k = keys[j];
          if ((k & mask) == prefix && k > floor_key) bin = (k >> shift) & (kBins - 1);
        }
        // one atomic per distinct bin and warp: a row's high digits are few, so the lanes mostly agree
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        if (bin == kNoBin) continue;
        const bool leader = lane == __ffs(peers) - 1;
        if (with_mass) {
          const unsigned long long m = fixed_mass(k, mx);  // < 2^45: three 22-bit pieces sum exactly in 32 bits
          const unsigned long long lo = __reduce_add_sync(peers, (uint32_t)(m & 0x3fffff));
          const unsigned long long mid = __reduce_add_sync(peers, (uint32_t)(m >> 22 & 0x3fffff));
          const unsigned long long hi = __reduce_add_sync(peers, (uint32_t)(m >> 44));
          if (leader) atomicAdd(&h_mass[buf][bin], lo + (mid << 22) + (hi << 44));
        }
        if (leader) atomicAdd(&h_cnt[buf][bin], (uint32_t)__popc(peers));
      }
      cluster_sync_all();
      for (int i = tid; i < kBins; i += kSampleThreads) {
        uint32_t c = 0;
        unsigned long long m = 0;
        for (int r = 0; r < kSampleCtas; ++r) {
          c += ld_cluster_u32(map_to_rank(smem_u32(&h_cnt[buf][i]), r));
          if (with_mass) m += ld_cluster_u64(map_to_rank(smem_u32(&h_mass[buf][i]), r));
        }
        g_cnt[i] = c;
        g_mass[i] = m;
      }
      __syncthreads();
      return buf;
    };

    // ---- top-p: the first key, in ascending (key, index) order, whose inclusive mass exceeds thr * total
    uint32_t kp = 0, tie_keep_from = 0, kept_ties = 0, kept_p = (uint32_t)a.vocab;
    if (a.top_p_on) {
      int buf = 0;
      for (int shift = 24; shift >= 0; shift -= 8) {
        buf = radix_pass(shift, true, 0u);
        if (warp == 0) {
          unsigned long long ms = 0;
          uint32_t cs = 0;
          for (int i = 0; i < 8; ++i) ms += g_mass[lane * 8 + i], cs += g_cnt[lane * 8 + i];
          const unsigned long long pm = warp_inclusive_scan(ms, lane);
          const uint32_t pc = warp_inclusive_scan(cs, lane);
          const unsigned long long tot_m = __shfl_sync(0xffffffffu, pm, 31);
          const uint32_t tot_c = __shfl_sync(0xffffffffu, pc, 31);
          // thr * total in double: exact enough for a fixed, deterministic threshold
          const unsigned long long rem = shift == 24 ? (unsigned long long)((double)a.thr * (double)tot_m) : st.rem;
          const bool keep_last = st.keep_last || tot_m <= rem;
          __syncwarp();
          if (!keep_last) {
            const int L = __ffs(__ballot_sync(0xffffffffu, pm > rem)) - 1;
            if (lane == L) {
              unsigned long long am = pm - ms;
              uint32_t ac = pc - cs;
              int d = lane * 8;
              while (am + g_mass[d] <= rem) am += g_mass[d], ac += g_cnt[d], ++d;
              st.rem = rem - am;
              st.above += tot_c - ac - g_cnt[d];
              st.prefix |= (uint32_t)d << shift;
              st.digit = d;
            }
          } else {
            const int L = 31 - __clz(__ballot_sync(0xffffffffu, cs > 0));
            if (lane == L) {
              int d = lane * 8 + 7;
              while (g_cnt[d] == 0) --d;
              st.keep_last = 1;
              st.prefix |= (uint32_t)d << shift;
              st.digit = d;
            }
          }
        }
        __syncthreads();
      }
      kp = st.prefix;
      const uint32_t ties = g_cnt[st.digit];
      // the ties at kp are removed in index order while their inclusive mass stays <= the threshold
      tie_keep_from = st.keep_last ? ties - 1 : (uint32_t)(st.rem / (g_mass[st.digit] / ties));
      kept_ties = ties - tie_keep_from;
      kept_p = st.above + kept_ties;
      if (tid == 0) {  // ties in the lower CTAs (the buffer is rewritten only two cluster barriers later)
        uint32_t t = 0;
        for (uint32_t r = 0; r < rank; ++r) t += ld_cluster_u32(map_to_rank(smem_u32(&h_cnt[buf][st.digit]), r));
        ties_before = t;
      }
      __syncthreads();
      if (tid == 0) st = RowState{0, 0, 0, 0, 0};
      __syncthreads();
    }

    // ---- top-k: the top_k-th largest key among the top-p survivors (keys > kp, and kept_ties keys == kp)
    uint32_t kk = 0;
    if (a.top_k > 0 && (uint32_t)a.top_k < kept_p) {
      if (tid == 0) st.rem = (unsigned long long)a.top_k;
      __syncthreads();
      for (int shift = 24; shift >= 0; shift -= 8) {
        radix_pass(shift, false, kp);
        const uint32_t mask = shift == 24 ? 0u : ~0u << (shift + 8);
        if (warp == 0) {
          uint32_t cs = 0;
          for (int i = 0; i < 8; ++i) {
            const int d = lane * 8 + i;
            uint32_t c = g_cnt[d];
            if (kept_ties && (kp & mask) == st.prefix && ((kp >> shift) & (kBins - 1)) == (uint32_t)d) c += kept_ties;
            g_cnt[d] = c;
            cs += c;
          }
          const uint32_t pc = warp_inclusive_scan(cs, lane);
          const uint32_t tot_c = __shfl_sync(0xffffffffu, pc, 31);
          const uint32_t rem = (uint32_t)st.rem;
          __syncwarp();
          // the largest digit whose keys and all keys above it number at least rem
          const int L = 31 - __clz(__ballot_sync(0xffffffffu, pc - cs <= tot_c - rem));
          if (lane == L) {
            uint32_t below = pc - cs;
            int d = lane * 8;
            while (d < lane * 8 + 7 && below + g_cnt[d] <= tot_c - rem) below += g_cnt[d], ++d;
            st.rem = rem - (tot_c - below - g_cnt[d]);
            st.prefix |= (uint32_t)d << shift;
          }
        }
        __syncthreads();
      }
      kk = st.prefix;
    }

    // ---- the draw: weights of the kept keys in index order, the target over the cluster, the CTA that holds it
    unsigned long long total;
    uint32_t tie_rank = ties_before;
    if (a.top_p_on) {
      uint32_t t = 0;
      for (int j = c0; j < c1; ++j) t += keys[j] == kp;
      tie_rank += (uint32_t)block_exclusive_scan(t, warp_sums, total);
    }
    auto weight = [&](uint32_t k, uint32_t& rank_in_ties) -> unsigned long long {
      const bool tie = k == kp;
      const bool kept = (k > kp || (tie && rank_in_ties >= tie_keep_from)) && k >= kk;
      rank_in_ties += tie;
      if (!kept) return 0;
      if (a.greedy) return k == kmax;
      return fixed_mass(k, mx);
    };
    unsigned long long w = 0;
    {
      uint32_t r = tie_rank;
      for (int j = c0; j < c1; ++j) w += weight(keys[j], r);
    }
    const unsigned long long w_before = block_exclusive_scan(w, warp_sums, total);
    if (tid == 0) cta_total = total;
    cluster_sync_all();
    if (warp == 0) {
      const unsigned long long t = lane < kSampleCtas ? ld_cluster_u64(map_to_rank(smem_u32(&cta_total), lane)) : 0;
      const unsigned long long incl = warp_inclusive_scan(t, lane);
      const unsigned long long sum = __shfl_sync(0xffffffffu, incl, 31);  // > 0: a kept maximum weighs >= 1
      const unsigned long long lo = __shfl_sync(0xffffffffu, incl - t, rank);
      if (lane == 0) {
        unsigned long long target = 0;  // greedy: the first kept maximum
        if (!a.greedy) {
          const float u = a.uniforms[b];
          target = u > 0.f ? (unsigned long long)((double)u * (double)sum) : 0ull;
          target = min(target, sum - 1);
        }
        draw_lo = lo;
        draw_target = target;
      }
    }
    __syncthreads();
    const unsigned long long target = draw_target - draw_lo;  // wraps for CTAs below the target: no thread matches
    if (draw_target >= draw_lo && target >= w_before && target < w_before + w) {
      uint32_t r = tie_rank;
      unsigned long long acc = w_before;
      for (int j = c0; j < c1; ++j) {
        acc += weight(keys[j], r);
        if (acc > target) {
          a.tokens[b] = base + j;
          break;
        }
      }
    }
    cluster_sync_all();  // no CTA leaves the row while its shared memory may still be read
  }
}

}  // namespace

int launch_sample_next_token(const float* logits, long long logits_stride, int batch, int vocab, const long long* prev_ids,
                             long long prev_stride, int n_prev, float temperature, float penalty, float top_p, int top_k,
                             int greedy, const float* uniforms, long long* tokens, bool pdl, cudaStream_t stream) {
  SampleArgs a{};
  a.logits = logits, a.logits_stride = logits_stride, a.prev = prev_ids, a.prev_stride = prev_stride;
  a.uniforms = uniforms, a.tokens = tokens;
  a.batch = batch, a.vocab = vocab, a.n_prev = n_prev;
  a.slice = ((vocab + kSampleCtas - 1) / kSampleCtas + 31) / 32 * 32;
  a.temperature = temperature, a.penalty = penalty;
  a.top_p_on = top_p < 1.f;
  a.thr = (float)(1.0 - (double)top_p);
  a.top_k = top_k, a.greedy = greedy != 0;
  const int max_smem = (B200AWQ_SAMPLE_MAX_VOCAB / kSampleCtas) * 4 + (B200AWQ_SAMPLE_MAX_VOCAB / kSampleCtas) / 8;
  if (cudaError_t e = ensure_dyn_smem<sample_next_token_kernel>(max_smem)) return (int)e;
  const size_t smem = (size_t)a.slice * 4 + (size_t)a.slice / 8;
  const int clusters = std::min(batch, 65535);
  return launch_kernel(sample_next_token_kernel, dim3((unsigned)(clusters * kSampleCtas)), dim3(kSampleThreads), smem,
                       stream, pdl, kSampleCtas, a);
}

}  // namespace b200awq
