// Attention of few queries over many keys for sm_90a (long-context decode, chunks over a KV cache): the key range is
// split over CTAs, each CTA packs the query rows that read one KV head into wgmma tiles.
//
//   O = softmax(scale * Q K^T + mask) V        fp16 / bf16, head size D in {64, 128}
//
// Two launches share the kernel:
//   * flash_attn_func's split-key route (kWG = 1): Sq * (H / Hkv) <= 64, one 64-row tile, K and V [B][Sk][Hkv][D] with
//     the caller's strides.
//   * kv_cache_attention (kWG = 2): any Sq.  Each CTA takes a row tile of 128 packed rows in two consumer warpgroups
//     of 64 that share one K / V ring, so each K / V tile is read once per 128 rows; a CTA whose rows fit in 64 runs
//     one warpgroup.  With kFtK, K is tinychat's FasterTransformer cache [B][Hkv][D / 8][Lmax][8], read in place by a
//     4-D map {8, Sk, D / 8, B * Hkv}: a 128-key box lands as [D / 8][128 keys][8], wgmma's K-major no-swizzle operand
//     (core matrices of 8 keys x 16 B; 128 x 16 B between k-adjacent ones, 128 B between 8-key groups).  Under causal
//     masking a row tile loads no key tile past the horizon of its last row.
//
// Numerics as prefill_attention.cu (S in fp32 from T operands, p = exp2(scale * log2(e) * (s - max)) as one FFMA + ex2,
// P rounded to T, O in fp32), plus the combine of the splits below.
//
// Tile: one CTA = (key split, row tile, KV head, batch row).  The R = Sq * G query rows (G = H / Hkv) of a KV head are
// packed, row s * G + g = query s of head hk * G + g, into row tiles of kWG * 64 rows; rows past R are zero and never
// stored.
//   * Q is read once with 16-byte loads from the caller's strides and stored with the 128-byte swizzle TMA would use.
//   * K and V tiles of 128 keys arrive by 4-D TMA from the caller's strides (views into a larger cache are read in
//     place; the maps' token extent is Sk, so slots past the view are never read) into a full / empty mbarrier ring
//     of 192 KB (D = 128: 3 stages of K + V, D = 64: 6), which keeps the HBM requests of one SM in flight.
//   * S = Q K^T with wgmma.m64n128k16, O += P V with P from registers, as in prefill_attention.cu; the P V of tile n and
//     the Q K^T of tile n + 1 go to the tensor core as one batch.
//   * Causal (bottom-right, per packed row: query s sees keys j <= s + Sk - Sq): masked keys select -inf.
// Splits: the number of splits follows from the shape and the SM count (plan_splits).  Each split writes fp32
// partials (unnormalised O, the row max m of the raw scores, the row sum l) to the workspace and counts its arrival;
// the last CTA of a cell (row tile, KV head, batch row) to arrive combines them in split order:
//   O = sum_s w_s O_s / sum_s w_s l_s,  w_s = exp2(scale * log2(e) * (m_s - M)),  M = max_s m_s,
// rounded once to T.  A split in which a row sees no key has m_s = -inf and weighs 0; a row that sees no key at all is
// zero.  The counter is only an arrival count: which CTA combines varies, the arithmetic and its order do not, so
// every call returns the same bits.  With one split the CTA writes O / l directly and the workspace is not touched.
// Warp roles (one CTA per SM): warps 0 .. 4 kWG - 1 = the consumer warpgroups (wgmma, softmax, epilogue, combine); warp
// 4 kWG = TMA producer (one thread).  kWG = 2 adds three idle warps to the producer's warpgroup and moves registers
// from it to the consumers (setmaxnreg: 232 each, 40 for the producer).
#include <algorithm>

#include "attention_wgmma.cuh"

namespace b200awq {
namespace {

constexpr int kRows = 64;       // packed query rows per consumer warpgroup
constexpr int kBN = 128;        // keys per pipeline stage
constexpr int kRingBytes = 192 * 1024;  // K / V tiles in flight
constexpr int kMaxSms = 256;    // the split rule and the workspace bound assume at most this many SMs

template <int D, int kWG = 1>
struct SplitCfg {
  // consumer warpgroups + producer warp; kWG = 2: a producer warpgroup, so that setmaxnreg can move its registers to
  // the consumers (at the 168 registers of 384 threads ptxas would serialise the wgmma batches)
  static constexpr int kThreads = kWG == 1 ? 160 : kWG * 128 + 128;
  static constexpr int kStages = D == 64 ? 6 : 3;    // 192 KB of K / V tiles in flight
  static constexpr int kQBytes = kRows * D * 2;      // Q block of one warpgroup
  static constexpr int kKBytes = kBN * D * 2;        // K tile; the V tile follows it
  static constexpr int kStageBytes = 2 * kKBytes;
  static constexpr int kSmem = kWG * kQBytes + kStages * kStageBytes + 1024 /*align*/ + 128 /*barriers*/;
  static_assert(kQBytes % 1024 == 0 && kKBytes % 1024 == 0, "tiles must stay aligned to the swizzle repeat");
  static_assert(kStages * kStageBytes == kRingBytes, "the combine scratch bound assumes this ring");
  static_assert(kSmem <= 232448, "over the sm_90 shared-memory limit per block");
};

// Largest split count whose combine scratch fits in the ring: row maxima / weights and row sums (splits x rows floats
// each) and inverse row sums (rows floats), for `rows` packed rows per cell.  383 for rows <= 64 (above kMaxSms).
constexpr int max_splits(int rows) { return (kRingBytes / 4 - rows) / (2 * rows); }
static_assert(max_splits(kRows) >= kMaxSms, "a 64-row cell must take any split count the SM count allows");

struct SplitArgs {
  const void* q;
  void* out;                  // [B][Sq][H][D] contiguous
  float* part;                // [cells][splits][crows][D] O of each split, then [cells][splits][crows][2] (m, l)
  unsigned int* count;        // [cells] arrival counters (zero between launches)
  long long qs0, qs1, qs2;    // q strides (batch, token, head) in elements
  int sq, sk, heads, kv_heads, group, rows, splits, tiles_per_split;
  float scale_log2;
  int causal;
};

// Rows of the cell starting at packed row r0, and the row stride of a cell's partials (kWG = 1: one cell of all rows)
template <int kWG>
__device__ __forceinline__ int cell_rows_at(const SplitArgs& a, int r0) {
  return kWG == 1 ? a.rows : min(kWG * kRows, a.rows - r0);
}
template <int kWG>
__device__ __forceinline__ int cell_stride(const SplitArgs& a) {
  return kWG == 1 ? a.rows : min(kWG * kRows, a.rows);
}
// Keys the rows from r0 can see: causal stops at the horizon of the cell's last row
template <int kWG>
__device__ __forceinline__ int cell_key_end(const SplitArgs& a, int r0) {
  return kWG == 1 || !a.causal ? a.sk : max(0, min(a.sk, (r0 + cell_rows_at<kWG>(a, r0) - 1) / a.group + a.sk - a.sq + 1));
}
// bar.sync 1 for the consumers of kWG = 1; kWG = 2: 1 + wg per warpgroup, 3 for all consumer threads
template <int kWG>
__device__ __forceinline__ void sync_warpgroup(int wg) {
  if constexpr (kWG == 1) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}
template <int kWG>
__device__ __forceinline__ void sync_consumers(int n_threads) {
  if constexpr (kWG == 1) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 3, %0;" ::"r"(n_threads) : "memory");
}

template <typename T, int D, int kWG = 1, bool kFtK = false>
__global__ void __launch_bounds__(SplitCfg<D, kWG>::kThreads, 1)
splitkv_attention_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                         const __grid_constant__ SplitArgs a) {
  using C = SplitCfg<D, kWG>;
  constexpr int kStages = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ unsigned int s_last;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* qs = smem;                              // Q blocks of the warpgroups: D / 64 blocks [64][64], 128-byte swizzle
  uint8_t* kvs = qs + kWG * C::kQBytes;            // stage s: K tile, then V tile
  uint64_t* full = reinterpret_cast<uint64_t*>(kvs + kStages * C::kStageBytes);  // [kStages] TMA -> consumers
  uint64_t* empty = full + kStages;                // [kStages] consumer warps -> TMA

  // this CTA's cell: KV head hk of batch row b, packed rows from r0 (kWG = 1: all R rows, grid (split, hk, b))
  const int split = blockIdx.x;
  const int hk = kWG == 1 ? (int)blockIdx.y : (int)(blockIdx.z % a.kv_heads);
  const int b = kWG == 1 ? (int)blockIdx.z : (int)(blockIdx.z / a.kv_heads);
  const int r0 = kWG == 1 ? 0 : blockIdx.y * kWG * kRows;
  const int t0 = split * a.tiles_per_split;
  const int n_tiles = max(0, min((cell_key_end<kWG>(a, r0) + kBN - 1) / kBN, t0 + a.tiles_per_split) - t0);
  const int n_wg = kWG == 1 ? 1 : (cell_rows_at<kWG>(a, r0) + kRows - 1) / kRows;  // consumer warpgroups with rows
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4 * n_wg);
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (kWG == 1 ? warp == 4 : warp >= 4 * kWG) {
    // =========================================================== TMA producer
    if constexpr (kWG > 1) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if ((kWG == 1 || warp == 4 * kWG) && lane == 0 && n_tiles > 0) {
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      int s = 0;
      uint32_t ph = 0;
      for (int n = 0; n < n_tiles; ++n) {
        const int row = (t0 + n) * kBN;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], C::kStageBytes);
        uint8_t* st = kvs + s * C::kStageBytes;
        if constexpr (kFtK) tma_load_4d(st, &tm_k, &full[s], 0, row, 0, b * a.kv_heads + hk);  // [D / 8][128][8]
#pragma unroll
        for (int c = 0; c < D / 64; ++c) {
          if constexpr (!kFtK) tma_load_4d(st + c * kBN * 128, &tm_k, &full[s], c * 64, row, hk, b);
          tma_load_4d(st + C::kKBytes + c * kBN * 128, &tm_v, &full[s], c * 64, row, hk, b);
        }
        if (++s == kStages) s = 0, ph ^= 1;
      }
    }
    return;
  }

  // =========================================================== consumer warpgroups
  if constexpr (kWG > 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = kWG == 1 ? 0 : warp >> 2;
  if (wg >= n_wg) return;  // no rows for this warpgroup (it never arrives on the ring's barriers)
  const int tid = kWG == 1 ? threadIdx.x : threadIdx.x & 127;  // thread of the warpgroup
  const int wr0 = r0 + wg * kRows;        // this warpgroup's first packed row
  uint8_t* qw = qs + wg * C::kQBytes;     // and its Q block
  {
    // packed Q tile, 16-byte chunks: chunk c of row r lands at block c / 8, row r, position (c % 8) ^ (r % 8)
    const T* qg = static_cast<const T*>(a.q) + (long long)b * a.qs0;
    constexpr int kChunks = D / 8;
    for (int e = tid; e < kRows * kChunks; e += 128) {
      const int r = e / kChunks, c = e % kChunks;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (wr0 + r < a.rows) {
        const int s = (wr0 + r) / a.group, h = hk * a.group + (wr0 + r) % a.group;
        val = __ldg(reinterpret_cast<const uint4*>(qg + s * a.qs1 + h * a.qs2 + c * 8));
      }
      *reinterpret_cast<uint4*>(qw + (c / 8) * kRows * 128 + r * 128 + (((c % 8) ^ (r & 7)) * 16)) = val;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> wgmma operand reads
    sync_warpgroup<kWG>(wg);
  }

  const int g = lane >> 2, t = lane & 3;
  const int r_lo = r0 + wg * kRows + (kWG == 1 ? warp : warp & 3) * 16 + g;  // this thread's packed rows: r_lo, r_lo + 8
  // keys below lim are seen by the row: all Sk, or causal s + Sk - Sq + 1 (<= 0: none)
  const int diag = a.sk - a.sq;
  const int lim_lo = a.causal ? min(a.sk, r_lo / a.group + diag + 1) : a.sk;
  const int lim_hi = a.causal ? min(a.sk, (r_lo + 8) / a.group + diag + 1) : a.sk;
  // accumulator element 4 j + e: row r_lo + 8 (e >> 1), column 8 j + 2 t + (e & 1)
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;  // running max (raw scores), partial sums
  const uint32_t q_addr = smem_u32(qw);
  uint32_t pa[kBN / 16][4];  // P of the current tile as the A fragments of the 8 k16 steps of O += P V
  float sc[64];              // S of the next tile
  const float scale_log2 = a.scale_log2;

  auto issue_qk = [&](int stage) {
    const uint32_t k_addr = smem_u32(kvs + stage * C::kStageBytes);
    // FT K: no swizzle, 8-column blocks kBN * 16 bytes apart (two per k16 step), 8-key groups 128 bytes apart
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)  // k16 step kk: block kk / 4, +32 bytes per step inside the block
      wgmma_ss<T>(sc, make_smem_desc(q_addr + (kk / 4) * kRows * 128 + (kk % 4) * 32, 1, 16, 1024),
                  kFtK ? make_smem_desc(k_addr + kk * 2 * kBN * 16, 0, kBN * 16, 128)
                       : make_smem_desc(k_addr + (kk / 4) * kBN * 128 + (kk % 4) * 32, 1, 16, 1024),
                  kk > 0 ? 1u : 0u);
  };
  auto issue_pv = [&](int stage) {
    const uint32_t v_addr = smem_u32(kvs + stage * C::kStageBytes + C::kKBytes);
    // V is MN-major: 64-column blocks kBN * 128 bytes apart, 8-key groups 1024 bytes apart
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk)
      wgmma_rs<T, D, true>(o, pa[kk], make_smem_desc(v_addr + kk * 16 * 128, 1, kBN * 128, 1024), 1u);
  };
  // mask and online softmax of tile n's S: P into pa, O rescaled
  auto softmax = [&](int n) {
    const int k0 = (t0 + n) * kBN;
    if (k0 + kBN > min(lim_lo, lim_hi)) {  // on the raw scores: scale_log2 > 0 keeps -inf the smallest value
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int key = k0 + 8 * (i >> 2) + 2 * t + (i & 1);
        sc[i] = key < ((i & 2) ? lim_hi : lim_lo) ? sc[i] : -INFINITY;
      }
    }
    online_softmax<T>(sc, pa, o, m_lo, m_hi, l_lo, l_hi, scale_log2);
  };
  consume_tiles<kStages>(n_tiles, full, empty, lane, sc, o, NoTurns{}, issue_qk, issue_pv, softmax);
  row_sums(l_lo, l_hi);

  const int lr_lo = r_lo - r0;        // this thread's rows in the cell: lr_lo, lr_lo + 8
  const int ctid = threadIdx.x;       // thread of the CTA's consumers
  const int n_threads = 128 * n_wg;   // consumer threads of this CTA
  T* out = static_cast<T*>(a.out);
  auto out_row = [&](int r) {  // packed row r = query r / G of head hk * G + r % G
    return out + (((size_t)b * a.sq + r / a.group) * a.heads + hk * a.group + r % a.group) * D;
  };
  if (a.splits == 1) {  // ------------------------------------------------ O / l, rounded once, written directly
    const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f, inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
    T* lo = r_lo < a.rows ? out_row(r_lo) : nullptr;
    T* hi = r_lo + 8 < a.rows ? out_row(r_lo + 8) : nullptr;
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int col = 8 * j + 2 * t;
      if (lo) *reinterpret_cast<uint32_t*>(lo + col) = pack2<T>(o[4 * j] * inv_lo, o[4 * j + 1] * inv_lo);
      if (hi) *reinterpret_cast<uint32_t*>(hi + col) = pack2<T>(o[4 * j + 2] * inv_hi, o[4 * j + 3] * inv_hi);
    }
    return;
  }

  // ------------------------------------------------ partials of this split
  const int cell = kWG == 1 ? b * a.kv_heads + hk : blockIdx.z * gridDim.y + blockIdx.y;
  const size_t per_cell = (size_t)a.splits * cell_stride<kWG>(a);  // (split, row) pairs of one cell
  float* part = a.part + cell * per_cell * D;
  float* ml = a.part + (size_t)gridDim.y * gridDim.z * per_cell * D + cell * per_cell * 2;
  {
    float* p_lo = part + ((size_t)split * cell_stride<kWG>(a) + lr_lo) * D;
    float* p_hi = p_lo + 8 * D;
    const bool st_lo = lr_lo < cell_rows_at<kWG>(a, r0), st_hi = lr_lo + 8 < cell_rows_at<kWG>(a, r0);
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int col = 8 * j + 2 * t;
      if (st_lo) *reinterpret_cast<float2*>(p_lo + col) = make_float2(o[4 * j], o[4 * j + 1]);
      if (st_hi) *reinterpret_cast<float2*>(p_hi + col) = make_float2(o[4 * j + 2], o[4 * j + 3]);
    }
    float* q_lo = ml + ((size_t)split * cell_stride<kWG>(a) + lr_lo) * 2;
    if (t == 0 && st_lo) *reinterpret_cast<float2*>(q_lo) = make_float2(m_lo, l_lo);
    if (t == 0 && st_hi) *reinterpret_cast<float2*>(q_lo + 16) = make_float2(m_hi, l_hi);
  }
  __threadfence();
  sync_consumers<kWG>(n_threads);
  if (ctid == 0) s_last = atomicAdd(&a.count[cell], 1u) == (unsigned)a.splits - 1 ? 1u : 0u;
  sync_consumers<kWG>(n_threads);
  if (!s_last) return;
  __threadfence();

  // ------------------------------------------------ the last CTA of this cell combines, in split order
  // (every TMA write to the ring has landed: its shared memory holds the scratch).  The loads of the partials are
  // independent of each other; only the sums run in split order.
  const int n_pairs = (int)per_cell;
  float* wts = reinterpret_cast<float*>(kvs);  // [splits][crows]: row maxima, then weights
  float* sums = wts + n_pairs;                 // [splits][crows]
  float* inv = sums + n_pairs;                 // [crows]
  for (int e = ctid; e < n_pairs; e += n_threads) {
    const float2 x = __ldcg(reinterpret_cast<const float2*>(ml) + e);
    wts[e] = x.x, sums[e] = x.y;
  }
  sync_consumers<kWG>(n_threads);
  for (int r = ctid; r < cell_rows_at<kWG>(a, r0); r += n_threads) {
    float M = -INFINITY;
    for (int sp = 0; sp < a.splits; ++sp) M = fmaxf(M, wts[sp * cell_stride<kWG>(a) + r]);
    const float nb = M == -INFINITY ? 0.f : -M * scale_log2;
    float den = 0.f;
    for (int sp = 0; sp < a.splits; ++sp) {
      const float w = ex2(fmaf(wts[sp * cell_stride<kWG>(a) + r], scale_log2, nb));
      wts[sp * cell_stride<kWG>(a) + r] = w;
      den = fmaf(w, sums[sp * cell_stride<kWG>(a) + r], den);
    }
    inv[r] = den > 0.f ? 1.f / den : 0.f;
  }
  sync_consumers<kWG>(n_threads);
  if constexpr (kWG == 1) {
    for (int e = ctid; e < cell_rows_at<kWG>(a, r0) * (D / 4); e += n_threads) {
      const int r = e / (D / 4), col = 4 * (e % (D / 4));
      float x0 = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f;
  #pragma unroll 8
      for (int sp = 0; sp < a.splits; ++sp) {
        const float w = wts[sp * cell_stride<kWG>(a) + r];
        const float4 v = __ldcg(reinterpret_cast<const float4*>(part + ((size_t)sp * cell_stride<kWG>(a) + r) * D + col));
        x0 = fmaf(w, v.x, x0), x1 = fmaf(w, v.y, x1), x2 = fmaf(w, v.z, x2), x3 = fmaf(w, v.w, x3);
      }
      const float iv = inv[r];
      *reinterpret_cast<uint2*>(out_row(r0 + r) + col) =
          make_uint2(pack2<T>(x0 * iv, x1 * iv), pack2<T>(x2 * iv, x3 * iv));
    }
  } else {
    // the same sums, kItems (row, 4 columns) items per thread at once: the combine of a 128-row cell is one CTA's
    // reads of splits x 64 KB from L2, which one item per thread leaves latency-bound
    constexpr int kItems = 4;
    const int n_items = cell_rows_at<kWG>(a, r0) * (D / 4), stride = cell_stride<kWG>(a);
    for (int e0 = ctid; e0 < n_items; e0 += kItems * n_threads) {
      float4 x[kItems];
#pragma unroll
      for (int u = 0; u < kItems; ++u) x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
      for (int sp = 0; sp < a.splits; ++sp) {
#pragma unroll
        for (int u = 0; u < kItems; ++u) {
          const int e = min(e0 + u * n_threads, n_items - 1);  // past the end: a duplicate, never stored
          const int r = e / (D / 4), col = 4 * (e % (D / 4));
          const float w = wts[sp * stride + r];
          const float4 v = __ldcg(reinterpret_cast<const float4*>(part + ((size_t)sp * stride + r) * D + col));
          x[u].x = fmaf(w, v.x, x[u].x), x[u].y = fmaf(w, v.y, x[u].y);
          x[u].z = fmaf(w, v.z, x[u].z), x[u].w = fmaf(w, v.w, x[u].w);
        }
      }
#pragma unroll
      for (int u = 0; u < kItems; ++u) {
        const int e = e0 + u * n_threads;
        if (e >= n_items) break;
        const int r = e / (D / 4), col = 4 * (e % (D / 4));
        const float iv = inv[r];
        *reinterpret_cast<uint2*>(out_row(r0 + r) + col) =
            make_uint2(pack2<T>(x[u].x * iv, x[u].y * iv), pack2<T>(x[u].z * iv, x[u].w * iv));
      }
    }
  }
  if (ctid == 0) a.count[cell] = 0u;  // ready for the next launch (graph replay included)
}

// Splits of the key range: enough CTAs to cover every SM (at most ceil(SMs / cells) splits, at least one 128-key tile
// each, at most max_splits), chosen by the estimated time waves x tiles per split; fewer splits win ties (less to
// combine).  More cells than counters: one split.
void plan_splits(int cells, int n_tiles, int sms, int max_splits, int& splits, int& tiles_per_split) {
  splits = 1, tiles_per_split = n_tiles;
  if (n_tiles < 2 || cells > kAttentionCounters) return;
  const int cap = std::min(std::min(n_tiles, (sms + cells - 1) / cells), max_splits);
  long long best = n_tiles;  // one split: one wave as long as cells <= sms
  best *= (cells + sms - 1) / sms;
  for (int sp = 2; sp <= cap; ++sp) {
    const int tps = (n_tiles + sp - 1) / sp, used = (n_tiles + tps - 1) / tps;
    const long long cost = (long long)((cells * used + sms - 1) / sms) * tps;
    if (cost < best) best = cost, splits = used, tiles_per_split = tps;
  }
}

// [counters: kAttentionCounters x u32 at offset 0] [partials: D floats (O), then 2 (m, l), per packed row, split and
// cell].  A plan has splits <= min(n_tiles, ceil(SMs / cells)), so cells * splits <= min(cells * n_tiles,
// cells + kMaxSms - 1).  0 when no plan can split: one key tile, more cells than counters, or more than max_cells.
size_t workspace_bound(long long cells, long long cell_rows, int seqlen_k, int head_dim, long long max_cells) {
  const long long n_tiles = ((long long)seqlen_k + kBN - 1) / kBN;
  if (n_tiles < 2 || cells > std::min<long long>(kAttentionCounters, max_cells)) return 0;
  const long long cs = std::min(cells * n_tiles, cells + kMaxSms);
  return (size_t)kAttentionCounters * sizeof(unsigned int) + (size_t)cs * cell_rows * (head_dim + 2) * sizeof(float);
}

// tinychat's FasterTransformer K cache [batch][kv_heads][D / 8][max_len][8] as the 4-D map {8, tokens, D / 8,
// batch * kv_heads}, box {8, rows, D / 8, 1}, no swizzle: a box lands as [D / 8][rows][8]
template <typename T>
int encode_ft_k(EncodeTiledFn enc, CUtensorMap* tm, const void* p, int head_dim, int tokens, long long max_len,
                int batch_heads, int rows) {
  cuuint64_t dims[4] = {8, (cuuint64_t)(tokens > 0 ? tokens : 1), (cuuint64_t)(head_dim / 8), (cuuint64_t)batch_heads};
  cuuint64_t strides[3] = {16, (cuuint64_t)max_len * 16, (cuuint64_t)max_len * head_dim * sizeof(T)};
  cuuint32_t box[4] = {8, (cuuint32_t)rows, (cuuint32_t)(head_dim / 8), 1};
  cuuint32_t ones[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, TypeTraits<T>::kIsBf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                   const_cast<void*>(p), dims, strides, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : B200AWQ_ERR_DRIVER;
}

// kWG = 1: flash_attn_func's route (R <= 64, one cell per (batch, KV head)); kWG = 2: kv_cache_attention.  kFtK: K is
// the FT cache of max_len slots (ks unused), else [B][Sk][Hkv][D] with strides ks.
template <typename T, int D, int kWG, bool kFtK>
int launch_t(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k, int heads,
             int kv_heads, const long long* qs, const long long* ks, const long long* vs, long long max_len,
             float softmax_scale, bool causal, void* workspace, size_t workspace_bytes, size_t workspace_need,
             cudaStream_t stream) {
  using C = SplitCfg<D, kWG>;
  const int sms = std::min(sm_count(), kMaxSms);
  if (sms == 0) return B200AWQ_ERR_DEVICE;
  SplitArgs a{};
  a.q = q, a.out = out;
  a.qs0 = qs[0], a.qs1 = qs[1], a.qs2 = qs[2];
  a.sq = seqlen_q, a.sk = seqlen_k, a.heads = heads, a.kv_heads = kv_heads, a.group = heads / kv_heads;
  a.rows = seqlen_q * a.group;
  const int row_tiles = (a.rows + kWG * kRows - 1) / (kWG * kRows);  // kWG = 1: R <= 64, one
  plan_splits(row_tiles * batch * kv_heads, (seqlen_k + kBN - 1) / kBN, sms, max_splits(std::min(a.rows, kWG * kRows)), a.splits,
              a.tiles_per_split);
  if (a.splits > 1) {
    // the plan never needs more than workspace_need (whatever the SM count up to kMaxSms)
    if (!workspace || workspace_bytes < workspace_need) return B200AWQ_ERR_WORKSPACE;
    a.count = static_cast<unsigned int*>(workspace);
    a.part = reinterpret_cast<float*>(static_cast<char*>(workspace) + kAttentionCounters * sizeof(unsigned int));
  }
  a.scale_log2 = softmax_scale * 1.4426950408889634f;
  a.causal = causal ? 1 : 0;
  EncodeTiledFn enc = get_encoder();
  if (!enc) return B200AWQ_ERR_DRIVER;
  CUtensorMap tm[2];
  if constexpr (kFtK) {
    if (int e = encode_ft_k<T>(enc, &tm[0], k, D, seqlen_k, max_len, batch * kv_heads, kBN)) return e;
  } else {
    if (int e = encode_bthd<T>(enc, &tm[0], k, D, seqlen_k, kv_heads, batch, ks, 64, kBN)) return e;
  }
  if (int e = encode_bthd<T>(enc, &tm[1], v, D, seqlen_k, kv_heads, batch, vs, 64, kBN)) return e;
  auto kernel = splitkv_attention_kernel<T, D, kWG, kFtK>;
  if (cudaError_t ea = ensure_dyn_smem<splitkv_attention_kernel<T, D, kWG, kFtK>>(C::kSmem)) return (int)ea;
  const dim3 grid = kWG == 1 ? dim3((unsigned)a.splits, (unsigned)kv_heads, (unsigned)batch)
                             : dim3((unsigned)a.splits, (unsigned)row_tiles, (unsigned)(batch * kv_heads));
  // no programmatic dependent launch: the kernel never waits on the previous grid
  return launch_kernel(kernel, grid, dim3(C::kThreads), (size_t)C::kSmem, stream, false, 1, tm[0], tm[1], a);
}

template <typename T, int kWG, bool kFtK>
int launch_d(int head_dim, const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
             int heads, int kv_heads, const long long* qs, const long long* ks, const long long* vs, long long max_len,
             float scale, bool causal, void* ws, size_t ws_bytes, size_t ws_need, cudaStream_t st) {
  switch (head_dim) {
    case 64: return launch_t<T, 64, kWG, kFtK>(q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs, max_len, scale, causal, ws, ws_bytes, ws_need, st);
    case 128: return launch_t<T, 128, kWG, kFtK>(q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs, max_len, scale, causal, ws, ws_bytes, ws_need, st);
    default: return B200AWQ_ERR_SHAPE;
  }
}

template <int kWG, bool kFtK>
int launch_dt(int dtype, int head_dim, const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q,
              int seqlen_k, int heads, int kv_heads, const long long* qs, const long long* ks, const long long* vs,
              long long max_len, float scale, bool causal, void* ws, size_t ws_bytes, size_t ws_need, cudaStream_t st) {
  if (dtype == B200AWQ_DTYPE_F16)
    return launch_d<__half, kWG, kFtK>(head_dim, q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs, max_len,
                                       scale, causal, ws, ws_bytes, ws_need, st);
  return launch_d<__nv_bfloat16, kWG, kFtK>(head_dim, q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs,
                                            max_len, scale, causal, ws, ws_bytes, ws_need, st);
}

}  // namespace

size_t splitkv_attention_workspace_bytes(int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim) {
  if (batch < 1 || seqlen_q < 1 || seqlen_k < 1 || heads < 1 || kv_heads < 1 || heads % kv_heads ||
      (head_dim != 64 && head_dim != 128))
    return 0;
  const long long rows = (long long)seqlen_q * (heads / kv_heads);
  if (rows > kRows) return 0;
  return workspace_bound((long long)batch * kv_heads, rows, seqlen_k, head_dim, kAttentionCounters);
}

// Cells are (row tile of 128 packed rows, KV head, batch row).  A plan splits only when 2 * cells <= SMs (with more
// cells, two splits take two waves and save nothing), so the bound is 0 exactly when no SM count up to kMaxSms splits:
// one key tile or more than kMaxSms / 2 cells.
size_t kv_cache_attention_workspace_bytes(int layout, int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads,
                                          int head_dim) {
  if ((layout != B200AWQ_KV_FT && layout != B200AWQ_KV_BTHD) || batch < 1 || seqlen_q < 1 || seqlen_k < 1 || heads < 1 ||
      kv_heads < 1 || heads % kv_heads || (head_dim != 64 && head_dim != 128))
    return 0;
  const long long rows = (long long)seqlen_q * (heads / kv_heads), tile = 2 * kRows;
  const long long cells = (rows + tile - 1) / tile * batch * kv_heads;
  return workspace_bound(cells, std::min(rows, tile), seqlen_k, head_dim, kMaxSms / 2);
}

int launch_splitkv_attention(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
                             int heads, int kv_heads, int head_dim, const long long* q_strides, const long long* k_strides,
                             const long long* v_strides, float softmax_scale, bool causal, int dtype, void* workspace,
                             size_t workspace_bytes, cudaStream_t stream) {
  return launch_dt<1, false>(dtype, head_dim, q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides, k_strides,
                             v_strides, 0, softmax_scale, causal, workspace, workspace_bytes,
                             splitkv_attention_workspace_bytes(batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim), stream);
}

int launch_kv_cache_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int layout, int batch,
                              int seqlen_q, int seqlen_k, int max_len, int heads, int kv_heads, int head_dim,
                              const long long* q_strides, float softmax_scale, bool causal, int dtype, void* workspace,
                              size_t workspace_bytes, cudaStream_t stream) {
  const size_t need = kv_cache_attention_workspace_bytes(layout, batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim);
  const long long L = max_len, D = head_dim;
  if (layout == B200AWQ_KV_FT) {  // v_cache [B][Hkv][Lmax][D]: (batch, token, head) strides
    const long long vs[3] = {kv_heads * L * D, D, L * D};
    return launch_dt<2, true>(dtype, head_dim, q, k_cache, v_cache, out, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides,
                              nullptr, vs, L, softmax_scale, causal, workspace, workspace_bytes, need, stream);
  }
  const long long kvs[3] = {L * kv_heads * D, kv_heads * D, D};  // [B][Lmax][Hkv][D]
  return launch_dt<2, false>(dtype, head_dim, q, k_cache, v_cache, out, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides,
                             kvs, kvs, L, softmax_scale, causal, workspace, workspace_bytes, need, stream);
}

}  // namespace b200awq
