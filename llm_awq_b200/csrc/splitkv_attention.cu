// Attention of few queries over many keys for sm_90a (long-context decode, few-token chunks): the key range is split
// over CTAs, each CTA packs every query row that reads one KV head into one wgmma tile.
//
//   O = softmax(scale * Q K^T + mask) V        fp16 / bf16, head size D in {64, 128}, Sq * (H / Hkv) <= 64
//
// Numerics as prefill_attention.cu (S in fp32 from T operands, p = exp2(scale * log2(e) * (s - max)) as one FFMA + ex2,
// P rounded to T, O in fp32), plus the combine of the splits below.
//
// Tile: one CTA = (key split, KV head, batch row).  Its R = Sq * G query rows (G = H / Hkv) are packed into one 64-row
// tile, row s * G + g = query s of head hk * G + g; rows R..63 are zero and never stored.
//   * Q is read once with 16-byte loads from the caller's strides and stored with the 128-byte swizzle TMA would use.
//   * K and V tiles of 128 keys arrive by 4-D TMA from the caller's strides (views into a larger cache are read in
//     place; the maps' token extent is Sk, so slots past the view are never read) into a full / empty mbarrier ring
//     of 192 KB (D = 128: 3 stages of K + V, D = 64: 6), which keeps the HBM requests of one SM in flight.
//   * S = Q K^T with wgmma.m64n128k16, O += P V with P from registers, as in prefill_attention.cu; the P V of tile n and
//     the Q K^T of tile n + 1 go to the tensor core as one batch.
//   * Causal (bottom-right, per packed row: query s sees keys j <= s + Sk - Sq): masked keys select -inf.
// Splits: the number of splits follows from the shape and the SM count (plan_splits).  Each split writes fp32
// partials (unnormalised O, the row max m of the raw scores, the row sum l) to the workspace and counts its arrival;
// the last CTA of a (batch, KV head) to arrive combines them in split order:
//   O = sum_s w_s O_s / sum_s w_s l_s,  w_s = exp2(scale * log2(e) * (m_s - M)),  M = max_s m_s,
// rounded once to T.  A split in which a row sees no key has m_s = -inf and weighs 0; a row that sees no key at all is
// zero.  The counter is only an arrival count: which CTA combines varies, the arithmetic and its order do not, so
// every call returns the same bits.  With one split the CTA writes O / l directly and the workspace is not touched.
// Warp roles (160 threads, one CTA per SM): warps 0-3 = the consumer warpgroup (wgmma, softmax, epilogue, combine);
// warp 4 = TMA producer (one thread).
#include <algorithm>

#include "attention_wgmma.cuh"

namespace b200awq {
namespace {

constexpr int kRows = 64;       // packed query rows per CTA
constexpr int kBN = 128;        // keys per pipeline stage
constexpr int kThreads = 160;   // consumer warpgroup + producer warp
constexpr int kMaxSms = 256;    // the split rule and the workspace bound assume at most this many SMs

template <int D>
struct SplitCfg {
  static constexpr int kStages = D == 64 ? 6 : 3;    // 192 KB of K / V tiles in flight
  static constexpr int kQBytes = kRows * D * 2;
  static constexpr int kKBytes = kBN * D * 2;        // K tile; the V tile follows it
  static constexpr int kStageBytes = 2 * kKBytes;
  static constexpr int kSmem = kQBytes + kStages * kStageBytes + 1024 /*align*/ + 128 /*barriers*/;
  static_assert(kQBytes % 1024 == 0 && kKBytes % 1024 == 0, "tiles must stay aligned to the swizzle repeat");
  // the combine's row maxima / weights and row sums (splits x rows floats each) and inverse row sums reuse the ring
  static_assert(kStages * kStageBytes >= (2 * kMaxSms * kRows + kRows) * 4, "combine scratch must fit in the ring");
};

struct SplitArgs {
  const void* q;
  void* out;                  // [B][Sq][H][D] contiguous
  float* part;                // [B * Hkv][splits][rows][D] O of each split, then [B * Hkv][splits][rows][2] (m, l)
  unsigned int* count;        // [B * Hkv] arrival counters (zero between launches)
  long long qs0, qs1, qs2;    // q strides (batch, token, head) in elements
  int sq, sk, heads, kv_heads, group, rows, splits, tiles_per_split;
  float scale_log2;
  int causal;
};

template <typename T, int D>
__global__ void __launch_bounds__(kThreads, 1)
splitkv_attention_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                         const __grid_constant__ SplitArgs a) {
  using C = SplitCfg<D>;
  constexpr int kStages = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ unsigned int s_last;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* qs = smem;                              // Q tile: D / 64 blocks [64][64], 128-byte swizzle
  uint8_t* kvs = qs + C::kQBytes;                  // stage s: K tile, then V tile
  uint64_t* full = reinterpret_cast<uint64_t*>(kvs + kStages * C::kStageBytes);  // [kStages] TMA -> consumers
  uint64_t* empty = full + kStages;                // [kStages] consumer warps -> TMA

  const int split = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int t0 = split * a.tiles_per_split;
  const int n_tiles = max(0, min((a.sk + kBN - 1) / kBN, t0 + a.tiles_per_split) - t0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);
    }
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 4) {
    // =========================================================== TMA producer
    if (lane == 0 && n_tiles > 0) {
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      int s = 0;
      uint32_t ph = 0;
      for (int n = 0; n < n_tiles; ++n) {
        const int row = (t0 + n) * kBN;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], C::kStageBytes);
        uint8_t* st = kvs + s * C::kStageBytes;
#pragma unroll
        for (int c = 0; c < D / 64; ++c) {
          tma_load_4d(st + c * kBN * 128, &tm_k, &full[s], c * 64, row, hk, b);
          tma_load_4d(st + C::kKBytes + c * kBN * 128, &tm_v, &full[s], c * 64, row, hk, b);
        }
        if (++s == kStages) s = 0, ph ^= 1;
      }
    }
    return;
  }

  // =========================================================== consumer warpgroup
  const int tid = threadIdx.x;  // 0..127
  {
    // packed Q tile, 16-byte chunks: chunk c of row r lands at block c / 8, row r, position (c % 8) ^ (r % 8)
    const T* qg = static_cast<const T*>(a.q) + (long long)b * a.qs0;
    constexpr int kChunks = D / 8;
    for (int e = tid; e < kRows * kChunks; e += 128) {
      const int r = e / kChunks, c = e % kChunks;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (r < a.rows) {
        const int s = r / a.group, h = hk * a.group + r % a.group;
        val = __ldg(reinterpret_cast<const uint4*>(qg + s * a.qs1 + h * a.qs2 + c * 8));
      }
      *reinterpret_cast<uint4*>(qs + (c / 8) * kRows * 128 + r * 128 + (((c % 8) ^ (r & 7)) * 16)) = val;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> wgmma operand reads
    asm volatile("bar.sync 1, 128;" ::: "memory");
  }

  const int g = lane >> 2, t = lane & 3;
  const int r_lo = warp * 16 + g;  // this thread's packed rows: r_lo, r_lo + 8
  // keys below lim are seen by the row: all Sk, or causal s + Sk - Sq + 1 (<= 0: none)
  const int diag = a.sk - a.sq;
  const int lim_lo = a.causal ? min(a.sk, r_lo / a.group + diag + 1) : a.sk;
  const int lim_hi = a.causal ? min(a.sk, (r_lo + 8) / a.group + diag + 1) : a.sk;
  // accumulator element 4 j + e: row r_lo + 8 (e >> 1), column 8 j + 2 t + (e & 1)
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;  // running max (raw scores), partial sums
  const uint32_t q_addr = smem_u32(qs);
  uint32_t pa[kBN / 16][4];  // P of the current tile as the A fragments of the 8 k16 steps of O += P V
  float sc[64];              // S of the next tile
  const float scale_log2 = a.scale_log2;

  auto issue_qk = [&](int stage) {
    const uint32_t k_addr = smem_u32(kvs + stage * C::kStageBytes);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)  // k16 step kk: block kk / 4, +32 bytes per step inside the block
      wgmma_qk<T>(sc, make_smem_desc(q_addr + (kk / 4) * kRows * 128 + (kk % 4) * 32, 1, 16, 1024),
                  make_smem_desc(k_addr + (kk / 4) * kBN * 128 + (kk % 4) * 32, 1, 16, 1024), kk > 0 ? 1u : 0u);
  };
  auto issue_pv = [&](int stage) {
    const uint32_t v_addr = smem_u32(kvs + stage * C::kStageBytes + C::kKBytes);
    // V is MN-major: 64-column blocks kBN * 128 bytes apart, 8-key groups 1024 bytes apart
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk)
      wgmma_pv<T, D>(o, pa[kk], make_smem_desc(v_addr + kk * 16 * 128, 1, kBN * 128, 1024), 1u);
  };
  // scale, mask and online softmax of tile n's S: P into pa, O rescaled
  auto softmax = [&](int n) {
    const int k0 = (t0 + n) * kBN;
    if (k0 + kBN > min(lim_lo, lim_hi)) {  // on the raw scores: scale_log2 > 0 keeps -inf the smallest value
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int key = k0 + 8 * (i >> 2) + 2 * t + (i & 1);
        sc[i] = key < ((i & 2) ? lim_hi : lim_lo) ? sc[i] : -INFINITY;
      }
    }
    float mx_lo = m_lo, mx_hi = m_hi;
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
      mx_lo = fmaxf(mx_lo, fmaxf(sc[i], sc[i + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(sc[i + 2], sc[i + 3]));
    }
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, d));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, d));
    }
    // a row that has seen no key yet keeps max -inf: its probabilities are exp2(-inf) = 0 and nothing is rescaled
    const float nb_lo = mx_lo == -INFINITY ? 0.f : -mx_lo * scale_log2;
    const float nb_hi = mx_hi == -INFINITY ? 0.f : -mx_hi * scale_log2;
    const float alpha_lo = ex2(fmaf(m_lo, scale_log2, nb_lo)), alpha_hi = ex2(fmaf(m_hi, scale_log2, nb_hi));
    m_lo = mx_lo, m_hi = mx_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
      const float p0 = ex2(fmaf(sc[i], scale_log2, nb_lo)), p1 = ex2(fmaf(sc[i + 1], scale_log2, nb_lo));
      const float p2 = ex2(fmaf(sc[i + 2], scale_log2, nb_hi)), p3 = ex2(fmaf(sc[i + 3], scale_log2, nb_hi));
      sum_lo += p0 + p1, sum_hi += p2 + p3;
      const int kk = i >> 3, half = (i >> 2) & 1;  // columns 8 (i / 4) + 2 t: k16 step i / 8, k + 8 when half
      pa[kk][2 * half] = pack2<T>(p0, p1);
      pa[kk][2 * half + 1] = pack2<T>(p2, p3);
    }
    l_lo = l_lo * alpha_lo + sum_lo, l_hi = l_hi * alpha_hi + sum_hi;
#pragma unroll
    for (int i = 0; i < D / 2; i += 4) {
      o[i] *= alpha_lo, o[i + 1] *= alpha_lo;
      o[i + 2] *= alpha_hi, o[i + 3] *= alpha_hi;
    }
  };

  if (n_tiles > 0) {
    mbar_wait(&full[0], 0);
    wgmma_fence();
    issue_qk(0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(sc);
    softmax(0);
  }
  int s = 0;
  uint32_t ph = 0;
  for (int n = 0; n + 1 < n_tiles; ++n) {
    const int s1 = s + 1 == kStages ? 0 : s + 1;
    const uint32_t ph1 = s1 == 0 ? ph ^ 1 : ph;
    mbar_wait(&full[s1], ph1);
    wgmma_fence();
    issue_pv(s);
    issue_qk(s1);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(o);
    acc_fence(sc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);  // tile n's K and V have been read
    softmax(n + 1);
    s = s1, ph = ph1;
  }
  if (n_tiles > 0) {  // P V of the last tile
    wgmma_fence();
    issue_pv(s);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(o);
  }
#pragma unroll
  for (int d = 1; d <= 2; d <<= 1) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, d);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, d);
  }

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
  const int cell = b * a.kv_heads + hk;
  const size_t per_cell = (size_t)a.splits * a.rows;  // (split, row) pairs of one cell
  float* part = a.part + cell * per_cell * D;
  float* ml = a.part + (size_t)gridDim.y * gridDim.z * per_cell * D + cell * per_cell * 2;
  {
    float* p_lo = part + ((size_t)split * a.rows + r_lo) * D;
    float* p_hi = p_lo + 8 * D;
    const bool st_lo = r_lo < a.rows, st_hi = r_lo + 8 < a.rows;
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int col = 8 * j + 2 * t;
      if (st_lo) *reinterpret_cast<float2*>(p_lo + col) = make_float2(o[4 * j], o[4 * j + 1]);
      if (st_hi) *reinterpret_cast<float2*>(p_hi + col) = make_float2(o[4 * j + 2], o[4 * j + 3]);
    }
    float* q_lo = ml + ((size_t)split * a.rows + r_lo) * 2;
    if (t == 0 && st_lo) *reinterpret_cast<float2*>(q_lo) = make_float2(m_lo, l_lo);
    if (t == 0 && st_hi) *reinterpret_cast<float2*>(q_lo + 16) = make_float2(m_hi, l_hi);
  }
  __threadfence();
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (tid == 0) s_last = atomicAdd(&a.count[cell], 1u) == (unsigned)a.splits - 1 ? 1u : 0u;
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (!s_last) return;
  __threadfence();

  // ------------------------------------------------ the last CTA of this (batch, KV head) combines, in split order
  // (every TMA write to the ring has landed: its shared memory holds the scratch).  The loads of the partials are
  // independent of each other; only the sums run in split order.
  const int n_pairs = (int)per_cell;
  float* wts = reinterpret_cast<float*>(kvs);  // [splits][rows]: row maxima, then weights
  float* sums = wts + n_pairs;                 // [splits][rows]
  float* inv = sums + n_pairs;                 // [rows]
  for (int e = tid; e < n_pairs; e += 128) {
    const float2 x = __ldcg(reinterpret_cast<const float2*>(ml) + e);
    wts[e] = x.x, sums[e] = x.y;
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  for (int r = tid; r < a.rows; r += 128) {
    float M = -INFINITY;
    for (int sp = 0; sp < a.splits; ++sp) M = fmaxf(M, wts[sp * a.rows + r]);
    const float nb = M == -INFINITY ? 0.f : -M * scale_log2;
    float den = 0.f;
    for (int sp = 0; sp < a.splits; ++sp) {
      const float w = ex2(fmaf(wts[sp * a.rows + r], scale_log2, nb));
      wts[sp * a.rows + r] = w;
      den = fmaf(w, sums[sp * a.rows + r], den);
    }
    inv[r] = den > 0.f ? 1.f / den : 0.f;
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  for (int e = tid; e < a.rows * (D / 4); e += 128) {
    const int r = e / (D / 4), col = 4 * (e % (D / 4));
    float x0 = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f;
#pragma unroll 8
    for (int sp = 0; sp < a.splits; ++sp) {
      const float w = wts[sp * a.rows + r];
      const float4 v = __ldcg(reinterpret_cast<const float4*>(part + ((size_t)sp * a.rows + r) * D + col));
      x0 = fmaf(w, v.x, x0), x1 = fmaf(w, v.y, x1), x2 = fmaf(w, v.z, x2), x3 = fmaf(w, v.w, x3);
    }
    const float iv = inv[r];
    *reinterpret_cast<uint2*>(out_row(r) + col) = make_uint2(pack2<T>(x0 * iv, x1 * iv), pack2<T>(x2 * iv, x3 * iv));
  }
  if (tid == 0) a.count[cell] = 0u;  // ready for the next launch (graph replay included)
}

// Splits of the key range: enough CTAs to cover every SM (at most ceil(SMs / (B * Hkv)) splits, at least one 128-key
// tile each), chosen by the estimated time waves x tiles per split; fewer splits win ties (less to combine).  More
// (batch, KV head) cells than counters: one split.
void plan_splits(int cells, int n_tiles, int sms, int& splits, int& tiles_per_split) {
  splits = 1, tiles_per_split = n_tiles;
  if (n_tiles < 2 || cells > kAttentionCounters) return;
  const int cap = std::min(n_tiles, (sms + cells - 1) / cells);
  long long best = n_tiles;  // one split: one wave as long as cells <= sms
  best *= (cells + sms - 1) / sms;
  for (int sp = 2; sp <= cap; ++sp) {
    const int tps = (n_tiles + sp - 1) / sp, used = (n_tiles + tps - 1) / tps;
    const long long cost = (long long)((cells * used + sms - 1) / sms) * tps;
    if (cost < best) best = cost, splits = used, tiles_per_split = tps;
  }
}

template <typename T, int D>
int launch_t(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k, int heads,
             int kv_heads, const long long* qs, const long long* ks, const long long* vs, float softmax_scale, bool causal,
             void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  using C = SplitCfg<D>;
  const int sms = std::min(sm_count(), kMaxSms);
  if (sms == 0) return B200AWQ_ERR_DEVICE;
  SplitArgs a{};
  a.q = q, a.out = out;
  a.qs0 = qs[0], a.qs1 = qs[1], a.qs2 = qs[2];
  a.sq = seqlen_q, a.sk = seqlen_k, a.heads = heads, a.kv_heads = kv_heads, a.group = heads / kv_heads;
  a.rows = seqlen_q * a.group;
  plan_splits(batch * kv_heads, (seqlen_k + kBN - 1) / kBN, sms, a.splits, a.tiles_per_split);
  if (a.splits > 1) {
    // the plan never needs more than splitkv_attention_workspace_bytes (whatever the SM count up to kMaxSms)
    if (!workspace || workspace_bytes < splitkv_attention_workspace_bytes(batch, seqlen_q, seqlen_k, heads, kv_heads, D))
      return B200AWQ_ERR_WORKSPACE;
    a.count = static_cast<unsigned int*>(workspace);
    a.part = reinterpret_cast<float*>(static_cast<char*>(workspace) + kAttentionCounters * sizeof(unsigned int));
  }
  a.scale_log2 = softmax_scale * 1.4426950408889634f;
  a.causal = causal ? 1 : 0;
  EncodeTiledFn enc = get_encoder();
  if (!enc) return B200AWQ_ERR_DRIVER;
  CUtensorMap tm[2];
  if (int e = encode_bthd<T>(enc, &tm[0], k, D, seqlen_k, kv_heads, batch, ks, 64, kBN)) return e;
  if (int e = encode_bthd<T>(enc, &tm[1], v, D, seqlen_k, kv_heads, batch, vs, 64, kBN)) return e;
  if (cudaError_t ea = ensure_dyn_smem<splitkv_attention_kernel<T, D>>(C::kSmem)) return (int)ea;
  // no programmatic dependent launch: the kernel never waits on the previous grid
  return launch_kernel(splitkv_attention_kernel<T, D>, dim3((unsigned)a.splits, (unsigned)kv_heads, (unsigned)batch),
                       dim3(kThreads), (size_t)C::kSmem, stream, false, 1, tm[0], tm[1], a);
}

template <typename T>
int launch_d(int head_dim, const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
             int heads, int kv_heads, const long long* qs, const long long* ks, const long long* vs, float scale, bool causal,
             void* ws, size_t ws_bytes, cudaStream_t st) {
  switch (head_dim) {
    case 64: return launch_t<T, 64>(q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs, scale, causal, ws, ws_bytes, st);
    case 128: return launch_t<T, 128>(q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, qs, ks, vs, scale, causal, ws, ws_bytes, st);
    default: return B200AWQ_ERR_SHAPE;
  }
}

}  // namespace

// [counters: kAttentionCounters x u32 at offset 0] [partials: D floats (O), then 2 (m, l), per packed row, split and
// (batch, KV head)].
// A plan has splits <= min(n_tiles, ceil(SMs / cells)), so cells * splits <= min(cells * n_tiles, cells + kMaxSms - 1).
// 0 when every plan of the shape has one split (one key tile, or more cells than counters: plan_splits) or the shape is
// outside the envelope.
size_t splitkv_attention_workspace_bytes(int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim) {
  if (batch < 1 || seqlen_q < 1 || seqlen_k < 1 || heads < 1 || kv_heads < 1 || heads % kv_heads ||
      (head_dim != 64 && head_dim != 128))
    return 0;
  const long long rows = (long long)seqlen_q * (heads / kv_heads);
  const long long cells = (long long)batch * kv_heads, n_tiles = ((long long)seqlen_k + kBN - 1) / kBN;
  if (rows > kRows || n_tiles < 2 || cells > kAttentionCounters) return 0;
  const long long cs = std::min(cells * n_tiles, cells + kMaxSms);
  return (size_t)kAttentionCounters * sizeof(unsigned int) + (size_t)cs * rows * (head_dim + 2) * sizeof(float);
}

int launch_splitkv_attention(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
                             int heads, int kv_heads, int head_dim, const long long* q_strides, const long long* k_strides,
                             const long long* v_strides, float softmax_scale, bool causal, int dtype, void* workspace,
                             size_t workspace_bytes, cudaStream_t stream) {
  if (dtype == B200AWQ_DTYPE_F16)
    return launch_d<__half>(head_dim, q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides, k_strides,
                            v_strides, softmax_scale, causal, workspace, workspace_bytes, stream);
  return launch_d<__nv_bfloat16>(head_dim, q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides, k_strides,
                                 v_strides, softmax_scale, causal, workspace, workspace_bytes, stream);
}

}  // namespace b200awq
