// Forward attention over many queries for sm_90a: TMA -> swizzled shared memory -> wgmma, online softmax in registers.
//
//   O = softmax(scale * Q K^T + mask) V        fp16 / bf16, head size D in {64, 72, 128}
//
// Replaces flash-attn 2's forward kernels (Ampere cp.async + ldmatrix + mma.sync) behind flash_attn_func and
// flash_attn_varlen_qkvpacked_func: LLM prefill (causal, grouped-query) and the vision towers (non-causal).
//
// Numerics (flash-attn's own): S = Q K^T accumulated in fp32 from T operands; softmax in fp32 (running max of the raw
// scores, exp2(scale * log2(e) * (s - max)) as one FFMA + ex2, so the scale must be > 0; running row sum of the fp32
// probabilities); P rounded to T for O += P V; O
// accumulated in fp32, divided by the row sum and rounded once to T.  A row that sees no key is written as zeros.
//
// Tile: one CTA = 128 query rows of one (sequence, query head); query head h reads KV head h / (H / Hkv).
//   * Q [128 x D] arrives once by TMA; K and V tiles of 128 keys arrive by TMA into a full / empty mbarrier ring (4 stages, D = 128: 2).
//   * Shared-memory layout: 64-column blocks with the 128-byte swizzle; D = 72 runs as 80, its columns 64..79 in one
//     16-column block with the 32-byte swizzle (that tensor map's inner extent is 72: TMA zero-fills columns 72..79).
//   * S = Q K^T: wgmma.m64n128k16, both operands K-major shared-memory descriptors.  O += P V: P (the S accumulator
//     layout is the A-fragment layout) from registers, V as the MN-major (transposed) shared-memory B operand.
//   * Causal (bottom-right: query i sees keys j <= i + Sk - Sq): key tiles past the tile's last row's horizon are not
//     loaded; partial tiles select -inf for masked keys (a NaN or inf in a masked key cannot leak into the row).
//     Query tiles are scheduled heaviest first.
//   * Varlen (cu_seqlens in device memory): tile coordinates are offsets into the packed token dimension.  The tensor
//     maps do not know the packed length, so a sequence's last Q / K / V tile is shifted back to END at the sequence's
//     end (rows before the tensor's start arrive as zeros): no tile reads past its sequence.  Keys outside the tile's
//     own range and other sequences' rows are masked; query rows outside the tile's range are not stored.
//   * No split over keys, no atomics, no workspace: deterministic, and output row r depends only on query r and the
//     keys it sees.
// Warp roles (384 threads, one CTA per SM): warpgroup 0 = TMA producer (one thread; its registers are handed to the
// consumers with setmaxnreg); warpgroups 1, 2 = query rows [0, 64) / [64, 128) of the tile (wgmma, softmax, epilogue
// through shared memory into 16-byte stores).
#include "attention_wgmma.cuh"

namespace b200awq {
namespace {

constexpr int kBM = 128;        // query rows per CTA
constexpr int kBN = 128;        // keys per pipeline stage
constexpr int kThreads = 384;   // producer warpgroup + 2 consumer warpgroups

// DP = head size as computed (72 -> 80).  An operand tile of R rows is stored as kMain / 64 blocks [R][64] (128-byte
// swizzle, R * 128 bytes each), then, when kTail = 16, one block [R][16] (32-byte swizzle).
template <int DP>
struct AttnCfg {
  static constexpr int kMain = DP / 64 * 64;
  static constexpr int kTail = DP - kMain;
  static_assert(kTail == 0 || kTail == 16, "head sizes 64, 80, 128");
  // K / V ring depth: as deep as shared memory allows (4 stages hide the load latency of the short vision-tower calls;
  // D = 128 fits 2 next to Q and the output staging)
  static constexpr int kStages = DP <= 80 ? 4 : 2;
  static constexpr int kQBytes = kBM * DP * 2;
  static constexpr int kKBytes = kBN * DP * 2;                // K tile; the V tile follows it
  static constexpr int kStageBytes = 2 * kKBytes;
  static constexpr int kOutRow = DP * 2 + 16;                 // staged output row (+ pad against bank conflicts)
  static constexpr int kSmem = kQBytes + kStages * kStageBytes + kBM * kOutRow + 1024 /*align*/ + 128 /*barriers*/;
  static_assert(kQBytes % 1024 == 0 && kKBytes % 1024 == 0, "tiles must stay aligned to the swizzle repeat");
};

// The two consumer warpgroups take turns at the tensor core (named barriers 3 and 4): one issues its wgmmas (P V of
// tile n and Q K^T of tile n + 1, one batch) while the other runs its softmax.  Warpgroup 1 lets warpgroup 0 go first
// and skips its last hand-over, so that every barrier phase completes.  Both wait for the Q tile before the first.
struct Turns {
  int wg;
  uint64_t* qfull;
  __device__ __forceinline__ void first() const {
    if (wg == 1) asm volatile("bar.arrive 3, 256;" ::: "memory");
    mbar_wait(qfull, 0);
  }
  __device__ __forceinline__ void wait() const { asm volatile("bar.sync %0, 256;" ::"r"(3 + wg) : "memory"); }
  __device__ __forceinline__ void pass(bool last) const {
    if (!last || wg == 0) asm volatile("bar.arrive %0, 256;" ::"r"(4 - wg) : "memory");
  }
};

// first row of the K / V tile n in the sequence: n * kBN, or, for packed sequences, shifted back to end at the
// sequence's end (see the file comment)
__device__ __forceinline__ int key_tile_start(int n, int sk, bool varlen) {
  return varlen ? min(n * kBN, sk - kBN) : n * kBN;
}

template <typename T, int DP>
__global__ void __launch_bounds__(kThreads, 1)
prefill_attention_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                         const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_qt,
                         const __grid_constant__ CUtensorMap tm_kt, const __grid_constant__ CUtensorMap tm_vt,
                         T* __restrict__ out, const int* __restrict__ cu_q,
                         const int* __restrict__ cu_k, int seqlen_q, int seqlen_k, int heads, int group, int head_dim,
                         float scale_log2, int causal) {
  using C = AttnCfg<DP>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* qs = smem;                              // Q tile (blocks as in AttnCfg)
  uint8_t* kvs = qs + C::kQBytes;                  // stage s: K tile, then V tile
  constexpr int kStages = C::kStages;
  uint8_t* stage_out = kvs + kStages * C::kStageBytes;  // [kBM][kOutRow] T
  uint64_t* full = reinterpret_cast<uint64_t*>(stage_out + kBM * C::kOutRow);  // [kStages] TMA -> consumers
  uint64_t* empty = full + kStages;                // [kStages] consumers (8 warps) -> TMA
  uint64_t* qfull = empty + kStages;               // the Q tile has landed

  const int h = blockIdx.x, b = blockIdx.y;
  const int m0 = (gridDim.z - 1 - blockIdx.z) * kBM;  // heaviest (causal) query tiles first
  const bool varlen = cu_q != nullptr;
  int sq = seqlen_q, sk = seqlen_k, q_tok = 0, k_tok = 0;  // q_tok / k_tok: first token of the sequence (packed)
  if (varlen) {
    q_tok = __ldg(cu_q + b), sq = __ldg(cu_q + b + 1) - q_tok;
    k_tok = __ldg(cu_k + b), sk = __ldg(cu_k + b + 1) - k_tok;
  }
  if (m0 >= sq) return;  // uniform over the CTA
  const int q0 = varlen ? min(m0, sq - kBM) : m0;  // sequence row of the tile's first loaded query row
  const int diag = sk - sq;                        // causal: query i sees keys j <= i + diag
  int n_tiles = (sk + kBN - 1) / kBN;
  if (causal) {
    const int horizon = min(m0 + kBM, sq) - 1 + diag;  // of the tile's last stored row
    n_tiles = min(n_tiles, horizon < 0 ? 0 : horizon / kBN + 1);
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    mbar_init(qfull, 1);
    mbar_fence_init();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // =========================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (threadIdx.x == 0 && n_tiles > 0) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      if constexpr (C::kTail) {
        tma_prefetch_desc(&tm_qt);
        tma_prefetch_desc(&tm_kt);
        tma_prefetch_desc(&tm_vt);
      }
      const int hk = h / group, bz = varlen ? 0 : b;
      mbar_expect_tx(qfull, C::kQBytes);
#pragma unroll
      for (int c = 0; c < C::kMain / 64; ++c) tma_load_4d(qs + c * kBM * 128, &tm_q, qfull, c * 64, q_tok + q0, h, bz);
      if constexpr (C::kTail) tma_load_4d(qs + C::kMain * kBM * 2, &tm_qt, qfull, C::kMain, q_tok + q0, h, bz);
      int s = 0;
      uint32_t ph = 0;
      for (int n = 0; n < n_tiles; ++n) {
        const int row = k_tok + key_tile_start(n, sk, varlen);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], C::kStageBytes);
        uint8_t* st = kvs + s * C::kStageBytes;
#pragma unroll
        for (int c = 0; c < C::kMain / 64; ++c) {
          tma_load_4d(st + c * kBN * 128, &tm_k, &full[s], c * 64, row, hk, bz);
          tma_load_4d(st + C::kKBytes + c * kBN * 128, &tm_v, &full[s], c * 64, row, hk, bz);
        }
        if constexpr (C::kTail) {
          tma_load_4d(st + C::kMain * kBN * 2, &tm_kt, &full[s], C::kMain, row, hk, bz);
          tma_load_4d(st + C::kKBytes + C::kMain * kBN * 2, &tm_vt, &full[s], C::kMain, row, hk, bz);
        }
        if (++s == kStages) s = 0, ph ^= 1;
      }
    }
    return;
  }

  // =========================================================== consumers (warpgroups 1, 2)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
  const int wg = (warp >> 2) - 1, g = lane >> 2, t = lane & 3;
  const int r_lo = wg * 64 + (warp & 3) * 16 + g;  // this thread's tile rows: r_lo, r_lo + 8
  const int i_lo = q0 + r_lo;                      // their sequence rows: i_lo, i_lo + 8
  // accumulator element 4 j + e: row r_lo + 8 (e >> 1), column 8 j + 2 t + (e & 1)
  float o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;  // running max (scaled, log2 units), partial sums
  const uint32_t q_addr = smem_u32(qs) + wg * 64 * 128;                                   // 64-column blocks
  const uint32_t qt_addr = smem_u32(qs) + C::kMain * kBM * 2 + wg * 64 * 32;               // 16-column block
  uint32_t pa[kBN / 16][4];  // P of the current tile as the A fragments of the 8 k16 steps of O += P V
  float sc[64];              // S of the next tile

  auto issue_qk = [&](int stage) {
    const uint32_t k_addr = smem_u32(kvs + stage * C::kStageBytes);
#pragma unroll
    for (int kk = 0; kk < C::kMain / 16; ++kk)  // k16 step kk: block kk / 4, +32 bytes per step inside the block
      wgmma_ss<T>(sc, make_smem_desc(q_addr + (kk / 4) * kBM * 128 + (kk % 4) * 32, 1, 16, 1024),
                  make_smem_desc(k_addr + (kk / 4) * kBN * 128 + (kk % 4) * 32, 1, 16, 1024), kk > 0 ? 1u : 0u);
    if constexpr (C::kTail)
      wgmma_ss<T>(sc, make_smem_desc(qt_addr, 3, 16, 256), make_smem_desc(k_addr + C::kMain * kBN * 2, 3, 16, 256), 1u);
  };
  auto issue_pv = [&](int stage) {
    const uint32_t v_addr = smem_u32(kvs + stage * C::kStageBytes + C::kKBytes);
    // V is MN-major: 64-column blocks kBN * 128 bytes apart, 8-key groups 1024 (tail: 256) bytes apart
    float(&o_main)[C::kMain / 2] = *reinterpret_cast<float(*)[C::kMain / 2]>(o);
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk) {
      wgmma_rs<T, C::kMain, true>(o_main, pa[kk], make_smem_desc(v_addr + kk * 16 * 128, 1, kBN * 128, 1024), 1u);
      if constexpr (C::kTail)
        wgmma_rs<T, 16, true>(*reinterpret_cast<float(*)[8]>(o + C::kMain / 2), pa[kk],
                              make_smem_desc(v_addr + C::kMain * kBN * 2 + kk * 16 * 32, 3, kBN * 32, 256), 1u);
    }
  };
  // mask and online softmax of tile n's S: P into pa, O rescaled
  auto softmax = [&](int n) {
    const int ks = key_tile_start(n, sk, varlen);
    const int k_lo = n * kBN;  // keys below k_lo belong to earlier tiles
    const bool masked = ks != k_lo || k_lo + kBN > sk || (causal && k_lo + kBN - 1 > q0 + diag);
    if (masked) {  // on the raw scores: scale_log2 > 0 keeps -inf the smallest value
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int key = ks + 8 * (i >> 2) + 2 * t + (i & 1);
        const int row = i_lo + ((i & 2) ? 8 : 0);
        const bool ok = key >= k_lo && key < sk && (!causal || key <= row + diag);
        sc[i] = ok ? sc[i] : -INFINITY;
      }
    }
    online_softmax<T>(sc, pa, o, m_lo, m_hi, l_lo, l_hi, scale_log2);
  };
  consume_tiles<kStages>(n_tiles, full, empty, lane, sc, o, Turns{wg, qfull}, issue_qk, issue_pv, softmax);

  // ------------------------------------------------ epilogue: O / l, rounded once, staged, 16-byte stores
  row_sums(l_lo, l_hi);
  const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f, inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
#pragma unroll
  for (int j = 0; j < DP / 8; ++j) {
    const int col = 8 * j + 2 * t;
    *reinterpret_cast<uint32_t*>(stage_out + r_lo * C::kOutRow + col * 2) = pack2<T>(o[4 * j] * inv_lo, o[4 * j + 1] * inv_lo);
    *reinterpret_cast<uint32_t*>(stage_out + (r_lo + 8) * C::kOutRow + col * 2) =
        pack2<T>(o[4 * j + 2] * inv_hi, o[4 * j + 3] * inv_hi);
  }
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
  const int chunks = head_dim / 8;  // 16-byte pieces of an output row (the true head size)
  const size_t row0 = varlen ? (size_t)q_tok : (size_t)b * seqlen_q;
  for (int e = threadIdx.x & 127; e < 64 * chunks; e += 128) {
    const int r = wg * 64 + e / chunks, cc = e % chunks;
    const int i = q0 + r;
    if (i >= m0 && i < sq)
      *reinterpret_cast<uint4*>(out + ((row0 + i) * heads + h) * head_dim + cc * 8) =
          *reinterpret_cast<const uint4*>(stage_out + r * C::kOutRow + cc * 16);
  }
}

template <typename T, int DP>
int launch_t(const void* q, const void* k, const void* v, void* out, const int* cu_q, const int* cu_k, int batch,
             int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim, const long long* qs, const long long* ks,
             const long long* vs, float softmax_scale, bool causal, cudaStream_t stream) {
  using C = AttnCfg<DP>;
  EncodeTiledFn enc = get_encoder();
  if (!enc) return B200AWQ_ERR_DRIVER;
  // packed sequences: one "batch" of batch * max-length tokens, an upper bound of the packed length that no tile
  // reaches past (tiles end at their sequence's end)
  const bool varlen = cu_q != nullptr;
  const int nb = varlen ? 1 : batch;
  const long long tq = varlen ? (long long)batch * seqlen_q : seqlen_q;
  const long long tk = varlen ? (long long)batch * seqlen_k : seqlen_k;
  CUtensorMap tm[6];  // q, k, v; their 16-column tails (D = 72; otherwise unused copies)
  if (int e = encode_bthd<T>(enc, &tm[0], q, head_dim, tq, heads, nb, qs, 64, kBM)) return e;
  if (int e = encode_bthd<T>(enc, &tm[1], k, head_dim, tk, kv_heads, nb, ks, 64, kBN)) return e;
  if (int e = encode_bthd<T>(enc, &tm[2], v, head_dim, tk, kv_heads, nb, vs, 64, kBN)) return e;
  for (int i = 0; i < 3; ++i) tm[3 + i] = tm[i];
  if constexpr (C::kTail) {
    if (int e = encode_bthd<T>(enc, &tm[3], q, head_dim, tq, heads, nb, qs, 16, kBM)) return e;
    if (int e = encode_bthd<T>(enc, &tm[4], k, head_dim, tk, kv_heads, nb, ks, 16, kBN)) return e;
    if (int e = encode_bthd<T>(enc, &tm[5], v, head_dim, tk, kv_heads, nb, vs, 16, kBN)) return e;
  }
  if (cudaError_t ea = ensure_dyn_smem<prefill_attention_kernel<T, DP>>(C::kSmem)) return (int)ea;
  const dim3 grid((unsigned)heads, (unsigned)batch, (unsigned)((seqlen_q + kBM - 1) / kBM));
  const float scale_log2 = softmax_scale * 1.4426950408889634f;
  // no programmatic dependent launch: the kernel never waits on the previous grid
  return launch_kernel(prefill_attention_kernel<T, DP>, grid, dim3(kThreads), (size_t)C::kSmem, stream, false, 1, tm[0], tm[1],
                       tm[2], tm[3], tm[4], tm[5], out, cu_q, cu_k, seqlen_q, seqlen_k, heads, heads / kv_heads, head_dim,
                       scale_log2, causal ? 1 : 0);
}

template <typename T>
int launch_d(int head_dim, const void* q, const void* k, const void* v, void* out, const int* cu_q, const int* cu_k, int batch,
             int seqlen_q, int seqlen_k, int heads, int kv_heads, const long long* qs, const long long* ks, const long long* vs,
             float scale, bool causal, cudaStream_t st) {
  switch (head_dim) {
    case 64: return launch_t<T, 64>(q, k, v, out, cu_q, cu_k, batch, seqlen_q, seqlen_k, heads, kv_heads, 64, qs, ks, vs, scale, causal, st);
    case 72: return launch_t<T, 80>(q, k, v, out, cu_q, cu_k, batch, seqlen_q, seqlen_k, heads, kv_heads, 72, qs, ks, vs, scale, causal, st);
    case 128: return launch_t<T, 128>(q, k, v, out, cu_q, cu_k, batch, seqlen_q, seqlen_k, heads, kv_heads, 128, qs, ks, vs, scale, causal, st);
    default: return B200AWQ_ERR_SHAPE;
  }
}

}  // namespace

int launch_prefill_attention(const void* q, const void* k, const void* v, void* out, const int* cu_q, const int* cu_k, int batch,
                             int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim, const long long* q_strides,
                             const long long* k_strides, const long long* v_strides, float softmax_scale, bool causal, int dtype,
                             cudaStream_t stream) {
  if (dtype == B200AWQ_DTYPE_F16)
    return launch_d<__half>(head_dim, q, k, v, out, cu_q, cu_k, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides, k_strides,
                            v_strides, softmax_scale, causal, stream);
  return launch_d<__nv_bfloat16>(head_dim, q, k, v, out, cu_q, cu_k, batch, seqlen_q, seqlen_k, heads, kv_heads, q_strides,
                                 k_strides, v_strides, softmax_scale, causal, stream);
}

}  // namespace b200awq
