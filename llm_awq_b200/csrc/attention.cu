// Decode-step attention and rotary embedding around the W4A16 linears (SURVEY.md §8f-3).
//
//  * single-query attention with the KV-cache layout tinychat's callers fix
//      k_cache [B, Hkv, D / 8, L, 8]   v_cache [B, Hkv, L, D]       (tinychat/modules/fused_attn.py:195-223)
//    replaces `single_query_attention` (awq/kernels/csrc/attention/ft_attention.cpp:112-184 ->
//    decoder_masked_multihead_attention_template.hpp:880-1500, FasterTransformer's masked MHA): per (batch, head)
//      tlength = length_per_sample ? length_per_sample[b] : timestep                        (:975-978)
//      q, k of the current step are rotated at position tlength (RoPE, angle = tlength * scale / base^(2i / rot_dim),
//      utils.h:1282-1287; neox style pairs (i, i + rot_dim / 2), else (2i, 2i + 1)) and ROUNDED to T        (:1080-1135)
//      k, v are written to the cache at slot tlength % L                                   (:1148-1175, :1424-1440)
//      out = softmax(q . K^T / sqrt(D)) V over positions max(0, tlength + 1 - L) .. tlength  (:1177-1500), fp32 math
//    ALiBi slopes and fp32 tensors are not supported here (Llama-family callers pass None / fp16, bf16).
//    Any G = H / Hkv >= 1, any head size D % 8 == 0 up to 256.
//    Design: the query heads that share a KV head are served by head groups of at most 8 heads, one CTA per group (the
//    KV bytes are read once per group, 16-byte loads: K coalesces over positions, V over channels; G <= 8 is one group,
//    larger G re-reads the KV head once per extra group, concurrently, so mostly from L2), and long contexts are SPLIT
//    over CTAs (flash-decoding): every CTA writes (max, sum, unnormalised output) of its chunk to the workspace, the last
//    one to arrive combines in a fixed order.  HBM-bound: algorithmic bytes = 2 * n_pos * D * sizeof(T) per KV head.
//  * fused_rope_with_pos_forward_func (awq/kernels/csrc/rope_new/fused_rope_with_pos.cu:33-75,243-285): RoPE over a
//    strided [s, b, h, d] tensor with per-(s, b) angles `freqs`, fp32 math, one rounding.
#include <algorithm>
#include <cfloat>

#include "rope_kv_store.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 p;
    if constexpr (TypeTraits<T>::kIsBf16) p = __bfloat1622float2(u32_as_b2(w[i]));
    else p = __half22float2(u32_as_h2(w[i]));
    f[2 * i] = p.x, f[2 * i + 1] = p.y;
  }
}

constexpr int kAttThreads = 256;
constexpr int kAttMaxGS = 8;   // query heads per CTA (a head group); G = H / Hkv > 8 takes ceil(G / 8) groups
constexpr int kAttMaxD = 256;  // head dimension
constexpr int kAttCounters = kAttentionCounters;  // batch * kv_heads * groups the workspace's counter block is sized for

// Head groups of a KV head: ceil(G / 8) groups of near-equal size gs = ceil(G / groups) <= 8; the last group's heads
// past G are masked.  For G <= 8: one group of G heads.
inline int att_groups(int G) { return (G + kAttMaxGS - 1) / kAttMaxGS; }
inline int att_group_size(int G) { return (G + att_groups(G) - 1) / att_groups(G); }

struct AttArgs {
  const void* q;
  const void* k;
  const void* v;
  void* k_cache;
  void* v_cache;
  void* out;
  const int* length_per_sample;
  float* ws;            // [B][Hkv][groups][splits][GS][D + 2] partials (after the counters)
  unsigned int* count;  // [B][Hkv][groups] arrival counters at the START of the workspace (zero between launches)
  long long q_stride, k_stride, v_stride;  // elements between batches of q / k / v
  int B, H, Hkv, G, groups, D, L, timestep, rot_dim, neox, splits, chunk;
  float base, scale, inv_sqrt_d;
};

// rotate (x, y) by the angle of pair `pair_idx` at position t
__device__ __forceinline__ void rope_pair(float& x, float& y, int pair_idx, int rot_dim, int t, float base, float scale) {
  const float ang = ((float)t * scale) / powf(base, (float)(2 * pair_idx) / (float)rot_dim);
  float s, c;
  sincosf(ang, &s, &c);
  const float rx = c * x - s * y, ry = c * y + s * x;
  x = rx, y = ry;
}

// logits of one position for all GS heads: k at kp + c * cstep (c = 8-channel chunk), four 16-byte loads in flight; the
// same fma order wherever k comes from (the cache or this CTA's copy of the current step)
template <typename T, int GS>
__device__ __forceinline__ void att_logits(const T* kp, size_t cstep, int nch, const float* qs, int D, float (&acc)[GS]) {
#pragma unroll
  for (int g = 0; g < GS; ++g) acc[g] = 0.f;
  for (int c0 = 0; c0 < nch; c0 += 4) {  // the tail is guarded
    uint4 kv4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      kv4[j] = c0 + j < nch ? *reinterpret_cast<const uint4*>(kp + (size_t)(c0 + j) * cstep) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c0 + j >= nch) break;
      const int c = c0 + j;
      float kf[8];
      unpack8<T>(kv4[j], kf);
#pragma unroll
      for (int g = 0; g < GS; ++g) {
        const float4 qa = *reinterpret_cast<const float4*>(qs + g * D + c * 8);
        const float4 qb = *reinterpret_cast<const float4*>(qs + g * D + c * 8 + 4);
        acc[g] = fmaf(qa.x, kf[0], acc[g]), acc[g] = fmaf(qa.y, kf[1], acc[g]);
        acc[g] = fmaf(qa.z, kf[2], acc[g]), acc[g] = fmaf(qa.w, kf[3], acc[g]);
        acc[g] = fmaf(qb.x, kf[4], acc[g]), acc[g] = fmaf(qb.y, kf[5], acc[g]);
        acc[g] = fmaf(qb.z, kf[6], acc[g]), acc[g] = fmaf(qb.w, kf[7], acc[g]);
      }
    }
  }
}

// One CTA = (split, KV head x head group, batch).  GS = query heads per CTA; heads of the group past G are masked.
// Two CTAs per SM: <= 128 registers, and without the bound ptxas spills at GS = 1 (-Xptxas -v).
template <typename T, int GS>
__global__ void __launch_bounds__(kAttThreads, 2) single_query_attention_kernel(const AttArgs a) {
  extern __shared__ __align__(16) float att_smem[];
  const int D = a.D, L = a.L;
  float* qs = att_smem;                                     // [GS][D] rotated, rounded queries
  T* kcur = reinterpret_cast<T*>(qs + GS * D);              // [D] rotated, rounded key of the current step
  T* vcur = kcur + D;                                       // [D] value of the current step
  float* red = qs + GS * D + D;                             // [8 warps][GS] reduction scratch, then [GS] max, [GS] sum
  float* sc = red + kAttThreads / 32 * GS + 2 * GS;         // [GS][chunk] logits -> probabilities
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int split = blockIdx.x, kvh = blockIdx.y / a.groups, grp = blockIdx.y % a.groups, b = blockIdx.z;
  const int h0 = grp * GS, ng = min(GS, a.G - h0);         // this CTA's heads: kvh * G + h0 .. + ng - 1
  const T* q = static_cast<const T*>(a.q) + (size_t)b * a.q_stride;
  const T* kin = static_cast<const T*>(a.k) + (size_t)b * a.k_stride;
  const T* vin = static_cast<const T*>(a.v) + (size_t)b * a.v_stride;
  T* kc = static_cast<T*>(a.k_cache) + (size_t)(b * a.Hkv + kvh) * L * D;
  T* vc = static_cast<T*>(a.v_cache) + (size_t)(b * a.Hkv + kvh) * L * D;
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const int tlength = a.length_per_sample ? a.length_per_sample[b] : a.timestep;
  const int first = max(0, tlength + 1 - L);
  const int npos = tlength + 1 - first;                   // positions attended to, the current one last
  const int p0 = first + split * a.chunk, p1 = min(first + npos, p0 + a.chunk);
  const bool has_current = p0 <= tlength && tlength < p0 + a.chunk;  // this CTA's chunk holds the current step
  const bool writes_cache = has_current && grp == 0;      // one CTA per (batch, KV head) stores the step in the cache
  const int pc = has_current ? tlength : p1;              // cache positions p0 .. pc - 1; the current one from kcur / vcur
  const int half_rot = a.rot_dim >> 1;

  // ---- current step: rotate q (every CTA) and k (every CTA whose chunk holds the current step: the same arithmetic in
  // each, so all head groups see the same bits), round to T like the reference.  No CTA reads the cache slot of the
  // current step, which another CTA may be writing.
  // Pair slot j of a head: neox style -> elements (j, j + rot_dim / 2) for j < rot_dim / 2, angle index j; interleaved ->
  // elements (2 j, 2 j + 1), angle index j while 2 j < rot_dim; the remaining elements are copied.
  for (int i = tid; i < (GS + 1) * (D / 2); i += kAttThreads) {
    const int g = i / (D / 2), j = i % (D / 2);            // g == GS: the key
    if (g == GS && !has_current) continue;
    if (g < GS && g >= ng) {                               // masked head: zero query, output never stored
      qs[g * D + 2 * j] = 0.f, qs[g * D + 2 * j + 1] = 0.f;
      continue;
    }
    const T* src = g < GS ? q + (size_t)(kvh * a.G + h0 + g) * D : kin + (size_t)kvh * D;
    int i0, i1;
    bool rot;
    if (a.neox) {
      rot = j < half_rot;
      i0 = rot ? j : a.rot_dim + 2 * (j - half_rot);
      i1 = rot ? j + half_rot : i0 + 1;
    } else {
      rot = 2 * j < a.rot_dim;
      i0 = 2 * j, i1 = 2 * j + 1;
    }
    float x = to_float<T>(src[i0]), y = to_float<T>(src[i1]);
    if (rot) rope_pair(x, y, j, a.rot_dim, tlength, a.base, a.scale);
    const T xr = from_float<T>(x), yr = from_float<T>(y);
    if (g < GS) {
      qs[g * D + i0] = to_float<T>(xr), qs[g * D + i1] = to_float<T>(yr);
    } else {
      kcur[i0] = xr, kcur[i1] = yr;
      if (writes_cache) {                                  // k -> cache [D / 8][L][8] at slot tlength % L
        const int slot = tlength % L;
        kc[((size_t)(i0 >> 3) * L + slot) * 8 + (i0 & 7)] = xr;
        kc[((size_t)(i1 >> 3) * L + slot) * 8 + (i1 & 7)] = yr;
      }
    }
  }
  if (has_current)
    for (int i = tid; i < D; i += kAttThreads) {
      const T x = vin[(size_t)kvh * D + i];
      vcur[i] = x;
      if (writes_cache) vc[(size_t)(tlength % L) * D + i] = x;
    }
  __syncthreads();  // qs, kcur, vcur complete

  // ---- logits of this chunk: lane = position (K coalesces over positions), all GS heads against one load of K
  float mx[GS];
#pragma unroll
  for (int g = 0; g < GS; ++g) mx[g] = -FLT_MAX;
  const int nch = D >> 3;
  auto store_logits = [&](int p, const float (&acc)[GS]) {
#pragma unroll
    for (int g = 0; g < GS; ++g) {
      const float s = acc[g] * a.inv_sqrt_d;
      sc[g * a.chunk + (p - p0)] = s;
      mx[g] = fmaxf(mx[g], s);
    }
  };
  for (int p = p0 + tid; p < pc; p += kAttThreads) {
    float acc[GS];
    att_logits<T, GS>(kc + (size_t)(p % L) * 8, (size_t)L * 8, nch, qs, D, acc);
    store_logits(p, acc);
  }
  if (has_current && (tlength - p0) % kAttThreads == tid) {  // the thread the current position falls to
    float acc[GS];
    att_logits<T, GS>(kcur, 8, nch, qs, D, acc);
    store_logits(tlength, acc);
  }
  // block max per head
#pragma unroll
  for (int g = 0; g < GS; ++g) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx[g] = fmaxf(mx[g], __shfl_xor_sync(0xffffffffu, mx[g], o));
    if (lane == 0) red[warp * GS + g] = mx[g];
  }
  __syncthreads();
  float* stat = red + kAttThreads / 32 * GS;  // [GS] max, [GS] sum
  if (tid < GS) {
    float m = -FLT_MAX;
    for (int w = 0; w < kAttThreads / 32; ++w) m = fmaxf(m, red[w * GS + tid]);
    stat[tid] = m;
  }
  __syncthreads();
  float sum[GS];
#pragma unroll
  for (int g = 0; g < GS; ++g) sum[g] = 0.f;
  for (int i = tid; i < p1 - p0; i += kAttThreads) {
#pragma unroll
    for (int g = 0; g < GS; ++g) {
      const float e = __expf(sc[g * a.chunk + i] - stat[g]);
      sc[g * a.chunk + i] = e;
      sum[g] += e;
    }
  }
  __syncthreads();  // stat[max] consumed by everybody; red reusable
#pragma unroll
  for (int g = 0; g < GS; ++g) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum[g] += __shfl_xor_sync(0xffffffffu, sum[g], o);
    if (lane == 0) red[warp * GS + g] = sum[g];
  }
  __syncthreads();
  if (tid < GS) {
    float s = 0.f;
    for (int w = 0; w < kAttThreads / 32; ++w) s += red[w * GS + tid];
    stat[GS + tid] = s;
  }
  __syncthreads();

  // ---- probabilities x V: thread = (row r of 256 / (D / 8) position rows, rounded down, 8 channels dc); V coalesces
  // over channels.  The spare threads of a head size that does not divide 2048 idle.
  const int tpr = D >> 3, rows = kAttThreads / tpr, r = tid / tpr, dc = tid % tpr;
  float o[GS][8];
#pragma unroll
  for (int g = 0; g < GS; ++g)
#pragma unroll
    for (int e = 0; e < 8; ++e) o[g][e] = 0.f;
  auto accumulate_v = [&](int p, const uint4& v4) {
    float vf[8];
    unpack8<T>(v4, vf);
#pragma unroll
    for (int g = 0; g < GS; ++g) {
      const float pr = sc[g * a.chunk + (p - p0)];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[g][e] = fmaf(pr, vf[e], o[g][e]);
    }
  };
  if (r < rows) {
    for (int pb = p0 + r; pb < pc; pb += 4 * rows) {  // four rows of V in flight per thread
      uint4 vv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int p = pb + j * rows;
        vv[j] = p < pc ? *reinterpret_cast<const uint4*>(vc + (size_t)(p % L) * D + dc * 8) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int p = pb + j * rows;
        if (p >= pc) break;
        accumulate_v(p, vv[j]);
      }
    }
    // the current step is the last position of its row: the same accumulation order as if it came from the cache
    if (has_current && (tlength - p0) % rows == r) accumulate_v(tlength, *reinterpret_cast<const uint4*>(vcur + dc * 8));
  }
  // reduce over the position rows through shared memory (reusing the logits' space: every probability has been read)
  __syncthreads();
  float* pv = sc;  // [rows][GS][D]
  if (r < rows) {
#pragma unroll
    for (int g = 0; g < GS; ++g)
#pragma unroll
      for (int e = 0; e < 8; ++e) pv[(r * GS + g) * D + dc * 8 + e] = o[g][e];
  }
  __syncthreads();
  const size_t cell = (size_t)(b * a.Hkv + kvh) * a.groups + grp;  // (batch, KV head, head group)
  float* part = a.ws + (cell * a.splits + split) * GS * (D + 2);
  T* out = static_cast<T*>(a.out) + ((size_t)b * a.H + (size_t)kvh * a.G + h0) * D;
  for (int i = tid; i < GS * D; i += kAttThreads) {
    float s = 0.f;
    for (int rr = 0; rr < rows; ++rr) s += pv[rr * GS * D + i];
    if (a.splits == 1) {
      if (i < ng * D) out[i] = from_float<T>(s / stat[GS + i / D]);
    } else {
      part[(i / D) * (D + 2) + (i % D)] = s;
    }
  }
  if (a.splits == 1) return;
  if (tid < GS) part[tid * (D + 2) + D] = stat[tid], part[tid * (D + 2) + D + 1] = stat[GS + tid];
  // ---- the last CTA of this (batch, KV head, head group) combines the chunks
  __threadfence();
  __syncthreads();
  __shared__ unsigned int s_last;
  if (tid == 0) s_last = atomicAdd(&a.count[cell], 1u) == (unsigned)a.splits - 1 ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* all = a.ws + cell * a.splits * GS * (D + 2);
  for (int i = tid; i < ng * D; i += kAttThreads) {
    const int g = i / D, d = i % D;
    float M = -FLT_MAX;
    for (int s = 0; s < a.splits; ++s) M = fmaxf(M, all[((size_t)s * GS + g) * (D + 2) + D]);
    float num = 0.f, den = 0.f;
    for (int s = 0; s < a.splits; ++s) {
      const float* ps = all + ((size_t)s * GS + g) * (D + 2);
      const float w = __expf(ps[D] - M);
      num = fmaf(w, ps[d], num), den = fmaf(w, ps[D + 1], den);
    }
    out[i] = from_float<T>(num / den);
  }
  if (tid == 0) a.count[cell] = 0u;  // ready for the next launch (graph replay included)
}

template <typename T, int GS>
int launch_att_gs(const AttArgs& a, size_t smem, bool pdl, cudaStream_t stream) {
  // The size follows the shape (head size, positions per split), so the opt-in is set on every launch that needs it
  // rather than once per device.
  if (smem > 48 * 1024) {
    if (cudaError_t e = cudaFuncSetAttribute(single_query_attention_kernel<T, GS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem))
      return (int)e;
  }
  return launch_kernel(single_query_attention_kernel<T, GS>, dim3((unsigned)a.splits, (unsigned)(a.Hkv * a.groups), (unsigned)a.B),
                       dim3(kAttThreads), smem, stream, pdl, 1, a);
}

template <typename T>
int launch_att_g(const AttArgs& a, int GS, size_t smem, bool pdl, cudaStream_t stream) {
  switch (GS) {
    case 1: return launch_att_gs<T, 1>(a, smem, pdl, stream);
    case 2: return launch_att_gs<T, 2>(a, smem, pdl, stream);
    case 3: return launch_att_gs<T, 3>(a, smem, pdl, stream);
    case 4: return launch_att_gs<T, 4>(a, smem, pdl, stream);
    case 5: return launch_att_gs<T, 5>(a, smem, pdl, stream);
    case 6: return launch_att_gs<T, 6>(a, smem, pdl, stream);
    case 7: return launch_att_gs<T, 7>(a, smem, pdl, stream);
    case 8: return launch_att_gs<T, 8>(a, smem, pdl, stream);
    default: return B200AWQ_ERR_SHAPE;
  }
}

// ------------------------------------------------------------------------------------------------ RoPE over [s, b, h, d]
struct RopeArgs {
  const void* x;
  const float* freqs;
  void* y;
  int s, b, h, d, d2;
  long long ss, sb, sh, sd, os, ob, oh, od;
};

template <typename T>
__global__ void __launch_bounds__(256) rope_with_pos_kernel(const RopeArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const int s_id = blockIdx.x, b_id = blockIdx.y;
  const T* src = static_cast<const T*>(a.x) + s_id * a.ss + b_id * a.sb;
  T* dst = static_cast<T*>(a.y) + s_id * a.os + b_id * a.ob;
  const float* fr = a.freqs + ((size_t)b_id * a.s + s_id) * a.d2;  // fused_rope_with_pos.cu:46
  for (int i = threadIdx.x; i < a.h * a.d; i += blockDim.x) {
    const int h_id = i / a.d, d_id = i % a.d;
    const T* sp = src + h_id * a.sh;
    float v = to_float<T>(sp[d_id * a.sd]);
    if (d_id < a.d2) {
      const RopeAngle ang = rope_angle(fr[d_id]);
      const float rot = (d_id + a.d2 / 2 < a.d2) ? -to_float<T>(sp[(d_id + a.d2 / 2) * a.sd]) : to_float<T>(sp[(d_id - a.d2 / 2) * a.sd]);
      v = rope_apply(v, rot, ang);  // fused_rope_with_pos.cu:52-57
    }
    dst[h_id * a.oh + d_id * a.od] = from_float<T>(v);
  }
}

}  // namespace

size_t attention_workspace_bytes(int batch, int heads, int kv_heads, int head_dim, int max_len) {
  if (batch < 1 || kv_heads < 1 || heads < kv_heads || head_dim < 8) return 0;
  const int G = heads / kv_heads;
  const size_t max_splits = 64;
  (void)max_len;
  // [counters: kAttCounters x u32, always at offset 0 whatever the shape -- partials of an earlier launch with another
  // shape must never alias them] [partials: G (head_dim + 2) floats per head and split, the masked heads of the last
  // head group included]
  const size_t padded_g = (size_t)att_groups(G) * att_group_size(G);
  return kAttCounters * sizeof(unsigned int) + (size_t)batch * kv_heads * (max_splits * padded_g * (head_dim + 2) * sizeof(float));
}

int launch_single_query_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, void* out,
                                  const int* length_per_sample, int batch, int heads, int kv_heads, int head_dim, int max_len,
                                  int timestep, long long q_batch_stride, long long k_batch_stride, long long v_batch_stride, int rotary_dim, float rotary_base, float rotary_scale,
                                  int neox, int dtype, void* workspace, size_t workspace_bytes, bool pdl, cudaStream_t stream) {
  if (batch < 1 || kv_heads < 1 || heads < kv_heads || heads % kv_heads || head_dim < 8 || head_dim % 8 || head_dim > kAttMaxD ||
      max_len < 1 || timestep < 0 || rotary_dim < 0 || rotary_dim > head_dim || (rotary_dim & 1) || (neox && rotary_dim % 2))
    return B200AWQ_ERR_SHAPE;
  const int G = heads / kv_heads, groups = att_groups(G), GS = att_group_size(G);
  if ((long long)batch * kv_heads * groups > kAttCounters) return B200AWQ_ERR_SHAPE;
  if (workspace_bytes < attention_workspace_bytes(batch, heads, kv_heads, head_dim, max_len) || !workspace)
    return B200AWQ_ERR_WORKSPACE;
  AttArgs a{};
  a.q = q, a.k = k, a.v = v, a.k_cache = k_cache, a.v_cache = v_cache, a.out = out;
  a.length_per_sample = length_per_sample;
  a.B = batch, a.H = heads, a.Hkv = kv_heads, a.G = G, a.groups = groups, a.D = head_dim, a.L = max_len, a.timestep = timestep;
  a.q_stride = q_batch_stride, a.k_stride = k_batch_stride, a.v_stride = v_batch_stride;
  a.rot_dim = rotary_dim, a.neox = neox, a.base = rotary_base, a.scale = rotary_scale;
  a.inv_sqrt_d = 1.f / sqrtf((float)head_dim);
  // worst-case positions (length_per_sample is on the device): the chunking must cover up to min(timestep, max_len - 1) + 1
  const int npos_max = std::min(length_per_sample ? max_len : timestep + 1, max_len);
  const int nsm = sm_count();
  if (nsm == 0) return B200AWQ_ERR_DEVICE;
  const int chunk_cap = std::max(256, (48 * 1024 / 4) / GS / 32 * 32);  // logits of a chunk: GS * chunk floats <= 48 KB
  int splits = std::max(1, std::min(64, 2 * nsm / std::max(1, batch * kv_heads * groups)));
  splits = std::min(splits, (npos_max + 127) / 128);                  // >= 128 positions per CTA
  splits = std::max(splits, (npos_max + chunk_cap - 1) / chunk_cap);
  if (splits > 64) return B200AWQ_ERR_SHAPE;
  a.splits = std::max(1, splits);
  a.chunk = ((npos_max + a.splits - 1) / a.splits + 31) / 32 * 32;
  a.count = static_cast<unsigned int*>(workspace);
  a.ws = reinterpret_cast<float*>(static_cast<char*>(workspace) + kAttCounters * sizeof(unsigned int));
  const int rows = kAttThreads / (head_dim / 8);  // rounded down
  const size_t sc_floats = std::max((size_t)GS * a.chunk, (size_t)rows * GS * head_dim);
  // [GS][D] queries, [D] key + [D] value of the current step as T (D floats), reduction scratch, logits / PV partials
  const size_t smem = ((size_t)GS * head_dim + head_dim + kAttThreads / 32 * GS + 2 * GS + sc_floats) * sizeof(float) + 16;
  if (smem > 200 * 1024) return B200AWQ_ERR_SHAPE;
  if (dtype == B200AWQ_DTYPE_F16) return launch_att_g<__half>(a, GS, smem, pdl, stream);
  return launch_att_g<__nv_bfloat16>(a, GS, smem, pdl, stream);
}

int launch_rope_with_pos(const void* x, const float* freqs, void* y, int s, int b, int h, int d, int d2, const long long* in_strides,
                         const long long* out_strides, int dtype, bool pdl, cudaStream_t stream) {
  if (s < 1 || b < 1 || h < 1 || d < 1 || d2 < 0 || d2 > d || (d2 & 1)) return B200AWQ_ERR_SHAPE;
  RopeArgs a{x, freqs, y, s, b, h, d, d2, in_strides[0], in_strides[1], in_strides[2], in_strides[3],
             out_strides[0], out_strides[1], out_strides[2], out_strides[3]};
  const dim3 grid((unsigned)s, (unsigned)b);
  if (dtype == B200AWQ_DTYPE_F16) return launch_kernel(rope_with_pos_kernel<__half>, grid, dim3(256), 0, stream, pdl, 1, a);
  return launch_kernel(rope_with_pos_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, pdl, 1, a);
}

}  // namespace b200awq
