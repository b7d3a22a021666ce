// Internal launcher interface between the C ABI (api.cu) and the kernel translation units, and the host launch path
// every launcher shares.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <atomic>

#include "../../include/b200awq.h"

namespace b200awq {

inline bool aligned16(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Per-device host caches hold this many devices; a device with a higher ordinal is served uncached.
constexpr int kMaxCachedDevices = 64;

// The current device's SM count, cached per device; 0 if the query fails.
inline int sm_count() {
  static std::atomic<int> cache[kMaxCachedDevices];
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (dev < kMaxCachedDevices && (n = cache[dev].load(std::memory_order_relaxed)) > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 0) return 0;
  if (dev < kMaxCachedDevices) cache[dev].store(n, std::memory_order_relaxed);
  return n;
}

// Opt kernel `Kern` into `bytes` of dynamic shared memory once per device (function attributes are per device, and
// several GPUs may be driven from one process); `max_shared_carveout` also asks for the largest shared-memory carveout.
template <auto Kern>
inline cudaError_t ensure_dyn_smem(int bytes, bool max_shared_carveout = false) {
  static std::atomic<bool> done[kMaxCachedDevices];
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  const bool cached = dev < kMaxCachedDevices;
  if (cached && done[dev].load(std::memory_order_acquire)) return cudaSuccess;
  if (cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)) return e;
  if (max_shared_carveout)
    cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (cached) done[dev].store(true, std::memory_order_release);
  return cudaSuccess;
}

// Launches `kern` with programmatic dependent launch when `pdl` and in clusters of `cluster_x` CTAs when > 1.
// Returns 0 or the launch's cudaError_t.
template <typename... KArgs, typename... Args>
int launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                  unsigned cluster_x, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  if (cluster_x > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = cluster_x;
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
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  return e == cudaSuccess ? 0 : (int)e;
}

// Every launcher below picks its kernel configuration (instantiation, k split, grid, ring depth, shared-memory size)
// from the shape and the device's SM count alone; the constants behind those choices live in the launchers.  The one
// exception is DecodeTuning: a test-only override of the decode kernel's plan (include/b200awq.h).

// Row-parallel tensor parallelism: the GEMV epilogue exchanges fp32 partial sums with the peer GPUs through
// symmetric (peer-mapped) buffers over NVLink and reduces them in the same kernel (w4a16_stream.cu).
struct PeerArgs {
  unsigned long long* data[8];  // data[r]: rank r's exchange buffer ({fp32, epoch} words) as mapped in this process
  unsigned int* epoch;          // this rank's per-row-block epoch counters (device memory, zero-initialised once)
  int rank, world;              // world <= 1: no exchange
  int cap;                      // words per (parity, source) region  (= tok_cap * n_max)
  int tok_cap;                  // tokens a region is laid out for: word slot = channel * tok_cap + token
};

// Bias / residual epilogue of a W4A16 launch (b200awq_w4a16_linear): y = rn_T(rn_T(rn_T(acc) + bias[n]) + residual[i, n]),
// either pointer may be null.  Both null (the default) launches the plain instantiation of the kernel, the one the
// other entries run; otherwise the launcher picks the instantiation that loads them after griddepcontrol.wait.
struct Epilogue {
  const void* bias = nullptr;      // [N] of the activation dtype
  const void* residual = nullptr;  // [M, N] of the activation dtype
  bool on() const { return bias || residual; }
};

// RMSNorm prologue of a one-token / few-token W4A16 launch (b200awq_w4a16_norm_linear, b200awq_w4a16_norm_mlp_front):
// the kernel multiplies x^ = RMSNorm(x, gamma, eps) (rmsnorm_stat.cuh), bit-identical to launch_rmsnorm's output, instead
// of x.  Only launch_decode, launch_decode_mlp_front and launch_ring take one; with gamma null (the default) they launch
// the instantiation the other entries run.
struct NormPrologue {
  const void* gamma = nullptr;  // [K] of the activation dtype, 16-byte aligned
  float eps = 0.f;
  bool on() const { return gamma != nullptr; }
};

// HBM-bound streaming kernel, 1 <= M <= 16 (w4a16_stream.cu); the epilogue does not apply to the all-reduce (peers)
int launch_stream(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                  bool pdl, cudaStream_t stream, const PeerArgs* peers = nullptr, const Epilogue& epi = Epilogue{});

// TMA + wgmma tensor-core kernel, any M, N % 128 == 0 (w4a16_wgmma.cu)
int launch_umma(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi = Epilogue{});

// persistent warp-specialised decode kernel, 1 <= M <= 4 (w4a16_ring.cu); returns B200AWQ_ERR_SHAPE when the
// activations do not fit next to a useful ring (the caller falls back to the kernels below)
int launch_ring(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi = Epilogue{}, const NormPrologue& norm = NormPrologue{});

// Test-only override of the decode kernel's plan (env B200AWQ_DECODE_SPLIT / B200AWQ_DECODE_SLOTS, api.cu): the
// default-constructed value means "pick from the shape".
struct DecodeTuning {
  int split = 0;   // 0 = auto, else CTAs per cluster = k split (1 to 8)
  int slots = 0;   // 0 = as many ring slots as fit next to a second CTA, else a cap
};

// one-token fp16 decode kernel: 8 KB bulk copies, int8-digit tensor-core MACs (w4a16_decode.cu); returns
// B200AWQ_ERR_SHAPE for bf16 and when the activations do not fit next to a useful ring (the caller falls back)
int launch_decode(const void* x, const void* qw, const void* sc, const void* sz, void* y, int N, int K, int dtype, bool pdl,
                  const DecodeTuning& tune, cudaStream_t stream, const Epilogue& epi = Epilogue{},
                  const NormPrologue& norm = NormPrologue{});

// one-token fused MLP front half: y = silu(x Wgate~^T) * (x Wup~^T), both weight sets through one ring (w4a16_decode.cu)
int launch_decode_mlp_front(const void* x, const void* gqw, const void* gsc, const void* gsz, const void* uqw, const void* usc,
                            const void* usz, void* y, int N, int K, int dtype, bool pdl, const DecodeTuning& tune,
                            cudaStream_t stream, const NormPrologue& norm = NormPrologue{});

// out = silu(gate) * up over rows x cols elements, the reference's roundings; gate / up rows are in_pitch elements
// apart, out is dense (silu_mul.cu)
int launch_silu_mul(const void* gate, const void* up, void* out, size_t rows, size_t cols, size_t in_pitch, int dtype, bool pdl,
                    cudaStream_t stream);

// Both attention workspaces (single-query decode and split-key attention) start with the same block of kAttentionCounters
// u32 arrival counters, which every launch leaves zero, so that one zero-initialised buffer per stream can serve both:
// the partials of one entry never alias the other's counters.
constexpr int kAttentionCounters = 4096;

// single-query (decode-step) attention over tinychat's KV-cache layout + RoPE over [s, b, h, d] (attention.cu)
size_t attention_workspace_bytes(int batch, int heads, int kv_heads, int head_dim, int max_len);
int launch_single_query_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, void* out,
                                  const int* length_per_sample, int batch, int heads, int kv_heads, int head_dim, int max_len,
                                  int timestep, long long q_batch_stride, long long k_batch_stride, long long v_batch_stride, int rotary_dim, float rotary_base, float rotary_scale,
                                  int neox, int dtype, void* workspace, size_t workspace_bytes, bool pdl, cudaStream_t stream);
int launch_rope_with_pos(const void* x, const float* freqs, void* y, int s, int b, int h, int d, int d2, const long long* in_strides,
                         const long long* out_strides, int dtype, bool pdl, cudaStream_t stream);
// in-place NeoX RoPE from a cos|sin table (rope_neox.cu)
int launch_rope_neox(const long long* positions, void* query, void* key, const void* cos_sin, int tokens, int q_heads,
                     int k_heads, int head_size, int rot_dim, long long q_stride, long long k_stride, int dtype, bool pdl,
                     cudaStream_t stream);
// RoPE of a chunk's q / k in the fused qkv output with the store of k / v into a KV cache; arguments as
// b200awq_rope_kv_store, validated (rope_kv_store.cu)
int launch_rope_kv_store(void* qkv, const float* freqs, void* k_cache, void* v_cache, int layout, int batch, int seqlen,
                         int heads, int kv_heads, int head_dim, int max_len, int start_pos, const long long* qkv_strides,
                         int dtype, bool pdl, cudaStream_t stream);

// the next token from fp32 logits (temperature, repetition penalty, top-p, top-k, draw); arguments as
// b200awq_sample_next_token, validated (sampling.cu)
int launch_sample_next_token(const float* logits, long long logits_stride, int batch, int vocab, const long long* prev_ids,
                             long long prev_stride, int n_prev, float temperature, float penalty, float top_p, int top_k,
                             int greedy, const float* uniforms, long long* tokens, bool pdl, cudaStream_t stream);

// the LM head's fp32 logits of 1 <= m <= kLmHeadMaxM rows, RMSNorm prologue when gamma is non-null; arguments as
// b200awq_lm_head, validated (lm_head.cu)
constexpr int kLmHeadMaxM = 8;
int launch_lm_head(const void* x, long long x_row_stride, const void* gamma, float eps, const void* weight, float* logits,
                   int m, int vocab, int k, int dtype, bool pdl, cudaStream_t stream);

// forward attention over many queries, D in {64, 72, 128}; arguments as b200awq_prefill_attention (prefill_attention.cu)
int launch_prefill_attention(const void* q, const void* k, const void* v, void* out, const int* cu_q, const int* cu_k, int batch,
                             int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim, const long long* q_strides,
                             const long long* k_strides, const long long* v_strides, float softmax_scale, bool causal, int dtype,
                             cudaStream_t stream);

// attention of few queries over many keys, seqlen_q * (heads / kv_heads) <= 64, D in {64, 128}, split over keys;
// arguments as b200awq_splitkv_attention (splitkv_attention.cu)
size_t splitkv_attention_workspace_bytes(int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim);
int launch_splitkv_attention(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
                             int heads, int kv_heads, int head_dim, const long long* q_strides, const long long* k_strides,
                             const long long* v_strides, float softmax_scale, bool causal, int dtype, void* workspace,
                             size_t workspace_bytes, cudaStream_t stream);
// the same kernel over a KV cache in either of tinychat's layouts, any seqlen_q; arguments as b200awq_kv_cache_attention
size_t kv_cache_attention_workspace_bytes(int layout, int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads,
                                          int head_dim);
int launch_kv_cache_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int layout, int batch,
                              int seqlen_q, int seqlen_k, int max_len, int heads, int kv_heads, int head_dim,
                              const long long* q_strides, float softmax_scale, bool causal, int dtype, void* workspace,
                              size_t workspace_bytes, cudaStream_t stream);

// the same kernel for skinny batches, 1 <= M <= 16, N % 128 == 0: one CTA per tile and k slice (w4a16_wgmma.cu)
int launch_flat(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, cudaStream_t stream, const Epilogue& epi = Epilogue{});

// RMSNorm over the last dimension, one CTA per row (rmsnorm.cu)
int launch_rmsnorm(const void* x, const void* gamma, void* y, float eps, int m, int n, int dtype, bool pdl, cudaStream_t stream);

// W8A8 GEMM, int8 x [M, K] and w [N, K], fp16 y [M, N] with the reference's epilogue; bias may be null
// (w8a8_wgmma.cu).  M >= 1, N % 8 == 0, K % 16 == 0.  With a layer scale [N] or a residual [M, N] (fp16, 16-byte
// aligned, either may be null) the epilogue kernel multiplies the stored values by the layer scale and adds the
// residual (b200awq_w8a8_linear); with both null this launches the plain kernel.
int launch_w8a8_gemm(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias, void* y,
                     int M, int N, int K, bool pdl, cudaStream_t stream, const void* layer_scale = nullptr,
                     const void* residual = nullptr);

// W8A8 row kernels, one CTA per row, rows of at most w8a8_row_limit() elements (w8a8_rowops.cu)
int w8a8_row_limit();
int launch_quant_per_token(const void* x, void* q, void* scales, int m, int n, int dtype, bool pdl, cudaStream_t st);
int launch_layernorm_quant(const void* x, const void* gamma, const void* beta, void* q, void* scale, int m, int n, float eps,
                           bool per_token, int dtype, bool pdl, cudaStream_t st);
int launch_gelu_quant(const void* x, void* q, void* scales, void* tmp, int m, int n, bool pdl, cudaStream_t st);

}  // namespace b200awq
