// Internal launcher interface between the C ABI (api.cu) and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/b200awq.h"

namespace b200awq {

// Opt a kernel into a large dynamic shared-memory size once PER DEVICE (several GPUs may be driven from one process;
// function attributes are per device).  `flags` is a function-local static array of the caller.
template <typename K>
inline cudaError_t ensure_dyn_smem(K kern, int bytes, bool (&flags)[32]) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  dev &= 31;
  if (flags[dev]) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) flags[dev] = true;
  return e;
}

struct StreamTuning {
  int mode = -1;  // -1 = auto (fp16: 2, bf16: 0); 0 operand-exact, 2 group-factored    [env B200AWQ_STREAM_MODE]
  int kc = 0;     // 0 = auto, else input channels per CTA (K / kc in {1,2,4,8})       [env B200AWQ_STREAM_KC]
  int rpb = 0;    // 0 = auto, else 1024-k rounds per prefetch barrier (copy = 2 rpb KB) [env B200AWQ_STREAM_RPB]
  int rbs = 0;    // 0 = auto, else row blocks per CTA (1 or 2)                        [env B200AWQ_STREAM_RBS]
  int warps = 0;  // 0 = auto, else 8 or 16 warps per CTA                              [env B200AWQ_STREAM_WARPS]
  int pad = 0;    // extra dynamic smem bytes per CTA (co-residency limiter, tuning)     [env B200AWQ_STREAM_PAD]
};

struct UmmaTuning {
  int tn = 0;      // 0 = auto, else token tile (16 / 32 / 64 / 128)    [env B200AWQ_UMMA_TN]
  int max_ctas = 0;  // 0 = one per SM                                   [env B200AWQ_UMMA_CTAS]
  int split = 0;     // 0 = auto, 1 = never, 2/4/8 = split k over a cluster [env B200AWQ_UMMA_SPLIT]
};

// Row-parallel tensor parallelism: the GEMV epilogue exchanges fp32 partial sums with the peer GPUs through
// symmetric (peer-mapped) buffers over NVLink and reduces them in the same kernel (w4a16_stream.cu).
struct PeerArgs {
  unsigned long long* data[8];  // data[r]: rank r's exchange buffer ({fp32, epoch} words) as mapped in this process
  unsigned int* epoch;          // this rank's per-row-block epoch counters (device memory, zero-initialised once)
  int rank, world;              // world <= 1: no exchange
  int cap;                      // words per (parity, source) region  (= tok_cap * n_max)
  int tok_cap;                  // tokens a region is laid out for: word slot = channel * tok_cap + token
};

struct FlatTuning {
  int kc = 0;  // 0 = auto, else input channels per CTA (K / kc <= 8)   [env B200AWQ_FLAT_KC]
};

// HBM-bound streaming kernel, 1 <= M <= 16 (w4a16_stream.cu)
int launch_stream(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                  bool pdl, const StreamTuning& tune, cudaStream_t stream, const PeerArgs* peers = nullptr);

// TMA + wgmma tensor-core kernel, any M, N % 128 == 0 (w4a16_wgmma.cu)
int launch_umma(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, const UmmaTuning& tune, cudaStream_t stream);

struct RingTuning {
  int mode = -1;   // -1 = auto (fp16: 2, bf16: 0); 0 or 2                               [env B200AWQ_RING_MODE]
  int split = 0;   // 0 = auto, 1 = no k split, 2 = k split over a 2-CTA cluster      [env B200AWQ_RING_SPLIT]
  int slots = 0;   // 0 = as many ring slots as fit next to a second CTA, else a cap  [env B200AWQ_RING_SLOTS]
};

// persistent warp-specialised decode kernel, 1 <= M <= 8 (w4a16_ring.cu); returns B200AWQ_ERR_SHAPE when the
// activations do not fit next to a useful ring (the caller falls back to the kernels below)
int launch_ring(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, const RingTuning& tune, cudaStream_t stream);

struct DecodeTuning {
  int split = 0;   // 0 = auto, else CTAs per cluster = k split (1, 2, 4, 8)            [env B200AWQ_DECODE_SPLIT]
  int slots = 0;   // 0 = as many ring slots as fit next to a second CTA, else a cap    [env B200AWQ_DECODE_SLOTS]
  int warps = 0;   // consumer warps per CTA: 8, else 16                                  [env B200AWQ_DECODE_WARPS]
};

// one-token decode kernel: 8 KB bulk copies, int8-digit tensor-core MACs (w4a16_decode.cu); returns
// B200AWQ_ERR_SHAPE when the activations do not fit next to a useful ring (the caller falls back)
int launch_decode(const void* x, const void* qw, const void* sc, const void* sz, void* y, int N, int K, int dtype, bool pdl,
                  const DecodeTuning& tune, cudaStream_t stream);

// one-token fused MLP front half: y = silu(x Wgate~^T) * (x Wup~^T), both weight sets through one ring (w4a16_decode.cu)
int launch_decode_mlp_front(const void* x, const void* gqw, const void* gsc, const void* gsz, const void* uqw, const void* usc,
                            const void* usz, void* y, int N, int K, int dtype, bool pdl, const DecodeTuning& tune,
                            cudaStream_t stream);

// out = silu(gate) * up over `count` elements, the reference's roundings (silu_mul.cu)
int launch_silu_mul(const void* gate, const void* up, void* out, size_t count, int dtype, bool pdl, cudaStream_t stream);

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

// the same kernel for skinny batches, 1 <= M <= 64, N % 128 == 0: one CTA per tile and k slice (w4a16_wgmma.cu)
int launch_flat(const void* x, const void* qw, const void* sc, const void* sz, void* y, int M, int N, int K, int dtype,
                bool pdl, const FlatTuning& tune, cudaStream_t stream);

// RMSNorm over the last dimension, one CTA per row (rmsnorm.cu)
int launch_rmsnorm(const void* x, const void* gamma, void* y, float eps, int m, int n, int dtype, bool pdl, cudaStream_t stream);

}  // namespace b200awq
