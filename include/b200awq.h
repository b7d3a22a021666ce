/*
 * b200awq.h — C ABI of the H100-native (sm_90a) W4A16 (AWQ v2 layout) quantized-linear path.
 *
 * This is the drop-in boundary: the two launchers below are what the reference's
 * extension entry points bind to,
 *
 *   gemv_forward_cuda_new(in_feats, kernel, scaling_factors, zeros, m, n, k, group_size)
 *       reference: awq/kernels/csrc/quantization_new/gemv/gemv_cuda.h:4-12,
 *                  host code gemv_cuda.cu:245-338, exported at csrc/pybind.cpp:23
 *   gemm_forward_cuda_new(in_feats, kernel, scales, zeros)
 *       reference: awq/kernels/csrc/quantization_new/gemm/gemm_cuda.h:3,
 *                  host code gemm_cuda.cu:1126-1236, exported at csrc/pybind.cpp:22
 *
 * called from awq/quantize/qmodule.py:207,218 (WQLinear.forward) and
 * tinychat/modules/fused_mlp.py:40,51,65,72.
 *
 * Conventions: plain pointers and sizes, no torch types.  All pointers are DEVICE
 * pointers.  Inputs are borrowed for the duration of the (asynchronous) launch; nothing
 * is retained, nothing is allocated, the calling thread is never synchronised with the
 * device.  Work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = legacy
 * default stream).  Return value: 0 on success, a negative B200AWQ_ERR_* for rejected
 * arguments (nothing was launched), or a positive cudaError_t if the launch failed.
 *
 * Tensor layouts (exactly the reference's WQLinear buffers, awq/quantize/qmodule.py:98-137):
 *   x        [m, k]            fp16 / bf16, row-major, 16-byte aligned
 *   qweight  [n/4, k]          int16, the interleaved 4-bit packing of pack_intweight
 *                              (qmodule.py:26-65), 16-byte aligned
 *   scales   [>= k/group, n]   same dtype as x; rows beyond k/group are padding
 *   szeros   [>= k/group, n]   same dtype as x  (= -scale * zero_point, qmodule.py:194-196)
 *   y        [m, n]            same dtype as x, row-major
 * Semantics: y[i,j] = sum_k x[i,k] * rn_T( q[j,k] * scales[k/group, j] + szeros[k/group, j] )
 * with q the unsigned nibble 0..15, accumulated in fp32, rounded once to T.
 */
#ifndef B200AWQ_H_
#define B200AWQ_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200AWQ_DTYPE_F16 0
#define B200AWQ_DTYPE_BF16 1

#define B200AWQ_OK 0
#define B200AWQ_ERR_SHAPE (-1)     /* n % 8 (gemv) / n % 128 (gemm), k % 128 (w8a8: k % 16), m out of range */
#define B200AWQ_ERR_GROUP (-2)     /* group_size != 128 (reference: gemv_cuda.cu:289,332-335) */
#define B200AWQ_ERR_ALIGN (-3)     /* a pointer is NULL or not 16-byte aligned (w8a8_linear: residual overlaps y) */
#define B200AWQ_ERR_DTYPE (-4)     /* dtype is not F16 / BF16 (reference: dispatch_utils.cuh:7-18) */
#define B200AWQ_ERR_BATCH (-5)     /* gemv with m outside 1..7 (reference: gemv_cuda.cu:291-330) */
#define B200AWQ_ERR_WORKSPACE (-6) /* workspace smaller than b200awq_w4a16_gemm_workspace_bytes */
#define B200AWQ_ERR_DRIVER (-7)    /* CUDA driver entry point for TMA descriptors unavailable */
#define B200AWQ_ERR_DEVICE (-8)    /* current device is not compute capability 9.x */
#define B200AWQ_ERR_PEERS (-9)     /* bad peer description (world, rank, capacities, null buffers) */

/* Decode path: 1 <= m <= 7 (the reference's GEMV envelope).  n % 8 == 0, k % 128 == 0,
 * group_size == 128. */
int b200awq_w4a16_gemv(const void* x, const void* qweight, const void* scales, const void* szeros,
                       void* y, int m, int n, int k, int group_size, int dtype, void* stream);

/* Prefill / batched path: any m >= 1.  n % 128 == 0, k % 128 == 0, group 128 (the
 * reference GEMM hard-codes G = 128, gemm_cuda.cu:1157).  `workspace` may be NULL when
 * b200awq_w4a16_gemm_workspace_bytes(m, n, k) == 0. */
int b200awq_w4a16_gemm(const void* x, const void* qweight, const void* scales, const void* szeros,
                       void* y, int m, int n, int k, int group_size, int dtype,
                       void* workspace, size_t workspace_bytes, void* stream);

size_t b200awq_w4a16_gemm_workspace_bytes(int m, int n, int k);

/* The quantised linear with its bias and residual adds in the same launch:
 *   y[i, j] = rn_T( rn_T( rn_T(acc[i, j]) + bias[j] ) + residual[i, j] )
 * with acc the sum of b200awq_w4a16_gemv / gemm and each + done in fp32 and rounded once to T: bit-identical to those
 * entries followed by PyTorch's `out + bias`, then `residual + out` (WQLinear.forward, awq/quantize/qmodule.py:221,
 * and the decoder blocks' `residual + x`).  Either operand may be NULL; with both NULL this launches exactly what
 * gemv / gemm launch.  bias [n] and residual [m, n] (row-major) are of the activation dtype, 16-byte aligned, and
 * must not overlap y.  The reference's dispatch rule (qmodule.py:206): m < 8 takes the gemv routes (n % 8 == 0),
 * m >= 8 the gemm routes (n % 128 == 0).  bias and residual are read only after the launch's dependency wait, so
 * either may be written by the launch right before it in the stream.  One launch, no workspace, deterministic. */
int b200awq_w4a16_linear(const void* x, const void* qweight, const void* scales, const void* szeros,
                         const void* bias, const void* residual, void* y, int m, int n, int k, int group_size,
                         int dtype, void* stream);

/* Row-parallel tensor parallelism (new work, SURVEY.md §8e; the reference has no multi-GPU path): the decode
 * GEMV of THIS rank's k-slice fused with the sum all-reduce of the [m, n] partial outputs over NVLink peer
 * memory, in one kernel.  Every rank calls it with its own shard and the same (m, n); on return (stream order)
 * y holds the full sum on every rank, bit-identical across ranks.
 *   data[r]   rank r's exchange buffer as mapped in this process (symmetric / peer-mapped allocation):
 *             8-byte words {fp32 partial, epoch}, >= 2 * world * cap_words of them, ZERO before the first call
 *   epoch     this rank's private counters (device memory, uint32, n_max / 8 elements, ZERO before first use)
 *   n_max     widest layer (out_features) the buffers are sized for, a multiple of 8
 *   cap_words words per (parity, source rank) region = tok_cap * n_max for some tok_cap >= m; a word's slot is
 *             channel * tok_cap + token and its epoch counter is the channel's row block, so layers of
 *             DIFFERENT n (<= n_max) may share one set of buffers.
 *   1 <= m <= 8, world <= 8.  n > n_max or m > cap_words / n_max is rejected with B200AWQ_ERR_PEERS.  All ranks
 *   must issue the same sequence of calls on these buffers.  Safe under CUDA-graph capture / replay (no
 *   host-side state).  A rank whose peer delivers nothing for 10 s gives up: its outputs of that call are NaN and
 *   every later exchange of the process returns NaN at once (the kernel never spins for ever). */
typedef struct b200awq_peers {
  void* data[8];
  void* epoch;
  int rank, world;
  int cap_words;
  int n_max;
} b200awq_peers;

int b200awq_w4a16_gemv_allreduce(const void* x, const void* qweight, const void* scales, const void* szeros,
                                 void* y, int m, int n, int k, int group_size, int dtype,
                                 const b200awq_peers* peers, void* stream);

/* Front half of the gated MLP (SURVEY.md §8f-1): y = silu(x Wgate~^T) * (x Wup~^T), i.e. what
 * QuantLlamaMLP.our_llama_mlp computes with two engine calls, F.silu and a multiply
 *   reference: tinychat/modules/fused_mlp.py:36-83 (both branches use the zeros tensor they are GIVEN; the GEMM
 *   branch's `scaled_zeros - 8 * scales` is the caller's business).
 * Same tensor layouts as b200awq_w4a16_gemv / gemm for each weight set; y is [m, n].  Roundings are the reference's:
 * gate and up products rounded to T, silu (fp32) rounded to T, product rounded to T.
 *   m == 1, fp16: ONE kernel -- x read once, the two weight streams share one shared-memory ring, one [1, n] write
 *                 (no workspace needed).
 *   otherwise:    the two products through the GEMV / GEMM path into `workspace` (>= b200awq_w4a16_mlp_front_workspace_bytes
 *                 = 2 * m * n * 2 bytes, 16-byte aligned), then one elementwise kernel.  n % 128 == 0 for m >= 8. */
int b200awq_w4a16_mlp_front(const void* x, const void* gate_qweight, const void* gate_scales, const void* gate_szeros,
                            const void* up_qweight, const void* up_scales, const void* up_szeros, void* y, int m, int n, int k,
                            int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream);
size_t b200awq_w4a16_mlp_front_workspace_bytes(int m, int n, int k);

/* RMSNorm prologues of the decoder's norm -> linear launches (DESIGN §3.5c): the attention block's
 * `input_layernorm -> qkv_proj` and the MLP's `post_attention_layernorm -> gate/up`.  With x^ = the output of
 * b200awq_rmsnorm(x, gamma, eps) (fp16 clamp included), bit for bit:
 *   b200awq_w4a16_norm_linear(x, gamma, eps, W, bias)     == b200awq_w4a16_linear(x^, W, bias, residual = NULL)
 *   b200awq_w4a16_norm_mlp_front(x, gamma, eps, Wg, Wu)  == b200awq_w4a16_mlp_front(x^, Wg, Wu)
 * for every m, dtype and shape the plain entries take.  One fp16 token (and the ring kernel's m = 2..4 / bf16 m = 1 for
 * norm_linear) computes the row statistic and x^ inside the W4A16 launch: one kernel, the plain launch's plan.  Every
 * other shape writes x^ into the workspace with b200awq_rmsnorm and runs the plain route on it.
 *   gamma     [k] of the activation dtype, 16-byte aligned (else B200AWQ_ERR_ALIGN); a model constant: it is read
 *             before the dependency wait, so it must not be written by the launch right before
 *   eps       finite and >= 0 (else B200AWQ_ERR_SHAPE)
 *   workspace 16-byte aligned, required on every call, also when the one-kernel route needs none (else
 *             B200AWQ_ERR_WORKSPACE): norm_linear needs m * k * 2 bytes (8 KB for one token at k = 4096), norm_mlp_front
 *             b200awq_w4a16_norm_workspace_bytes(m, n, k) = m * k * 2 + 2 * m * n * 2, which also serves norm_linear.
 *             It must not overlap x, y or the weights.
 * Otherwise the return codes of b200awq_w4a16_linear / b200awq_w4a16_mlp_front.  No residual operand. */
int b200awq_w4a16_norm_linear(const void* x, const void* gamma, float eps, const void* qweight, const void* scales,
                              const void* szeros, const void* bias, void* y, int m, int n, int k, int group_size, int dtype,
                              void* workspace, size_t workspace_bytes, void* stream);
int b200awq_w4a16_norm_mlp_front(const void* x, const void* gamma, float eps, const void* gate_qweight,
                                 const void* gate_scales, const void* gate_szeros, const void* up_qweight,
                                 const void* up_scales, const void* up_szeros, void* y, int m, int n, int k, int group_size,
                                 int dtype, void* workspace, size_t workspace_bytes, void* stream);
size_t b200awq_w4a16_norm_workspace_bytes(int m, int n, int k);

/* RMSNorm of the decoder layers around the quantised linears (SURVEY.md §8f-2): y[i, :] = x[i, :] *
 * rsqrt(mean(x[i, :]^2) + eps) * gamma, statistics in fp32, one rounding to the element type (fp16 results are
 * clamped to +-(65504 - 1000) like the reference).  Replaces layernorm_forward_cuda(input, gamma, out, eps)
 *   reference: awq/kernels/csrc/layernorm/layernorm.cu:38-64 (kernel), :111-131 (host), csrc/pybind.cpp:17.
 * x, y: [m, n] row-major, gamma: [n]; any n >= 1 (16-byte aligned pointers and n % 8 == 0 take the one-pass
 * kernel).  m == 0 is a no-op. */
int b200awq_rmsnorm(const void* x, const void* gamma, void* y, int m, int n, float eps, int dtype, void* stream);

/* Decode-step attention over tinychat's KV-cache layout (SURVEY.md §8f-3).  Replaces
 *   single_query_attention(q, k, v, k_cache, v_cache, length_per_sample, alibi_slopes, timestep, rotary_embedding_dim,
 *                          rotary_base, rotary_scale, neox_rotary_style)
 *   reference: awq/kernels/csrc/attention/ft_attention.cpp:112-184, exported at csrc/pybind.cpp:24-27, called from
 *              tinychat/modules/fused_attn.py:308-321.
 * q [batch, heads, head_dim], k / v [batch, kv_heads, head_dim] with their own batch strides in ELEMENTS (they are
 * usually views into the fused QKV output; the reference applies q's stride to all three, template.hpp:967-969), head
 * stride head_dim, unit element stride; k_cache [batch, kv_heads, head_dim / 8,
 * max_len, 8], v_cache [batch, kv_heads, max_len, head_dim], out [batch, heads, head_dim] contiguous.  The current
 * step's q and k are rotated at position t = length_per_sample ? length_per_sample[b] : timestep (angle t * scale /
 * base^(2i / rotary_dim); neox != 0 pairs (i, i + rotary_dim / 2), else (2i, 2i + 1)) and rounded to the element type;
 * k and v are stored at cache slot t % max_len; out = softmax(q K^T / sqrt(head_dim)) V over the last min(t + 1,
 * max_len) positions.  heads % kv_heads == 0 (any ratio; query head h reads KV head h / (heads / kv_heads)),
 * head_dim % 8 == 0 and head_dim <= 256.
 * `workspace`: >= b200awq_single_query_attention_workspace_bytes(...) bytes of device memory, ZERO before the first
 * use, then owned by the kernels (they leave it zero where it matters); one workspace per stream.  ALiBi is not
 * supported (the reference's alibi_slopes argument must be None). */
int b200awq_single_query_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, void* out,
                                   const int* length_per_sample, int batch, int heads, int kv_heads, int head_dim,
                                   int max_len, int timestep, long long q_batch_stride, long long k_batch_stride,
                                   long long v_batch_stride, int rotary_dim, float rotary_base,
                                   float rotary_scale, int neox, int dtype, void* workspace, size_t workspace_bytes,
                                   void* stream);
size_t b200awq_single_query_attention_workspace_bytes(int batch, int heads, int kv_heads, int head_dim, int max_len);

/* RoPE with explicit angles over a strided [s, b, h, d] tensor (prefill).  Replaces
 *   fused_rope_with_pos_forward_func(input, freqs, transpose_output_memory)
 *   reference: awq/kernels/csrc/rope_new/fused_rope_with_pos.cu:33-75,243-285, csrc/pybind.cpp:28, called from
 *              tinychat/modules/fused_attn.py:253-254.
 * y[s, b, h, i] = x[i] cos(f_i) + rot(x)[i] sin(f_i) for i < d2 with f_i = freqs[(b * S + s) * d2 + i] (fp32) and
 * rot(x)[i] = -x[i + d2 / 2] for i < d2 / 2, x[i - d2 / 2] otherwise; elements i >= d2 are copied.  Strides in ELEMENTS
 * for s, b, h, d of the input and of the output. */
int b200awq_rope_with_pos(const void* x, const float* freqs, void* y, int s, int b, int h, int d, int d2,
                          const long long in_strides[4], const long long out_strides[4], int dtype, void* stream);

/* In-place NeoX-style RoPE on query and key from a table of cosines and sines (the HF-attention branch).  Replaces
 *   rotary_embedding_neox(positions, query, key, head_size, cos_sin_cache)
 *   reference: awq/kernels/csrc/position_embedding/pos_encoding_kernels.cu:13-88, csrc/pybind.cpp:24, called from
 *              tinychat/modules/fused_attn.py:61-79 (QuantLlamaRotaryEmbedding, table built at :43-59).
 * For every token t and head: with p = positions[t] (int64) and row = cos_sin_cache[p] ([rot_dim] of T: rot_dim / 2
 * cosines, then rot_dim / 2 sines), the pairs (x, y) = (head[r], head[rot_dim / 2 + r]), r < rot_dim / 2, become
 * (x cos_r - y sin_r, y cos_r + x sin_r); elements beyond rot_dim are untouched.  Products in fp32, one rounding to T
 * (the reference multiplies and adds in T: <= 2 ulp apart).  query [tokens, q_heads, head_size] and key
 * [tokens, k_heads, head_size] with token strides in ELEMENTS; the reference rotates key with query's head count
 * (pos_encoding_kernels.cu:61,64 -- equal for the models that take this branch), here each tensor has its own;
 * key may be NULL with k_heads == 0.  positions are not range-checked (as in the reference). */
int b200awq_rotary_embedding_neox(const long long* positions, void* query, void* key, const void* cos_sin_cache, int tokens,
                                  int q_heads, int k_heads, int head_size, int rot_dim, long long q_token_stride,
                                  long long k_token_stride, int dtype, void* stream);

/* Forward attention over many queries (prefill, vision towers).  Replaces flash-attn 2's flash_attn_func and
 * flash_attn_varlen_qkvpacked_func (called from tinychat/modules/fused_attn.py, models/llama.py, models/qwen2.py,
 * modules/fused_siglipdecoder.py and models/internvl/internvit.py) for the parameters those callers pass:
 *   out = softmax(softmax_scale * q k^T + mask) v per (sequence, query head); query head h reads KV head
 *   h / (heads / kv_heads).  causal != 0 aligns the mask bottom-right: query i sees keys j <= i + Sk - Sq; a row that
 *   sees no key is zero.  S in fp32 from T operands, softmax in fp32, P rounded to T, O in fp32 rounded once to T.
 * q [.., Sq, H, D], k / v [.., Sk, Hkv, D]: strides in ELEMENTS for (batch, token, head), unit element stride;
 * out [batch * Sq or total_q, H, D] contiguous.  cu_seqlens_q / cu_seqlens_k: NULL for fixed lengths, else batch + 1
 * int32 offsets into the token dimension in DEVICE memory, read by the kernel only (batch strides ignored; seqlen_q /
 * seqlen_k are then the maxima).  head_dim in {64, 72, 128}, heads % kv_heads == 0 and a finite softmax_scale > 0
 * (else B200AWQ_ERR_SHAPE);
 * q, k, v, out 16-byte aligned and strides multiples of 8 elements (else B200AWQ_ERR_ALIGN).  seqlen_q == 0 or
 * batch == 0 is a no-op.  Deterministic: no split over keys, no atomics, no workspace. */
int b200awq_prefill_attention(const void* q, const void* k, const void* v, void* out,
                              const int* cu_seqlens_q, const int* cu_seqlens_k,
                              int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim,
                              const long long q_strides[3], const long long k_strides[3], const long long v_strides[3],
                              float softmax_scale, int causal, int dtype, void* stream);

/* Attention of few queries over many keys (long-context decode, few-token chunks): flash_attn_func's fixed-length
 * call as tinychat's long_forward makes it (tinychat/modules/fused_attn.py, q [B, 1, H, D] over views
 * cache[:, :start_pos + 1] of [B, Lmax, Hkv, D] caches), with the key range split over CTAs.  Same semantics, layouts,
 * strides, alignment rules and return codes as b200awq_prefill_attention for fixed lengths (no cu_seqlens), within a
 * narrower envelope: head_dim in {64, 128} and seqlen_q * (heads / kv_heads) <= 64 (else B200AWQ_ERR_SHAPE; callers
 * fall through to b200awq_prefill_attention).  k / v are read only for tokens < seqlen_k, whatever lies past them.
 * `workspace`: >= b200awq_splitkv_attention_workspace_bytes(...) bytes of 16-byte aligned device memory (else
 * B200AWQ_ERR_WORKSPACE), ZERO before the first use, then owned by the kernel, which leaves its counters zero; one
 * workspace per stream.  The workspace of b200awq_single_query_attention on the same stream may serve both (their
 * counters share one block at offset 0).  A size of 0 means no workspace is needed (NULL is fine): the shape always
 * runs as one split (one 128-key tile, or batch * kv_heads > 4096, more cells than the counter block holds).  A CUDA
 * graph that captured a call keeps using the workspace it captured: it must stay allocated, and zero in its counter
 * block, for as long as the graph is replayed (the launches leave it so).  Deterministic: the splits are combined in a fixed order, no atomics in the arithmetic. */
int b200awq_splitkv_attention(const void* q, const void* k, const void* v, void* out,
                              int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim,
                              const long long q_strides[3], const long long k_strides[3], const long long v_strides[3],
                              float softmax_scale, int causal, int dtype, void* workspace, size_t workspace_bytes,
                              void* stream);
size_t b200awq_splitkv_attention_workspace_bytes(int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads,
                                                 int head_dim);

/* Attention of a chunk of queries over a KV cache, read in place (tinychat's chunked prefill and multi-round chat:
 * the chunk's k / v are already stored in the cache, the history is not copied out of it).  For the caller's
 * `flash_attn_func(q, cache_k[:B, :seqlen_k], cache_v[:B, :seqlen_k], causal)` in either cache layout:
 *   B200AWQ_KV_FT    k_cache [>= batch, kv_heads, head_dim / 8, max_len, 8], v_cache [>= batch, kv_heads, max_len,
 *                    head_dim] (the decode caches of b200awq_single_query_attention)
 *   B200AWQ_KV_BTHD  k_cache, v_cache [>= batch, max_len, kv_heads, head_dim] (long_forward's caches)
 * both contiguous.  Semantics as b200awq_splitkv_attention over keys [0, seqlen_k) of cache rows [0, batch): q
 * [batch, seqlen_q, heads, head_dim] with strides q_strides (batch, token, head) in ELEMENTS, out [batch, seqlen_q,
 * heads, head_dim] contiguous; causal != 0 aligns the mask bottom-right (query i sees keys j <= i + seqlen_k -
 * seqlen_q; a row that sees no key is zero).  Cache slots >= seqlen_k and cache rows >= batch are never read.
 * Any seqlen_q >= 1; head_dim in {64, 128}, heads % kv_heads == 0, 1 <= max_len, seqlen_k <= max_len and a finite
 * softmax_scale > 0 (else B200AWQ_ERR_SHAPE).  q, caches and out 16-byte aligned, q_strides multiples of 8
 * (else B200AWQ_ERR_ALIGN).  batch == 0 or seqlen_q == 0 is a no-op.
 * `workspace`: as for b200awq_splitkv_attention, >= b200awq_kv_cache_attention_workspace_bytes(...) bytes (0: the
 * shape never splits the keys, NULL is fine), and the same per-stream buffer may serve all three attention entries.
 * One kernel launch per call (the splits are combined inside it); deterministic; safe under graph capture. */
#define B200AWQ_KV_FT 0
#define B200AWQ_KV_BTHD 1
int b200awq_kv_cache_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int layout,
                               int batch, int seqlen_q, int seqlen_k, int max_len, int heads, int kv_heads,
                               int head_dim, const long long q_strides[3], float softmax_scale, int causal, int dtype,
                               void* workspace, size_t workspace_bytes, void* stream);
size_t b200awq_kv_cache_attention_workspace_bytes(int layout, int batch, int seqlen_q, int seqlen_k, int heads,
                                                  int kv_heads, int head_dim);

/* RoPE of a chunk's q and k with the store of k and v into a KV cache, in one launch: for tinychat's chunked prefill
 * and long_forward's decode, what the caller's two fused_rope_with_pos_forward_func calls (the second on k) and its
 * k / v cache stores compute.
 *   qkv      the fused qkv linear's output as [batch, seqlen, heads + 2 kv_heads, head_dim]: heads 0 .. heads - 1 are
 *            q, the next kv_heads are k, the last kv_heads are v; strides in ELEMENTS for (batch, token, head), unit
 *            element stride
 *   freqs    fp32 [seqlen, head_dim]: angle f_i of token s is freqs[s * head_dim + i], the same for every batch row
 *   k_cache, v_cache  in `layout` (B200AWQ_KV_FT or B200AWQ_KV_BTHD), as b200awq_kv_cache_attention reads them
 * Every q and k head becomes y[i] = x[i] cos f_i + rot(x)[i] sin f_i in fp32, rounded once to T, with rot as in
 * b200awq_rope_with_pos (d2 = head_dim): bit-identical to b200awq_rope_with_pos.  Rotated q is written back into the q
 * heads of qkv; rotated k and the v heads are stored into cache slots [start_pos, start_pos + seqlen) of cache rows
 * [0, batch).  The k and v heads of qkv, every other cache slot and every cache row >= batch are left as they were.
 * heads % kv_heads == 0, head_dim % 8 == 0 and <= 256, max_len >= 1, start_pos >= 0 and start_pos + seqlen <= max_len
 * (the ring of the decode cache does not wrap here), layout one of the two (else B200AWQ_ERR_SHAPE); qkv, freqs and
 * the caches 16-byte aligned and qkv_strides multiples of 8 (else B200AWQ_ERR_ALIGN).  batch == 0 or seqlen == 0 is a
 * no-op.  One launch, no workspace, no atomics; qkv and freqs are read after the launch's dependency wait, so either
 * may be written by the launch right before it in the stream. */
int b200awq_rope_kv_store(void* qkv, const float* freqs, void* k_cache, void* v_cache, int layout, int batch, int seqlen,
                          int heads, int kv_heads, int head_dim, int max_len, int start_pos,
                          const long long qkv_strides[3], int dtype, void* stream);

/* The choice of the next token from fp32 logits, in one launch: what tinychat's per-token block computes
 * (tinychat/stream_generators/stream_gen.py: TemperatureLogitsWarper, RepetitionPenaltyLogitsProcessor,
 * TopPLogitsWarper, TopKLogitsWarper, then argmax or softmax + torch.multinomial).  For each row b < batch, with x the
 * row's vocab logits (logits + b * logits_row_stride; rows may alias, e.g. a stride of 0):
 *   1. temperature != 1: x = x / temperature (an fp32 division);
 *   2. repetition_penalty > 1: every DISTINCT id of prev_ids[b * prev_row_stride + i], i < n_prev, that lies in
 *      [0, vocab) becomes x < 0 ? x * penalty : x / penalty (ids outside are ignored);
 *   3. 0 < top_p < 1: in ascending order of (x, index) -- a stable sort -- tokens whose inclusive cumulative softmax
 *      probability is <= fp32(1 - top_p) are removed; the last token in that order is always kept;
 *   4. 0 < top_k < vocab: tokens below the top_k-th largest value left after 3 are removed (ties at it are kept);
 *   5. greedy != 0: the token is the smallest index among the maxima of the kept tokens (uniforms may be NULL);
 *      otherwise, with u = uniforms[b] in [0, 1) and p_i = exp(x_i - max) over the kept tokens, the smallest index i
 *      whose cumulative kept mass through i (in index order) exceeds u * sum p -- the inverse CDF;
 *   6. tokens[b] = that index (int64).
 * Probabilities are fp32 exp(x - max) in 2^-44 fixed point, summed exactly: the top-p rule may decide differently from
 * float64 arithmetic only for tokens whose cumulative probability lies within 1e-5 of 1 - top_p (DESIGN §3.12).  NaN
 * logits count as -inf; -inf entries of a row with a finite maximum are never drawn; every row, even an all -inf or NaN
 * one, gets an id in [0, vocab).
 * B200AWQ_ERR_SHAPE: batch < 0, vocab < 1 or > B200AWQ_SAMPLE_MAX_VOCAB, n_prev < 0, temperature not finite or <= 0,
 * repetition_penalty not finite or < 1, top_p outside (0, 1] (1 = off), top_k < 0 (0 = off).  B200AWQ_ERR_ALIGN: logits
 * or tokens NULL or misaligned, uniforms when !greedy, prev_ids when n_prev > 0 and repetition_penalty > 1 (4-, 8-, 4-
 * and 8-byte alignment).  batch == 0 is a no-op.  One launch, no workspace, no global atomics, deterministic, safe under
 * graph capture; logits, prev_ids and uniforms are read after the launch's dependency wait. */
#define B200AWQ_SAMPLE_MAX_VOCAB 262144
int b200awq_sample_next_token(const float* logits, long long logits_row_stride, int batch, int vocab,
                              const long long* prev_ids, long long prev_row_stride, int n_prev, float temperature,
                              float repetition_penalty, float top_p, int top_k, int greedy, const float* uniforms,
                              long long* tokens, void* stream);

/* The LM head: the decoder's final RMSNorm and the vocabulary projection in one launch, fp32 logits for
 * b200awq_sample_next_token (tinychat/models/llama.py:353-354, 395, 412-413: `norm(h[:, -1:, :])`, `lm_head(h)`,
 * `.float()`; DESIGN §3.13).  For i < m, v < vocab:
 *   logits[i * vocab + v] = (float) rn_T( sum_j x^[i, j] * weight[v * k + j] )
 * where x^ = x, or with gamma non-NULL exactly what b200awq_rmsnorm(x, gamma, eps) writes (fp16 clamp included); the
 * sum is accumulated in fp32 in an order that depends on k alone (not on vocab, v, m, the other rows or the device),
 * rounded once to T (fp16 overflow gives +-inf) and widened exactly.
 *   x         [m, k] of T, row i at x + i * x_row_stride elements; x_row_stride >= k (else B200AWQ_ERR_SHAPE) and a
 *             multiple of 8 (else B200AWQ_ERR_ALIGN), so that h[:, -1, :] of a [B, S, k] hidden state is read in place
 *   gamma     [k] of T or NULL (no norm); eps finite and >= 0 when gamma is given (else B200AWQ_ERR_SHAPE)
 *   weight    [vocab, k] of T, contiguous (an untied lm_head or a tied embedding)
 *   logits    [m, vocab] fp32, contiguous; must not overlap x, gamma or weight (else B200AWQ_ERR_ALIGN)
 * 1 <= m <= 8 (else B200AWQ_ERR_BATCH); vocab >= 1, 8 <= k <= 8192, k % 8 == 0 (else B200AWQ_ERR_SHAPE); x, gamma,
 * weight and logits 16-byte aligned (else B200AWQ_ERR_ALIGN).  One launch, no workspace, no atomics, deterministic,
 * safe under graph capture; x and gamma are read after the launch's dependency wait (the previous launch may write
 * them), weight is a model constant streamed from before it, so the launch right before must not write it. */
int b200awq_lm_head(const void* x, long long x_row_stride, const void* gamma, float eps, const void* weight, float* logits,
                    int m, int vocab, int k, int dtype, void* stream);

/* ---- W8A8 (int8 weights, int8 per-token activations): the vision-tower ops of the reference's extension
 * (csrc/pybind.cpp:30-37), called by awq/quantize/w8a8_linear.py and tinychat's QuantSiglipEncoder /
 * QuantInternVisionEncoder.  Scales are fp16 everywhere (the reference reads them as at::Half).  fp32 activations,
 * which the reference also dispatches, are rejected with B200AWQ_ERR_DTYPE.  The row ops take rows of at most
 * 32768 elements, 8192 when n % 8 != 0 or a row pointer is not 16-byte aligned (B200AWQ_ERR_SHAPE beyond); m == 0
 * is a no-op. */

/* y[i, j] = rn_f16(f32(acc) * (wscales[j] * ascales[i]))                    bias == NULL
 *         = rn_f16(fma(ascales[i], f32(acc) * wscales[j], bias[j]))         otherwise
 * with acc = sum_k x[i, k] w[j, k] exact in int32, every fp32 product flushing denormals.  Replaces
 *   w8a8_gemm_forward_cuda(in_feats, kernel, wscales, ascales, out_feats)             w8a8/w8a8_gemm_cuda.cu:907-953
 *   w8a8_gemm_fuse_bias_forward_cuda(in_feats, kernel, wscales, ascales, out, bias)   w8a8/w8a8_gemm_cuda.cu:586-633
 * x [m, k] int8, w [n, k] int8 (the plain [OC, IC] matrix of W8A8OF16LinearDynamicInputScale, not repacked), both
 * row-major and 16-byte aligned; wscales [n], ascales [m], bias [n] fp16; y [m, n] fp16, 16-byte aligned.
 * m >= 1, n % 8 == 0, k % 16 == 0 (any k tail is exact). */
int b200awq_w8a8_gemm(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias, void* y,
                      int m, int n, int k, void* stream);

/* The W8A8 linear with the vision towers' layer scale and residual in the same launch:
 *   v = the b200awq_w8a8_gemm formula above (with or without bias), unchanged
 *   y0 = rn_f16(v)
 *   y1 = layer_scale ? rn_f16(f32(y0) * f32(layer_scale[j])) : y0
 *   y[i, j] = residual ? rn_f16(f32(residual[i, j]) + f32(y1)) : y1
 * each operation in fp32 and rounded once: bit-identical to b200awq_w8a8_gemm followed by PyTorch's fp16 `out * ls`
 * and then `residual + out` (tinychat's QuantInternVisionEncoderLayer: `residual + out * self.ls1`;
 * QuantSiglipEncoderLayer: `residual + out`).  The arguments and their checks are b200awq_w8a8_gemm's; layer_scale
 * [n] and residual [m, n] (row-major) are fp16 and 16-byte aligned, and any of bias, layer_scale and residual may be
 * NULL.  With layer_scale and residual both NULL this launches exactly what b200awq_w8a8_gemm launches.  residual
 * must not overlap y (B200AWQ_ERR_ALIGN): the residual stream is written out of place, since the encoders keep every
 * layer's input.  layer_scale and residual are read only after the launch's dependency wait, so either may be written
 * by the launch right before it in the stream.  Every argument error returns before the device is touched.  One
 * launch, no workspace, deterministic. */
int b200awq_w8a8_linear(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias,
                        const void* layer_scale, const void* residual, void* y, int m, int n, int k, void* stream);

/* Per-token int8 quantisation: scales[i] = rn_f16(amax_i / 127), q[i, j] = cvt.rni.sat(x[i, j] * (127 / amax_i)),
 * amax_i = max_j |x[i, j]| (a zero row gives codes 0 and scale 0).  Replaces invoke_quant(out, input, scale),
 * w8a8/quantization.cu:54-112.  x [m, n] of dtype, q [m, n] int8, scales [m] fp16. */
int b200awq_quant_per_token(const void* x, void* q, void* scales, int m, int n, int dtype, void* stream);

/* LayerNorm + int8 quantisation.  Replaces rms_norm_general(out, input, weight, bias, scaling, epsilon,
 * use_per_token_quant), w8a8/layernorm.cu:55-231 -- a LayerNorm (mean, E[x^2] - E[x]^2, rsqrt) despite the name.
 *   per_token != 0: y = (x - mean) rstd gamma + beta (beta may be NULL); amax over rn_T(y) starting from 1e-6;
 *                   q = cvt.rni.sat(y * (127 / amax)) from the unrounded y; scale[i] = rn_f16(amax / 127)  [m]
 *   per_token == 0: the reference's per-tensor branch: beta is IGNORED and q = cvt.rni.sat(rn_T(y) * scale[0])
 *                   (scale[0] multiplies); scale is read, not written.
 * x [m, n], gamma / beta [n] of dtype, q [m, n] int8. */
int b200awq_layernorm_quant(const void* x, const void* gamma, const void* beta, void* q, void* scale, int m, int n,
                            float eps, int per_token, int dtype, void* stream);

/* GELU (tanh form, the reference's fp16 operation chain around tanh.approx) + per-token int8 quantisation, fp16 only
 * like the reference.  tmp[i, j] = gelu(x[i, j]); amax_i over |tmp| except values in (0, 1e-4], which enter negated;
 * scales[i] = rn_f16(amax_i / 127); q = cvt.rni.sat(f32(rn_f16(rn_f16(127 / amax_i) * tmp))).  Replaces
 * gelu_and_quant(out, input, scale_out, tmp), w8a8/act.cu:22-96.  x, tmp [m, n] fp16, q [m, n] int8, scales [m]. */
int b200awq_gelu_quant(const void* x, void* q, void* scales, void* tmp, int m, int n, void* stream);

/* y[i, j] = rn_T(rn_T(silu(x[i, j])) * x[i, d + j]) for x [m, 2d], y [m, d] of dtype.  Replaces
 * silu_and_mul(input), w8a8/act.cu:107-140 (same kernel as the MLP front half's tail, with a row pitch). */
int b200awq_silu_and_mul(const void* x, void* y, int m, int d, int dtype, void* stream);

/* Names used by BASELINE.json's north_star; identical to the two launchers above. */
int gemv_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros,
                      void* y, int m, int n, int k, int group_size, int dtype, void* stream);
int gemm_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros,
                      void* y, int m, int n, int k, int group_size, int dtype,
                      void* workspace, size_t workspace_bytes, void* stream);

/* Programmatic dependent launch between consecutive launches of this library on one
 * stream (weights of launch i+1 are prefetched while launch i drains).  Default on;
 * b200awq_set_pdl(0) turns it off.  Returns the previous setting. */
int b200awq_set_pdl(int enable);

/* Test-only override of the one-token decode kernel's plan, for tests that must run that kernel with a k split or a
 * ring depth the shape alone would not pick:
 *   B200AWQ_DECODE_SPLIT  CTAs per cluster = k split (1 to 8) instead of the choice from the shape
 *   B200AWQ_DECODE_SLOTS  cap on the ring slots; below 3 the kernel declines and the next kernel takes the call
 * Unset or 0 means "pick from the shape".  Every other kernel configuration is fixed in code.  The library reads the
 * two variables once, at the first one-token launch; this reads them again (thread-safe). */
void b200awq_reload_config(void);

/* Number of kernels this library has launched since load (monotonic, per process). */
unsigned long long b200awq_launch_count(void);

/* Human-readable text for a return value of the functions above. */
const char* b200awq_strerror(int code);

/* "b200awq <version> sm_90a" */
const char* b200awq_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200AWQ_H_ */
