// C ABI of libb200awq.so (declared in include/b200awq.h): argument validation, dispatch
// between the HBM-bound streaming kernels and the wgmma tensor-core kernel, the PDL switch.
// No torch types, no allocation, no synchronisation.
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <initializer_list>

#include "w4a16_kernels.h"

namespace {

std::atomic<unsigned long long> g_launches{0};

// Test-only override of the decode kernel's plan (B200AWQ_DECODE_SPLIT, B200AWQ_DECODE_SLOTS; include/b200awq.h), read
// once on the first one-token launch and again by b200awq_reload_config().  Double-buffered so that a reload never
// races a reader: readers take a pointer with acquire, writers publish a fully built copy.
b200awq::DecodeTuning read_decode_tuning() {
  auto env_int = [](const char* name) {
    const char* v = std::getenv(name);
    return v && *v ? std::atoi(v) : 0;
  };
  b200awq::DecodeTuning t;
  t.split = env_int("B200AWQ_DECODE_SPLIT");
  t.slots = env_int("B200AWQ_DECODE_SLOTS");
  return t;
}

b200awq::DecodeTuning g_decode_store[2];
std::atomic<const b200awq::DecodeTuning*> g_decode{nullptr};

const b200awq::DecodeTuning& decode_tuning() {
  const b200awq::DecodeTuning* t = g_decode.load(std::memory_order_acquire);
  if (!t) {
    static const b200awq::DecodeTuning first = read_decode_tuning();  // thread-safe one-time initialisation
    g_decode.store(&first, std::memory_order_release);
    t = &first;
  }
  return *t;
}

std::atomic<bool> g_pdl{true};  // programmatic dependent launch, b200awq_set_pdl()

bool pdl_enabled() { return g_pdl.load(std::memory_order_relaxed); }

using b200awq::aligned16;

// `r` passed through; a successful entry that launched a kernel counts one launch (b200awq_launch_count)
int counted(int r, bool launched = true) {
  if (r == 0 && launched) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

// A positive result is the cudaError_t of a launch that could not be configured (e.g. an unschedulable cluster shape):
// not the caller's problem.  The error is cleared and the result becomes B200AWQ_ERR_SHAPE, so that the next kernel
// in line gets the shape.
int next_on_config_error(int r) {
  if (r <= 0) return r;
  (void)cudaGetLastError();
  return B200AWQ_ERR_SHAPE;
}

int check_dtype(int dtype) { return dtype == B200AWQ_DTYPE_F16 || dtype == B200AWQ_DTYPE_BF16 ? 0 : B200AWQ_ERR_DTYPE; }

int check_device() {
  static std::atomic<signed char> ok[32];  // per device: 0 unknown, 1 ok, -1 wrong device
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200AWQ_ERR_DEVICE;
  dev &= 31;
  signed char v = ok[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    v = (major == 9) ? 1 : -1;
    ok[dev].store(v, std::memory_order_relaxed);
  }
  return v == 1 ? 0 : B200AWQ_ERR_DEVICE;
}

// the W4A16 entries' argument checks that need no device
int check_args(const void* x, const void* qw, const void* sc, const void* sz, void* y, int m, int n, int k, int group_size,
               int dtype) {
  if (int e = check_dtype(dtype)) return e;
  if (group_size != 128) return B200AWQ_ERR_GROUP;
  if (m < 1 || n < 8 || k < 128 || (n % 8) || (k % 128)) return B200AWQ_ERR_SHAPE;
  if (!aligned16(x) || !aligned16(qw) || !aligned16(sc) || !aligned16(sz) || !aligned16(y)) return B200AWQ_ERR_ALIGN;
  return 0;
}

int check_common(const void* x, const void* qw, const void* sc, const void* sz, void* y, int m, int n, int k,
                 int group_size, int dtype) {
  if (int e = check_args(x, qw, sc, sz, y, m, n, k, group_size, dtype)) return e;
  return check_device();
}

// Routing of small token counts.  The one-token decode kernel takes fp16 only: bf16 stays operand-exact in the ring
// kernel (dropping the bf16 rounding of q s + z would move results by ~1e-3 against the reference).
constexpr int kRingMaxM = 4;         // largest token count served by the ring kernel
constexpr int kFlatMinM = 5;         // the wgmma skinny launch from 5 tokens ...
constexpr int kFlatMinMLongK = 3;    // ... from 3 when k is long enough to need a cluster split (k > 8192) ...
constexpr int kFlatMaxM = 16;        // ... up to 16; the wgmma tile launch above
constexpr int kStreamMaxM = 16;      // largest token count served by the streaming kernel

bool use_decode(int m, int dtype) { return m == 1 && dtype == B200AWQ_DTYPE_F16; }

// which kernel serves small token counts beyond the ring kernel's range
bool use_flat(int m, int n, int k) {
  const int min_m = k > 8192 ? kFlatMinMLongK : kFlatMinM;
  return n % 128 == 0 && m >= min_m && m <= kFlatMaxM;
}

// One W4A16 product y = x W~^T (+ epilogue), or x^ W~^T with x^ = RMSNorm(x) (+ epilogue), as validated by the entry.
struct W4Operands {
  const void *x, *qw, *sc, *sz;
  void* y;
  int m, n, k, dtype;
  cudaStream_t st;
  b200awq::Epilogue epi;
  b200awq::NormPrologue norm;  // b200awq_w4a16_norm_linear; gamma null: none
  void* xhat = nullptr;        // with a prologue: [m, k] of workspace for x^ on the routes without one
};

// The kernels an entry may route to.
enum class Envelope {
  kGemv,           // the small-token kernels only (b200awq_w4a16_gemv; b200awq_w4a16_linear below 8 tokens)
  kGemm,           // the small-token kernels, else the wgmma tile kernel (b200awq_w4a16_gemm; linear from 8 tokens)
  kMlpProjection,  // as kGemm, but without kGemm's 9..16-token big-layer rule (each of mlp_front's two projections)
};

// Routing of every W4A16 entry.  Small token counts take decode (one fp16 token) -> ring -> flat -> stream, each returning
// B200AWQ_ERR_SHAPE (or, for the cluster kernels, a launch-configuration error) when it cannot take the shape; outside
// kGemv, a shape none of them takes goes to the 128-channel wgmma tiles (split-k over a cluster for small token counts).
// An RMSNorm prologue rides along with decode and ring; before any later route, one RMSNorm launch (counted here) writes
// x^ into o.xhat and the route reads it, which is bit-identical by construction.
int launch_w4a16(const W4Operands& o, Envelope env) {
  const auto& [x_in, qw, sc, sz, y, m, n, k, dtype, st, epi, norm, xhat] = o;
  const bool pdl = pdl_enabled();
  const void* x = x_in;
  bool composed = !norm.on();
  auto compose = [&o, &x, &composed, pdl]() {
    if (composed) return 0;
    composed = true;
    x = o.xhat;
    return counted(b200awq::launch_rmsnorm(o.x, o.norm.gamma, o.xhat, o.norm.eps, o.m, o.k, o.dtype, pdl, o.st));
  };
  // kGemm: 9..16 tokens on the large layers (>= 48 M weights) take the persistent tile launch (split-k) directly
  const bool big_mid = env == Envelope::kGemm && m > 8 && (long long)n * k >= 48ll * 1000 * 1000;
  int r = B200AWQ_ERR_SHAPE;
  if (!big_mid) {
    if (use_decode(m, dtype))
      r = next_on_config_error(b200awq::launch_decode(x, qw, sc, sz, y, n, k, dtype, pdl, decode_tuning(), st, epi, norm));
    if (r != 0 && m <= kRingMaxM)
      r = next_on_config_error(b200awq::launch_ring(x, qw, sc, sz, y, m, n, k, dtype, pdl, st, epi, norm));
    if (r != 0 && (use_flat(m, n, k) || m <= kStreamMaxM))
      if (int e = compose()) return e;
    if (r != 0 && use_flat(m, n, k)) r = next_on_config_error(b200awq::launch_flat(x, qw, sc, sz, y, m, n, k, dtype, pdl, st, epi));
    if (r != 0 && m <= kStreamMaxM) r = b200awq::launch_stream(x, qw, sc, sz, y, m, n, k, dtype, pdl, st, nullptr, epi);
  }
  if (env != Envelope::kGemv && r == B200AWQ_ERR_SHAPE && n % 128 == 0) {
    if (int e = compose()) return e;
    r = b200awq::launch_umma(x, qw, sc, sz, y, m, n, k, dtype, pdl, st, epi);
  }
  return r;
}

// The RMSNorm entries' own checks, all without a device: gamma, eps and a workspace of at least `need` bytes.
int check_norm(const void* gamma, float eps, const void* workspace, size_t workspace_bytes, size_t need) {
  if (!aligned16(gamma)) return B200AWQ_ERR_ALIGN;
  if (!(std::isfinite(eps) && eps >= 0.f)) return B200AWQ_ERR_SHAPE;
  if (!aligned16(workspace) || workspace_bytes < need) return B200AWQ_ERR_WORKSPACE;
  return 0;
}

// mlp_front's composed path: the two projections into `workspace` (2 m n elements) and silu_mul, one count per kernel
int mlp_front_composed(const void* x, const void* gate_qweight, const void* gate_scales, const void* gate_szeros,
                       const void* up_qweight, const void* up_scales, const void* up_szeros, void* y, int m, int n, int k,
                       int dtype, void* workspace, cudaStream_t st) {
  const size_t half = (size_t)m * n * 2;
  void* g = workspace;
  void* u = static_cast<char*>(workspace) + half;
  const W4Operands gate{x, gate_qweight, gate_scales, gate_szeros, g, m, n, k, dtype, st};
  const W4Operands up{x, up_qweight, up_scales, up_szeros, u, m, n, k, dtype, st};
  for (const W4Operands* o : {&gate, &up})
    if (int r = counted(launch_w4a16(*o, Envelope::kMlpProjection))) return r;
  return counted(b200awq::launch_silu_mul(g, u, y, 1, (size_t)m * n, (size_t)m * n, dtype, pdl_enabled(), st));
}

// The TMA attention entries' common checks: dtype, sizes, head ratio and scale (the softmax runs on the raw scores'
// max: scale > 0).  kv_heads >= 1 once this passes.
int check_attention(int dtype, int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, float softmax_scale) {
  if (int e = check_dtype(dtype)) return e;
  if (batch < 0 || seqlen_q < 0 || seqlen_k < 0 || heads < 1 || kv_heads < 1 || heads % kv_heads ||
      !(std::isfinite(softmax_scale) && softmax_scale > 0.f))
    return B200AWQ_ERR_SHAPE;
  return 0;
}

// q, k, v, out and the strides of the operands read through TMA (16-byte multiples; Q is read in 16-byte pieces)
int check_attention_operands(const void* q, const void* k, const void* v, const void* out,
                             std::initializer_list<const long long*> strides) {
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(out)) return B200AWQ_ERR_ALIGN;
  for (const long long* s : strides)
    if (!s || s[0] % 8 || s[1] % 8 || s[2] % 8) return B200AWQ_ERR_ALIGN;
  return 0;
}

int check_workspace(const void* workspace, size_t workspace_bytes, size_t need) {
  if (workspace && !aligned16(workspace)) return B200AWQ_ERR_ALIGN;
  if (workspace_bytes < need || (workspace_bytes && !workspace)) return B200AWQ_ERR_WORKSPACE;
  return 0;
}

}  // namespace

extern "C" {

int b200awq_w4a16_gemv(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                       int k, int group_size, int dtype, void* stream) {
  if (int e = check_common(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (m > 7) return B200AWQ_ERR_BATCH;  // reference envelope: gemv_cuda.cu:291-330
  const W4Operands o{x, qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream)};
  return counted(launch_w4a16(o, Envelope::kGemv));
}

int b200awq_w4a16_linear(const void* x, const void* qweight, const void* scales, const void* szeros, const void* bias,
                         const void* residual, void* y, int m, int n, int k, int group_size, int dtype, void* stream) {
  if (int e = check_args(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if ((bias && !aligned16(bias)) || (residual && !aligned16(residual))) return B200AWQ_ERR_ALIGN;
  if (m >= 8 && n % 128) return B200AWQ_ERR_SHAPE;  // the GEMM envelope (b200awq_w4a16_gemm)
  if (int e = check_device()) return e;
  const W4Operands o{x, qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream), {bias, residual}};
  // the reference's dispatch rule (awq/quantize/qmodule.py:206): the GEMV's routes below 8 tokens, the GEMM's from 8
  return counted(launch_w4a16(o, m < 8 ? Envelope::kGemv : Envelope::kGemm));
}

int b200awq_w4a16_gemv_allreduce(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m,
                                 int n, int k, int group_size, int dtype, const b200awq_peers* peers, void* stream) {
  if (int e = check_common(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (m > 8) return B200AWQ_ERR_BATCH;
  if (!peers || peers->world < 1 || peers->world > 8 || peers->rank < 0 || peers->rank >= peers->world || !peers->epoch ||
      peers->n_max < 8 || peers->n_max % 8 || n > peers->n_max || peers->cap_words / peers->n_max < m)
    return B200AWQ_ERR_PEERS;
  b200awq::PeerArgs pa{};
  for (int r = 0; r < peers->world; ++r) {
    if (!peers->data[r]) return B200AWQ_ERR_PEERS;
    pa.data[r] = static_cast<unsigned long long*>(peers->data[r]);
  }
  pa.epoch = static_cast<unsigned int*>(peers->epoch);
  pa.rank = peers->rank;
  pa.world = peers->world;
  pa.tok_cap = peers->cap_words / peers->n_max;
  pa.cap = pa.tok_cap * peers->n_max;
  return counted(b200awq::launch_stream(x, qweight, scales, szeros, y, m, n, k, dtype, pdl_enabled(),
                                        static_cast<cudaStream_t>(stream), &pa));
}

size_t b200awq_w4a16_mlp_front_workspace_bytes(int m, int n, int) { return m > 0 && n > 0 ? (size_t)2 * m * n * 2 : 0; }

int b200awq_w4a16_mlp_front(const void* x, const void* gate_qweight, const void* gate_scales, const void* gate_szeros,
                            const void* up_qweight, const void* up_scales, const void* up_szeros, void* y, int m, int n, int k,
                            int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = check_common(x, gate_qweight, gate_scales, gate_szeros, y, m, n, k, group_size, dtype)) return e;
  if (!aligned16(up_qweight) || !aligned16(up_scales) || !aligned16(up_szeros)) return B200AWQ_ERR_ALIGN;
  if (m >= 8 && n % 128) return B200AWQ_ERR_SHAPE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the fused one-token kernel, else the composed path below: two projections and silu_mul, one count per kernel
  if (use_decode(m, dtype) &&
      next_on_config_error(b200awq::launch_decode_mlp_front(x, gate_qweight, gate_scales, gate_szeros, up_qweight, up_scales,
                                                            up_szeros, y, n, k, dtype, pdl_enabled(), decode_tuning(), st)) == 0)
    return counted(0);
  const size_t half = (size_t)m * n * 2;
  if (!workspace || workspace_bytes < 2 * half || !aligned16(workspace)) return B200AWQ_ERR_WORKSPACE;
  return mlp_front_composed(x, gate_qweight, gate_scales, gate_szeros, up_qweight, up_scales, up_szeros, y, m, n, k, dtype,
                            workspace, st);
}

size_t b200awq_w4a16_norm_workspace_bytes(int m, int n, int k) {
  return m > 0 && n > 0 && k > 0 ? (size_t)m * k * 2 + (size_t)2 * m * n * 2 : 0;
}

int b200awq_w4a16_norm_linear(const void* x, const void* gamma, float eps, const void* qweight, const void* scales,
                              const void* szeros, const void* bias, void* y, int m, int n, int k, int group_size, int dtype,
                              void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = check_args(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (bias && !aligned16(bias)) return B200AWQ_ERR_ALIGN;
  if (m >= 8 && n % 128) return B200AWQ_ERR_SHAPE;  // as b200awq_w4a16_linear
  if (int e = check_norm(gamma, eps, workspace, workspace_bytes, (size_t)m * k * 2)) return e;
  if (int e = check_device()) return e;
  const W4Operands o{x,  qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream), {bias, nullptr},
                     {gamma, eps}, workspace};
  return counted(launch_w4a16(o, m < 8 ? Envelope::kGemv : Envelope::kGemm));
}

int b200awq_w4a16_norm_mlp_front(const void* x, const void* gamma, float eps, const void* gate_qweight,
                                 const void* gate_scales, const void* gate_szeros, const void* up_qweight,
                                 const void* up_scales, const void* up_szeros, void* y, int m, int n, int k, int group_size,
                                 int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = check_args(x, gate_qweight, gate_scales, gate_szeros, y, m, n, k, group_size, dtype)) return e;
  if (!aligned16(up_qweight) || !aligned16(up_scales) || !aligned16(up_szeros)) return B200AWQ_ERR_ALIGN;
  if (m >= 8 && n % 128) return B200AWQ_ERR_SHAPE;
  if (int e = check_norm(gamma, eps, workspace, workspace_bytes, b200awq_w4a16_norm_workspace_bytes(m, n, k))) return e;
  if (int e = check_device()) return e;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool pdl = pdl_enabled();
  // the fused one-token kernel with the prologue, else x^ into the workspace and mlp_front's composed path behind it
  if (use_decode(m, dtype) &&
      next_on_config_error(b200awq::launch_decode_mlp_front(x, gate_qweight, gate_scales, gate_szeros, up_qweight, up_scales,
                                                            up_szeros, y, n, k, dtype, pdl, decode_tuning(), st,
                                                            {gamma, eps})) == 0)
    return counted(0);
  void* xhat = workspace;
  if (int r = counted(b200awq::launch_rmsnorm(x, gamma, xhat, eps, m, k, dtype, pdl, st))) return r;
  return mlp_front_composed(xhat, gate_qweight, gate_scales, gate_szeros, up_qweight, up_scales, up_szeros, y, m, n, k, dtype,
                            static_cast<char*>(workspace) + (size_t)m * k * 2, st);
}

size_t b200awq_single_query_attention_workspace_bytes(int batch, int heads, int kv_heads, int head_dim, int max_len) {
  return b200awq::attention_workspace_bytes(batch, heads, kv_heads, head_dim, max_len);
}

int b200awq_single_query_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, void* out,
                                   const int* length_per_sample, int batch, int heads, int kv_heads, int head_dim,
                                   int max_len, int timestep, long long q_batch_stride, long long k_batch_stride,
                                   long long v_batch_stride, int rotary_dim, float rotary_base,
                                   float rotary_scale, int neox, int dtype, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (!q || !k || !v || !aligned16(k_cache) || !aligned16(v_cache) || !out) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_single_query_attention(q, k, v, k_cache, v_cache, out, length_per_sample, batch, heads, kv_heads,
                                                        head_dim, max_len, timestep, q_batch_stride, k_batch_stride, v_batch_stride,
                                                        rotary_dim, rotary_base, rotary_scale, neox, dtype, workspace,
                                                        workspace_bytes, pdl_enabled(), static_cast<cudaStream_t>(stream)));
}

int b200awq_prefill_attention(const void* q, const void* k, const void* v, void* out, const int* cu_seqlens_q,
                              const int* cu_seqlens_k, int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads,
                              int head_dim, const long long q_strides[3], const long long k_strides[3],
                              const long long v_strides[3], float softmax_scale, int causal, int dtype, void* stream) {
  if (int e = check_attention(dtype, batch, seqlen_q, seqlen_k, heads, kv_heads, softmax_scale)) return e;
  if (head_dim != 64 && head_dim != 72 && head_dim != 128) return B200AWQ_ERR_SHAPE;
  if (int e = check_attention_operands(q, k, v, out, {q_strides, k_strides, v_strides})) return e;
  if ((cu_seqlens_q == nullptr) != (cu_seqlens_k == nullptr)) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  if (batch == 0 || seqlen_q == 0) return 0;
  return counted(b200awq::launch_prefill_attention(q, k, v, out, cu_seqlens_q, cu_seqlens_k, batch, seqlen_q, seqlen_k, heads,
                                                   kv_heads, head_dim, q_strides, k_strides, v_strides, softmax_scale, causal != 0,
                                                   dtype, static_cast<cudaStream_t>(stream)));
}

size_t b200awq_splitkv_attention_workspace_bytes(int batch, int seqlen_q, int seqlen_k, int heads, int kv_heads, int head_dim) {
  return b200awq::splitkv_attention_workspace_bytes(batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim);
}

int b200awq_splitkv_attention(const void* q, const void* k, const void* v, void* out, int batch, int seqlen_q, int seqlen_k,
                              int heads, int kv_heads, int head_dim, const long long q_strides[3],
                              const long long k_strides[3], const long long v_strides[3], float softmax_scale, int causal,
                              int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = check_attention(dtype, batch, seqlen_q, seqlen_k, heads, kv_heads, softmax_scale)) return e;
  if ((long long)seqlen_q * (heads / kv_heads) > 64 || (head_dim != 64 && head_dim != 128)) return B200AWQ_ERR_SHAPE;
  if (int e = check_attention_operands(q, k, v, out, {q_strides, k_strides, v_strides})) return e;
  if (int e = check_workspace(workspace, workspace_bytes,
                              b200awq::splitkv_attention_workspace_bytes(batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim)))
    return e;
  if (int e = check_device()) return e;
  if (batch == 0 || seqlen_q == 0) return 0;
  return counted(b200awq::launch_splitkv_attention(q, k, v, out, batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim, q_strides,
                                                   k_strides, v_strides, softmax_scale, causal != 0, dtype, workspace,
                                                   workspace_bytes, static_cast<cudaStream_t>(stream)));
}

size_t b200awq_kv_cache_attention_workspace_bytes(int layout, int batch, int seqlen_q, int seqlen_k, int heads,
                                                  int kv_heads, int head_dim) {
  return b200awq::kv_cache_attention_workspace_bytes(layout, batch, seqlen_q, seqlen_k, heads, kv_heads, head_dim);
}

int b200awq_kv_cache_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int layout, int batch,
                               int seqlen_q, int seqlen_k, int max_len, int heads, int kv_heads, int head_dim,
                               const long long q_strides[3], float softmax_scale, int causal, int dtype, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (int e = check_attention(dtype, batch, seqlen_q, seqlen_k, heads, kv_heads, softmax_scale)) return e;
  if ((layout != B200AWQ_KV_FT && layout != B200AWQ_KV_BTHD) || max_len < 1 || seqlen_k > max_len ||
      (head_dim != 64 && head_dim != 128))
    return B200AWQ_ERR_SHAPE;
  if (int e = check_attention_operands(q, k_cache, v_cache, out, {q_strides})) return e;  // the caches are not strided
  if (int e = check_workspace(workspace, workspace_bytes,
                              b200awq::kv_cache_attention_workspace_bytes(layout, batch, seqlen_q, seqlen_k, heads,
                                                                          kv_heads, head_dim)))
    return e;
  if (batch == 0 || seqlen_q == 0) return 0;  // unlike the two entries above, before the device check
  if (int e = check_device()) return e;
  return counted(b200awq::launch_kv_cache_attention(q, k_cache, v_cache, out, layout, batch, seqlen_q, seqlen_k, max_len, heads,
                                                    kv_heads, head_dim, q_strides, softmax_scale, causal != 0, dtype,
                                                    workspace, workspace_bytes, static_cast<cudaStream_t>(stream)));
}

int b200awq_rope_kv_store(void* qkv, const float* freqs, void* k_cache, void* v_cache, int layout, int batch, int seqlen,
                          int heads, int kv_heads, int head_dim, int max_len, int start_pos, const long long qkv_strides[3],
                          int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if ((layout != B200AWQ_KV_FT && layout != B200AWQ_KV_BTHD) || batch < 0 || seqlen < 0 || heads < 1 || kv_heads < 1 ||
      heads % kv_heads || head_dim < 8 || head_dim % 8 || head_dim > 256 || max_len < 1 || start_pos < 0 ||
      (long long)start_pos + seqlen > max_len)
    return B200AWQ_ERR_SHAPE;
  if (!aligned16(qkv) || !aligned16(freqs) || !aligned16(k_cache) || !aligned16(v_cache)) return B200AWQ_ERR_ALIGN;
  if (!qkv_strides || qkv_strides[0] % 8 || qkv_strides[1] % 8 || qkv_strides[2] % 8) return B200AWQ_ERR_ALIGN;
  if (batch == 0 || seqlen == 0) return 0;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_rope_kv_store(qkv, freqs, k_cache, v_cache, layout, batch, seqlen, heads, kv_heads, head_dim,
                                               max_len, start_pos, qkv_strides, dtype, pdl_enabled(),
                                               static_cast<cudaStream_t>(stream)));
}

int b200awq_sample_next_token(const float* logits, long long logits_row_stride, int batch, int vocab,
                              const long long* prev_ids, long long prev_row_stride, int n_prev, float temperature,
                              float repetition_penalty, float top_p, int top_k, int greedy, const float* uniforms,
                              long long* tokens, void* stream) {
  if (batch < 0 || vocab < 1 || vocab > B200AWQ_SAMPLE_MAX_VOCAB || n_prev < 0 ||
      !(std::isfinite(temperature) && temperature > 0.f) ||
      !(std::isfinite(repetition_penalty) && repetition_penalty >= 1.f) || !(top_p > 0.f && top_p <= 1.f) || top_k < 0)
    return B200AWQ_ERR_SHAPE;
  auto aligned = [](const void* p, uintptr_t bytes) { return p && (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; };
  if (!aligned(logits, 4) || !aligned(tokens, 8) || (!greedy && !aligned(uniforms, 4)) ||
      (n_prev > 0 && repetition_penalty > 1.f && !aligned(prev_ids, 8)))
    return B200AWQ_ERR_ALIGN;
  if (batch == 0) return 0;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_sample_next_token(logits, logits_row_stride, batch, vocab, prev_ids, prev_row_stride, n_prev,
                                                   temperature, repetition_penalty, top_p, top_k, greedy, uniforms, tokens,
                                                   pdl_enabled(), static_cast<cudaStream_t>(stream)));
}

int b200awq_lm_head(const void* x, long long x_row_stride, const void* gamma, float eps, const void* weight, float* logits,
                    int m, int vocab, int k, int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (m < 1 || m > b200awq::kLmHeadMaxM) return B200AWQ_ERR_BATCH;
  if (vocab < 1 || k < 8 || k > 8192 || k % 8 || x_row_stride < k) return B200AWQ_ERR_SHAPE;
  if (!aligned16(x) || !aligned16(weight) || !aligned16(logits) || (gamma && !aligned16(gamma)) || x_row_stride % 8)
    return B200AWQ_ERR_ALIGN;
  if (gamma && !(std::isfinite(eps) && eps >= 0.f)) return B200AWQ_ERR_SHAPE;
  // the logits are written while the inputs are read: they must not share a byte with any of them
  const uintptr_t o = reinterpret_cast<uintptr_t>(logits), o_end = o + (uintptr_t)m * (uintptr_t)vocab * 4u;
  auto overlaps = [o, o_end](const void* p, uintptr_t bytes) {
    const uintptr_t b = reinterpret_cast<uintptr_t>(p);
    return p && b < o_end && o < b + bytes;
  };
  if (overlaps(x, ((uintptr_t)(m - 1) * (uintptr_t)x_row_stride + (uintptr_t)k) * 2u) ||
      overlaps(weight, (uintptr_t)vocab * (uintptr_t)k * 2u) || overlaps(gamma, (uintptr_t)k * 2u))
    return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_lm_head(x, x_row_stride, gamma, eps, weight, logits, m, vocab, k, dtype, pdl_enabled(),
                                         static_cast<cudaStream_t>(stream)));
}

int b200awq_rope_with_pos(const void* x, const float* freqs, void* y, int s, int b, int h, int d, int d2,
                          const long long in_strides[4], const long long out_strides[4], int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (!x || !freqs || !y || !in_strides || !out_strides) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_rope_with_pos(x, freqs, y, s, b, h, d, d2, in_strides, out_strides, dtype, pdl_enabled(),
                                               static_cast<cudaStream_t>(stream)));
}

int b200awq_rotary_embedding_neox(const long long* positions, void* query, void* key, const void* cos_sin_cache, int tokens,
                                  int q_heads, int k_heads, int head_size, int rot_dim, long long q_token_stride,
                                  long long k_token_stride, int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (!positions || !cos_sin_cache || (q_heads > 0 && !query) || (k_heads > 0 && !key)) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_rope_neox(positions, query, key, cos_sin_cache, tokens, q_heads, k_heads, head_size, rot_dim,
                                           q_token_stride, k_token_stride, dtype, pdl_enabled(), static_cast<cudaStream_t>(stream)),
                 tokens > 0 && q_heads + k_heads > 0);
}

int b200awq_rmsnorm(const void* x, const void* gamma, void* y, int m, int n, float eps, int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (m < 0 || n < 1) return B200AWQ_ERR_SHAPE;
  if (!x || !gamma || !y) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  if (m == 0) return 0;
  return counted(b200awq::launch_rmsnorm(x, gamma, y, eps, m, n, dtype, pdl_enabled(), static_cast<cudaStream_t>(stream)));
}

size_t b200awq_w4a16_gemm_workspace_bytes(int, int, int) { return 0; }

int b200awq_w4a16_gemm(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                       int k, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  (void)workspace;
  (void)workspace_bytes;
  if (int e = check_common(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (n % 128) return B200AWQ_ERR_SHAPE;  // reference: N / CTA_N with CTA_N = 128, gemm_cuda.cu:38,1225
  const W4Operands o{x, qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream)};
  return counted(launch_w4a16(o, Envelope::kGemm));
}

// ---------------------------------------------------------------- W8A8
namespace {
// b200awq_w8a8_gemm's argument checks that need no device
int check_w8a8_gemm(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias, const void* y,
                    int m, int n, int k) {
  if (m < 1 || n < 8 || k < 16 || n % 8 || k % 16) return B200AWQ_ERR_SHAPE;
  if (!aligned16(x) || !aligned16(w) || !aligned16(y) || !wscales || !ascales) return B200AWQ_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(wscales) | reinterpret_cast<uintptr_t>(ascales) | reinterpret_cast<uintptr_t>(bias)) & 1u)
    return B200AWQ_ERR_ALIGN;
  return 0;
}
}  // namespace

int b200awq_w8a8_gemm(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias, void* y,
                      int m, int n, int k, void* stream) {
  if (int e = check_w8a8_gemm(x, w, wscales, ascales, bias, y, m, n, k)) return e;
  if (int e = check_device()) return e;
  return counted(b200awq::launch_w8a8_gemm(x, w, wscales, ascales, bias, y, m, n, k, pdl_enabled(), static_cast<cudaStream_t>(stream)));
}

int b200awq_w8a8_linear(const void* x, const void* w, const void* wscales, const void* ascales, const void* bias,
                        const void* layer_scale, const void* residual, void* y, int m, int n, int k, void* stream) {
  if (int e = check_w8a8_gemm(x, w, wscales, ascales, bias, y, m, n, k)) return e;
  if ((layer_scale && !aligned16(layer_scale)) || (residual && !aligned16(residual))) return B200AWQ_ERR_ALIGN;
  if (residual) {  // the residual is read and y written by different threads: the two must not share a byte
    const uintptr_t r = reinterpret_cast<uintptr_t>(residual), o = reinterpret_cast<uintptr_t>(y);
    const uintptr_t bytes = (uintptr_t)m * (uintptr_t)n * 2u;
    if (r < o + bytes && o < r + bytes) return B200AWQ_ERR_ALIGN;
  }
  if (int e = check_device()) return e;
  return counted(b200awq::launch_w8a8_gemm(x, w, wscales, ascales, bias, y, m, n, k, pdl_enabled(),
                                           static_cast<cudaStream_t>(stream), layer_scale, residual));
}

namespace {
// common checks of the W8A8 row ops: 16-bit activations, rows the kernels hold in registers, non-null 2-byte aligned
// pointers (the int8 codes are written one byte at a time when not 16-byte aligned, so any even address will do)
int check_rows(int m, int n, int dtype, std::initializer_list<const void*> ptrs) {
  if (int e = check_dtype(dtype)) return e;
  if (m < 0 || n < 1 || n > b200awq::w8a8_row_limit()) return B200AWQ_ERR_SHAPE;
  for (const void* p : ptrs)
    if (!p || (reinterpret_cast<uintptr_t>(p) & 1u)) return B200AWQ_ERR_ALIGN;
  return check_device();
}
}  // namespace

int b200awq_quant_per_token(const void* x, void* q, void* scales, int m, int n, int dtype, void* stream) {
  if (int e = check_rows(m, n, dtype, {x, scales, q})) return e;
  return counted(b200awq::launch_quant_per_token(x, q, scales, m, n, dtype, pdl_enabled(), static_cast<cudaStream_t>(stream)), m > 0);
}

int b200awq_layernorm_quant(const void* x, const void* gamma, const void* beta, void* q, void* scale, int m, int n,
                            float eps, int per_token, int dtype, void* stream) {
  if (reinterpret_cast<uintptr_t>(beta) & 1u) return B200AWQ_ERR_ALIGN;
  if (int e = check_rows(m, n, dtype, {x, gamma, scale, q})) return e;
  return counted(b200awq::launch_layernorm_quant(x, gamma, beta, q, scale, m, n, eps, per_token != 0, dtype, pdl_enabled(),
                                                 static_cast<cudaStream_t>(stream)),
                 m > 0);
}

int b200awq_gelu_quant(const void* x, void* q, void* scales, void* tmp, int m, int n, void* stream) {
  if (int e = check_rows(m, n, B200AWQ_DTYPE_F16, {x, scales, tmp, q})) return e;
  return counted(b200awq::launch_gelu_quant(x, q, scales, tmp, m, n, pdl_enabled(), static_cast<cudaStream_t>(stream)), m > 0);
}

int b200awq_silu_and_mul(const void* x, void* y, int m, int d, int dtype, void* stream) {
  if (int e = check_dtype(dtype)) return e;
  if (m < 0 || d < 1) return B200AWQ_ERR_SHAPE;
  if (!x || !y || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 1u)) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  const char* xb = static_cast<const char*>(x);
  return counted(b200awq::launch_silu_mul(xb, xb + (size_t)d * 2, y, (size_t)m, (size_t)d, (size_t)2 * d, dtype, pdl_enabled(),
                                          static_cast<cudaStream_t>(stream)),
                 m > 0);
}

int gemv_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                      int k, int group_size, int dtype, void* stream) {
  return b200awq_w4a16_gemv(x, qweight, scales, szeros, y, m, n, k, group_size, dtype, stream);
}
int gemm_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                      int k, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  return b200awq_w4a16_gemm(x, qweight, scales, szeros, y, m, n, k, group_size, dtype, workspace, workspace_bytes, stream);
}

int b200awq_set_pdl(int enable) { return g_pdl.exchange(enable != 0, std::memory_order_relaxed) ? 1 : 0; }

void b200awq_reload_config(void) {
  static std::atomic<int> which{0};
  const int w = which.fetch_add(1, std::memory_order_relaxed) & 1;
  g_decode_store[w] = read_decode_tuning();
  g_decode.store(&g_decode_store[w], std::memory_order_release);
}

unsigned long long b200awq_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

const char* b200awq_strerror(int code) {
  switch (code) {
    case B200AWQ_OK: return "ok";
    case B200AWQ_ERR_SHAPE:
      return "unsupported shape (need n % 8 == 0 [gemm: n % 128 == 0], k % 128 == 0 [w8a8 gemm: k % 16 == 0], m >= 1)";
    case B200AWQ_ERR_GROUP: return "unsupported group size (only 128)";
    case B200AWQ_ERR_ALIGN: return "null or misaligned pointer (16-byte alignment required), or a residual overlapping y";
    case B200AWQ_ERR_DTYPE: return "unsupported dtype (fp16 / bf16 only; gelu_quant: fp16 only)";
    case B200AWQ_ERR_BATCH: return "unsupported batch size for gemv kernel (1..7)";
    case B200AWQ_ERR_WORKSPACE: return "workspace too small";
    case B200AWQ_ERR_DRIVER: return "cuTensorMapEncodeTiled unavailable or failed";
    case B200AWQ_ERR_DEVICE: return "device is not compute capability 9.x (sm_90a kernels only)";
    case B200AWQ_ERR_PEERS: return "bad peer description for the fused all-reduce";
    default: return code > 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : "unknown error";
  }
}

const char* b200awq_version(void) { return "b200awq 0.1 sm_90a"; }

}  // extern "C"
