// C ABI of libb200awq.so (declared in include/b200awq.h): argument validation, dispatch
// between the HBM-bound streaming kernel and the wgmma tensor-core kernel, process-wide
// switches.  No torch types, no allocation, no synchronisation.
#include <atomic>
#include <cstdint>
#include <cstdlib>

#include "w4a16_kernels.h"

namespace {

std::atomic<unsigned long long> g_launches{0};

int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return v && *v ? std::atoi(v) : dflt;
}

// Every environment knob of the library, read ONCE (first launch, or b200awq_reload_config()): the decode path is a
// few microseconds per call, a dozen getenv() per launch is not free, and the tunings are plain values handed to the
// launchers -- no mutable globals on the call path.
struct Config {
  bool pdl;
  bool decode;        // B200AWQ_DECODE=0: never use the one-token decode kernel (fp16; bf16 with B200AWQ_DECODE=2)
  bool decode_bf16;
  b200awq::DecodeTuning decode_t;
  bool ring;          // B200AWQ_RING=0: never use the persistent ring kernel
  int ring_max_m;     // largest token count served by the ring kernel
  bool flat;          // B200AWQ_SKINNY=stream: never use the wgmma skinny launch
  int flat_min_m, flat_min_m_longk, flat_max_m;
  int stream_max_m;
  b200awq::RingTuning ring_t;
  b200awq::StreamTuning stream_t;
  b200awq::FlatTuning flat_t;
  b200awq::UmmaTuning umma_t;
};

Config read_config() {
  Config c;
  c.pdl = env_int("B200AWQ_PDL", 1) != 0;
  c.decode = env_int("B200AWQ_DECODE", 1) != 0;
  c.decode_bf16 = env_int("B200AWQ_DECODE", 1) == 2;
  c.decode_t.split = env_int("B200AWQ_DECODE_SPLIT", 0);
  c.decode_t.slots = env_int("B200AWQ_DECODE_SLOTS", 0);
  c.decode_t.warps = env_int("B200AWQ_DECODE_WARPS", 0);
  c.ring = env_int("B200AWQ_RING", 1) != 0;
  c.ring_max_m = env_int("B200AWQ_RING_MAX_M", 4);
  const char* sk = std::getenv("B200AWQ_SKINNY");
  c.flat = !(sk && sk[0] == 's');
  // crossovers: the wgmma skinny launch from 5 tokens (from 3 when k is long enough to need a cluster split), the
  // wgmma tile launch above 16
  c.flat_min_m = env_int("B200AWQ_FLAT_MIN_M", 5);
  c.flat_min_m_longk = env_int("B200AWQ_FLAT_MIN_M", 3);
  c.flat_max_m = env_int("B200AWQ_FLAT_MAX_M", 16);
  c.stream_max_m = env_int("B200AWQ_STREAM_MAX_M", 16);
  c.ring_t.mode = env_int("B200AWQ_RING_MODE", -1);
  c.ring_t.split = env_int("B200AWQ_RING_SPLIT", 0);
  c.ring_t.slots = env_int("B200AWQ_RING_SLOTS", 0);
  c.stream_t.mode = env_int("B200AWQ_STREAM_MODE", -1);
  c.stream_t.kc = env_int("B200AWQ_STREAM_KC", 0);
  c.stream_t.rpb = env_int("B200AWQ_STREAM_RPB", 0);
  c.stream_t.pad = env_int("B200AWQ_STREAM_PAD", 0);
  c.stream_t.rbs = env_int("B200AWQ_STREAM_RBS", 0);
  c.stream_t.warps = env_int("B200AWQ_STREAM_WARPS", 0);
  c.flat_t.kc = env_int("B200AWQ_FLAT_KC", 0);
  c.umma_t.tn = env_int("B200AWQ_UMMA_TN", 0);
  c.umma_t.max_ctas = env_int("B200AWQ_UMMA_CTAS", 0);
  c.umma_t.split = env_int("B200AWQ_UMMA_SPLIT", 0);
  return c;
}

// Double-buffered so that a reload never races a reader: readers take a pointer with acquire, writers publish a
// fully built copy.
Config g_cfg_store[2];
std::atomic<const Config*> g_cfg{nullptr};
std::atomic<int> g_pdl_override{-1};  // b200awq_set_pdl(): -1 = follow the environment

const Config& cfg() {
  const Config* c = g_cfg.load(std::memory_order_acquire);
  if (!c) {
    static const Config first = read_config();  // thread-safe one-time initialisation
    g_cfg.store(&first, std::memory_order_release);
    c = &first;
  }
  return *c;
}

bool pdl_enabled() {
  const int o = g_pdl_override.load(std::memory_order_relaxed);
  return o < 0 ? cfg().pdl : o != 0;
}

bool aligned16(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

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

int check_common(const void* x, const void* qw, const void* sc, const void* sz, void* y, int m, int n, int k,
                 int group_size, int dtype) {
  if (dtype != B200AWQ_DTYPE_F16 && dtype != B200AWQ_DTYPE_BF16) return B200AWQ_ERR_DTYPE;
  if (group_size != 128) return B200AWQ_ERR_GROUP;
  if (m < 1 || n < 8 || k < 128 || (n % 8) || (k % 128)) return B200AWQ_ERR_SHAPE;
  if (!aligned16(x) || !aligned16(qw) || !aligned16(sc) || !aligned16(sz) || !aligned16(y)) return B200AWQ_ERR_ALIGN;
  return check_device();
}

// which kernel serves small token counts beyond the ring kernel's range
bool use_flat(const Config& c, int m, int n, int k) {
  const int min_m = k > 8192 ? c.flat_min_m_longk : c.flat_min_m;
  return c.flat && n % 128 == 0 && m >= min_m && m <= c.flat_max_m;
}

// Small token counts (decode and the bottom of the batch sweep): decode (one token) -> ring -> flat -> stream, each returning
// B200AWQ_ERR_SHAPE (or, for the cluster kernels, a launch-configuration error) when it cannot take the shape.
int launch_small(const Config& c, const void* x, const void* qw, const void* sc, const void* sz, void* y, int m, int n,
                 int k, int dtype, cudaStream_t st) {
  int r = B200AWQ_ERR_SHAPE;
  // one token: fp16 through the int8-digit decode kernel (bf16 stays operand-exact: dropping the bf16 rounding of
  // q s + z would move results by ~1e-3 against the reference)
  if (m == 1 && c.decode && (dtype == B200AWQ_DTYPE_F16 || c.decode_bf16))
    r = b200awq::launch_decode(x, qw, sc, sz, y, n, k, dtype, pdl_enabled(), c.decode_t, st);
  if (r > 0) {  // a launch-configuration error (e.g. an unschedulable cluster): the kernels below can take the shape
    (void)cudaGetLastError();
    r = B200AWQ_ERR_SHAPE;
  }
  if (r != 0 && c.ring && m <= c.ring_max_m) r = b200awq::launch_ring(x, qw, sc, sz, y, m, n, k, dtype, pdl_enabled(), c.ring_t, st);
  if (r != 0 && use_flat(c, m, n, k)) {
    r = b200awq::launch_flat(x, qw, sc, sz, y, m, n, k, dtype, pdl_enabled(), c.flat_t, st);
    if (r > 0) {  // e.g. an unschedulable cluster shape: not the caller's problem, the streaming kernel can take it
      (void)cudaGetLastError();
      r = B200AWQ_ERR_SHAPE;
    }
  }
  if (r != 0 && m <= 16 && m <= c.stream_max_m) {
    if (r > 0) (void)cudaGetLastError();
    r = b200awq::launch_stream(x, qw, sc, sz, y, m, n, k, dtype, pdl_enabled(), c.stream_t, st);
  }
  return r;
}

}  // namespace

extern "C" {

int b200awq_w4a16_gemv(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                       int k, int group_size, int dtype, void* stream) {
  if (int e = check_common(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (m > 7) return B200AWQ_ERR_BATCH;  // reference envelope: gemv_cuda.cu:291-330
  const int r = launch_small(cfg(), x, qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream));
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
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
  int r = b200awq::launch_stream(x, qweight, scales, szeros, y, m, n, k, dtype, pdl_enabled(), cfg().stream_t,
                                 static_cast<cudaStream_t>(stream), &pa);
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

size_t b200awq_w4a16_mlp_front_workspace_bytes(int m, int n, int) { return m > 0 && n > 0 ? (size_t)2 * m * n * 2 : 0; }

int b200awq_w4a16_mlp_front(const void* x, const void* gate_qweight, const void* gate_scales, const void* gate_szeros,
                            const void* up_qweight, const void* up_scales, const void* up_szeros, void* y, int m, int n, int k,
                            int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = check_common(x, gate_qweight, gate_scales, gate_szeros, y, m, n, k, group_size, dtype)) return e;
  if (!aligned16(up_qweight) || !aligned16(up_scales) || !aligned16(up_szeros)) return B200AWQ_ERR_ALIGN;
  if (m >= 8 && n % 128) return B200AWQ_ERR_SHAPE;
  const Config& c = cfg();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (m == 1 && c.decode && (dtype == B200AWQ_DTYPE_F16 || c.decode_bf16)) {
    const int r = b200awq::launch_decode_mlp_front(x, gate_qweight, gate_scales, gate_szeros, up_qweight, up_scales, up_szeros, y,
                                                   n, k, dtype, pdl_enabled(), c.decode_t, st);
    if (r == 0) {
      g_launches.fetch_add(1, std::memory_order_relaxed);
      return 0;
    }
    if (r > 0) (void)cudaGetLastError();  // launch-configuration error: the composed path below can take the shape
  }
  const size_t half = (size_t)m * n * 2;
  if (!workspace || workspace_bytes < 2 * half || !aligned16(workspace)) return B200AWQ_ERR_WORKSPACE;
  void* g = workspace;
  void* u = static_cast<char*>(workspace) + half;
  for (int t = 0; t < 2; ++t) {
    const void* qw = t ? up_qweight : gate_qweight;
    const void* sc = t ? up_scales : gate_scales;
    const void* sz = t ? up_szeros : gate_szeros;
    int r = B200AWQ_ERR_SHAPE;
    if (m <= 16) r = launch_small(c, x, qw, sc, sz, t ? u : g, m, n, k, dtype, st);
    if (r == B200AWQ_ERR_SHAPE && n % 128 == 0)
      r = b200awq::launch_umma(x, qw, sc, sz, t ? u : g, m, n, k, dtype, pdl_enabled(), c.umma_t, st);
    if (r != 0) return r;
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  const int r = b200awq::launch_silu_mul(g, u, y, (size_t)m * n, dtype, pdl_enabled(), st);
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
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
  if (dtype != B200AWQ_DTYPE_F16 && dtype != B200AWQ_DTYPE_BF16) return B200AWQ_ERR_DTYPE;
  if (!q || !k || !v || !aligned16(k_cache) || !aligned16(v_cache) || !out) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  const int r = b200awq::launch_single_query_attention(q, k, v, k_cache, v_cache, out, length_per_sample, batch, heads, kv_heads,
                                                       head_dim, max_len, timestep, q_batch_stride, k_batch_stride, v_batch_stride, rotary_dim,
                                                       rotary_base,
                                                       rotary_scale, neox, dtype, workspace, workspace_bytes, pdl_enabled(),
                                                       static_cast<cudaStream_t>(stream));
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

int b200awq_rope_with_pos(const void* x, const float* freqs, void* y, int s, int b, int h, int d, int d2,
                          const long long in_strides[4], const long long out_strides[4], int dtype, void* stream) {
  if (dtype != B200AWQ_DTYPE_F16 && dtype != B200AWQ_DTYPE_BF16) return B200AWQ_ERR_DTYPE;
  if (!x || !freqs || !y || !in_strides || !out_strides) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  const int r = b200awq::launch_rope_with_pos(x, freqs, y, s, b, h, d, d2, in_strides, out_strides, dtype, pdl_enabled(),
                                              static_cast<cudaStream_t>(stream));
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

int b200awq_rotary_embedding_neox(const long long* positions, void* query, void* key, const void* cos_sin_cache, int tokens,
                                  int q_heads, int k_heads, int head_size, int rot_dim, long long q_token_stride,
                                  long long k_token_stride, int dtype, void* stream) {
  if (dtype != B200AWQ_DTYPE_F16 && dtype != B200AWQ_DTYPE_BF16) return B200AWQ_ERR_DTYPE;
  if (!positions || !cos_sin_cache || (q_heads > 0 && !query) || (k_heads > 0 && !key)) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  const int r = b200awq::launch_rope_neox(positions, query, key, cos_sin_cache, tokens, q_heads, k_heads, head_size, rot_dim,
                                          q_token_stride, k_token_stride, dtype, pdl_enabled(), static_cast<cudaStream_t>(stream));
  if (r == 0 && tokens > 0 && q_heads + k_heads > 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

int b200awq_rmsnorm(const void* x, const void* gamma, void* y, int m, int n, float eps, int dtype, void* stream) {
  if (dtype != B200AWQ_DTYPE_F16 && dtype != B200AWQ_DTYPE_BF16) return B200AWQ_ERR_DTYPE;
  if (m < 0 || n < 1) return B200AWQ_ERR_SHAPE;
  if (!x || !gamma || !y) return B200AWQ_ERR_ALIGN;
  if (int e = check_device()) return e;
  if (m == 0) return 0;
  const int r = b200awq::launch_rmsnorm(x, gamma, y, eps, m, n, dtype, pdl_enabled(), static_cast<cudaStream_t>(stream));
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

size_t b200awq_w4a16_gemm_workspace_bytes(int, int, int) { return 0; }

int b200awq_w4a16_gemm(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                       int k, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  (void)workspace;
  (void)workspace_bytes;
  if (int e = check_common(x, qweight, scales, szeros, y, m, n, k, group_size, dtype)) return e;
  if (n % 128) return B200AWQ_ERR_SHAPE;  // reference: N / CTA_N with CTA_N = 128, gemm_cuda.cu:38,1225
  const Config& c = cfg();
  int r = B200AWQ_ERR_SHAPE;
  // 9..16 tokens on the large layers (>= 48 M weights): the persistent tile launch (split-k); everything else below
  // 17 tokens: the small-token kernels
  const bool big_mid = m > 8 && (long long)n * k >= 48ll * 1000 * 1000;
  if (m <= 16 && !big_mid) r = launch_small(c, x, qweight, scales, szeros, y, m, n, k, dtype, static_cast<cudaStream_t>(stream));
  if (r == B200AWQ_ERR_SHAPE)  // 128-channel wgmma tiles; split-k over a cluster for small token counts
    r = b200awq::launch_umma(x, qweight, scales, szeros, y, m, n, k, dtype, pdl_enabled(), c.umma_t,
                             static_cast<cudaStream_t>(stream));
  if (r == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  return r;
}

int gemv_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                      int k, int group_size, int dtype, void* stream) {
  return b200awq_w4a16_gemv(x, qweight, scales, szeros, y, m, n, k, group_size, dtype, stream);
}
int gemm_forward_4bit(const void* x, const void* qweight, const void* scales, const void* szeros, void* y, int m, int n,
                      int k, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  return b200awq_w4a16_gemm(x, qweight, scales, szeros, y, m, n, k, group_size, dtype, workspace, workspace_bytes, stream);
}

int b200awq_set_pdl(int enable) {
  const int prev = pdl_enabled() ? 1 : 0;
  g_pdl_override.store(enable ? 1 : 0, std::memory_order_relaxed);
  return prev;
}

void b200awq_reload_config(void) {
  static std::atomic<int> which{0};
  const int w = which.fetch_add(1, std::memory_order_relaxed) & 1;
  g_cfg_store[w] = read_config();
  g_cfg.store(&g_cfg_store[w], std::memory_order_release);
}

unsigned long long b200awq_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

const char* b200awq_strerror(int code) {
  switch (code) {
    case B200AWQ_OK: return "ok";
    case B200AWQ_ERR_SHAPE: return "unsupported shape (need n % 8 == 0 [gemm: n % 128 == 0], k % 128 == 0, m >= 1)";
    case B200AWQ_ERR_GROUP: return "unsupported group size (only 128)";
    case B200AWQ_ERR_ALIGN: return "null or misaligned pointer (16-byte alignment required)";
    case B200AWQ_ERR_DTYPE: return "unsupported dtype (fp16 / bf16 only)";
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
