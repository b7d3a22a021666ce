// Python module `awq_inference_engine`: the reference's extension name and the two entry
// points WQLinear / tinychat call (awq/kernels/csrc/pybind.cpp:22-23), as a thin shim over
// the C ABI in include/b200awq.h.  Same positional signatures, same return tensors, same
// exception types as the reference host functions (gemv_cuda.cu:245-338,
// gemm_cuda.cu:1126-1236); additionally: launches on the CURRENT stream of the input's
// device (the reference uses the legacy default stream and no device guard), checks
// contiguity / shapes, and surfaces launch errors.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <algorithm>
#include <initializer_list>
#include <map>
#include <stdexcept>
#include <vector>

#include "../../include/b200awq.h"

namespace {

int dtype_code(const torch::Tensor& t, const char* fn) {
  if (t.scalar_type() == at::ScalarType::Half) return B200AWQ_DTYPE_F16;
  if (t.scalar_type() == at::ScalarType::BFloat16) return B200AWQ_DTYPE_BF16;
  // reference: dispatch_utils.cuh:13-17
  TORCH_CHECK(false, fn, " failed to dispatch data type ", t.scalar_type());
}

// Operands of one W4A16 product: in_feats [..., k] (m rows), qweight int16 [n / 4, k], scales / zeros [>= k / group, n]
// of in_feats' dtype, all CUDA and contiguous.  The output has in_feats' shape with n channels.
struct W4Shape {
  int64_t m, n, k;
  int dt;
  std::vector<int64_t> out_shape;
};

W4Shape w4a16_shape(const torch::Tensor& in, const torch::Tensor& kernel, const torch::Tensor& scales,
                    const torch::Tensor& zeros, int64_t group_size, const char* fn) {
  TORCH_CHECK(in.is_cuda() && kernel.is_cuda() && scales.is_cuda() && zeros.is_cuda(), "all tensors must be CUDA tensors");
  TORCH_CHECK(scales.scalar_type() == in.scalar_type());  // reference: gemv_cuda.cu:260, gemm_cuda.cu:1145
  TORCH_CHECK(zeros.scalar_type() == in.scalar_type());   // reference: gemv_cuda.cu:261, gemm_cuda.cu:1146
  TORCH_CHECK(kernel.scalar_type() == at::ScalarType::Short, "qweight must be int16 [N/4, K]");
  TORCH_CHECK(in.is_contiguous() && kernel.is_contiguous() && scales.is_contiguous() && zeros.is_contiguous(),
              "inputs must be contiguous");
  TORCH_CHECK(kernel.dim() == 2 && scales.dim() == 2 && zeros.dim() == 2 && in.dim() >= 1, "bad tensor ranks");
  const int dt = dtype_code(in, fn);
  const int64_t n = kernel.size(0) * 4, k = in.size(-1);  // n: reference gemm_cuda.cu:1133
  TORCH_CHECK(k > 0, fn, ": in_feats must have a non-empty last dimension");
  TORCH_CHECK(kernel.size(1) == k, "qweight does not match in_feats");
  TORCH_CHECK(scales.size(1) == n && zeros.size(1) == n && scales.size(0) * group_size >= k && zeros.size(0) * group_size >= k,
              "scales / zeros do not match (n, k, group)");
  std::vector<int64_t> out_shape = in.sizes().vec();
  out_shape.back() = n;
  return {in.numel() / k, n, k, dt, out_shape};
}

void raise(int code, bool is_gemv = false) {
  if (code == 0) return;
  // the reference throws std::runtime_error for unsupported batch / group (gemv_cuda.cu:329,334)
  if (is_gemv && code == B200AWQ_ERR_BATCH) throw std::runtime_error("Unsupported batch size for gemv kernel.\n");
  if (is_gemv && code == B200AWQ_ERR_GROUP) throw std::runtime_error("Unsupported group size for gemv kernel.\n");
  TORCH_CHECK(false, "b200awq: ", b200awq_strerror(code), " (code ", code, ")");
}

void* current_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

}  // namespace

torch::Tensor gemv_forward_cuda_new(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _scaling_factors,
                                    torch::Tensor _zeros, int m, int n, int k, int group_size) {
  const W4Shape s = w4a16_shape(_in_feats, _kernel, _scaling_factors, _zeros, group_size, "gemv_forward_cuda_new");
  TORCH_CHECK(s.k == k && s.m == m, "in_feats does not match (m, k)");
  TORCH_CHECK(s.n == n, "qweight does not match (n, k)");
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  raise(b200awq_w4a16_gemv(_in_feats.data_ptr(), _kernel.data_ptr(), _scaling_factors.data_ptr(), _zeros.data_ptr(),
                           out.data_ptr(), m, n, k, group_size, s.dt, current_stream()),
        true);
  return out;
}

torch::Tensor gemm_forward_cuda_new(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _scales,
                                    torch::Tensor _zeros) {
  const W4Shape s = w4a16_shape(_in_feats, _kernel, _scales, _zeros, 128, "gemm_forward_cuda_new");
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  if (s.m == 0) return out;
  const size_t ws_bytes = b200awq_w4a16_gemm_workspace_bytes((int)s.m, (int)s.n, (int)s.k);
  at::Tensor ws;
  if (ws_bytes) ws = torch::empty({(int64_t)ws_bytes}, _in_feats.options().dtype(torch::kUInt8));
  raise(b200awq_w4a16_gemm(_in_feats.data_ptr(), _kernel.data_ptr(), _scales.data_ptr(), _zeros.data_ptr(), out.data_ptr(),
                           (int)s.m, (int)s.n, (int)s.k, 128, s.dt, ws_bytes ? ws.data_ptr() : nullptr, ws_bytes, current_stream()));
  return out;
}

// New entry (no counterpart in the reference's extension): WQLinear.forward's engine call with its `out + bias`
// (awq/quantize/qmodule.py:205-221) and the decoder block's `residual + out` in one launch, bit-identical to the
// engine call followed by those two adds.  The reference's dispatch rule picks the GEMV (m < 8) or GEMM routes.
// bias [N] and residual (the output's shape) must have in_feats' dtype and device and be contiguous.
torch::Tensor w4a16_linear_forward_cuda(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _scales,
                                        torch::Tensor _zeros, int64_t group_size, c10::optional<torch::Tensor> bias,
                                        c10::optional<torch::Tensor> residual) {
  const char* fn = "w4a16_linear_forward_cuda";
  const W4Shape s = w4a16_shape(_in_feats, _kernel, _scales, _zeros, group_size, fn);
  for (const c10::optional<torch::Tensor>* t : {&bias, &residual}) {
    if (!t->has_value()) continue;
    const torch::Tensor& v = t->value();
    TORCH_CHECK(v.is_cuda() && v.device() == _in_feats.device(), fn, ": bias / residual must be on in_feats' device");
    TORCH_CHECK(v.scalar_type() == _in_feats.scalar_type(), fn, ": bias / residual must have in_feats' dtype");
    TORCH_CHECK(v.is_contiguous(), fn, ": bias / residual must be contiguous");
  }
  if (bias.has_value()) TORCH_CHECK(bias->dim() == 1 && bias->size(0) == s.n, fn, ": bias must be [", s.n, "]");
  if (residual.has_value())
    TORCH_CHECK(residual->sizes() == torch::IntArrayRef(s.out_shape), fn, ": residual must have the output's shape ",
                torch::IntArrayRef(s.out_shape));
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  if (s.m == 0) return out;
  raise(b200awq_w4a16_linear(_in_feats.data_ptr(), _kernel.data_ptr(), _scales.data_ptr(), _zeros.data_ptr(),
                             bias.has_value() ? bias->data_ptr() : nullptr,
                             residual.has_value() ? residual->data_ptr() : nullptr, out.data_ptr(), (int)s.m, (int)s.n,
                             (int)s.k, (int)group_size, s.dt, current_stream()));
  return out;
}

// New entry (no counterpart in the reference's extension): the whole of QuantLlamaMLP.our_llama_mlp
// (tinychat/modules/fused_mlp.py:36-83) in one call.  The zeros tensors are used as given.
torch::Tensor mlp_front_forward_cuda(torch::Tensor _in_feats, torch::Tensor _gate_kernel, torch::Tensor _gate_scales,
                                     torch::Tensor _gate_zeros, torch::Tensor _up_kernel, torch::Tensor _up_scales,
                                     torch::Tensor _up_zeros) {
  const char* fn = "mlp_front_forward_cuda";
  const W4Shape s = w4a16_shape(_in_feats, _gate_kernel, _gate_scales, _gate_zeros, 128, fn);
  TORCH_CHECK(w4a16_shape(_in_feats, _up_kernel, _up_scales, _up_zeros, 128, fn).n == s.n, "qweights do not match");
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  if (s.m == 0) return out;
  // One fp16 token first tries the fused kernel, which needs no workspace; B200AWQ_ERR_WORKSPACE means that it declined
  // the shape and the composed path needs one.
  auto call = [&](bool with_workspace) {
    const size_t bytes = with_workspace ? b200awq_w4a16_mlp_front_workspace_bytes((int)s.m, (int)s.n, (int)s.k) : 0;
    const at::Tensor ws = bytes ? torch::empty({(int64_t)bytes}, _in_feats.options().dtype(torch::kUInt8)) : at::Tensor();
    return b200awq_w4a16_mlp_front(_in_feats.data_ptr(), _gate_kernel.data_ptr(), _gate_scales.data_ptr(),
                                   _gate_zeros.data_ptr(), _up_kernel.data_ptr(), _up_scales.data_ptr(), _up_zeros.data_ptr(),
                                   out.data_ptr(), (int)s.m, (int)s.n, (int)s.k, 128, s.dt, bytes ? ws.data_ptr() : nullptr,
                                   bytes, current_stream());
  };
  const bool fused_first = s.m == 1 && s.dt == B200AWQ_DTYPE_F16;
  int rc = call(!fused_first);
  if (fused_first && rc == B200AWQ_ERR_WORKSPACE) rc = call(true);
  raise(rc);
  return out;
}

namespace {
// gamma [k] of in_feats' dtype and device, contiguous (the checks of layernorm_forward_cuda); a workspace of `bytes` from
// the caching allocator
at::Tensor norm_workspace(const torch::Tensor& in, const torch::Tensor& gamma, int64_t k, size_t bytes, const char* fn) {
  TORCH_CHECK(gamma.is_cuda() && gamma.device() == in.device(), fn, ": gamma must be on in_feats' device");
  TORCH_CHECK(gamma.scalar_type() == in.scalar_type(), fn, ": gamma must have in_feats' dtype");
  TORCH_CHECK(gamma.is_contiguous() && gamma.numel() == k, fn, ": gamma must be contiguous with ", k, " elements");
  return torch::empty({(int64_t)std::max<size_t>(bytes, 16)}, in.options().dtype(torch::kUInt8));
}
}  // namespace

// New entry: tinychat's `input_layernorm(x)` followed by the q/k/v projection (+ bias) in one call, bit-identical to
// layernorm_forward_cuda followed by w4a16_linear_forward_cuda (include/b200awq.h, b200awq_w4a16_norm_linear).
torch::Tensor rmsnorm_w4a16_linear_forward_cuda(torch::Tensor _in_feats, torch::Tensor _gamma, double eps, torch::Tensor _kernel,
                                                torch::Tensor _scales, torch::Tensor _zeros, int64_t group_size,
                                                c10::optional<torch::Tensor> bias) {
  const char* fn = "rmsnorm_w4a16_linear_forward_cuda";
  const W4Shape s = w4a16_shape(_in_feats, _kernel, _scales, _zeros, group_size, fn);
  if (bias.has_value()) {
    TORCH_CHECK(bias->is_cuda() && bias->device() == _in_feats.device(), fn, ": bias must be on in_feats' device");
    TORCH_CHECK(bias->scalar_type() == _in_feats.scalar_type(), fn, ": bias must have in_feats' dtype");
    TORCH_CHECK(bias->is_contiguous() && bias->dim() == 1 && bias->size(0) == s.n, fn, ": bias must be contiguous [", s.n, "]");
  }
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  const size_t bytes = (size_t)s.m * (size_t)s.k * 2;  // x^ for the routes without the prologue (include/b200awq.h)
  const at::Tensor ws = norm_workspace(_in_feats, _gamma, s.k, bytes, fn);
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  if (s.m == 0) return out;
  raise(b200awq_w4a16_norm_linear(_in_feats.data_ptr(), _gamma.data_ptr(), (float)eps, _kernel.data_ptr(), _scales.data_ptr(),
                                  _zeros.data_ptr(), bias.has_value() ? bias->data_ptr() : nullptr, out.data_ptr(), (int)s.m,
                                  (int)s.n, (int)s.k, (int)group_size, s.dt, ws.data_ptr(), bytes, current_stream()));
  return out;
}

// New entry: tinychat's `post_attention_layernorm(x)` followed by QuantLlamaMLP.our_llama_mlp in one call, bit-identical
// to layernorm_forward_cuda followed by mlp_front_forward_cuda (b200awq_w4a16_norm_mlp_front).
torch::Tensor rmsnorm_mlp_front_forward_cuda(torch::Tensor _in_feats, torch::Tensor _gamma, double eps,
                                             torch::Tensor _gate_kernel, torch::Tensor _gate_scales, torch::Tensor _gate_zeros,
                                             torch::Tensor _up_kernel, torch::Tensor _up_scales, torch::Tensor _up_zeros) {
  const char* fn = "rmsnorm_mlp_front_forward_cuda";
  const W4Shape s = w4a16_shape(_in_feats, _gate_kernel, _gate_scales, _gate_zeros, 128, fn);
  TORCH_CHECK(w4a16_shape(_in_feats, _up_kernel, _up_scales, _up_zeros, 128, fn).n == s.n, "qweights do not match");
  const c10::cuda::CUDAGuard guard(_in_feats.device());
  const size_t bytes = b200awq_w4a16_norm_workspace_bytes((int)s.m, (int)s.n, (int)s.k);
  const at::Tensor ws = norm_workspace(_in_feats, _gamma, s.k, bytes, fn);
  at::Tensor out = torch::empty(s.out_shape, _in_feats.options());
  if (s.m == 0) return out;
  raise(b200awq_w4a16_norm_mlp_front(_in_feats.data_ptr(), _gamma.data_ptr(), (float)eps, _gate_kernel.data_ptr(),
                                     _gate_scales.data_ptr(), _gate_zeros.data_ptr(), _up_kernel.data_ptr(),
                                     _up_scales.data_ptr(), _up_zeros.data_ptr(), out.data_ptr(), (int)s.m, (int)s.n, (int)s.k,
                                     128, s.dt, ws.data_ptr(), bytes, current_stream()));
  return out;
}

// reference: awq/kernels/csrc/layernorm/layernorm.cu:111-131 (input [b, s, c], gamma [c], out like input; returns
// nothing).  Same dtype checks; additionally any rank >= 1 is accepted (rows = numel / last dim), the launch goes to
// the current stream, and contiguity is checked instead of assumed.
void layernorm_forward_cuda(torch::Tensor _input, torch::Tensor _gamma, torch::Tensor _out, float eps) {
  TORCH_CHECK(_input.is_cuda() && _gamma.is_cuda() && _out.is_cuda(), "all tensors must be CUDA tensors");
  const int dt = dtype_code(_input, "layernorm_forward_cuda");
  TORCH_CHECK(_gamma.scalar_type() == _input.scalar_type());  // layernorm.cu:122
  TORCH_CHECK(_out.scalar_type() == _input.scalar_type());    // layernorm.cu:123
  TORCH_CHECK(_input.dim() >= 1 && _input.is_contiguous() && _out.is_contiguous() && _gamma.is_contiguous(),
              "inputs must be contiguous");
  const int64_t n = _input.size(-1);
  TORCH_CHECK(_gamma.numel() == n && _out.numel() == _input.numel(), "gamma / out do not match input");
  if (_input.numel() == 0) return;
  const c10::cuda::CUDAGuard guard(_input.device());
  raise(b200awq_rmsnorm(_input.data_ptr(), _gamma.data_ptr(), _out.data_ptr(), (int)(_input.numel() / n), (int)n, eps, dt,
                        current_stream()));
}

namespace {

// The attention workspace of the current stream on `like`'s device, at least `need` bytes: one zero-initialised buffer
// per (device, stream), shared by single_query_attention and the split-key attention behind flash_attn_func (their
// counter blocks coincide and every launch leaves its counters zero).  When a call needs more, a new zeroed buffer of
// at least twice the size takes over, and the ones it replaces are kept, never freed: a CUDA graph that captured a call
// on this stream keeps launching with the buffer it captured, which must stay valid (its counters stay zero, since
// every launch leaves them so).  The doubling bounds how many buffers are kept.
// Leaked on purpose: CUDA tensors must not be destroyed by static destructors at interpreter exit.
const torch::Tensor& attention_workspace(const torch::Tensor& like, size_t need) {
  struct Buffers {
    torch::Tensor current;
    std::vector<torch::Tensor> replaced;  // still referenced by graphs captured before a growth
  };
  static auto& workspaces = *new std::map<std::pair<int, void*>, Buffers>();
  Buffers& w = workspaces[std::make_pair((int)like.get_device(), current_stream())];
  const size_t have = w.current.defined() ? (size_t)w.current.numel() : 0;
  if (have < need) {
    if (w.current.defined()) w.replaced.push_back(w.current);
    w.current = torch::zeros({(int64_t)std::max(need, 2 * have)}, like.options().dtype(torch::kUInt8));
  }
  return w.current;
}

}  // namespace

// reference: awq/kernels/csrc/attention/ft_attention.cpp:112-184 (same checks, same argument order and defaults,
// pybind.cpp:24-27).  alibi_slopes must be None; fp32 tensors are not dispatched.  Like the reference, any
// nheads % nheads_kv == 0 and any headdim % 8 == 0 up to 256 run.
torch::Tensor single_query_attention(const torch::Tensor q, const torch::Tensor k, const torch::Tensor v, torch::Tensor k_cache,
                                     torch::Tensor v_cache, c10::optional<const torch::Tensor> length_per_sample_,
                                     c10::optional<const torch::Tensor> alibi_slopes_, const int timestep,
                                     const int rotary_embedding_dim, const float rotary_base, const float rotary_scale,
                                     const bool neox_rotary_style) {
  TORCH_CHECK(q.is_cuda() && k.is_cuda() && v.is_cuda() && k_cache.is_cuda() && v_cache.is_cuda(), "tensors must be on CUDA");
  const int batch_size = v_cache.size(0), nheads = q.size(1), nheads_kv = v_cache.size(1);
  const int memory_max_seqlen = v_cache.size(2), headdim = v_cache.size(3);
  TORCH_CHECK(q.sizes() == torch::IntArrayRef({batch_size, nheads, headdim}), "q must have shape (batch, nheads, headdim)");
  TORCH_CHECK(k.sizes() == torch::IntArrayRef({batch_size, nheads_kv, headdim}), "k must have shape (batch, nheads_kv, headdim)");
  TORCH_CHECK(v.sizes() == torch::IntArrayRef({batch_size, nheads_kv, headdim}), "v must have shape (batch, nheads_kv, headdim)");
  TORCH_CHECK(k_cache.sizes() == torch::IntArrayRef({batch_size, nheads_kv, headdim / 8, memory_max_seqlen, 8}),
              "k_cache must have shape (batch, nheads_kv, headdim / 8, max_seqlen, 8)");
  TORCH_CHECK(q.stride(2) == 1 && q.stride(1) == headdim);
  TORCH_CHECK(k.stride(2) == 1 && k.stride(1) == headdim);
  TORCH_CHECK(v.stride(2) == 1 && v.stride(1) == headdim);
  TORCH_CHECK(v_cache.is_contiguous() && k_cache.is_contiguous(), "caches must be contiguous");
  const int dt = dtype_code(q, "single_query_attention");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type() &&
              k_cache.scalar_type() == q.scalar_type() && v_cache.scalar_type() == q.scalar_type());
  TORCH_CHECK(!alibi_slopes_.has_value(), "b200awq: alibi_slopes is not supported by this build");
  const int* lps = nullptr;
  if (length_per_sample_.has_value()) {
    const auto& l = length_per_sample_.value();
    TORCH_CHECK(l.is_cuda() && l.is_contiguous() && l.dtype() == torch::kInt32 && l.numel() == batch_size);
    lps = l.data_ptr<int>();
  }
  const c10::cuda::CUDAGuard guard(q.device());
  torch::Tensor out = torch::empty({batch_size, nheads, headdim}, q.options());
  const torch::Tensor& ws = attention_workspace(
      q, b200awq_single_query_attention_workspace_bytes(batch_size, nheads, nheads_kv, headdim, memory_max_seqlen));
  raise(b200awq_single_query_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                       out.data_ptr(), lps, batch_size, nheads, nheads_kv, headdim, memory_max_seqlen, timestep,
                                       (long long)q.stride(0), (long long)k.stride(0), (long long)v.stride(0), rotary_embedding_dim, rotary_base, rotary_scale,
                                       neox_rotary_style ? 1 : 0, dt, ws.data_ptr(), (size_t)ws.numel(), current_stream()));
  return out;
}

// reference: awq/kernels/csrc/rope_new/fused_rope_with_pos.cu:243-285
at::Tensor fused_rope_with_pos_forward_func(const at::Tensor& input, const at::Tensor& freqs, const bool transpose_output_memory) {
  TORCH_CHECK(input.is_cuda() && freqs.is_cuda() && input.dim() == 4, "input must be a CUDA tensor [s, b, h, d]");
  TORCH_CHECK(freqs.scalar_type() == at::ScalarType::Float && freqs.is_contiguous(), "freqs must be contiguous float32");
  const int dt = dtype_code(input, "fused_rope_with_pos_forward_func");
  const int s = input.size(0), b = input.size(1), h = input.size(2), d = input.size(3), d2 = freqs.size(-1);
  TORCH_CHECK(freqs.numel() >= (int64_t)s * b * d2, "freqs must hold s * b * d2 angles");
  auto opts = input.options().requires_grad(false);
  at::Tensor output = transpose_output_memory ? torch::empty({b, s, h, d}, opts).transpose(0, 1) : torch::empty({s, b, h, d}, opts);
  const long long is[4] = {input.stride(0), input.stride(1), input.stride(2), input.stride(3)};
  const long long os[4] = {output.stride(0), output.stride(1), output.stride(2), output.stride(3)};
  const c10::cuda::CUDAGuard guard(input.device());
  raise(b200awq_rope_with_pos(input.data_ptr(), freqs.data_ptr<float>(), output.data_ptr(), s, b, h, d, d2, is, os, dt,
                              current_stream()));
  return output;
}

// reference: awq/kernels/csrc/position_embedding/pos_encoding_kernels.cu:56-88 (in place, returns nothing)
void rotary_embedding_neox(at::Tensor& positions, at::Tensor& query, at::Tensor& key, int head_size, at::Tensor& cos_sin_cache) {
  TORCH_CHECK(positions.is_cuda() && query.is_cuda() && key.is_cuda() && cos_sin_cache.is_cuda(), "all tensors must be CUDA tensors");
  TORCH_CHECK(positions.scalar_type() == at::ScalarType::Long && positions.is_contiguous(), "positions must be contiguous int64");
  const int dt = dtype_code(query, "rotary_embedding_neox");
  TORCH_CHECK(key.scalar_type() == query.scalar_type() && cos_sin_cache.scalar_type() == query.scalar_type(),
              "query, key and cos_sin_cache must have one dtype");
  TORCH_CHECK(query.is_contiguous() && key.is_contiguous() && cos_sin_cache.is_contiguous(), "tensors must be contiguous");
  TORCH_CHECK(query.dim() >= 3 && key.dim() >= 3 && cos_sin_cache.dim() == 2, "query / key [b, tokens, ..., heads, head_size]");
  TORCH_CHECK(query.size(-1) == head_size && key.size(-1) == head_size, "last dimension must be head_size");
  const int64_t tokens = query.size(0) * query.size(1);  // reference :63
  const int64_t q_heads = query.size(-2), k_heads = key.size(-2);
  const int64_t rot_dim = cos_sin_cache.size(1);         // reference :64
  TORCH_CHECK(query.numel() == tokens * q_heads * head_size && key.numel() == tokens * k_heads * head_size,
              "query / key must hold tokens x heads x head_size elements");
  TORCH_CHECK(positions.numel() >= tokens, "one position per token");
  const c10::cuda::CUDAGuard guard(query.device());
  raise(b200awq_rotary_embedding_neox(reinterpret_cast<const long long*>(positions.data_ptr<int64_t>()), query.data_ptr(),
                                      key.data_ptr(), cos_sin_cache.data_ptr(), (int)tokens, (int)q_heads, (int)k_heads,
                                      head_size, (int)rot_dim, q_heads * head_size, k_heads * head_size, dt, current_stream()));
}

// ---------------------------------------------------------------- W8A8 (w8a8/*.cu of the reference)
// Same argument order, return values and keyword names as the reference (csrc/pybind.cpp:30-37).  Unlike the
// reference, shapes, dtypes and contiguity are checked, and the launches go to the current stream of the input's
// device under a device guard.  fp32 activations are not dispatched.
namespace {

void check_cuda_contig(std::initializer_list<const torch::Tensor*> ts, const char* fn) {
  for (const torch::Tensor* t : ts) {
    TORCH_CHECK(t->is_cuda(), fn, ": all tensors must be CUDA tensors");
    TORCH_CHECK(t->is_contiguous(), fn, ": all tensors must be contiguous");
  }
}
void check_dtype(const torch::Tensor& t, at::ScalarType want, const char* fn, const char* what) {
  TORCH_CHECK(t.scalar_type() == want, fn, ": ", what, " must be ", want, ", got ", t.scalar_type());
}

// layer_scale / residual: w8a8_linear_forward_cuda's operands (b200awq_w8a8_linear); without either this is the
// reference's GEMM call (b200awq_w8a8_gemm).
void w8a8_gemm(const torch::Tensor& in, const torch::Tensor& kernel, const torch::Tensor& wscales, const torch::Tensor& ascales,
               torch::Tensor& out, const torch::Tensor* bias, const char* fn, const torch::Tensor* layer_scale = nullptr,
               const torch::Tensor* residual = nullptr) {
  std::initializer_list<const torch::Tensor*> all = {&in, &kernel, &wscales, &ascales, &out};
  check_cuda_contig(all, fn);
  if (bias) check_cuda_contig({bias}, fn);
  check_dtype(in, at::ScalarType::Char, fn, "in_feats");
  check_dtype(kernel, at::ScalarType::Char, fn, "kernel");
  check_dtype(wscales, at::ScalarType::Half, fn, "wscales");
  check_dtype(ascales, at::ScalarType::Half, fn, "ascales");
  check_dtype(out, at::ScalarType::Half, fn, "out_feats");
  if (bias) check_dtype(*bias, at::ScalarType::Half, fn, "bias");
  TORCH_CHECK(in.dim() == 2 && kernel.dim() == 2 && out.dim() >= 2, fn, ": in_feats / kernel must be 2-D, out_feats >= 2-D");
  // reference: M, N from out_feats, K from in_feats (w8a8_gemm_cuda.cu:907-927)
  const int64_t m = out.size(-2), n = out.size(-1), k = in.size(1);
  TORCH_CHECK(out.numel() == m * n, fn, ": out_feats must be [M, N]");
  TORCH_CHECK(in.size(0) == m, fn, ": in_feats has ", in.size(0), " rows, out_feats ", m);
  TORCH_CHECK(kernel.size(0) == n && kernel.size(1) == k, fn, ": kernel must be [N, K] = [", n, ", ", k, "]");
  TORCH_CHECK(wscales.numel() >= n && ascales.numel() >= m, fn, ": wscales needs N, ascales M elements");
  if (bias) TORCH_CHECK(bias->numel() >= n, fn, ": bias needs N elements");
  for (const torch::Tensor* t : {layer_scale, residual}) {
    if (!t) continue;
    check_cuda_contig({t}, fn);
    TORCH_CHECK(t->device() == out.device(), fn, ": layer_scale / residual must be on out_feats' device");
    check_dtype(*t, at::ScalarType::Half, fn, t == layer_scale ? "layer_scale" : "residual");
  }
  if (layer_scale) TORCH_CHECK(layer_scale->dim() == 1 && layer_scale->size(0) == n, fn, ": layer_scale must be [", n, "]");
  if (residual) {
    TORCH_CHECK(residual->sizes() == out.sizes(), fn, ": residual must have out_feats' shape ", out.sizes());
    const uintptr_t r = reinterpret_cast<uintptr_t>(residual->data_ptr()), o = reinterpret_cast<uintptr_t>(out.data_ptr());
    const uintptr_t bytes = (uintptr_t)out.numel() * 2u;
    TORCH_CHECK(bytes == 0 || r >= o + bytes || o >= r + bytes, fn, ": residual must not share memory with out_feats");
  }
  if (m == 0 || n == 0) return;
  const c10::cuda::CUDAGuard guard(in.device());
  void* bp = bias ? bias->data_ptr() : nullptr;
  if (layer_scale || residual)
    raise(b200awq_w8a8_linear(in.data_ptr(), kernel.data_ptr(), wscales.data_ptr(), ascales.data_ptr(), bp,
                              layer_scale ? layer_scale->data_ptr() : nullptr, residual ? residual->data_ptr() : nullptr,
                              out.data_ptr(), (int)m, (int)n, (int)k, current_stream()));
  else
    raise(b200awq_w8a8_gemm(in.data_ptr(), kernel.data_ptr(), wscales.data_ptr(), ascales.data_ptr(), bp, out.data_ptr(),
                            (int)m, (int)n, (int)k, current_stream()));
}

int act_dtype(const torch::Tensor& t, const char* fn) {
  TORCH_CHECK(t.scalar_type() != at::ScalarType::Float, fn, ": fp32 activations are not supported by this build");
  return dtype_code(t, fn);
}

}  // namespace

// reference: w8a8/w8a8_gemm_cuda.cu:907-953
void w8a8_gemm_forward_cuda(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _wscales, torch::Tensor _ascales,
                            torch::Tensor _out_feats) {
  w8a8_gemm(_in_feats, _kernel, _wscales, _ascales, _out_feats, nullptr, "w8a8_gemm_forward_cuda");
}

// reference: w8a8/w8a8_gemm_cuda.cu:586-633
void w8a8_gemm_fuse_bias_forward_cuda(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _wscales,
                                      torch::Tensor _ascales, torch::Tensor _out_feats, torch::Tensor _bias) {
  w8a8_gemm(_in_feats, _kernel, _wscales, _ascales, _out_feats, &_bias, "w8a8_gemm_fuse_bias_forward_cuda");
}

// New entry (no counterpart in the reference's extension): w8a8_gemm[_fuse_bias]_forward_cuda followed by the vision
// encoder layers' `out * ls` and `residual + out`, in the GEMM's launch and bit-identical to those PyTorch ops.  Writes
// out_feats like the reference's W8A8 entries.  layer_scale [N] and residual (out_feats' shape) are fp16, contiguous and
// on out_feats' device; residual must not share memory with out_feats.
void w8a8_linear_forward_cuda(torch::Tensor _in_feats, torch::Tensor _kernel, torch::Tensor _wscales, torch::Tensor _ascales,
                              torch::Tensor _out_feats, c10::optional<torch::Tensor> bias,
                              c10::optional<torch::Tensor> layer_scale, c10::optional<torch::Tensor> residual) {
  w8a8_gemm(_in_feats, _kernel, _wscales, _ascales, _out_feats, bias.has_value() ? &*bias : nullptr, "w8a8_linear_forward_cuda",
            layer_scale.has_value() ? &*layer_scale : nullptr, residual.has_value() ? &*residual : nullptr);
}

// reference: w8a8/quantization.cu:97-112 (out int8 like input, scale fp16 [tokens])
void invoke_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& scale) {
  const char* fn = "invoke_quant";
  check_cuda_contig({&out, &input, &scale}, fn);
  const int dt = act_dtype(input, fn);
  check_dtype(out, at::ScalarType::Char, fn, "out");
  check_dtype(scale, at::ScalarType::Half, fn, "scale");
  TORCH_CHECK(input.dim() >= 1 && input.size(-1) > 0, fn, ": input must have a last dimension");
  const int64_t n = input.size(-1), m = input.numel() / n;
  TORCH_CHECK(out.numel() == input.numel() && scale.numel() >= m, fn, ": out must match input, scale needs one per token");
  const c10::cuda::CUDAGuard guard(input.device());
  raise(b200awq_quant_per_token(input.data_ptr(), out.data_ptr(), scale.data_ptr(), (int)m, (int)n, dt, current_stream()));
}

// reference: w8a8/layernorm.cu:193-231
void rms_norm_general(torch::Tensor& out, torch::Tensor& input, torch::Tensor& weight, torch::Tensor& bias, torch::Tensor& scaling,
                      float epsilon, bool use_per_token_quant) {
  const char* fn = "rms_norm_general";
  check_cuda_contig({&out, &input, &weight, &scaling}, fn);
  const int dt = act_dtype(input, fn);
  check_dtype(out, at::ScalarType::Char, fn, "out");
  check_dtype(scaling, at::ScalarType::Half, fn, "scaling");
  check_dtype(weight, input.scalar_type(), fn, "weight");
  TORCH_CHECK(input.dim() >= 1 && input.size(-1) > 0, fn, ": input must have a last dimension");
  const int64_t n = input.size(-1), m = input.numel() / n;
  TORCH_CHECK(out.numel() == input.numel() && weight.numel() == n, fn, ": out must match input, weight must be [hidden]");
  const void* beta = nullptr;
  if (use_per_token_quant) {  // the per-tensor branch of the reference ignores bias
    check_cuda_contig({&bias}, fn);
    check_dtype(bias, input.scalar_type(), fn, "bias");
    TORCH_CHECK(bias.numel() == n, fn, ": bias must be [hidden]");
    beta = bias.data_ptr();
    TORCH_CHECK(scaling.numel() >= m, fn, ": scaling needs one element per token");
  } else {
    TORCH_CHECK(scaling.numel() >= 1, fn, ": scaling needs one element");
  }
  const c10::cuda::CUDAGuard guard(input.device());
  raise(b200awq_layernorm_quant(input.data_ptr(), weight.data_ptr(), beta, out.data_ptr(), scaling.data_ptr(), (int)m, (int)n,
                                epsilon, use_per_token_quant ? 1 : 0, dt, current_stream()));
}

// reference: w8a8/act.cu:120-141 (input [..., 2d] -> new tensor [..., d])
torch::Tensor silu_and_mul(torch::Tensor& input) {
  const char* fn = "silu_and_mul";
  check_cuda_contig({&input}, fn);
  const int dt = act_dtype(input, fn);
  TORCH_CHECK(input.dim() >= 1 && input.size(-1) % 2 == 0, fn, ": last dimension must be even");
  const int64_t d = input.size(-1) / 2, m = d ? input.numel() / (2 * d) : 0;
  std::vector<int64_t> shape = input.sizes().vec();
  shape.back() = d;
  torch::Tensor out = torch::empty(shape, input.options());
  if (m == 0 || d == 0) return out;
  const c10::cuda::CUDAGuard guard(input.device());
  raise(b200awq_silu_and_mul(input.data_ptr(), out.data_ptr(), (int)m, (int)d, dt, current_stream()));
  return out;
}

// reference: w8a8/act.cu:82-95 (fp16 only)
void gelu_and_quant(torch::Tensor& out, torch::Tensor& input, torch::Tensor& scale_out, torch::Tensor& tmp) {
  const char* fn = "gelu_and_quant";
  check_cuda_contig({&out, &input, &scale_out, &tmp}, fn);
  check_dtype(input, at::ScalarType::Half, fn, "input");
  check_dtype(tmp, at::ScalarType::Half, fn, "tmp");
  check_dtype(scale_out, at::ScalarType::Half, fn, "scale_out");
  check_dtype(out, at::ScalarType::Char, fn, "out");
  TORCH_CHECK(input.dim() >= 1 && input.size(-1) > 0, fn, ": input must have a last dimension");
  const int64_t n = input.size(-1), m = input.numel() / n;
  TORCH_CHECK(out.numel() == input.numel() && tmp.numel() >= input.numel() && scale_out.numel() >= m, fn,
              ": out / tmp must match input, scale_out needs one per token");
  const c10::cuda::CUDAGuard guard(input.device());
  raise(b200awq_gelu_quant(input.data_ptr(), out.data_ptr(), scale_out.data_ptr(), tmp.data_ptr(), (int)m, (int)n,
                           current_stream()));
}

// ---------------------------------------------------------------- attention over many queries
// flash-attn 2.8.3's flash_attn_func / flash_attn_varlen_qkvpacked_func (flash_attn/flash_attn_interface.py): same
// names, positional order and keyword names for the parameters tinychat's callers pass.  Fixed-length calls with few
// queries per KV head (decode over a long context) take the split-key kernel, everything else the prefill kernel.  Like flash-attn, an operand
// whose last dimension is not contiguous, or whose strides or pointer the TMA cannot take, is copied contiguous first;
// views into a fused qkv buffer are used in place.
namespace {

torch::Tensor tma_ready(const torch::Tensor& t) {
  const bool ok = t.stride(-1) == 1 && (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15u) == 0 &&
                  t.stride(0) % 8 == 0 && t.stride(1) % 8 == 0 && t.stride(2) % 8 == 0;
  return ok ? t : t.clone(at::MemoryFormat::Contiguous);  // a fresh allocation: aligned, dense strides
}

void check_attention_args(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v, double dropout_p,
                          const char* fn) {
  TORCH_CHECK(q.is_cuda() && k.is_cuda() && v.is_cuda(), fn, ": q, k, v must be CUDA tensors");
  TORCH_CHECK(dropout_p == 0.0, fn, ": dropout is not supported by this build (dropout_p must be 0)");
  TORCH_CHECK(q.scalar_type() == at::ScalarType::Half || q.scalar_type() == at::ScalarType::BFloat16, fn,
              ": only fp16 and bf16 are supported");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(), fn,
              ": query and key / value must have the same dtype");
}

// What both attention wrappers hand the C entries for q, under the device guard: q as the TMA can read it, its strides,
// the softmax scale (flash-attn's default 1 / sqrt(head_dim)) and the dtype code.
struct AttentionQuery {
  torch::Tensor q;
  long long strides[3];
  float scale;
  int dt;
};

AttentionQuery attention_query(const torch::Tensor& q_in, c10::optional<double> softmax_scale, const char* fn) {
  torch::Tensor q = tma_ready(q_in);
  const float scale = softmax_scale.has_value() ? (float)softmax_scale.value() : 1.0f / std::sqrt((float)q.size(-1));
  return {q, {q.stride(0), q.stride(1), q.stride(2)}, scale, dtype_code(q, fn)};
}

// attention_workspace() when a call needs one: (nullptr, 0) for need == 0
std::pair<void*, size_t> attention_workspace_if(const torch::Tensor& like, size_t need) {
  if (!need) return {nullptr, 0};
  const torch::Tensor& ws = attention_workspace(like, need);
  return {ws.data_ptr(), (size_t)ws.numel()};
}

torch::Tensor run_prefill_attention(const torch::Tensor& q_in, const torch::Tensor& k_in, const torch::Tensor& v_in,
                                    torch::Tensor& out, const int* cu_seqlens, int batch, int seqlen_q, int seqlen_k,
                                    c10::optional<double> softmax_scale, bool causal, const char* fn) {
  const c10::cuda::CUDAGuard guard(q_in.device());
  const AttentionQuery a = attention_query(q_in, softmax_scale, fn);
  const torch::Tensor& q = a.q;
  const torch::Tensor k = tma_ready(k_in), v = tma_ready(v_in);
  const int heads = q.size(-2), kv_heads = k.size(-2), d = q.size(-1);
  const long long ks[3] = {k.stride(0), k.stride(1), k.stride(2)};
  const long long vs[3] = {v.stride(0), v.stride(1), v.stride(2)};
  int rc = B200AWQ_ERR_SHAPE;
  if (!cu_seqlens) {  // few queries per KV head: the split-key kernel; outside its envelope the prefill kernel
    const auto ws = attention_workspace_if(
        q, b200awq_splitkv_attention_workspace_bytes(batch, seqlen_q, seqlen_k, heads, kv_heads, d));
    rc = b200awq_splitkv_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), batch, seqlen_q, seqlen_k, heads,
                                   kv_heads, d, a.strides, ks, vs, a.scale, causal ? 1 : 0, a.dt, ws.first, ws.second,
                                   current_stream());
  }
  if (rc == B200AWQ_ERR_SHAPE)
    rc = b200awq_prefill_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), cu_seqlens, cu_seqlens, batch,
                                   seqlen_q, seqlen_k, heads, kv_heads, d, a.strides, ks, vs, a.scale, causal ? 1 : 0, a.dt,
                                   current_stream());
  raise(rc);
  return out;
}

// The KV caches of kv_cache_attention and rope_kv_store on `like`'s device, for head_dim d: the layout follows from
// k_cache's rank (5-D: tinychat's decode cache k [Bc, Hkv, D / 8, Lmax, 8], v [Bc, Hkv, Lmax, D]; 4-D: long_forward's
// [Bc, Lmax, Hkv, D] both), caches contiguous.
struct KvCaches {
  int layout, kv_heads;
  int64_t rows, max_len;
};

KvCaches kv_caches(const torch::Tensor& like, const torch::Tensor& k_cache, const torch::Tensor& v_cache, int64_t d,
                   const char* fn) {
  TORCH_CHECK(k_cache.is_contiguous() && v_cache.is_contiguous(), fn, ": caches must be contiguous");
  TORCH_CHECK(k_cache.device() == like.device() && v_cache.device() == like.device(), fn, ": tensors must be on one device");
  KvCaches c;
  if (k_cache.dim() == 5) {
    c.layout = B200AWQ_KV_FT;
    c.rows = k_cache.size(0), c.kv_heads = (int)k_cache.size(1), c.max_len = k_cache.size(3);
    TORCH_CHECK(k_cache.size(2) * 8 == d && k_cache.size(4) == 8, fn, ": k_cache must be [batch, kv_heads, head_dim / 8, max_len, 8]");
    TORCH_CHECK(v_cache.dim() == 4 && v_cache.sizes() == torch::IntArrayRef({c.rows, c.kv_heads, c.max_len, d}), fn,
                ": v_cache must be [batch, kv_heads, max_len, head_dim]");
  } else {
    TORCH_CHECK(k_cache.dim() == 4, fn, ": k_cache must be 5-D (FasterTransformer layout) or 4-D [batch, max_len, kv_heads, head_dim]");
    c.layout = B200AWQ_KV_BTHD;
    c.rows = k_cache.size(0), c.max_len = k_cache.size(1), c.kv_heads = (int)k_cache.size(2);
    TORCH_CHECK(k_cache.size(3) == d && v_cache.sizes() == k_cache.sizes(), fn, ": k_cache / v_cache must be [batch, max_len, kv_heads, head_dim]");
  }
  return c;
}

}  // namespace

// q [B, Sq, H, D], k / v [B, Sk, Hkv, D] -> out [B, Sq, H, D]
torch::Tensor flash_attn_func(const torch::Tensor& q, const torch::Tensor& k, const torch::Tensor& v, double dropout_p,
                              c10::optional<double> softmax_scale, bool causal) {
  const char* fn = "flash_attn_func";
  check_attention_args(q, k, v, dropout_p, fn);
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && v.dim() == 4, fn, ": q, k, v must be [batch, seqlen, heads, head_dim]");
  TORCH_CHECK(k.sizes() == v.sizes(), fn, ": k and v must have the same shape");
  TORCH_CHECK(k.size(0) == q.size(0) && k.size(3) == q.size(3), fn, ": k / v batch and head_dim must match q");
  torch::Tensor out = torch::empty(q.sizes(), q.options());
  return run_prefill_attention(q, k, v, out, nullptr, q.size(0), q.size(1), k.size(1), softmax_scale, causal, fn);
}

// qkv [total, 3, H, D], cu_seqlens int32 [batch + 1] -> out [total, H, D]
torch::Tensor flash_attn_varlen_qkvpacked_func(const torch::Tensor& qkv, const torch::Tensor& cu_seqlens, int64_t max_seqlen,
                                               double dropout_p, c10::optional<double> softmax_scale, bool causal) {
  const char* fn = "flash_attn_varlen_qkvpacked_func";
  TORCH_CHECK(qkv.dim() == 4 && qkv.size(1) == 3, fn, ": qkv must be [total_tokens, 3, heads, head_dim]");
  const torch::Tensor q = qkv.select(1, 0), k = qkv.select(1, 1), v = qkv.select(1, 2);
  check_attention_args(q, k, v, dropout_p, fn);
  TORCH_CHECK(cu_seqlens.is_cuda() && cu_seqlens.scalar_type() == at::ScalarType::Int && cu_seqlens.dim() == 1 &&
                  cu_seqlens.is_contiguous() && cu_seqlens.numel() >= 1,
              fn, ": cu_seqlens must be a contiguous int32 CUDA tensor [batch + 1]");
  TORCH_CHECK(cu_seqlens.device() == qkv.device(), fn, ": cu_seqlens must be on qkv's device");
  TORCH_CHECK(max_seqlen >= 0 && max_seqlen <= INT32_MAX, fn, ": bad max_seqlen");
  torch::Tensor out = torch::empty({qkv.size(0), qkv.size(2), qkv.size(3)}, qkv.options());
  // [total, H, D] views as [1, total, H, D]: the batch stride is ignored for packed sequences
  return run_prefill_attention(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), out, cu_seqlens.data_ptr<int>(),
                               (int)cu_seqlens.numel() - 1, (int)max_seqlen, (int)max_seqlen, softmax_scale, causal, fn);
}

// Attention of a chunk q [B, Sq, H, D] over keys [0, seqlen_k) of a KV cache, read in place -> out [B, Sq, H, D].  The
// layout follows from k_cache: 5-D is tinychat's decode cache (k_cache [Bc, Hkv, D / 8, Lmax, 8], v_cache [Bc, Hkv,
// Lmax, D]), 4-D long_forward's ([Bc, Lmax, Hkv, D] both); Bc >= B, caches contiguous.  q may be a strided view (as for
// flash_attn_func, one that the kernel cannot read is copied contiguous first).
torch::Tensor kv_cache_attention(const torch::Tensor& q_in, const torch::Tensor& k_cache, const torch::Tensor& v_cache,
                                 int64_t seqlen_k, c10::optional<double> softmax_scale, bool causal) {
  const char* fn = "kv_cache_attention";
  check_attention_args(q_in, k_cache, v_cache, 0.0, fn);
  TORCH_CHECK(q_in.dim() == 4, fn, ": q must be [batch, seqlen_q, heads, head_dim]");
  const int64_t d = q_in.size(3);
  const auto [layout, kv_heads, rows, max_len] = kv_caches(q_in, k_cache, v_cache, d, fn);
  TORCH_CHECK(q_in.size(0) <= rows, fn, ": q has ", q_in.size(0), " batch rows, the caches ", rows);
  TORCH_CHECK(seqlen_k >= 0 && seqlen_k <= max_len, fn, ": seqlen_k must be in [0, ", max_len, "]");
  TORCH_CHECK(max_len <= INT32_MAX && q_in.size(1) <= INT32_MAX, fn, ": sizes out of range");
  const c10::cuda::CUDAGuard guard(q_in.device());
  const AttentionQuery a = attention_query(q_in, softmax_scale, fn);
  const int batch = (int)a.q.size(0), seqlen_q = (int)a.q.size(1), heads = (int)a.q.size(2);
  torch::Tensor out = torch::empty({a.q.size(0), a.q.size(1), a.q.size(2), d}, a.q.options());
  const auto ws = attention_workspace_if(
      a.q, b200awq_kv_cache_attention_workspace_bytes(layout, batch, seqlen_q, (int)seqlen_k, heads, kv_heads, (int)d));
  raise(b200awq_kv_cache_attention(a.q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(), layout, batch,
                                   seqlen_q, (int)seqlen_k, (int)max_len, heads, kv_heads, (int)d, a.strides, a.scale,
                                   causal ? 1 : 0, a.dt, ws.first, ws.second, current_stream()));
  return out;
}

// RoPE of a chunk's q and k with the store of k and v into the caches, one launch (include/b200awq.h,
// b200awq_rope_kv_store).  qkv [B, S, H + 2 Hkv, D] is tinychat's xqkv view (last dimension contiguous); freqs fp32,
// contiguous, S * D angles ([S, D] or tinychat's [S, 1, 1, D] slice), shared by all batch rows; caches as for
// kv_cache_attention, Hkv read from them.  Returns the view qkv[:, :, :H], which holds the rotated q.
torch::Tensor rope_kv_store(const torch::Tensor& qkv, const torch::Tensor& freqs, torch::Tensor& k_cache,
                            torch::Tensor& v_cache, int64_t start_pos) {
  const char* fn = "rope_kv_store";
  TORCH_CHECK(qkv.is_cuda() && freqs.is_cuda() && k_cache.is_cuda() && v_cache.is_cuda(), fn, ": tensors must be CUDA tensors");
  TORCH_CHECK(qkv.dim() == 4 && qkv.stride(3) == 1, fn, ": qkv must be [batch, seqlen, heads + 2 kv_heads, head_dim] with a contiguous last dimension");
  const int dt = dtype_code(qkv, fn);
  TORCH_CHECK(k_cache.scalar_type() == qkv.scalar_type() && v_cache.scalar_type() == qkv.scalar_type(), fn,
              ": qkv and the caches must have the same dtype");
  TORCH_CHECK(freqs.device() == qkv.device(), fn, ": tensors must be on one device");
  TORCH_CHECK(freqs.scalar_type() == at::ScalarType::Float && freqs.is_contiguous(), fn, ": freqs must be contiguous float32");
  const int64_t B = qkv.size(0), S = qkv.size(1), D = qkv.size(3);
  TORCH_CHECK(freqs.numel() == S * D, fn, ": freqs must hold seqlen * head_dim = ", S * D, " angles, not ", freqs.numel());
  const auto [layout, kv_heads, rows, max_len] = kv_caches(qkv, k_cache, v_cache, D, fn);
  const int64_t H = qkv.size(2) - 2 * kv_heads;
  TORCH_CHECK(H >= 1, fn, ": qkv has ", qkv.size(2), " heads, fewer than 2 * kv_heads + 1 = ", 2 * kv_heads + 1);
  TORCH_CHECK(B <= rows, fn, ": qkv has ", B, " batch rows, the caches ", rows);
  TORCH_CHECK(start_pos >= 0 && start_pos + S <= max_len, fn, ": slots [", start_pos, ", ", start_pos + S,
              ") are not within the caches' ", max_len);
  TORCH_CHECK(max_len <= INT32_MAX, fn, ": sizes out of range");
  if (B == 0 || S == 0) return qkv.narrow(2, 0, H);
  const c10::cuda::CUDAGuard guard(qkv.device());
  const long long st[3] = {qkv.stride(0), qkv.stride(1), qkv.stride(2)};
  raise(b200awq_rope_kv_store(qkv.data_ptr(), freqs.data_ptr<float>(), k_cache.data_ptr(), v_cache.data_ptr(), layout, (int)B,
                              (int)S, (int)H, kv_heads, (int)D, (int)max_len, (int)start_pos, st, dt, current_stream()));
  return qkv.narrow(2, 0, H);
}

// The next token of each row, one launch (include/b200awq.h, b200awq_sample_next_token).  logits fp32 [B, V] with a
// contiguous last dimension (tinychat's logits[:, -1, :] view is read in place); prev_ids int64 [B, n] with a contiguous
// last dimension, or None; uniforms fp32 [B] in [0, 1), required unless greedy.  Returns int64 [B] on logits' device.
torch::Tensor sample_next_token(const torch::Tensor& logits, c10::optional<torch::Tensor> prev_ids, double temperature,
                                double repetition_penalty, double top_p, int64_t top_k, bool greedy,
                                c10::optional<torch::Tensor> uniforms) {
  const char* fn = "sample_next_token";
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::ScalarType::Float && logits.dim() == 2 &&
                  logits.stride(1) == 1,
              fn, ": logits must be a float32 CUDA tensor [batch, vocab] with a contiguous last dimension");
  const int64_t B = logits.size(0), V = logits.size(1);
  TORCH_CHECK(B <= INT32_MAX && V <= INT32_MAX && top_k >= 0 && top_k <= INT32_MAX, fn, ": sizes out of range");
  const long long* ids = nullptr;
  long long ids_stride = 0;
  int n_prev = 0;
  if (prev_ids.has_value()) {
    const torch::Tensor& p = prev_ids.value();
    TORCH_CHECK(p.device() == logits.device() && p.scalar_type() == at::ScalarType::Long && p.dim() == 2 &&
                    p.size(0) == B && (p.stride(1) == 1 || p.size(1) <= 1) && p.size(1) <= INT32_MAX,
                fn, ": prev_ids must be an int64 tensor [batch, n] on logits' device with a contiguous last dimension");
    ids = reinterpret_cast<const long long*>(p.data_ptr<int64_t>());
    ids_stride = p.stride(0);
    n_prev = (int)p.size(1);
  }
  const float* u = nullptr;
  if (uniforms.has_value()) {
    const torch::Tensor& t = uniforms.value();
    TORCH_CHECK(t.device() == logits.device() && t.scalar_type() == at::ScalarType::Float && t.dim() == 1 &&
                    t.numel() == B && t.is_contiguous(),
                fn, ": uniforms must be a contiguous float32 tensor [batch] on logits' device");
    u = t.data_ptr<float>();
  }
  TORCH_CHECK(greedy || u, fn, ": uniforms are required unless greedy");
  const c10::cuda::CUDAGuard guard(logits.device());
  torch::Tensor tokens = torch::empty({B}, logits.options().dtype(torch::kInt64));
  if (B == 0) return tokens;
  raise(b200awq_sample_next_token(logits.data_ptr<float>(), (long long)logits.stride(0), (int)B, (int)V, ids, ids_stride,
                                  n_prev, (float)temperature, (float)repetition_penalty, (float)top_p, (int)top_k,
                                  greedy ? 1 : 0, u, reinterpret_cast<long long*>(tokens.data_ptr<int64_t>()),
                                  current_stream()));
  return tokens;
}

// tinychat's tail in one launch (include/b200awq.h, b200awq_lm_head): the fp32 logits [m, vocab] of hidden [m, k]
// (any row stride that is a multiple of 8, so h[:, -1, :] is read in place) against weight [vocab, k], after the final
// RMSNorm when gamma [k] is given.  hidden, weight and gamma share one dtype and device.
torch::Tensor lm_head_forward_cuda(const torch::Tensor& hidden, const torch::Tensor& weight, c10::optional<torch::Tensor> gamma,
                                   double eps) {
  const char* fn = "lm_head_forward_cuda";
  TORCH_CHECK(hidden.is_cuda() && weight.is_cuda() && weight.device() == hidden.device(), fn,
              ": hidden and weight must be CUDA tensors on one device");
  const int dt = dtype_code(hidden, fn);
  TORCH_CHECK(weight.scalar_type() == hidden.scalar_type(), fn, ": weight must have hidden's dtype");
  TORCH_CHECK(hidden.dim() == 2 && (hidden.stride(1) == 1 || hidden.size(1) <= 1), fn,
              ": hidden must be [m, k] with a contiguous last dimension");
  TORCH_CHECK(weight.dim() == 2 && weight.is_contiguous() && weight.size(1) == hidden.size(1), fn,
              ": weight must be a contiguous [vocab, k] matching hidden");
  const int64_t m = hidden.size(0), k = hidden.size(1), vocab = weight.size(0);
  TORCH_CHECK(m <= 8, fn, ": at most 8 rows, got ", m);
  TORCH_CHECK(vocab <= INT32_MAX && k <= INT32_MAX, fn, ": sizes out of range");
  const void* g = nullptr;
  if (gamma.has_value()) {
    TORCH_CHECK(gamma->is_cuda() && gamma->device() == hidden.device(), fn, ": gamma must be on hidden's device");
    TORCH_CHECK(gamma->scalar_type() == hidden.scalar_type(), fn, ": gamma must have hidden's dtype");
    TORCH_CHECK(gamma->is_contiguous() && gamma->numel() == k, fn, ": gamma must be contiguous with ", k, " elements");
    g = gamma->data_ptr();
  }
  const c10::cuda::CUDAGuard guard(hidden.device());
  torch::Tensor logits = torch::empty({m, vocab}, hidden.options().dtype(torch::kFloat32));
  if (m == 0) return logits;
  const long long stride = m == 1 ? (long long)k : (long long)hidden.stride(0);  // a single row's stride is never used
  raise(b200awq_lm_head(hidden.data_ptr(), stride, g, (float)eps, weight.data_ptr(), logits.data_ptr<float>(), (int)m,
                        (int)vocab, (int)k, dt, current_stream()));
  return logits;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "H100 (sm_90a) drop-in for llm-awq's awq_inference_engine (W4A16 and W8A8 paths)";
  m.def("gemm_forward_cuda_new", &gemm_forward_cuda_new, "New quantized GEMM kernel.");
  m.def("gemv_forward_cuda_new", &gemv_forward_cuda_new, "New quantized GEMV kernel.");
  m.def("layernorm_forward_cuda", &layernorm_forward_cuda, "FasterTransformer layernorm kernel");
  m.def("single_query_attention", &single_query_attention, "Attention with a single query", py::arg("q"), py::arg("k"),
        py::arg("v"), py::arg("k_cache"), py::arg("v_cache"), py::arg("length_per_sample_"), py::arg("alibi_slopes_"),
        py::arg("timestep"), py::arg("rotary_embedding_dim") = 0, py::arg("rotary_base") = 10000.0f,
        py::arg("rotary_scale") = 1.0f, py::arg("neox_rotary_style") = true);
  m.def("fused_rope_with_pos_forward_func", &fused_rope_with_pos_forward_func,
        "Fused rope forward function with B,S,D embedding");
  m.def("rotary_embedding_neox", &rotary_embedding_neox, "Apply GPT-NeoX style rotary embedding to query and key");
  m.def("w4a16_linear_forward_cuda", &w4a16_linear_forward_cuda,
        "W4A16 linear with the bias and residual adds in the same launch", py::arg("in_feats"), py::arg("kernel"),
        py::arg("scales"), py::arg("zeros"), py::arg("group_size"), py::arg("bias") = py::none(),
        py::arg("residual") = py::none());
  m.def("mlp_front_forward_cuda", &mlp_front_forward_cuda, "silu(x Wgate^T) * (x Wup^T) for W4A16 weights, one call");
  m.def("rmsnorm_w4a16_linear_forward_cuda", &rmsnorm_w4a16_linear_forward_cuda,
        "RMSNorm(x) W^T (+ bias) for W4A16 weights, bit-identical to layernorm_forward_cuda + w4a16_linear_forward_cuda",
        py::arg("in_feats"), py::arg("gamma"), py::arg("eps"), py::arg("kernel"), py::arg("scales"), py::arg("zeros"),
        py::arg("group_size"), py::arg("bias") = py::none());
  m.def("rmsnorm_mlp_front_forward_cuda", &rmsnorm_mlp_front_forward_cuda,
        "silu(RMSNorm(x) Wgate^T) * (RMSNorm(x) Wup^T), bit-identical to layernorm_forward_cuda + mlp_front_forward_cuda",
        py::arg("in_feats"), py::arg("gamma"), py::arg("eps"), py::arg("gate_kernel"), py::arg("gate_scales"),
        py::arg("gate_zeros"), py::arg("up_kernel"), py::arg("up_scales"), py::arg("up_zeros"));
  m.def("w8a8_gemm_forward_cuda", &w8a8_gemm_forward_cuda, "our w8a8 gemm kernel");
  m.def("w8a8_gemm_fuse_bias_forward_cuda", &w8a8_gemm_fuse_bias_forward_cuda, "our w8a8 gemm fused bias kernel");
  m.def("w8a8_linear_forward_cuda", &w8a8_linear_forward_cuda,
        "W8A8 linear with the layer scale and residual in the same launch, into out_feats", py::arg("in_feats"),
        py::arg("kernel"), py::arg("wscales"), py::arg("ascales"), py::arg("out_feats"), py::arg("bias") = py::none(),
        py::arg("layer_scale") = py::none(), py::arg("residual") = py::none());
  m.def("invoke_quant", &invoke_quant, "fp16->int8 quantization");
  m.def("rms_norm_general", &rms_norm_general, py::arg("out"), py::arg("input"), py::arg("weight"), py::arg("bias"),
        py::arg("scaling"), py::arg("epsilon"), py::arg("use_per_token_quant") = true,
        "LayerNorm + int8 quantization (per token or per tensor)");
  m.def("silu_and_mul", &silu_and_mul, "Activation function.");
  m.def("gelu_and_quant", &gelu_and_quant, "Apply gelu act and quant output");
  m.def("flash_attn_func", &flash_attn_func, "Attention over many queries (flash-attn's flash_attn_func)", py::arg("q"),
        py::arg("k"), py::arg("v"), py::arg("dropout_p") = 0.0, py::arg("softmax_scale") = py::none(),
        py::arg("causal") = false);
  m.def("flash_attn_varlen_qkvpacked_func", &flash_attn_varlen_qkvpacked_func,
        "Attention over packed sequences of a fused qkv tensor (flash-attn's flash_attn_varlen_qkvpacked_func)",
        py::arg("qkv"), py::arg("cu_seqlens"), py::arg("max_seqlen"), py::arg("dropout_p") = 0.0,
        py::arg("softmax_scale") = py::none(), py::arg("causal") = false);
  m.def("kv_cache_attention", &kv_cache_attention,
        "Attention of a chunk of queries over a KV cache in either of tinychat's layouts, read in place", py::arg("q"),
        py::arg("k_cache"), py::arg("v_cache"), py::arg("seqlen_k"), py::arg("softmax_scale") = py::none(),
        py::arg("causal") = true);
  m.def("rope_kv_store", &rope_kv_store,
        "RoPE of a chunk's q and k in the fused qkv output with the store of k and v into a KV cache, one launch",
        py::arg("qkv"), py::arg("freqs"), py::arg("k_cache"), py::arg("v_cache"), py::arg("start_pos"));
  m.def("sample_next_token", &sample_next_token,
        "tinychat's temperature, repetition penalty, top-p, top-k and the choice of the next token, one launch",
        py::arg("logits"), py::arg("prev_ids"), py::arg("temperature"), py::arg("repetition_penalty"), py::arg("top_p"),
        py::arg("top_k"), py::arg("greedy"), py::arg("uniforms") = py::none());
  m.def("lm_head_forward_cuda", &lm_head_forward_cuda,
        "fp32 logits of the LM head, optionally after the final RMSNorm, one launch", py::arg("hidden"), py::arg("weight"),
        py::arg("gamma") = py::none(), py::arg("eps") = 1e-6);
  m.def("set_pdl",[](bool on) { return b200awq_set_pdl(on ? 1 : 0) != 0; }, "programmatic dependent launch on/off");
  m.def("launch_count", []() { return b200awq_launch_count(); }, "kernels launched by libb200awq so far");
  m.def("version", []() { return std::string(b200awq_version()); });
}
