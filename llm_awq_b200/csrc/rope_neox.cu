// rotary_embedding_neox: in-place NeoX-style RoPE on query and key from a cos|sin table (the HF-attention branch of
// tinychat, tinychat/modules/fused_attn.py:61-79 -> awq/kernels/csrc/position_embedding/pos_encoding_kernels.cu:13-88).
// HBM-bound elementwise pass: per token 2 * (q_heads + k_heads) * rot_dim elements are read and written once, plus one
// table row.  One CTA per token like the reference; 16-byte accesses (8 pairs per thread) when alignment allows.
#include <algorithm>

#include "rope_neox.cuh"
#include "w4a16_kernels.h"

namespace b200awq {

template <typename T, int V>
__global__ void rope_neox_kernel(const RopeNeoxArgs a) {
  // the table row and the pairs are inputs of this launch only if a previous kernel produced query / key: wait for it
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int items = rope_neox_items<V>(a);
  for (int token = blockIdx.x; token < a.tokens; token += gridDim.x)
    for (int i = threadIdx.x; i < items; i += blockDim.x) rope_neox_item<T, V>(a, token, i);
}

template <typename T>
static int launch_neox_t(const RopeNeoxArgs& a, bool pdl, cudaStream_t stream) {
  const bool vec = rope_neox_can_vectorise(a);
  const int items = vec ? rope_neox_items<8>(a) : rope_neox_items<1>(a);
  const dim3 grid((unsigned)std::min(a.tokens, 65535 * 8));
  const dim3 block((unsigned)std::min(512, std::max(32, (items + 31) / 32 * 32)));
  if (vec) return launch_kernel(rope_neox_kernel<T, 8>, grid, block, 0, stream, pdl, 1, a);
  return launch_kernel(rope_neox_kernel<T, 1>, grid, block, 0, stream, pdl, 1, a);
}

int launch_rope_neox(const long long* positions, void* query, void* key, const void* cos_sin, int tokens, int q_heads,
                     int k_heads, int head_size, int rot_dim, long long q_stride, long long k_stride, int dtype, bool pdl,
                     cudaStream_t stream) {
  if (tokens < 0 || q_heads < 0 || k_heads < 0 || head_size < 1 || rot_dim < 2 || (rot_dim & 1) || rot_dim > head_size ||
      q_stride < (long long)q_heads * head_size || (k_heads > 0 && k_stride < (long long)k_heads * head_size))
    return B200AWQ_ERR_SHAPE;
  if (tokens == 0 || q_heads + k_heads == 0) return 0;
  const RopeNeoxArgs a{positions, query, key, cos_sin, tokens, q_heads, k_heads, head_size, rot_dim, q_stride, k_stride};
  if (dtype == B200AWQ_DTYPE_F16) return launch_neox_t<__half>(a, pdl, stream);
  return launch_neox_t<__nv_bfloat16>(a, pdl, stream);
}

}  // namespace b200awq
