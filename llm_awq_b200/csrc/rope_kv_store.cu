// rope_kv_store: RoPE of a chunk's q and k heads in the fused qkv output, q rotated in place, rotated k and v stored into
// tinychat's KV caches (FT or BTHD layout), one launch.  HBM-bound: per token (heads + 2 kv_heads) head_dim elements are
// read once and written once, plus one row of angles.
//
// Thread mapping: a CTA of 256 threads owns one token tile of one batch row and 256 / tile columns (head, pair of
// V-element pieces); the token is the fastest index, so a warp covers 8 tokens x 4 columns.  Every warp-wide access is
// made of whole 32-byte sectors: per token it reads (and writes back, for q) 4 adjacent 16-byte pieces of a head, and in
// the FT k cache, where consecutive positions of one 8-channel block are consecutive 16-byte pieces, the 8 tokens of a
// column store one 128-byte run.  No shared memory and no barrier: the transposition into the FT layout is done by the
// lane-to-token mapping, not by a staging buffer (DESIGN §3.11).
#include <algorithm>

#include "rope_kv_store.cuh"
#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

constexpr int kRopeKvThreads = 256;
constexpr int kRopeKvTileLog2 = 3;  // 8-token tiles: FT k runs of 128 bytes

template <typename T, int V>
__global__ void __launch_bounds__(kRopeKvThreads) rope_kv_store_kernel(const RopeKvArgs a, int batch, int tiles) {
  pdl_launch_dependents();
  pdl_wait_prior_grid();  // qkv is normally the previous launch's output
  const int item = blockIdx.x * kRopeKvThreads + threadIdx.x;
  if (item >= rope_kv_tile_items<V>(a)) return;
  for (int b = blockIdx.z; b < batch; b += gridDim.z)
    for (int tile = blockIdx.y; tile < tiles; tile += gridDim.y) rope_kv_store_item<T, V>(a, b, tile, item);
}

template <typename T, int V>
int launch_rope_kv_t(const RopeKvArgs& a, int batch, bool pdl, cudaStream_t stream) {
  const int tiles = (a.seqlen + (1 << a.tile_log2) - 1) >> a.tile_log2;
  const dim3 grid((unsigned)((rope_kv_tile_items<V>(a) + kRopeKvThreads - 1) / kRopeKvThreads),
                  (unsigned)std::min(tiles, 65535), (unsigned)std::min(batch, 65535));
  return launch_kernel(rope_kv_store_kernel<T, V>, grid, dim3(kRopeKvThreads), 0, stream, pdl, 1, a, batch, tiles);
}

template <typename T>
int launch_rope_kv_v(const RopeKvArgs& a, int batch, bool pdl, cudaStream_t stream) {
  // 16-byte pieces when the two halves of a head start on 16-byte boundaries, else 8-byte pieces (head_dim % 16 == 8)
  if (a.head_dim % 16 == 0) return launch_rope_kv_t<T, 8>(a, batch, pdl, stream);
  return launch_rope_kv_t<T, 4>(a, batch, pdl, stream);
}

}  // namespace

int launch_rope_kv_store(void* qkv, const float* freqs, void* k_cache, void* v_cache, int layout, int batch, int seqlen,
                         int heads, int kv_heads, int head_dim, int max_len, int start_pos, const long long* qkv_strides,
                         int dtype, bool pdl, cudaStream_t stream) {
  RopeKvArgs a{qkv, freqs, k_cache, v_cache, layout, seqlen, heads, kv_heads, head_dim, max_len, start_pos, 0,
               qkv_strides[0], qkv_strides[1], qkv_strides[2]};
  // a short chunk (long_forward's decode: one token) takes a tile of its own size, rounded up to a power of two
  while (a.tile_log2 < kRopeKvTileLog2 && (1 << a.tile_log2) < seqlen) ++a.tile_log2;
  if (dtype == B200AWQ_DTYPE_F16) return launch_rope_kv_v<__half>(a, batch, pdl, stream);
  return launch_rope_kv_v<__nv_bfloat16>(a, batch, pdl, stream);
}

}  // namespace b200awq
