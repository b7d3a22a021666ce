// TEST INFRASTRUCTURE (tests/test_rope_kv_store_cpu.py): walks the work items of llm_awq_b200/csrc/rope_kv_store.cuh on
// the CPU as the kernel's grid does (batch row, token tile, item = CTA x 256 + thread), so that the cache addressing and
// the arithmetic of the kernel body can be checked where there is no GPU.  Not part of the product; nothing under
// llm_awq_b200/ builds, loads or calls this file.
#include "rope_kv_store.cuh"

using namespace b200awq;

template <typename T, int V>
static void walk(const RopeKvArgs& a, int batch) {
  const int tiles = (a.seqlen + (1 << a.tile_log2) - 1) >> a.tile_log2;
  for (int b = 0; b < batch; ++b)
    for (int tile = 0; tile < tiles; ++tile)
      for (int i = 0; i < rope_kv_tile_items<V>(a); ++i) rope_kv_store_item<T, V>(a, b, tile, i);
}

// dtype: 0 = fp16, 1 = bf16 (include/b200awq.h).  Returns the elements per access that were used (8 or 4), < 0 on error.
extern "C" int rope_kv_store_host(void* qkv, const float* freqs, void* k_cache, void* v_cache, int layout, int batch,
                                  int seqlen, int heads, int kv_heads, int head_dim, int max_len, int start_pos,
                                  long long sb, long long st, long long sh, int dtype, int tile_log2) {
  const RopeKvArgs a{qkv, freqs, k_cache, v_cache, layout, seqlen, heads, kv_heads, head_dim, max_len, start_pos, tile_log2,
                     sb, st, sh};
  const bool v8 = head_dim % 16 == 0;
  if (dtype == 0) {
    if (v8) walk<__half, 8>(a, batch); else walk<__half, 4>(a, batch);
  } else if (dtype == 1) {
    if (v8) walk<__nv_bfloat16, 8>(a, batch); else walk<__nv_bfloat16, 4>(a, batch);
  } else {
    return -1;
  }
  return v8 ? 8 : 4;
}
