// RoPE of a prefill chunk's q and k with the store of k and v into tinychat's KV caches: the per-work-item body,
// shared by the kernel (rope_kv_store.cu) and by the host harness of tests/test_rope_kv_store_cpu.py, which compiles
// THIS header with g++ and walks the same items on the CPU to check the cache addressing (the product has no CPU path).
//
// Replaces, per layer and chunk, tinychat's two fused_rope_with_pos_forward_func calls and its k / v cache stores
// (tinychat/modules/fused_attn.py, short_forward's and long_forward's prefill branches).
#pragma once
#include <math.h>

#include "../../include/b200awq.h"
#include "rope_neox.cuh"

namespace b200awq {

// One rotated element: v cos f + rot sin f in fp32 (rot = -x[i + d2 / 2] below d2 / 2, x[i - d2 / 2] above), as
// rope_apply(v, rot, rope_angle(f)).  The one copy of fused_rope_with_pos' arithmetic: rope_with_pos_kernel
// (attention.cu) and rope_kv_store_item call it, so that both round the same fp32 value.  Two steps so that
// rope_with_pos_kernel can keep its order (angle, then the partner's load).
struct RopeAngle {
  float sn, cs;
};

B200AWQ_HD RopeAngle rope_angle(float f) {
  RopeAngle a;
  sincosf(f, &a.sn, &a.cs);
  return a;
}

B200AWQ_HD float rope_apply(float v, float rot, RopeAngle a) { return v * a.cs + rot * a.sn; }

struct RopeKvArgs {
  void* qkv;           // [batch, seqlen, heads + 2 kv_heads, head_dim], strides sb / st / sh (elements), unit element stride
  const float* freqs;  // [seqlen, head_dim] angles, shared by all batch rows
  void* k_cache;       // FT: [>= batch, kv_heads, head_dim / 8, max_len, 8]; BTHD: [>= batch, max_len, kv_heads, head_dim]
  void* v_cache;       // FT: [>= batch, kv_heads, max_len, head_dim];        BTHD: as k_cache
  int layout;          // B200AWQ_KV_FT / B200AWQ_KV_BTHD
  int seqlen, heads, kv_heads, head_dim, max_len, start_pos;
  int tile_log2;       // log2 of the token tile: the fastest-varying index of the work items
  long long sb, st, sh;
};

// Work items of one token tile of one batch row: (column c = head * pairs + pair p, token t in the tile), t fastest,
// pairs = head_dim / (2 V).  Item (c, t) owns the V elements [p V, p V + V) of its head and their rotation partners
// head_dim / 2 further.  Items of tokens past seqlen (in the last tile) do nothing.
template <int V>
B200AWQ_HD int rope_kv_tile_items(const RopeKvArgs& a) {
  return ((a.heads + 2 * a.kv_heads) * (a.head_dim / (2 * V))) << a.tile_log2;
}

// Element offset of (row b, KV head h, position pos, channel d) in the k cache / the v cache.
B200AWQ_HD long long rope_kv_k_offset(const RopeKvArgs& a, int b, int h, int pos, int d) {
  if (a.layout == B200AWQ_KV_FT)
    return ((((long long)b * a.kv_heads + h) * (a.head_dim / 8) + d / 8) * a.max_len + pos) * 8 + d % 8;
  return (((long long)b * a.max_len + pos) * a.kv_heads + h) * a.head_dim + d;
}

B200AWQ_HD long long rope_kv_v_offset(const RopeKvArgs& a, int b, int h, int pos, int d) {
  if (a.layout == B200AWQ_KV_FT) return (((long long)b * a.kv_heads + h) * a.max_len + pos) * a.head_dim + d;
  return (((long long)b * a.max_len + pos) * a.kv_heads + h) * a.head_dim + d;
}

// Item `item` of token tile `tile` of batch row b.  q heads are rotated in place (both halves are read before either is
// written), k heads are rotated into the k cache, v heads are copied into the v cache; all accesses are V elements wide
// (V = 8: 16 bytes).
template <typename T, int V>
B200AWQ_HD void rope_kv_store_item(const RopeKvArgs& a, int b, int tile, int item) {
  using Vec = NeoxVec<T, V>;
  using F4 = NeoxVec<float, 4>;
  const int pairs = a.head_dim / (2 * V), half = a.head_dim / 2;
  const int s = (tile << a.tile_log2) + (item & ((1 << a.tile_log2) - 1));
  const int col = item >> a.tile_log2, h = col / pairs, d = (col - h * pairs) * V;
  if (s >= a.seqlen) return;
  T* src = static_cast<T*>(a.qkv) + b * a.sb + s * a.st + h * a.sh;
  Vec x = *reinterpret_cast<const Vec*>(src + d), y = *reinterpret_cast<const Vec*>(src + half + d);
  const int pos = a.start_pos + s;
  if (h >= a.heads + a.kv_heads) {  // v: stored as is
    T* dst = static_cast<T*>(a.v_cache);
    const int hv = h - a.heads - a.kv_heads;
    *reinterpret_cast<Vec*>(dst + rope_kv_v_offset(a, b, hv, pos, d)) = x;
    *reinterpret_cast<Vec*>(dst + rope_kv_v_offset(a, b, hv, pos, half + d)) = y;
    return;
  }
  const float* fr = a.freqs + (long long)s * a.head_dim;
  float fx[V], fy[V];
#pragma unroll
  for (int j = 0; j < V; j += 4) {
    const F4 lo = *reinterpret_cast<const F4*>(fr + d + j), hi = *reinterpret_cast<const F4*>(fr + half + d + j);
#pragma unroll
    for (int i = 0; i < 4; ++i) fx[j + i] = lo.v[i], fy[j + i] = hi.v[i];
  }
  Vec rx, ry;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float xf = neox_to_float(x.v[i]), yf = neox_to_float(y.v[i]);
    neox_from_float(rope_apply(xf, -yf, rope_angle(fx[i])), rx.v[i]);
    neox_from_float(rope_apply(yf, xf, rope_angle(fy[i])), ry.v[i]);
  }
  if (h < a.heads) {  // q: in place
    *reinterpret_cast<Vec*>(src + d) = rx;
    *reinterpret_cast<Vec*>(src + half + d) = ry;
    return;
  }
  T* dst = static_cast<T*>(a.k_cache);
  const int hk = h - a.heads;
  *reinterpret_cast<Vec*>(dst + rope_kv_k_offset(a, b, hk, pos, d)) = rx;
  *reinterpret_cast<Vec*>(dst + rope_kv_k_offset(a, b, hk, pos, half + d)) = ry;
}

}  // namespace b200awq
