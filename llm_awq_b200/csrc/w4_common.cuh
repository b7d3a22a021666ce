// Shared device helpers for the sm_90a W4A16 kernels: packed-format index math,
// exact int4 -> fp16/bf16 dequantisation, mbarrier / bulk-copy / PDL / cluster PTX.
//
// Packed format (closed form of the reference packer awq/quantize/qmodule.py:26-65):
// qweight is int16 [N/4, K].  Each 4-row x 64-k tile is one contiguous 128-byte segment
//     [row0: kblk0 (16 B) | kblk1 (16 B)] [row1 ...] [row2 ...] [row3 ...]
// and inside the 16-byte chunk of (row, 32-k block), viewed as four uint32 `u`, nibble
// `i` of word `u` holds  k_local = 8*(i % 4) + 2*u + i/4.
// Consequence used by every kernel here: the 32-bit value (nibble j | nibble j+4 << 16)
// of word u is the k-adjacent pair (8j + 2u, 8j + 2u + 1).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200awq {

constexpr int kGroup = 128;  // the only group size the reference kernels accept

template <typename T> struct TypeTraits;
template <> struct TypeTraits<__half> {
  static constexpr bool kIsBf16 = false;
};
template <> struct TypeTraits<__nv_bfloat16> {
  static constexpr bool kIsBf16 = true;
};

__device__ __forceinline__ uint32_t h2_as_u32(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __half2 u32_as_h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }
__device__ __forceinline__ uint32_t b2_as_u32(__nv_bfloat162 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __nv_bfloat162 u32_as_b2(uint32_t v) { return *reinterpret_cast<__nv_bfloat162*>(&v); }

// 16-bit scalar (raw bits) -> packed pair (v, v)
__device__ __forceinline__ uint32_t splat16(uint16_t v) { return (uint32_t)v * 0x00010001u; }

// (a & b) | c in ONE LOP3 (the compiler splits the C expression into two because both
// constants would have to be immediates).
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xea;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// One packed word -> four pairs of EXACT integers q in T, out[j] = pair (k = 8j + 2u, 8j + 2u + 1).
// Same magic-number construction as the reference (quantization_new/dequantize.cuh:39-79, :93-122).
template <typename T>
__device__ __forceinline__ void unpack_word(uint32_t w, uint32_t (&out)[4]) {
  if constexpr (!TypeTraits<T>::kIsBf16) {
    const uint32_t t = w >> 8;
    const uint32_t h0 = and_or(w, 0x000f000fu, 0x64006400u);  // 1024 + q
    const uint32_t h1 = and_or(w, 0x00f000f0u, 0x64006400u);  // 1024 + 16 q
    const uint32_t h2 = and_or(t, 0x000f000fu, 0x64006400u);
    const uint32_t h3 = and_or(t, 0x00f000f0u, 0x64006400u);
    const __half2 k1024 = u32_as_h2(0x64006400u);
    const __half2 k16th = u32_as_h2(0x2c002c00u);   // 1/16
    const __half2 kneg64 = u32_as_h2(0xd400d400u);  // -64
    out[0] = h2_as_u32(__hsub2(u32_as_h2(h0), k1024));
    out[1] = h2_as_u32(__hfma2(u32_as_h2(h1), k16th, kneg64));
    out[2] = h2_as_u32(__hsub2(u32_as_h2(h2), k1024));
    out[3] = h2_as_u32(__hfma2(u32_as_h2(h3), k16th, kneg64));
  } else {
    const uint32_t h0 = and_or(w, 0x000f000fu, 0x43004300u);  // 128 + q
    const uint32_t h1 = and_or(w >> 4, 0x000f000fu, 0x43004300u);
    const uint32_t h2 = and_or(w >> 8, 0x000f000fu, 0x43004300u);
    const uint32_t h3 = and_or(w >> 12, 0x000f000fu, 0x43004300u);
    const __nv_bfloat162 k128 = u32_as_b2(0x43004300u);
    out[0] = b2_as_u32(__hsub2(u32_as_b2(h0), k128));
    out[1] = b2_as_u32(__hsub2(u32_as_b2(h1), k128));
    out[2] = b2_as_u32(__hsub2(u32_as_b2(h2), k128));
    out[3] = b2_as_u32(__hsub2(u32_as_b2(h3), k128));
  }
}

// Raw biased forms, no arithmetic at all: fp16 -> (1024 + q) for j = 0, 2 (nibble in mantissa
// bits 0-3 under exponent 2^10) and (64 + q) for j = 1, 3 (nibble in mantissa bits 4-7 under
// exponent 2^6, magic 0x5400);  bf16 -> (128 + q) for every j.  Only for fp32-accumulating
// consumers that remove the bias algebraically (w4a16_stream.cu, MODE 2).
template <typename T>
__device__ __forceinline__ void unpack_word_biased(uint32_t w, uint32_t (&out)[4]) {
  if constexpr (!TypeTraits<T>::kIsBf16) {
    const uint32_t t = w >> 8;
    out[0] = and_or(w, 0x000f000fu, 0x64006400u);
    out[1] = and_or(w, 0x00f000f0u, 0x54005400u);
    out[2] = and_or(t, 0x000f000fu, 0x64006400u);
    out[3] = and_or(t, 0x00f000f0u, 0x54005400u);
  } else {
    out[0] = and_or(w, 0x000f000fu, 0x43004300u);
    out[1] = and_or(w >> 4, 0x000f000fu, 0x43004300u);
    out[2] = and_or(w >> 8, 0x000f000fu, 0x43004300u);
    out[3] = and_or(w >> 12, 0x000f000fu, 0x43004300u);
  }
}

// One packed word -> four pairs w~ = rn_T(q * s + z): exact q, then ONE FMA in T
// (gemv_cuda.cu:161,165; gemm_cuda.cu:911-918), so the operand bits equal the reference's.
template <typename T>
__device__ __forceinline__ void dequant_word(uint32_t w, uint32_t s2, uint32_t z2, uint32_t (&out)[4]) {
  uint32_t q[4];
  unpack_word<T>(w, q);
  if constexpr (!TypeTraits<T>::kIsBf16) {
    const __half2 s = u32_as_h2(s2), z = u32_as_h2(z2);
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = h2_as_u32(__hfma2(u32_as_h2(q[j]), s, z));
  } else {
    const __nv_bfloat162 s = u32_as_b2(s2), z = u32_as_b2(z2);
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = b2_as_u32(__hfma2(u32_as_b2(q[j]), s, z));
  }
}

__device__ __forceinline__ float bits16_to_float(uint16_t v, bool bf16) {
  if (bf16) return __uint_as_float((uint32_t)v << 16);
  return __half2float(__ushort_as_half(v));
}

template <typename T>
__device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// ---------------------------------------------------------------- shared-memory addresses
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- bulk async copy (UBLKCP)
// global -> this CTA's shared memory, completion counted in bytes on an mbarrier.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch
__device__ __forceinline__ void pdl_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- cluster
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// address of `local_smem_addr` in CTA `rank` of the cluster (shared::cluster window)
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local_smem_addr), "r"(rank));
  return a;
}
__device__ __forceinline__ float ld_cluster_f32(uint32_t cluster_addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr) : "memory");
  return v;
}

// ---------------------------------------------------------------- warp-level tensor-core MAC
// D[16 x 8] = A[16 x 16] * B[16 x 8] + C, fp32 accumulate.  Not `volatile`: a pure function of its register
// operands, so the compiler may interleave independent groups.  Used by the HBM-bound streaming
// kernel only: rows of A are output channels (dequantised in registers), columns of B are
// tokens.
template <typename T>
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1, const float (&c)[4]) {
  if constexpr (!TypeTraits<T>::kIsBf16) {
    asm(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
  } else {
    asm(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
  }
}

}  // namespace b200awq
