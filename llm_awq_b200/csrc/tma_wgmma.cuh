// Shared by the sm_90a TMA + wgmma kernels (w4a16_wgmma.cu, w8a8_wgmma.cu, prefill_attention.cu): TMA tile loads, the
// shared-memory matrix descriptors (128-byte-swizzled K-major; any swizzle, K- or MN-major), the wgmma fence / commit /
// wait instructions and the run-time lookup of the driver's cuTensorMapEncodeTiled.
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the encoder is resolved at run time)

#include "w4_common.cuh"

namespace b200awq {

// ---------------------------------------------------------------- TMA / wgmma PTX
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 4-D box at coordinates (c0 innermost .. c3); elements outside the tensor, negative coordinates included, arrive as zeros
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// K-major, 128-byte swizzle, rows of 128 B, 8-row groups 1024 B apart (what TMA SWIZZLE_128B writes); sm_90 layout
// type 1 = SWIZZLE_128B in bits 62-63, leading byte offset unused for swizzled K-major operands
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// Any sm_90 matrix descriptor: layout type 1 = SWIZZLE_128B, 2 = 64B, 3 = 32B in bits 62-63.  K-major swizzled
// operands: sbo = bytes between 8-row groups, lbo unused.  MN-major (transposed) swizzled operands: lbo = bytes between
// swizzle-wide column blocks along MN, sbo = bytes between 8-row groups along K.  Regions aligned to the swizzle repeat.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t layout, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry-point query (no link-time dependency on libcuda);
// nullptr when the driver does not provide it.  One lookup per process.
inline EncodeTiledFn get_encoder() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace b200awq
