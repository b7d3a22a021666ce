// Shared by the sm_90a TMA + wgmma kernels (w4a16_wgmma.cu, w8a8_wgmma.cu, prefill_attention.cu,
// splitkv_attention.cu): TMA tile loads, the shared-memory matrix descriptors (128-byte-swizzled K-major; any swizzle,
// K- or MN-major), the one copy of every wgmma.mma_async form the kernels issue with its fence / commit / wait
// instructions, and the run-time lookup of the driver's cuTensorMapEncodeTiled.
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

// ---------------------------------------------------------------- wgmma.mma_async
// An asm template must be a string literal, so the instruction text is pieced together here by the preprocessor, once:
// shape and types (TY "f16" / "bf16" as a macro argument), the NA accumulators d[0 .. NA-1] (operands %0 .. %NA-1,
// constraint C "+f" or "+r"), the A and B operands AB (4 registers or a descriptor, then a descriptor), the operand P
// that sets the scale-d predicate (accum = 0 overwrites D instead of adding to it) and the trailing immediates IMM.
#define B200AWQ_ACC8(C, d, i) \
  C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define B200AWQ_ACC16(C, d, i) B200AWQ_ACC8(C, d, i), B200AWQ_ACC8(C, d, i + 8)
#define B200AWQ_ACC32(C, d, i) B200AWQ_ACC16(C, d, i), B200AWQ_ACC16(C, d, i + 16)
#define B200AWQ_ACC64(C, d, i) B200AWQ_ACC32(C, d, i), B200AWQ_ACC32(C, d, i + 32)
#define B200AWQ_REGS8 "%0,%1,%2,%3,%4,%5,%6,%7"
#define B200AWQ_REGS16 B200AWQ_REGS8 ",%8,%9,%10,%11,%12,%13,%14,%15"
#define B200AWQ_REGS32 B200AWQ_REGS16 ",%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define B200AWQ_REGS64                                                                                 \
  B200AWQ_REGS32 ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52" \
                 ",%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define B200AWQ_WGMMA(SHAPE_TYPES, C, NA, AB, P, IMM, ...)                                                 \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\n"                                           \
               "wgmma.mma_async.sync.aligned." SHAPE_TYPES " {" B200AWQ_REGS##NA "}, " AB ", p" IMM ";\n}\n" \
               : B200AWQ_ACC##NA(C, d, 0)                                                                \
               : __VA_ARGS__)
// register A: scale-a, scale-b, transpose-B
#define B200AWQ_WGMMA_RS_TY(N, NA, AB, P, TY, TNSPB)                                                                 \
  B200AWQ_WGMMA("m64n" #N "k16.f32." TY "." TY, "+f", NA, AB, P, ", 1, 1, " TNSPB, "r"(a[0]), "r"(a[1]), "r"(a[2]), \
                "r"(a[3]), "l"(bdesc), "r"(accum))
#define B200AWQ_WGMMA_RS(N, NA, AB, P)                                                               \
  if constexpr (!TypeTraits<T>::kIsBf16 && !kTnspB) B200AWQ_WGMMA_RS_TY(N, NA, AB, P, "f16", "0"); \
  else if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_RS_TY(N, NA, AB, P, "f16", "1");       \
  else if constexpr (!kTnspB) B200AWQ_WGMMA_RS_TY(N, NA, AB, P, "bf16", "0");                      \
  else B200AWQ_WGMMA_RS_TY(N, NA, AB, P, "bf16", "1")
// shared A, N = 128: 64 accumulators, then the A and B descriptors and accum
#define B200AWQ_WGMMA_SS(SHAPE_TYPES, C, IMM) \
  B200AWQ_WGMMA(SHAPE_TYPES, C, 64, "%64, %65", "%66", IMM, "l"(adesc), "l"(bdesc), "r"(accum))

// D[64 x N] (+)= A[64 x 16] * B[16 x N], fp32 accumulate.  A from registers: per warp, the A fragment of an m16n8k16
// mma.sync over its 16 rows.  B from shared memory, K-major, or MN-major with kTnspB (which transposes it).
template <typename T, int N, bool kTnspB>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
  static_assert(N == 16 || N == 32 || N == 64 || N == 128, "register-A wgmma: N = 16, 32, 64 or 128");
  if constexpr (N == 16) {
    B200AWQ_WGMMA_RS(16, 8, "{%8,%9,%10,%11}, %12", "%13");
  } else if constexpr (N == 32) {
    B200AWQ_WGMMA_RS(32, 16, "{%16,%17,%18,%19}, %20", "%21");
  } else if constexpr (N == 64) {
    B200AWQ_WGMMA_RS(64, 32, "{%32,%33,%34,%35}, %36", "%37");
  } else {
    B200AWQ_WGMMA_RS(128, 64, "{%64,%65,%66,%67}, %68", "%69");
  }
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], fp32 accumulate, both operands K-major in shared memory
template <typename T>
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (!TypeTraits<T>::kIsBf16) B200AWQ_WGMMA_SS("m64n128k16.f32.f16.f16", "+f", ", 1, 1, 0, 0");
  else B200AWQ_WGMMA_SS("m64n128k16.f32.bf16.bf16", "+f", ", 1, 1, 0, 0");
}

// D[64 x 128] (+)= A[64 x 32] * B[32 x 128], int8 x int8 -> int32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_ss(int (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  B200AWQ_WGMMA_SS("m64n128k32.s32.s8.s8", "+r", "");
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
