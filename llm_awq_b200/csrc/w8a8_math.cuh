// The fp32 instructions of the reference's W8A8 kernels, which are built with --use_fast_math, spelled out in PTX so
// that this project's W8A8 kernels round exactly where the reference rounds: every division is div.approx.ftz,
// tanhf is tanh.approx, rsqrtf is rsqrt.approx.ftz, products and fused multiply-adds flush denormals, int8 codes are
// cvt.rni.sat.s8.f32 (round to nearest even, saturate; NaN -> 0).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace b200awq {

__device__ __forceinline__ float fdiv_approx(float a, float b) {
  float r;
  asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float fmul_ftz(float a, float b) {
  float r;
  asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float fadd_ftz(float a, float b) {
  float r;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float fsub_ftz(float a, float b) {
  float r;
  asm("sub.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float ffma_ftz(float a, float b, float c) {
  float r;
  asm("fma.rn.ftz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ float frsqrt_approx(float a) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
__device__ __forceinline__ float ftanh_approx(float a) {
  float r;
  asm("tanh.approx.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
__device__ __forceinline__ int8_t f2s8_rni_sat(float a) {
  uint32_t r;
  asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(r) : "f"(a));
  return (int8_t)r;
}
__device__ __forceinline__ float s32_to_f32(int a) {
  float r;
  asm("cvt.rn.f32.s32 %0, %1;" : "=f"(r) : "r"(a));
  return r;
}
// four codes -> one 32-bit word, code 0 in the low byte
__device__ __forceinline__ uint32_t pack_s8x4(int8_t a, int8_t b, int8_t c, int8_t d) {
  return (uint32_t)(uint8_t)a | ((uint32_t)(uint8_t)b << 8) | ((uint32_t)(uint8_t)c << 16) | ((uint32_t)(uint8_t)d << 24);
}

}  // namespace b200awq
