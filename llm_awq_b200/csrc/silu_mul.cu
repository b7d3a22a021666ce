// c = silu(gate) * up, elementwise over [m, n] tensors of T: the tail of the MLP front half when the two projections
// ran as separate GEMMs / GEMVs (prefill, several tokens, bf16).  Same roundings as the reference's composition
// `F.silu(gate_output) * up_output` (tinychat/modules/fused_mlp.py:50,78,80): silu evaluated in fp32 and rounded to T,
// the product rounded to T.  HBM-bound: 3 * m * n * sizeof(T) bytes, 16-byte loads / stores, grid-stride.
// A row pitch on the inputs also serves silu_and_mul, whose gate and up are the two halves of one [m, 2d] row.
#include <algorithm>

#include "w4_common.cuh"
#include "w4a16_kernels.h"

namespace b200awq {
namespace {

template <typename T>
__device__ __forceinline__ uint32_t silu_mul_pair(uint32_t g2, uint32_t u2) {
  float2 g, u;
  if constexpr (TypeTraits<T>::kIsBf16) g = __bfloat1622float2(u32_as_b2(g2)), u = __bfloat1622float2(u32_as_b2(u2));
  else g = __half22float2(u32_as_h2(g2)), u = __half22float2(u32_as_h2(u2));
  const T s0 = from_float<T>(g.x / (1.f + expf(-g.x))), s1 = from_float<T>(g.y / (1.f + expf(-g.y)));
  const T c0 = from_float<T>((float)s0 * u.x), c1 = from_float<T>((float)s1 * u.y);
  return (uint32_t)(*reinterpret_cast<const uint16_t*>(&c0)) | ((uint32_t)(*reinterpret_cast<const uint16_t*>(&c1)) << 16);
}

// rows x cols elements; gate / up rows are `in_pitch` elements apart, out rows `cols` (a flat tensor is one row).
// 16-byte accesses over the first 8 (cols / 8) elements of each row when `vec`, the rest one element at a time.
template <typename T>
__global__ void __launch_bounds__(256) silu_mul_kernel(const T* __restrict__ gate, const T* __restrict__ up, T* __restrict__ out,
                                                       size_t rows, size_t cols, size_t in_pitch, bool vec) {
  pdl_launch_dependents();
  pdl_wait_prior_grid();
  const size_t nvec_row = vec ? cols >> 3 : 0, nvec = rows * nvec_row, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const size_t r = rows == 1 ? 0 : i / nvec_row, c = i - r * nvec_row;
    const uint4 g = reinterpret_cast<const uint4*>(gate + r * in_pitch)[c], u = reinterpret_cast<const uint4*>(up + r * in_pitch)[c];
    reinterpret_cast<uint4*>(out + r * cols)[c] =
        make_uint4(silu_mul_pair<T>(g.x, u.x), silu_mul_pair<T>(g.y, u.y), silu_mul_pair<T>(g.z, u.z), silu_mul_pair<T>(g.w, u.w));
  }
  // the elements past the 16-byte part of each row (all of them when !vec)
  const size_t tail = cols - (nvec_row << 3), ntail = rows * tail;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < ntail; i += stride) {
    const size_t r = rows == 1 ? 0 : i / tail, c = (nvec_row << 3) + (i - r * tail);
    const float g = (float)gate[r * in_pitch + c];
    const T s = from_float<T>(g / (1.f + expf(-g)));
    out[r * cols + c] = from_float<T>((float)s * (float)up[r * in_pitch + c]);
  }
}

}  // namespace

int launch_silu_mul(const void* gate, const void* up, void* out, size_t rows, size_t cols, size_t in_pitch, int dtype, bool pdl,
                    cudaStream_t stream) {
  const size_t count = rows * cols;
  if (count == 0) return 0;
  auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  // 16-byte accesses need every row start aligned (a single row only needs the base pointers aligned)
  const bool vec = a16(gate) && a16(up) && a16(out) && (rows == 1 || (cols % 8 == 0 && in_pitch % 8 == 0));
  int dev = 0, nsm = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  const size_t want = ((vec ? count / 8 : count) + 255) / 256;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)std::max<size_t>(1, std::min<size_t>(want, (size_t)nsm * 8)));
  cfg.blockDim = dim3(256);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e;
  if (dtype == B200AWQ_DTYPE_F16)
    e = cudaLaunchKernelEx(&cfg, silu_mul_kernel<__half>, static_cast<const __half*>(gate), static_cast<const __half*>(up),
                           static_cast<__half*>(out), rows, cols, in_pitch, vec);
  else
    e = cudaLaunchKernelEx(&cfg, silu_mul_kernel<__nv_bfloat16>, static_cast<const __nv_bfloat16*>(gate),
                           static_cast<const __nv_bfloat16*>(up), static_cast<__nv_bfloat16*>(out), rows, cols, in_pitch, vec);
  return e == cudaSuccess ? 0 : (int)e;
}

}  // namespace b200awq
