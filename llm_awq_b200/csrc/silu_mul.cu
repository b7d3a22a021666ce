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
  // 16-byte accesses need every row start aligned (a single row only needs the base pointers aligned)
  const bool vec = aligned16(gate) && aligned16(up) && aligned16(out) && (rows == 1 || (cols % 8 == 0 && in_pitch % 8 == 0));
  const int nsm = sm_count();
  if (nsm == 0) return B200AWQ_ERR_DEVICE;
  const size_t want = ((vec ? count / 8 : count) + 255) / 256;
  const dim3 grid((unsigned)std::max<size_t>(1, std::min<size_t>(want, (size_t)nsm * 8)));
  if (dtype == B200AWQ_DTYPE_F16)
    return launch_kernel(silu_mul_kernel<__half>, grid, dim3(256), 0, stream, pdl, 1, gate, up, out, rows, cols, in_pitch, vec);
  return launch_kernel(silu_mul_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, pdl, 1, gate, up, out, rows, cols, in_pitch,
                       vec);
}

}  // namespace b200awq
