// Our own 4-function binding around the REFERENCE's W4A16 kernels (compiled from where
// they lie in the checkout named by $AWQ_REFERENCE by oracle/build_ref.py; sources are never copied).
// Module name: ref_awq_engine.  Test infrastructure only (GPU-side parity oracle and the
// "reference_on_gpu" timing column of bench.py).
#include <torch/extension.h>
#include "quantization_new/gemm/gemm_cuda.h"   // reference: gemm_forward_cuda_new
#include "quantization_new/gemv/gemv_cuda.h"   // reference: gemv_forward_cuda_new
#include "layernorm/layernorm.h"               // reference: layernorm_forward_cuda
#include "position_embedding/pos_encoding.h"   // reference: rotary_embedding_neox

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("gemm_forward_cuda_new", &gemm_forward_cuda_new, "reference W4A16 GEMM (quantization_new)");
  m.def("gemv_forward_cuda_new", &gemv_forward_cuda_new, "reference W4A16 GEMV (quantization_new)");
  m.def("layernorm_forward_cuda", &layernorm_forward_cuda, "reference RMSNorm (layernorm/layernorm.cu)");
  m.def("rotary_embedding_neox", &rotary_embedding_neox, "reference in-place NeoX RoPE (position_embedding/pos_encoding_kernels.cu)");
}
