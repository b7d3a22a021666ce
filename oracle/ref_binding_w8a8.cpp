// Our own binding around the REFERENCE's W8A8 kernels (compiled from where they lie in the checkout named by
// $AWQ_REFERENCE by oracle/build_ref_w8a8.py; sources are never copied).  Module name: ref_awq_w8a8.  Test
// infrastructure only (the stored reference outputs of tests/golden/reference_kernels_w8a8.npz and the
// "reference_on_gpu" column of bench_siglip.py).
#include <torch/extension.h>
#include "w8a8/w8a8_gemm_cuda.h"   // reference: w8a8_gemm_forward_cuda, w8a8_gemm_fuse_bias_forward_cuda
#include "w8a8/quantization.h"     // reference: invoke_quant
#include "w8a8/layernorm.h"        // reference: rms_norm_general
#include "w8a8/act.h"              // reference: gelu_and_quant, silu_and_mul

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("w8a8_gemm_forward_cuda", &w8a8_gemm_forward_cuda, "reference W8A8 GEMM (w8a8/w8a8_gemm_cuda.cu)");
  m.def("w8a8_gemm_fuse_bias_forward_cuda", &w8a8_gemm_fuse_bias_forward_cuda, "reference W8A8 GEMM + bias");
  m.def("invoke_quant", &invoke_quant, "reference per-token int8 quantisation (w8a8/quantization.cu)");
  m.def("rms_norm_general", &rms_norm_general, py::arg("out"), py::arg("input"), py::arg("weight"), py::arg("bias"),
        py::arg("scaling"), py::arg("epsilon"), py::arg("use_per_token_quant") = true,
        "reference LayerNorm + int8 quantisation (w8a8/layernorm.cu)");
  m.def("silu_and_mul", &silu_and_mul, "reference silu(x[..., :d]) * x[..., d:] (w8a8/act.cu)");
  m.def("gelu_and_quant", &gelu_and_quant, "reference gelu + per-token int8 quantisation (w8a8/act.cu)");
}
