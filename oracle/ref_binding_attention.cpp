// Our own binding around the REFERENCE's decode-attention kernel (compiled from where it lies in the checkout named
// by $AWQ_REFERENCE by oracle/build_ref_attention.py; sources are never copied).  Module name: ref_awq_attention.
// Test infrastructure only (the stored reference outputs of tests/golden/reference_kernels_attention.npz).
#include <torch/extension.h>
#include "attention/ft_attention.h"  // reference: single_query_attention (attention/ft_attention.cpp)

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("single_query_attention", &single_query_attention, "reference decode attention (attention/ft_attention.cpp)",
        py::arg("q"), py::arg("k"), py::arg("v"), py::arg("k_cache"), py::arg("v_cache"), py::arg("length_per_sample_"),
        py::arg("alibi_slopes_"), py::arg("timestep"), py::arg("rotary_embedding_dim") = 0,
        py::arg("rotary_base") = 10000.0f, py::arg("rotary_scale") = 1.0f, py::arg("neox_rotary_style") = true);
}
