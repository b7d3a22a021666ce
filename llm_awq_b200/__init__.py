"""llm_awq_b200: H100-native (sm_90a) W4A16 quantized-linear path behind llm-awq's WQLinear, and the W8A8 ops of
its vision towers.

Only what the hot path needs:
  csrc/      hand-written sm_90a CUDA + the C ABI (include/b200awq.h) + the pybind shim
  engine.py  locates / loads the built artefacts; makes `import awq_inference_engine` resolve here
  qmodule.py host-side mirror of awq/quantize/qmodule.py (WQLinear, packer)
  w8a8_linear.py  host-side mirror of awq/quantize/w8a8_linear.py (W8A8OF16LinearDynamicInputScale)
  tp.py      column / row sharding of the packed tensors + the one all-reduce
"""
from .engine import engine, install, lib  # noqa: F401
from .qmodule import WQLinear, calculate_zeros_width, pack_intweight, unpack_intweight  # noqa: F401
from .w8a8_linear import W8A8OF16LinearDynamicInputScale, quantize_weight_per_channel  # noqa: F401
