"""llm_awq_b200: H100-native (sm_90a) W4A16 quantized-linear path behind llm-awq's WQLinear.

Only what the hot path needs:
  csrc/      hand-written sm_90a CUDA + the C ABI (include/b200awq.h) + the pybind shim
  engine.py  locates / loads the built artefacts; makes `import awq_inference_engine` resolve here
  qmodule.py host-side mirror of awq/quantize/qmodule.py (WQLinear, packer)
  tp.py      column / row sharding of the packed tensors + the one all-reduce
"""
from .engine import engine, install, lib  # noqa: F401
from .qmodule import WQLinear, calculate_zeros_width, pack_intweight, unpack_intweight  # noqa: F401
