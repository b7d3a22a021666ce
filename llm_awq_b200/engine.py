"""Locate and load the built sm_90a artefacts.  There is NO fallback: if the library or
the extension is missing (or there is no CUDA device when a kernel is called) this raises."""
import ctypes
import importlib
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
PLUGIN_DIR = os.path.join(_HERE, "plugin")
LIB_PATH = os.path.join(_HERE, "lib", "libb200awq.so")

_lib = None
_engine = None


def lib() -> ctypes.CDLL:
    """ctypes handle of libb200awq.so (C ABI of include/b200awq.h)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is not built; run `python llm_awq_b200/build.py`")
        L = ctypes.CDLL(LIB_PATH)
        vp, ci, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
        L.b200awq_w4a16_gemv.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
        L.b200awq_w4a16_gemv.restype = ci
        L.b200awq_w4a16_gemm.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, sz, vp]
        L.b200awq_w4a16_gemm.restype = ci
        L.gemv_forward_4bit.argtypes = L.b200awq_w4a16_gemv.argtypes
        L.gemv_forward_4bit.restype = ci
        L.gemm_forward_4bit.argtypes = L.b200awq_w4a16_gemm.argtypes
        L.gemm_forward_4bit.restype = ci
        L.b200awq_w4a16_gemv_allreduce.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp]
        L.b200awq_w4a16_gemv_allreduce.restype = ci
        L.b200awq_w4a16_gemm_workspace_bytes.argtypes = [ci, ci, ci]
        L.b200awq_w4a16_gemm_workspace_bytes.restype = sz
        L.b200awq_w4a16_mlp_front.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, sz, vp]
        L.b200awq_w4a16_mlp_front.restype = ci
        L.b200awq_w4a16_mlp_front_workspace_bytes.argtypes = [ci, ci, ci]
        L.b200awq_w4a16_mlp_front_workspace_bytes.restype = sz
        ll, fl = ctypes.c_longlong, ctypes.c_float
        L.b200awq_single_query_attention.argtypes = [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ll, ll, ll, ci, fl, fl, ci, ci,
                                                     vp, sz, vp]
        L.b200awq_single_query_attention.restype = ci
        L.b200awq_single_query_attention_workspace_bytes.argtypes = [ci, ci, ci, ci, ci]
        L.b200awq_single_query_attention_workspace_bytes.restype = sz
        L.b200awq_rope_with_pos.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, ci, vp]
        L.b200awq_rope_with_pos.restype = ci
        L.b200awq_rotary_embedding_neox.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci, ci, ctypes.c_longlong, ctypes.c_longlong, ci, vp]
        L.b200awq_rotary_embedding_neox.restype = ci
        L.b200awq_rmsnorm.argtypes = [vp, vp, vp, ci, ci, ctypes.c_float, ci, vp]
        L.b200awq_rmsnorm.restype = ci
        L.b200awq_set_pdl.argtypes = [ci]
        L.b200awq_set_pdl.restype = ci
        L.b200awq_launch_count.restype = ctypes.c_ulonglong
        L.b200awq_strerror.argtypes = [ci]
        L.b200awq_strerror.restype = ctypes.c_char_p
        L.b200awq_version.restype = ctypes.c_char_p
        _lib = L
    return _lib


def install() -> str:
    """Put the directory holding `awq_inference_engine*.so` first on sys.path so that the
    reference's own `import awq_inference_engine` (awq/quantize/qmodule.py:4,
    tinychat/modules/fused_mlp.py:8) resolves to this build.  Returns that directory."""
    if PLUGIN_DIR not in sys.path:
        sys.path.insert(0, PLUGIN_DIR)
    return PLUGIN_DIR


def engine():
    """The `awq_inference_engine` extension module (imports torch)."""
    global _engine
    if _engine is None:
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        install()
        mod = importlib.import_module("awq_inference_engine")
        if not os.path.abspath(getattr(mod, "__file__", "")).startswith(PLUGIN_DIR):
            raise ImportError(f"another awq_inference_engine is shadowing this build: {mod.__file__}")
        _engine = mod
    return _engine
