"""In-tree build of the sm_90a library and the `awq_inference_engine` extension.

    python llm_awq_b200/build.py [--force]

Produces (git-ignored build products):
    llm_awq_b200/lib/libb200awq.so                         C ABI (include/b200awq.h), nvcc, no torch
    llm_awq_b200/plugin/awq_inference_engine<EXT>.so       pybind shim over it (g++ + torch headers)
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libb200awq.so")
EXT = os.path.join(HERE, "plugin", "awq_inference_engine" + sysconfig.get_config_var("EXT_SUFFIX"))
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

KERNEL_SRCS = ("api.cu", "w4a16_decode.cu", "w4a16_ring.cu", "w4a16_stream.cu", "w4a16_wgmma.cu", "rmsnorm.cu", "silu_mul.cu", "attention.cu", "rope_neox.cu")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC"]


def _newer(target, deps):
    return os.path.exists(target) and all(os.path.getmtime(target) >= os.path.getmtime(d) for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: " + " ".join(cmd) + "\n" + r.stdout[-3000:] + r.stderr[-6000:])
    return r


def build_lib(force=False):
    srcs = [os.path.join(CSRC, f) for f in KERNEL_SRCS]
    deps = srcs + [os.path.join(CSRC, f) for f in ("w4_common.cuh", "w4a16_kernels.h", "rope_neox.cuh")] + \
        [os.path.join(INCLUDE, "b200awq.h"), __file__]
    if not force and _newer(LIB, deps):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    _run([nvcc] + NVCC_FLAGS + ["-shared", "-Xlinker", "-soname=libb200awq.so", "-o", LIB] + srcs)
    return LIB


def build_trace_lib():
    """Debug variant with per-launch timestamps (-DB200AWQ_TRACE); not part of the product."""
    out = os.path.join(HERE, "lib", "libb200awq_trace.so")
    srcs = [os.path.join(CSRC, f) for f in KERNEL_SRCS]
    _run([os.environ.get("NVCC", "nvcc")] + NVCC_FLAGS + ["-DB200AWQ_TRACE", "-rdc=true", "-shared", "-o", out] + srcs)
    return out


def build_ext(force=False):
    src = os.path.join(CSRC, "torch_ext.cpp")
    if not force and _newer(EXT, [src, LIB, os.path.join(INCLUDE, "b200awq.h"), __file__]):
        return EXT
    from torch.utils import cpp_extension as ce
    os.makedirs(os.path.dirname(EXT), exist_ok=True)
    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}"]
    libdirs = ce.library_paths("cuda")
    cmd = (["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w",
            "-DTORCH_EXTENSION_NAME=awq_inference_engine", "-DTORCH_API_INCLUDE_EXTENSION_H",
            "-D_GLIBCXX_USE_CXX11_ABI=1"] + inc + [src, "-o", EXT, f"-L{os.path.dirname(LIB)}", "-lb200awq"]
           + [f"-L{d}" for d in libdirs] + [f"-Wl,-rpath,{d}" for d in libdirs]
           + ["-Wl,-rpath,$ORIGIN/../lib", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
              "-ltorch_python"])
    _run(cmd)
    return EXT


def build_all(force=False):
    return build_lib(force), build_ext(force)


if __name__ == "__main__":
    print(*build_all("--force" in sys.argv), sep="\n")
    if "--trace" in sys.argv:
        print(build_trace_lib())
