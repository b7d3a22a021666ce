"""Build oracle/_ref/ref_awq_engine*.so: the REFERENCE's own W4A16 kernels for sm_90a.

Compiles awq/kernels/csrc/quantization_new/{gemv/gemv_cuda.cu,gemm/gemm_cuda.cu}, layernorm/layernorm.cu and
position_embedding/pos_encoding_kernels.cu from
an llm-awq checkout named by $AWQ_REFERENCE (nothing is copied into this repo) with the
reference's nvcc flags (awq/kernels/setup.py:7-21) plus an explicit sm_90a gencode,
and links them with oracle/ref_binding.cpp.  Output goes to oracle/_ref/ (git-ignored).
Does not run the reference's setup.py.  The GPU tests do not need it: they compare with
the reference outputs stored under tests/golden/ (tests/golden/make_ref_kernel_golden.py).

Usage: AWQ_REFERENCE=<llm-awq checkout> python oracle/build_ref.py     (about 5 minutes; skipped if up to date)
"""
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("AWQ_REFERENCE", "")
CSRC = os.path.join(REF, "awq/kernels/csrc")
OUT = os.path.join(HERE, "_ref")
EXT = sysconfig.get_config_var("EXT_SUFFIX")
TARGET = os.path.join(OUT, "ref_awq_engine" + EXT)


def available() -> bool:
    return bool(REF) and os.path.isdir(CSRC)


def build(force: bool = False) -> str | None:
    if not available():
        return TARGET if os.path.exists(TARGET) else None
    srcs = [os.path.join(CSRC, "quantization_new/gemv/gemv_cuda.cu"),
            os.path.join(CSRC, "quantization_new/gemm/gemm_cuda.cu"),
            os.path.join(CSRC, "layernorm/layernorm.cu"),
            os.path.join(CSRC, "position_embedding/pos_encoding_kernels.cu")]
    bind = os.path.join(HERE, "ref_binding.cpp")
    if not force and os.path.exists(TARGET) and all(
            os.path.getmtime(TARGET) > os.path.getmtime(s) for s in srcs + [bind, __file__]):
        return TARGET
    os.makedirs(OUT, exist_ok=True)
    from torch.utils import cpp_extension as ce
    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}", f"-I{CSRC}"]
    common = ["-DTORCH_EXTENSION_NAME=ref_awq_engine", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-D_GLIBCXX_USE_CXX11_ABI=1", "-DENABLE_BF16"]
    nvcc = ["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
            "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
            "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
            "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
            "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
            "-Xcompiler", "-fPIC", "-w"] + common + inc
    objs = [os.path.join(OUT, "gemv_cuda.o"), os.path.join(OUT, "gemm_cuda.o"), os.path.join(OUT, "layernorm.o"),
            os.path.join(OUT, "pos_encoding_kernels.o"), os.path.join(OUT, "ref_binding.o")]
    cmds = [nvcc + ["-c", srcs[0], "-o", objs[0]],
            nvcc + ["-c", srcs[1], "-o", objs[1]],
            nvcc + ["-c", srcs[2], "-o", objs[2]],
            nvcc + ["-c", srcs[3], "-o", objs[3]],
            ["g++", "-O2", "-std=c++17", "-fPIC", "-w"] + common + inc + ["-c", bind, "-o", objs[4]]]
    with ThreadPoolExecutor(5) as ex:
        for r in ex.map(lambda c: subprocess.run(c, capture_output=True, text=True), cmds):
            if r.returncode != 0:
                raise RuntimeError("reference build failed:\n" + r.stderr[-4000:])
    libdirs = ce.library_paths("cuda")
    link = ["g++", "-shared", "-o", TARGET] + objs + [f"-L{d}" for d in libdirs] + \
           [f"-Wl,-rpath,{d}" for d in libdirs] + ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
                                                    "-ltorch_python", "-lcudart"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("reference link failed:\n" + r.stderr[-4000:])
    for o in objs:
        os.remove(o)
    return TARGET


if __name__ == "__main__":
    t = build(force="--force" in sys.argv)
    print("reference oracle:", t)
