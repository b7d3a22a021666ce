"""Build oracle/_ref/ref_awq_attention*.so: the REFERENCE's own decode-attention kernel for sm_90a.

Compiles awq/kernels/csrc/attention/{ft_attention.cpp,decoder_masked_multihead_attention.cu} (FasterTransformer's
masked multi-head attention, every head size it dispatches in one translation unit) from the llm-awq checkout named by
$AWQ_REFERENCE (nothing is copied into this repo) with the reference's flags (awq/kernels/setup.py:5-21, -DENABLE_BF16
included) plus an explicit sm_90a gencode, and links them with oracle/ref_binding_attention.cpp.  Output goes to
oracle/_ref/ (git-ignored).  The GPU tests do not need it: they compare with the reference outputs stored under
tests/golden/ (tests/golden/make_attention_ref_kernel_golden.py).

Usage: AWQ_REFERENCE=<llm-awq checkout> python oracle/build_ref_attention.py   (about 2 minutes; skipped if up to date)
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
TARGET = os.path.join(OUT, "ref_awq_attention" + sysconfig.get_config_var("EXT_SUFFIX"))
CU_SRC = "attention/decoder_masked_multihead_attention.cu"
CPP_SRC = "attention/ft_attention.cpp"


def available() -> bool:
    return bool(REF) and os.path.isfile(os.path.join(CSRC, CU_SRC))


def build(force: bool = False) -> str | None:
    if not available():
        return TARGET if os.path.exists(TARGET) else None
    cu, cpp = os.path.join(CSRC, CU_SRC), os.path.join(CSRC, CPP_SRC)
    bind = os.path.join(HERE, "ref_binding_attention.cpp")
    if not force and os.path.exists(TARGET) and all(
            os.path.getmtime(TARGET) > os.path.getmtime(s) for s in (cu, cpp, bind, __file__)):
        return TARGET
    os.makedirs(OUT, exist_ok=True)
    from torch.utils import cpp_extension as ce
    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}", f"-I{CSRC}",
                                                          f"-I{os.path.join(CSRC, 'attention')}"]
    common = ["-DTORCH_EXTENSION_NAME=ref_awq_attention", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-D_GLIBCXX_USE_CXX11_ABI=1", "-DENABLE_BF16"]
    nvcc = ["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
            "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
            "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
            "-U__CUDA_NO_BFLOAT162_OPERATORS__", "-U__CUDA_NO_BFLOAT162_CONVERSIONS__",
            "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
            "-Xcompiler", "-fPIC", "-w"] + common + inc
    cxx = ["g++", "-O3", "-std=c++17", "-fPIC", "-w"] + common + inc
    objs = [os.path.join(OUT, "attn_" + n + ".o") for n in ("mmha", "ft_attention", "ref_binding_attention")]
    cmds = [nvcc + ["-c", cu, "-o", objs[0]], cxx + ["-c", cpp, "-o", objs[1]], cxx + ["-c", bind, "-o", objs[2]]]
    with ThreadPoolExecutor(len(cmds)) as ex:
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
    print("reference attention oracle:", t)
