"""Build recipe for libdfq_sm90.so (hand-written sm_90a CUDA behind a C ABI).

The library is built IN-TREE next to this file so that the package is importable from the repository tree; it is
git-ignored.  nvcc cross-compiles for sm_90a without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("DFQ_LIB_OUT") or os.path.join(HERE, "libdfq_sm90.so")
SOURCES = ["tensor_ops.cu", "cle_engine.cu", "passes.cu", "distill.cu", "host_copy.cu", "int8_conv.cu"]
HEADERS = [os.path.join(CSRC, h) for h in ("common.cuh", "rowpipe.cuh", "colscan.cuh", "bc_stream.cuh")] + \
    [os.path.join(HERE, "..", "include", "dfq_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--fmad=false",          # every fp32 op of the reference is individually rounded: never contract
    "-Xcompiler", "-fPIC", "-shared",
    "-Xptxas", "-v",
]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("DFQ_NVCC_DEFS", "").split()      # tuning experiments, e.g. -DDFQ_PIPE_STAGES=5 -DDFQ_CTAS=2
    cmd = [nvcc] + NVCC_FLAGS + extra + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES] + ["-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libdfq_sm90.so")
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
