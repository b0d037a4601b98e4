"""Compile the CUDA library in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libaie_b200.so")
SOURCES = ["aie_abi.cu", "aie_expand_host.cpp"]
DEPS = ["aie_abi.cu", "aie_expand_host.cpp", "aie_abi.inl", "aie_core.cuh", "aie_obs.cuh", "aie_host.h", "aie_layout.h", "aie_covid_core.cuh", "aie_covid_abi.inl", "aie_compact.cuh", "aie_compact_host.h",
        "../../include/aie_b200.h"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--fmad=false",
              "-shared", "-Xcompiler", "-fPIC"]


def build_library(force=False, verbose=False, extra_flags=(), out=None):
    newest = max(os.path.getmtime(os.path.join(CSRC, d)) for d in DEPS)
    if not force and out is None and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest:
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    target = out or LIB
    cmd = [nvcc] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-o", target] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    return target
