"""Builds libssegpu.so (hand-written CUDA for sm_90a + the C ABI of include/sse_gpu.h) in-tree."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# SSE_LIB: load this prebuilt library instead (A/B runs of build-time knobs on the GPU box, tools/build_variants.sh); never rebuilt
LIB = os.environ.get("SSE_LIB") or os.path.join(HERE, "libssegpu.so")
SOURCES = ["sse_fused.cu", "sse_kernel.cu", "sse_kernel2.cu", "sse_long.cu", "sse_host.cu", "sse_fold.cpp", "sse_gateway.cpp"]
HEADERS = ["sse_device.cuh", "sse_common.cuh", "sse_v2.cuh", "sse_tables.h", os.path.join("..", "..", "include", "sse_gpu.h"),
           os.path.join("..", "..", "include", "sse_gateway.h")]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libssegpu.so cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if os.environ.get("SSE_LIB"):
        return False
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
           "-Xcompiler", "-fPIC,-O2,-Wall", "-shared", "-cudart", "static",
           "-o", LIB] + os.environ.get("SSE_NVCC_DEFS", "").split() + [os.path.join(CSRC, f) for f in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
