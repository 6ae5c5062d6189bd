"""Build recipe for libb200drr.so (hand-written sm_90a CUDA kernels + the C ABI of include/b200drr.h).

The library is built IN-TREE (diffdrr_b200/libb200drr.so) with nvcc, so the artefact travels with a
`gpurun` snapshot; nvcc cross-compiles without a GPU.  No torch headers are involved: the boundary is a
plain C ABI (pointers + sizes + a cudaStream_t), bound from Python with ctypes (diffdrr_b200/_lib.py).
"""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libb200drr.so")
SOURCES = ["siddon.cu", "siddon_brick.cu", "trilinear.cu", "literal.cu", "pose.cu", "ncc.cu", "local_ncc.cu", "sobel.cu", "capi.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libb200drr.so cannot be built")
    return nvcc


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(os.path.dirname(_HERE), "include", "b200drr.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA extension for sm_90a if it is missing or older than its sources."""
    if not force and not _stale():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH + ".tmp", *[os.path.join(CSRC, s) for s in SOURCES]]
    if os.environ.get("B200DRR_BUILD_EXPERIMENTS") == "1":  # rejected kernel experiments (include/b200drr_experimental.h)
        cmd.insert(1, "-DB200DRR_EXPERIMENTS")
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + proc.stdout + proc.stderr)
    if verbose:
        print(proc.stderr)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
