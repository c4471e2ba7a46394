"""Build the C-ABI CUDA library in-tree (nvcc, sm_90a only).  No JIT cache: the .so sits next
to this file, so an in-tree checkout is importable once built."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200bo.so")
SOURCES = ["b200bo.cu"]
HEADERS = ["common.cuh", "select.cuh", "tc_common.cuh", "potrf_block.cuh", "fit_kernels.cuh", "predict_kernels.cuh", "predict16.cuh", "paths.cuh", os.path.join("..", "..", "include", "b200bo.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-ldl",
]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(p) > t for p in deps if os.path.exists(p))


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu -> libb200bo.so for sm_90a.  Returns the library path."""
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed:\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build_library(force=True, verbose=True))
