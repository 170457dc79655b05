"""Builds the CUDA extension in-tree: localexpstereo_b200/liblexp_cuda.so (sm_90a only)."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "liblexp_cuda.so")
SRCS = [os.path.join(HERE, "csrc", "lexp_capi.cu")]
DEPS = SRCS + sorted(glob.glob(os.path.join(HERE, "csrc", "*.cuh"))) + [os.path.join(HERE, "..", "include", "lexp_cuda.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-Xptxas=-v",
]


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", SO] + SRCS
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building liblexp_cuda.so")
    with open(os.path.join(HERE, "build_ptxas.log"), "w") as f:
        f.write(res.stdout + res.stderr)
    return SO


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(SO)
