"""Builds the CUDA extension in-tree: localexpstereo_b200/liblexp_cuda.so (sm_90a only)."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "liblexp_cuda.so")
# the kernels of the bilateral filter and the unfiltered mode (csrc/lexp_filters.cu) are a library of their own that liblexp_cuda.so
# links (found next to it through its run path): liblexp_cuda.so keeps exactly the kernels it had before them
FILTERS_SO = os.path.join(HERE, "liblexp_filters.so")
# the kernels of the reference's debug images (csrc/lexp_vis.cu) likewise: liblexp_vis.so, linked the same way
VIS_SO = os.path.join(HERE, "liblexp_vis.so")
SRCS = [os.path.join(HERE, "csrc", "lexp_capi.cu")]
FILTERS_SRCS = [os.path.join(HERE, "csrc", "lexp_filters.cu")]
VIS_SRCS = [os.path.join(HERE, "csrc", "lexp_vis.cu")]
DEPS = SRCS + FILTERS_SRCS + VIS_SRCS + sorted(glob.glob(os.path.join(HERE, "csrc", "*.cuh"))) + [os.path.join(HERE, "..", "include", "lexp_cuda.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-Xptxas=-v",
]


def needs_build():
    if not all(os.path.exists(f) for f in (SO, FILTERS_SO, VIS_SO)):
        return True
    t = min(os.path.getmtime(f) for f in (SO, FILTERS_SO, VIS_SO))
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    log = ""
    for out, cmd in ((FILTERS_SO, [nvcc] + NVCC_FLAGS + ["-o", FILTERS_SO] + FILTERS_SRCS),
                     (VIS_SO, [nvcc] + NVCC_FLAGS + ["-o", VIS_SO] + VIS_SRCS),
                     (SO, [nvcc] + NVCC_FLAGS + ["-o", SO] + SRCS + ["-L", HERE, "-llexp_filters", "-llexp_vis", "-Xlinker", "-rpath,$ORIGIN"])):
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed building {os.path.basename(out)}")
        log += res.stdout + res.stderr
    with open(os.path.join(HERE, "build_ptxas.log"), "w") as f:
        f.write(log)
    return SO


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(SO)
