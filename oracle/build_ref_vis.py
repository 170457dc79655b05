"""TEST INFRASTRUCTURE ONLY.  Compile oracle/ref_vis_driver.cpp -- oracle/ref_run_driver.cpp (the reference's whole run and its real
Evaluator.h) with cv::imwrite captured -- into oracle/_ref/liblexp_ref_vis.so.

The recipe of oracle/build_ref_run.py: the reference's headers are read where they lie, under LEXP_REFERENCE_DIR, with the same dialect
fixes on scratch copies that exist only during the compiler run; nothing of them is copied into the repository.  When the reference is
absent (the GPU machines) build() returns the existing library, if any."""
import os
import shutil
import subprocess

from oracle import build_ref as B
from oracle import build_ref_run as BR

LIB = os.path.join(B.OUT_DIR, "liblexp_ref_vis.so")
SOURCES = BR.SOURCES + [os.path.join(B.HERE, "ref_vis_driver.cpp"), os.path.abspath(__file__)]


def available():
    return os.path.exists(LIB)


def build(force=False, verbose=False):
    """Returns the path of liblexp_ref_vis.so, or None when it neither exists nor can be built."""
    if not B.reference_present():
        return LIB if available() else None
    if available() and not force and os.path.getmtime(LIB) >= max(os.path.getmtime(p) for p in SOURCES):
        return LIB
    gen = os.path.join(B.OUT_DIR, "gen_vis")
    os.makedirs(gen, exist_ok=True)
    try:
        with open(os.path.join(B.REF_DIR, "GuidedFilter.h"), "r", encoding="latin-1") as f:
            fixed, n = B._dialect_fixed_guided_filter(f.read())
        if n != 17:
            raise RuntimeError(f"dialect fix touched {n} lines of GuidedFilter.h, expected 17: the reference changed")
        with open(os.path.join(gen, "GuidedFilter.h"), "w", encoding="latin-1") as f:
            f.write(fixed)
        for name, expect in (("PMStereoBase.h", 1), ("FastGCStereo.h", 3)):
            with open(os.path.join(B.REF_DIR, name), "r", encoding="latin-1") as f:
                fixed, n = B._dialect_fixed_optimiser(f.read())
            if n != expect:
                raise RuntimeError(f"dialect fix touched {n} lines of {name}, expected {expect}: the reference changed")
            with open(os.path.join(gen, name), "w", encoding="latin-1") as f:
                f.write(fixed)
        # oracle/ sits before -I- with the scratch copies: the driver's #include "ref_run_driver.cpp" is a quoted include
        cmd = [B.CXX, "-std=c++14", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fpermissive", "-w",
               "-I", gen, "-I", B.HERE, "-I-", "-I", os.path.join(B.HERE, "cvshim"), "-I", B.REF_DIR,
               os.path.join(B.HERE, "ref_vis_driver.cpp"), "-o", LIB + ".tmp"]
        if verbose:
            print(" ".join(cmd))
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("building oracle/_ref/liblexp_ref_vis.so failed:\n" + r.stderr[-6000:])
        os.replace(LIB + ".tmp", LIB)
    finally:
        shutil.rmtree(gen, ignore_errors=True)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
