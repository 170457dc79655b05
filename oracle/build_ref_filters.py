"""TEST INFRASTRUCTURE ONLY.  Compile the reference's own energies with the bilateral filter and without a filter
(CostVolumeEnergy "BL" / "", NaiveStereoEnergy "BF" / "": CostVolumeEnergy.h:23-42, StereoEnergy.h:666-686, GuidedFilter.h:329-373)
into oracle/_ref/liblexp_ref_filters.so, around oracle/ref_filter_driver.cpp.

Same recipe as oracle/build_ref.py (whose dialect fixes it reuses on scratch copies that exist only during the compiler run): the
reference's headers are read where they lie, under LEXP_REFERENCE_DIR; nothing of them is copied into the repository.  When the
reference is absent (the GPU machines) build() returns the existing library, if any."""
import os
import shutil
import subprocess

from oracle import build_ref as B

LIB = os.path.join(B.OUT_DIR, "liblexp_ref_filters.so")
SOURCES = [os.path.join(B.HERE, "ref_filter_driver.cpp"), os.path.join(B.HERE, "cvshim", "opencv2", "opencv.hpp"), os.path.abspath(__file__)]


def available():
    return os.path.exists(LIB)


def build(force=False, verbose=False):
    """Returns the path of liblexp_ref_filters.so, or None when it neither exists nor can be built."""
    if not B.reference_present():
        return LIB if available() else None
    if available() and not force and os.path.getmtime(LIB) >= max(os.path.getmtime(p) for p in SOURCES):
        return LIB
    gen = os.path.join(B.OUT_DIR, "gen_filters")
    os.makedirs(gen, exist_ok=True)
    try:
        with open(os.path.join(B.REF_DIR, "GuidedFilter.h"), "r", encoding="latin-1") as f:
            fixed, n = B._dialect_fixed_guided_filter(f.read())
        if n != 17:
            raise RuntimeError(f"dialect fix touched {n} lines of GuidedFilter.h, expected 17: the reference changed")
        with open(os.path.join(gen, "GuidedFilter.h"), "w", encoding="latin-1") as f:
            f.write(fixed)
        cmd = [B.CXX, "-std=c++14", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fpermissive", "-w",
               "-I", gen, "-I-", "-I", os.path.join(B.HERE, "cvshim"), "-I", os.path.join(B.HERE, "refstub"), "-I", B.REF_DIR,
               os.path.join(B.HERE, "ref_filter_driver.cpp"), "-o", LIB + ".tmp"]
        if verbose:
            print(" ".join(cmd))
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("building oracle/_ref/liblexp_ref_filters.so failed:\n" + r.stderr[-6000:])
        os.replace(LIB + ".tmp", LIB)
    finally:
        shutil.rmtree(gen, ignore_errors=True)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
