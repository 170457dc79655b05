"""TEST INFRASTRUCTURE ONLY.  Compile the reference's own RansacProposer (Proposer.h:155-312) into oracle/_ref/liblexp_ref_ransac.so,
around oracle/ref_ransac_driver.cpp.

Same recipe as oracle/build_ref_post.py: the reference's headers are read where they lie, under LEXP_REFERENCE_DIR; nothing of them is
copied into the repository.  Linked with -Bsymbolic so that std::random_shuffle inside the library calls the driver's rand().  When the
reference is absent (the GPU machines) build() returns the existing library, if any."""
import os
import subprocess

from oracle import build_ref as B

LIB = os.path.join(B.OUT_DIR, "liblexp_ref_ransac.so")
SOURCES = [os.path.join(B.HERE, "ref_ransac_driver.cpp"), os.path.join(B.HERE, "cvshim", "opencv2", "opencv.hpp"), os.path.abspath(__file__)]


def available():
    return os.path.exists(LIB)


def build(force=False, verbose=False):
    """Returns the path of liblexp_ref_ransac.so, or None when it neither exists nor can be built."""
    if not B.reference_present():
        return LIB if available() else None
    if available() and not force and os.path.getmtime(LIB) >= max(os.path.getmtime(p) for p in SOURCES):
        return LIB
    os.makedirs(B.OUT_DIR, exist_ok=True)
    cmd = [B.CXX, "-std=c++14", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fpermissive", "-w", "-Wl,-Bsymbolic",
           "-I", os.path.join(B.HERE, "cvshim"), "-I", os.path.join(B.HERE, "refstub"), "-I", B.REF_DIR,
           os.path.join(B.HERE, "ref_ransac_driver.cpp"), "-o", LIB + ".tmp"]
    if verbose:
        print(" ".join(cmd))
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building oracle/_ref/liblexp_ref_ransac.so failed:\n" + r.stderr[-6000:])
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
