"""Mints tests/golden/sass_kernels.json: a SHA-256 per kernel of the SASS that `cuobjdump -sass` prints for a liblexp_cuda.so (instruction
lines only).  The committed file holds the kernels the library had before the whole-run kernels (lexp_run.cuh) were added:
    python tests/golden/make_sass_hashes.py path/to/liblexp_cuda.so > tests/golden/sass_kernels.json"""
import hashlib
import json
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernel_hashes(so):
    text = subprocess.run([CUOBJDUMP, "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = hashlib.sha256()
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            funcs[cur].update(line.strip().encode() + b"\n")
    return {k: v.hexdigest() for k, v in sorted(funcs.items())}


if __name__ == "__main__":
    json.dump(kernel_hashes(sys.argv[1]), sys.stdout, indent=1)
    sys.stdout.write("\n")
