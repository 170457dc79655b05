"""The whole-run kernels (lexp_run.cuh) were added without touching any existing kernel: every kernel listed in
tests/golden/sass_kernels.json must compile to the same SASS instructions as when the list was minted (tests/golden/make_sass_hashes.py).
Needs cuobjdump and the library build() made; no GPU."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_sass_hashes as M   # noqa: E402

SO = os.path.join(os.path.dirname(HERE), "localexpstereo_b200", "liblexp_cuda.so")


@pytest.mark.skipif(not os.path.exists(M.CUOBJDUMP), reason="cuobjdump is not installed")
def test_existing_kernels_have_the_same_sass():
    if not os.path.exists(SO):
        from localexpstereo_b200 import build
        build.build()
    want = json.load(open(os.path.join(HERE, "golden", "sass_kernels.json")))
    got = M.kernel_hashes(SO)
    assert len(want) == 46
    changed = sorted(k for k in want if got.get(k) != want[k])
    assert not changed, changed
    assert sorted(set(got) - set(want)) == ["_ZN4lexp16lexp_eval_finishEPKxiPx", "_ZN4lexp16lexp_eval_kernelEPK6float4PKfPKhPxiiff",
                                            "_ZN4lexp24lexp_random_start_kernelEPKNS_8CallInfoEiPNS_6Plane4Eyff"]
