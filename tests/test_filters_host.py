"""The filter selection of the C-ABI and the adapters without a GPU: the lexp_params layout, and the reference's filter names in the
C++ adapter (tests/cxx/filter_name_check.cpp against the cv stub)."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_params_keep_their_size_and_a_zeroed_struct_selects_the_guided_filter():
    from localexpstereo_b200 import _capi
    assert C.sizeof(_capi.Params) == 16 * 4
    assert _capi.Params.filter.offset == 12 * 4 and _capi.Params().filter == _capi.FILTER_GF == 0
    assert (_capi.FILTER_BILATERAL, _capi.FILTER_NONE) == (1, 2)


def test_adapter_filter_names(tmp_path):
    from localexpstereo_b200 import _capi, build
    build.build()
    exe = tmp_path / "filter_name_check"
    so_dir = os.path.dirname(_capi.SO_PATH)
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "cxx"),
           os.path.join(ROOT, "tests", "cxx", "filter_name_check.cpp"), "-o", str(exe), "-L", so_dir, "-llexp_cuda", f"-Wl,-rpath,{so_dir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "filter names ok" in out.stdout, out.stdout + out.stderr
