"""CudaCostVolumeEnergy::setSaveDir (include/CudaCostVolumeEnergy.h), the C++ form of the run's debug images, compiles and links against
the library; the adapter's other checks (tests/cxx/adapter_check.cpp, adapter_run_check.cpp) still compile with it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_adapter_save_dir_compiles_and_links(tmp_path):
    from localexpstereo_b200 import _capi, build
    build.build()
    exe = tmp_path / "adapter_vis_check"
    so_dir = os.path.dirname(_capi.SO_PATH)
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "tests", "cxx"),
           os.path.join(ROOT, "tests", "cxx", "adapter_vis_check.cpp"), "-o", str(exe), "-L", so_dir, "-llexp_cuda", f"-Wl,-rpath,{so_dir}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "lexp version" in out.stdout, out.stderr
