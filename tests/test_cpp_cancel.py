"""GPU: the C++ adapter's tiles_job::cancel() / cancelled() (tests/cpp/test_cancel.cpp): a cancelled pool job is ready soon and its slot runs the next job
exactly; a handle destroyed right after cancel() waits only briefly; cancel() on a complete job changes nothing."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_adapter_cancel(tw, tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "test_cancel.cpp")
    exe = os.path.join(str(tmp_path), "test_cancel")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"), "-I", "/usr/local/cuda/include",
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe, "1000000"], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
