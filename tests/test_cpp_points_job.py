"""GPU: the C++ adapter's tw3d::get_exact_zvals_async and tw3d::heightmap_heights_async, on the thread's context and on a tile_job_pool slot beside a
heightmap frame (tests/cpp/test_points_job.cpp): the heights equal the synchronous calls', the frame is unchanged, and cancel() throws TW_ERR_STATE."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_adapter_points_job(tw, tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "test_points_job.cpp")
    exe = os.path.join(str(tmp_path), "test_points_job")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"), "-I", "/usr/local/cuda/include",
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
