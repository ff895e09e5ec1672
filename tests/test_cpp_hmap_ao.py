"""GPU: the C++ adapter's tw3d::hmap_tile_ao_async (tests/cpp/test_hmap_ao.cpp): tile_set::hmap_ao_async on a tile_job_pool slot right after a heightmap
frame on another slot, and tile_job_pool::hmap_tile_ao_async, against the blocking tw3d::hmap_tile_ao on the synchronous chain's zvals."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_adapter_hmap_ao(tw, tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "test_hmap_ao.cpp")
    exe = os.path.join(str(tmp_path), "test_hmap_ao")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           "-I", "/usr/local/cuda/include", src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
