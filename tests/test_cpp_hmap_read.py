"""GPU: the C++ adapter's tw3d::read_heightmap and read_heightmap_async (tests/cpp/test_hmap_read.cpp), blocking, asynchronous and on a tile_job_pool slot:
whole images and rects into host and device memory, the read after erode_heightmap_async against the synchronous chain, and the brush workflow."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("size,iters", [(256, 800), (1031, 3000)])
def test_adapter_hmap_read(tw, tmp_path, size, iters):
    src = os.path.join(ROOT, "tests", "cpp", "test_hmap_read.cpp")
    exe = os.path.join(str(tmp_path), "test_hmap_read")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           "-I", "/usr/local/cuda/include", src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe, str(size), str(iters)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
