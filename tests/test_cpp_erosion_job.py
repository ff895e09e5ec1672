"""GPU: the C++ adapter's tw3d::apply_erosion_async / apply_erosion_parallel_async / erode_heightmap_async (tests/cpp/test_erosion_job.cpp) equal byte for
byte to tw3d::apply_erosion, apply_erosion_parallel(..., 1) and the synchronous image chain, on the tile-style erosion path and on the speculative one."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_erosion_job.cpp")
    exe = os.path.join(str(out_dir), "test_erosion_job")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("size,iters", [(256, 800), (1024, 3000)])
def test_adapter_erosion_async(tw, tmp_path, size, iters):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(size), str(iters)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
