"""GPU: the C++ adapter's tw3d::proc_gen_heightmap_async (tests/cpp/test_heightmap_job.cpp) equal byte for byte to the adapter's synchronous
proc_gen_heightmap, without erosion, on the tile-style erosion path and on the speculative one, and with the image set for heightmap tiles."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_heightmap_job.cpp")
    exe = os.path.join(str(out_dir), "test_heightmap_job")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("mode,size,iters", [(1, 300, 0), (4, 256, 800), (4, 1024, 3000)])
def test_adapter_proc_gen_heightmap_async(tw, tmp_path, mode, size, iters):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(mode), str(size), str(iters)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
