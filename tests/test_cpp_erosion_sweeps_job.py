"""GPU: the C++ adapter's tw3d::apply_erosion_sweeps_async / erode_heightmap_sweeps_async (tests/cpp/test_erosion_sweeps_job.cpp) equal byte for byte to
tw3d::apply_erosion_sweeps and the synchronous image chain, and tiles_job::cancel() / cancelled() on a long job and on one that has ended."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_erosion_sweeps_job.cpp")
    exe = os.path.join(str(out_dir), "test_erosion_sweeps_job")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("size,iters,sweep,halo", [(256, 5000, 500, 44), (1024, 30000, 2048, 64)])
def test_adapter_erosion_sweeps_async(tw, tmp_path, size, iters, sweep, halo):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(size), str(iters), str(sweep), str(halo)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
