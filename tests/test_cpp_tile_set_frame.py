"""GPU: the C++ adapter's tw3d::tile_set::create_tiles_async (tests/cpp/test_tile_set_frame.cpp): six camera frames, each a far row evicted, a new row on the
sun's side created into the set and the stale tiles relit in one job - on the thread's context and on a tw3d::tile_job_pool with frames in flight together -
equal byte for byte to the same frames as separate calls on a second set."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_tile_set_frame.cpp")
    exe = os.path.join(str(out_dir), "test_tile_set_frame")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           "-I", "/usr/local/cuda/include", src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-L/usr/local/cuda/lib64", "-lcudart",
                           "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe])
    return exe


def test_adapter_frame_compiles(tw, tmp_path):
    assert os.access(build_exe(tw, tmp_path), os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,slots", [(0, 0), (4, 0), (4, 6)])
def test_adapter_tile_set_frames(tw, ctx, tmp_path, mode, slots):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(mode), str(slots)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
    assert int(re.search(r"(\d+) shadowed cells", r.stdout).group(1)) > 0
    assert int(re.search(r"(\d+) recomputed", r.stdout).group(1)) > 0
