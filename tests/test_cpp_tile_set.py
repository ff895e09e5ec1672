"""GPU: the C++ adapter's tw3d::tile_set (tests/cpp/test_tile_set.cpp): a job's device zvals put into the set, relit with two lights, then a new row of tiles
on the sun's side put and only the stale tiles relit - every relight equal byte for byte to the adapter's calc_mesh_shadows over all resident tiles."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_tile_set.cpp")
    exe = os.path.join(str(out_dir), "test_tile_set")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           "-I", "/usr/local/cuda/include", src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-L/usr/local/cuda/lib64", "-lcudart",
                           "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 4])
def test_adapter_tile_set_relight(tw, ctx, tmp_path, mode):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(mode)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
    assert int(re.search(r"(\d+) shadowed cells", r.stdout).group(1)) > 0
    assert int(re.search(r"(\d+) recomputed", r.stdout).group(1)) > 0
