"""GPU: the C++ adapter's tw3d::create_tiles_async_from_heightmap (tests/cpp/test_tiles_hmap.cpp): heights from the image set with tw3d::set_heightmap, erosion,
the normal map and the sun's mesh shadows from one job, equal byte for byte to create_zvals_from_heightmap followed by the adapter's synchronous calls."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_tiles_hmap.cpp")
    exe = os.path.join(str(out_dir), "test_tiles_hmap")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
def test_adapter_create_tiles_async_from_heightmap(tw, ctx, tmp_path):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
    m = re.search(r"(\d+) eroded cells, (\d+) shadowed cells", r.stdout)
    assert int(m.group(1)) > 0 and int(m.group(2)) > 0
