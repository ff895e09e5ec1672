"""GPU: the shadows overload of the C++ adapter's tw3d::create_tiles_async (tests/cpp/test_tiles_shadows.cpp): heights and the mesh shadows of two lights
from one job, equal byte for byte to the adapter's calc_mesh_shadows on the job's zvals."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_tiles_shadows.cpp")
    exe = os.path.join(str(out_dir), "test_tiles_shadows")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 4])
def test_adapter_create_tiles_async_with_shadows(tw, ctx, tmp_path, mode):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(mode)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
    assert int(re.search(r"(\d+) shadowed cells", r.stdout).group(1)) > 0
