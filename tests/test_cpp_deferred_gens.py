"""GPU: the C++ adapter's tw3d::set_deferred_gens(8) and tw3d::tile_job_pool (tests/cpp/test_deferred_gens.cpp) - eight deferred height generations in flight on
shared contexts and two frames' tile jobs on a pool, each equal value for value to the adapter's blocking calls."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_deferred_gens.cpp")
    exe = os.path.join(str(out_dir), "test_deferred_gens")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [3, 4])
def test_adapter_deferred_gens_and_pool(tw, ctx, tmp_path, mode):
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(mode)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
