"""The C++ adapter's voxel model jobs on tile_job_pool slots (tests/cpp/test_voxel_model_family.cpp): a build, brush edits and reads launched on the
slots of a pool of 4, none waited for until all are launched and then newest first, give the block tables, counts and reads of the same script on the
thread's context alone, with remove_unconnected 0 and 3; a read between two strokes sees the first only, and a box read equals the whole grid's slice.
The compile check runs without a GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_voxel_model_family.cpp")
    exe = os.path.join(str(out_dir), "test_voxel_model_family")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


def test_adapter_voxel_model_family_compiles(tw, tmp_path):
    assert os.access(build_exe(tw, tmp_path), os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("rm", [0, 3])
def test_adapter_voxel_model_family(tw, ctx, tmp_path, rm):
    g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
    for name, dt in (("edge_table", np.uint32), ("tri_table", np.int32), ("edge_to_vals", np.uint32)):
        np.ascontiguousarray(g[name], dt).tofile(str(tmp_path / (name + ".bin")))
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(tmp_path), str(rm)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
