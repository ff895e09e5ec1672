"""The C++ adapter's change list (tests/cpp/test_voxel_changes.cpp): tw3d::voxel_model::edit_async with a tw_voxel_changes, whose list patched into the
engine's copies of the field and flags gives voxel_model::read after every brush edit, byte for byte, with remove_unconnected 0 and 3; and an
overflowing list that reports its full count and is refused by apply_changes. The compile check runs without a GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_voxel_changes.cpp")
    exe = os.path.join(str(out_dir), "test_voxel_changes")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


def test_adapter_voxel_changes_compiles(tw, tmp_path):
    assert os.access(build_exe(tw, tmp_path), os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("rm", [0, 3])
def test_adapter_voxel_changes(tw, ctx, tmp_path, rm):
    g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
    for name, dt in (("edge_table", np.uint32), ("tri_table", np.int32), ("edge_to_vals", np.uint32)):
        np.ascontiguousarray(g[name], dt).tofile(str(tmp_path / (name + ".bin")))
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(tmp_path), str(rm)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
