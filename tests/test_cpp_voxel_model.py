"""GPU: the C++ adapter's tw3d::voxel_model (tests/cpp/test_voxel_model.cpp): a one-block model's mesh equal to tw3d::voxel_mesh, the blocked model's
field and flags equal to create_procedural + voxel_build, and brush edits whose re-meshed blocks equal a fresh model's, byte for byte, with
remove_unconnected 0 and 3."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_voxel_model.cpp")
    exe = os.path.join(str(out_dir), "test_voxel_model")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


def test_adapter_voxel_model_compiles(tw, tmp_path):
    assert os.access(build_exe(tw, tmp_path), os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("rm", [0, 3])
def test_adapter_voxel_model(tw, ctx, tmp_path, rm):
    g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
    for name, dt in (("edge_table", np.uint32), ("tri_table", np.int32), ("edge_to_vals", np.uint32)):
        np.ascontiguousarray(g[name], dt).tofile(str(tmp_path / (name + ".bin")))
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(tmp_path), str(rm)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
