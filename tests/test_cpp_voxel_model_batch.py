"""The C++ adapter's voxel model batches (tests/cpp/test_voxel_model_batch.cpp): six small GLM rocks built with voxel_model_build_batch_async and hit by
four frames of voxel_model_edit_batch_async (on the thread's context and on a tile_job_pool slot) give the block tables, counts, change list counts and
reads of twin models driven by voxel_model::build_async / edit_async, with remove_unconnected 0 and 3. The compile check runs without a GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_voxel_model_batch.cpp")
    exe = os.path.join(str(out_dir), "test_voxel_model_batch")
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
