"""GPU: the C++ adapter's tw3d::voxel_mesh and the voxel_build_async overload with mesh outputs (tests/cpp/test_voxel_mesh.cpp): one job's soup and welded
mesh equal byte for byte to the synchronous create_procedural + voxel_build + voxel_mesh, in sine and GLM simplex mode, with remove_unconnected 1 and 3."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_exe(tw, out_dir):
    src = os.path.join(ROOT, "tests", "cpp", "test_voxel_mesh.cpp")
    exe = os.path.join(str(out_dir), "test_voxel_mesh")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"),
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-o", exe])
    return exe


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rm", [(0, 3), (1, 1)])
def test_adapter_voxel_mesh(tw, ctx, tmp_path, mode, rm):
    g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
    for name, dt in (("edge_table", np.uint32), ("tri_table", np.int32), ("edge_to_vals", np.uint32)):
        np.ascontiguousarray(g[name], dt).tofile(str(tmp_path / (name + ".bin")))
    exe = build_exe(tw, tmp_path)
    r = subprocess.run([exe, str(tmp_path), str(mode), str(rm)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
