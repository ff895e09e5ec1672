"""GPU: the C++ adapter's tw3d::gen_mesh_async against tw3d::gen_mesh, on the thread's context and on a tile_job_pool slot (tests/cpp/test_gen_mesh_job.cpp):
the mesh, the z values, the step count and the scene_globals it leaves equal gen_mesh's, flat mesh included."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_adapter_gen_mesh_job(tw, tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "test_gen_mesh_job.cpp")
    exe = os.path.join(str(tmp_path), "test_gen_mesh_job")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"), "-I", "/usr/local/cuda/include",
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
