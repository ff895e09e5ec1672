"""GPU: the C++ adapter's mesh shadows of the ground-mode mesh (tests/cpp/test_mesh_shadows.cpp): the blocking calc_mesh_shadows overload, mesh_shadows_async
on the thread's context and on a tile_job_pool slot, and gen_mesh_async with lights, byte for byte against each other and against the oracle's
calc_mesh_shadows on a non-square mesh written here."""
import os
import subprocess

import numpy as np
import pytest

from cases import convert

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


@pytest.mark.gpu
def test_adapter_mesh_shadows(tw, oracle, tmp_path):
    xs, ys, xss, yss = 300, 170, 4.0, 3.0
    rng = np.random.default_rng(5)
    z = (F(0.5) * np.sin(np.arange(xs, dtype=F) * F(0.07))[None, :] + F(0.2) * rng.standard_normal((ys, xs)).astype(F)).astype(F)
    zmin, zmax = float(z.min()) - 0.5, float(z.max()) + 0.5
    lights = [(3.0, -2.0, 1.2), (-1.5, -4.0, 0.6), (2.0, 5.0, 0.3)]
    # the adapter keeps DX_VAL_INV = 1/DX_VAL and its mesh_shadow_params takes dx_val = 1/DX_VAL_INV, dx_val_inv = 1/dx_val
    dx, dy = (F(1.0) / (F(1.0) / (F(F(2.0) * F(ss)) / F(n))) for ss, n in ((xss, xs), (yss, ys)))
    for l, lp in enumerate(lights):
        sp = tw.ShadowParams()
        for d in range(3):
            sp.lpos[d] = lp[d]
        sp.x_scene_size, sp.y_scene_size, sp.dx_val, sp.dy_val = xss, yss, float(dx), float(dy)
        sp.dx_val_inv, sp.dy_val_inv = float(F(1.0) / dx), float(F(1.0) / dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = xs + ys, zmin, zmax, 0
        m, ox, oy = oracle.calc_mesh_shadows(convert(sp, oracle.ShadowParams), z)
        (tmp_path / ("oracle_%d.bin" % l)).write_bytes(m.tobytes() + ox.tobytes() + oy.tobytes())
    (tmp_path / "mesh.f32").write_bytes(z.tobytes())
    (tmp_path / "params.f32").write_bytes(np.array([xs, ys, xss, yss, zmin, zmax, len(lights)] + [v for lp in lights for v in lp], F).tobytes())
    src = os.path.join(ROOT, "tests", "cpp", "test_mesh_shadows.cpp")
    exe = os.path.join(str(tmp_path), "test_mesh_shadows")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"), "-I", "/usr/local/cuda/include",
                           src, "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200", "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
