"""CPU: mesh shadows of one whole mesh on the host side - the three entry points are exported and listed in ABI_SYMBOLS, the ctypes mirror of
tw_mesh_shadows_job matches the header, NULL contexts and bad sizes are refused; every kernel of the build before tw_mesh_shadows existed keeps its SASS
(tests/golden/sass_before_mesh_shadows.json) and the new kernels are exactly the mesh pass's; the oracle's calc_mesh_shadows on a square mesh equals its
tile batch of one tile; and, where oracle/_ref is built, the oracle's calc_mesh_shadows on non-square meshes equals the reference's own."""
import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from cases import convert

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
ENTRY_POINTS = ("tw_mesh_shadows", "tw_mesh_shadows_launch", "tw_gen_mesh_launch_shadows")


def test_entry_points_are_exported(tw):
    for name in ENTRY_POINTS:
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    assert tw.lib.tw_abi_version() == 1


def test_job_layout(tw, tmp_path):
    fields = [f for f, _ in tw.MeshShadowsJobArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tw3d.h"\nint main(void) {printf("%zu", sizeof(tw_mesh_shadows_job)); '
                   + "".join('printf(" %%zu", offsetof(tw_mesh_shadows_job, %s)); ' % f for f in fields) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(tw.MeshShadowsJobArgs)] + [getattr(tw.MeshShadowsJobArgs, f).offset for f in fields]


def test_null_context_and_bad_sizes_are_refused(tw):
    sp = tw.ShadowParams()
    m = np.zeros((4, 4), np.uint8)
    z = np.zeros((4, 4), F)
    for xs, ys in ((4, 4), (1, 4), (4, 1), (0, 0), (-3, 4)):
        assert tw.lib.tw_mesh_shadows(None, tw._ptr(z), xs, ys, C.byref(sp), None, None, tw._ptr(m), None, None) == tw.TW_ERR_ARG
    job = tw.MeshShadowsJobArgs(tw._ptr(z), 4, 4, 0, None)
    assert tw.lib.tw_mesh_shadows_launch(None, C.byref(job)) == tw.TW_ERR_ARG
    assert tw.lib.tw_mesh_shadows_launch(None, None) == tw.TW_ERR_ARG
    assert tw.lib.tw_gen_mesh_launch_shadows(None, None, 0, None) == tw.TW_ERR_ARG


SASS_CUDA = "12.9"
NEW_KERNELS = {"_ZNANON_tw_shadows23mesh_shadow_init_kernelEPK14twi_mesh_lightmi",
               "_ZNANON_tw_shadows23mesh_shadow_rays_kernelEPKfiiPK14twi_mesh_lightP13twi_job_words",
               "_ZNANON_tw_shadows25mesh_shadow_unpack_kernelEPK14twi_mesh_lighti",
               "_ZNANON_tw_shadows25mesh_shadow_zrange_kernelEP14twi_mesh_lightjPK16twi_gen_mesh_rec"}


def kernel_sass(lib):
    """{mangled kernel name with each translation unit's anonymous-namespace tag written ANON_<file>: SHA-256 of its SASS instruction words}."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, name, buf = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                res[name] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
            name, buf = re.sub(r"\d+_GLOBAL__N__[0-9a-f]{8}_\d+_(\w+?)_cu_[0-9a-f]{8}", r"ANON_\1", m.group(1)), []
        elif name:
            buf.extend(re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line))   # the instruction words only: section headers name source paths
    if name:
        res[name] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
    return res


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_existing_kernels_keep_their_sass(tw):
    """Among them shadow_rays_kernel, shadow_init_kernel, shadow_unpack_kernel, every kernel of the ground-mode mesh job and the headline's noise kernels."""
    release = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != SASS_CUDA:
        pytest.skip("the digests are those of CUDA %s" % SASS_CUDA)
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_mesh_shadows.json")) as f:
        parent = json.load(f)
    got = kernel_sass(tw.LIB_PATH)
    assert {k: got.get(k) for k in parent} == parent
    assert set(got) - set(parent) == NEW_KERNELS


def oracle_params(oracle, xs, ys, lpos, zmin, zmax, dx, dy, x_scene, y_scene):
    sp = oracle.ShadowParams()
    for d in range(3):
        sp.lpos[d] = lpos[d]
    sp.x_scene_size, sp.y_scene_size, sp.dx_val, sp.dy_val = x_scene, y_scene, dx, dy
    sp.dx_val_inv, sp.dy_val_inv = 1.0 / F(dx), 1.0 / F(dy)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = xs + ys, zmin, zmax, 0
    return sp


LIGHTS = [(3.0, 2.0, 1.0), (-4.0, 1.0, 0.5), (1.0, -5.0, 0.7), (-2.0, -2.0, 3.0), (0.3, 6.0, 0.2), (-6.0, -0.4, 0.15), (5.0, 0.0, 1.0), (0.0, -3.0, 2.0),
          (-2.0, 2.0, 1.0), (0.0, 0.0, 5.0)]


def test_oracle_mesh_equals_tile_batch_of_one(oracle):
    rng = np.random.default_rng(2)
    z = rng.normal(0.0, 0.4, (48, 48)).astype(F)
    for lp in LIGHTS + [(1.0, 1.0, -5.0)]:
        sp = oracle_params(oracle, 48, 48, lp, -2.0, 2.0, 0.0625, 0.046875, 2.0, 1.5)
        m, ox, oy = oracle.calc_mesh_shadows(sp, z)
        mt, oxt, oyt = oracle.tile_shadows_batch(z[None], [(0, 0)], sp)
        assert np.array_equal(m, mt[0]) and np.array_equal(ox.view(np.uint32), oxt[0].view(np.uint32)) and np.array_equal(oy.view(np.uint32), oyt[0].view(np.uint32))


def test_oracle_mesh_shadows_against_reference_non_square(oracle, ref):
    """The reference's own calc_mesh_shadows (cut out of src/visibility.cpp:411-517 at build time) on meshes the tile pin never builds: 64x200, 333x97,
    2x513 and 1000x37, lights in every octant, steep and grazing, on an axis, with and without incoming heights; 1 OpenMP thread."""
    if not ref.has_shadow_extract():
        pytest.skip("oracle/_ref was built without the visibility.cpp extraction")
    RL = ref.lib()
    RL.ref_set_threads(1)
    rng = np.random.default_rng(11)
    for xs, ys in ((64, 200), (333, 97), (2, 513), (1000, 37)):
        ref.setup(mesh=(xs, ys, 1), scene=(4.0, 3.0, 4.0))
        dx, dy = RL.ref_get_dx(), RL.ref_get_dy()
        z = (rng.normal(0.0, 0.3, (ys, xs)) + np.sin(np.arange(xs) * 0.05)[None, :]).astype(F)
        zlo, zhi = float(z.min()) - 0.5, float(z.max()) + 0.5
        for lp in LIGHTS + [(2.0, 1.0, zlo - 1.0)]:
            sp = oracle_params(oracle, xs, ys, lp, zlo, zhi, dx, dy, 4.0, 3.0)
            for with_in in (0, 1):
                six = siy = None
                if with_in:
                    six = np.where(rng.random(xs) < 0.3, -1.0e6, z[0] + rng.uniform(-0.2, 0.6, xs)).astype(F)
                    siy = np.where(rng.random(ys) < 0.3, -1.0e6, z[:, 0] + rng.uniform(-0.2, 0.6, ys)).astype(F)
                got = oracle.calc_mesh_shadows(sp, z, six, siy)
                want = ref.calc_mesh_shadows(lp, z, zlo, zhi, six, siy)
                assert np.array_equal(got[0], want[0]), (xs, ys, lp, with_in)
                for g, w in zip(got[1:], want[1:]):
                    assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), (xs, ys, lp, with_in)
