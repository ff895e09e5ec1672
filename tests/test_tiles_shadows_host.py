"""CPU: the mesh shadows of the tile job and tw_tile_shadows_batch_ex on the host side - exported, listed in ABI_SYMBOLS, the ctypes mirrors of
tw_tile_light / tw_tile_shadows match the header, every argument error returns TW_ERR_ARG before anything is enqueued, and the C++ adapter's shadows overload
compiles against the library."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ("tw_tile_shadows_batch_ex", "tw_create_tiles_launch_shadows"):
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


def _layout(tw, tmp_path, ctype, cls):
    src = tmp_path / ("%s.c" % ctype)
    fields = [f for f, _ in cls._fields_]
    src.write_text("#include <tw3d.h>\n#include <stdio.h>\n#include <stddef.h>\nint main(void) {printf(\"%%zu\", sizeof(%s));" % ctype +
                   "".join('printf(" %%zu", offsetof(%s, %s));' % (ctype, f) for f in fields) + "return 0;}\n")
    exe = str(tmp_path / ctype)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    nums = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    assert nums[0] == C.sizeof(cls)
    assert nums[1:] == [getattr(cls, f).offset for f in fields]


def test_mirrors_match_the_header(tw, tmp_path):
    _layout(tw, tmp_path, "tw_tile_light", tw.TileLight)
    _layout(tw, tmp_path, "tw_tile_shadows", tw.TileShadows)
    _layout(tw, tmp_path, "tw_shadow_params", tw.ShadowParams)


def test_argument_errors(tw):
    import numpy as np
    L = tw.lib
    hp, ep = tw.HeightParams(), tw.ErosionParams()
    hp.gen_mode = 1
    nt, zv = 2, 8
    org = (C.c_int32 * 4)(0, 0, 8, 0)
    z = (C.c_float * (nt * zv * zv))()
    outs = tw.TileOutputs(C.cast(z, C.c_void_p), None, None, None, None)
    txy = np.array([[0, 0], [1, 0]], np.int32)
    dup = np.array([[0, 0], [0, 0]], np.int32)
    m = np.empty((nt, zv, zv), np.uint8)

    def light(smask=m):
        li = tw.TileLight()
        li.sp.lpos[0], li.sp.lpos[1], li.sp.lpos[2] = 1.0, 1.0, 1.0
        li.smask = tw._ptr(smask) if smask is not None else None
        return li

    def launch(h, shadows, zvsize=zv):
        return L.tw_create_tiles_launch_shadows(h, org, nt, 16, 16, 0.1, 0.1, zvsize, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs), None,
                                                C.byref(shadows) if shadows is not None else None)
    one = (tw.TileLight * 1)(light())
    assert launch(None, tw.TileShadows(tw._ptr(txy), 1, C.cast(one, C.c_void_p))) == tw.TW_ERR_ARG
    import torch
    if not torch.cuda.is_available():
        return
    ctx = tw.Context(0)
    try:
        h = ctx._h

        def refused(shadows, what, zvsize=zv):
            assert launch(h, shadows, zvsize) == tw.TW_ERR_ARG, what
            assert L.tw_create_tiles_poll(h, 0) == tw.TW_OK, what                                   # nothing was enqueued
            assert L.tw_last_error(h), what
        refused(tw.TileShadows(None, 1, C.cast(one, C.c_void_p)), "no tile_xy")
        refused(tw.TileShadows(tw._ptr(txy), 0, C.cast(one, C.c_void_p)), "no lights")
        refused(tw.TileShadows(tw._ptr(txy), 1, None), "lights NULL")
        no_mask = (tw.TileLight * 2)(light(), light(None))
        refused(tw.TileShadows(tw._ptr(txy), 2, C.cast(no_mask, C.c_void_p)), "a light without smask")
        dm = torch.empty(nt * zv * zv + 4, dtype=torch.uint8, device="cuda")
        odd = (tw.TileLight * 1)(light())
        odd[0].smask = dm.data_ptr() + 1
        refused(tw.TileShadows(tw._ptr(txy), 1, C.cast(odd, C.c_void_p)), "misaligned device smask")
        refused(tw.TileShadows(tw._ptr(dup), 1, C.cast(one, C.c_void_p)), "duplicate tile_xy")
        assert b"twice" in L.tw_last_error(h)
        refused(tw.TileShadows(tw._ptr(txy), 1, C.cast(one, C.c_void_p)), "zvsize < 2", zvsize=1)
        sp = tw.ShadowParams()
        assert L.tw_tile_shadows_batch_ex(h, C.cast(z, C.c_void_p), tw._ptr(dup), nt, zv, C.byref(sp), None, None, tw._ptr(m), None, None) == tw.TW_ERR_ARG
    finally:
        ctx.close()


def test_adapter_shadows_overload_compiles(tw, tmp_path):
    from test_cpp_tiles_shadows import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
