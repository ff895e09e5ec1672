"""CPU: tw_create_tiles_launch_ex on the host side - exported, its argument checks return TW_ERR_ARG / TW_ERR_STATE instead of crashing, the ctypes
mirror of tw_tile_shading matches the header, and the C++ adapter's shading overload of create_tiles_async compiles against the library."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_launch_ex_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_create_tiles_launch_ex\n" in out
    assert "tw_create_tiles_launch_ex" in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


def _weight_params(tw):
    wp = tw.WeightParams()
    for i in range(5):
        wp.h_dirt[i], wp.tex_class[i] = 0.2 * (i + 1), i
    wp.zmin, wp.zmax = -1.0, 1.0
    return wp


def test_argument_errors(tw):
    L = tw.lib
    hp, ep = tw.HeightParams(), tw.ErosionParams()
    hp.gen_mode = 1
    org = (C.c_int32 * 2)(0, 0)
    z = (C.c_float * 64)()
    ao, w, f = (C.c_uint8 * 49)(), (C.c_uint8 * 196)(), (C.c_uint8 * 1)()
    tp = (C.c_float * 8)()
    outs = tw.TileOutputs(C.cast(z, C.c_void_p), None, None, None, None)
    wp = _weight_params(tw)

    def shading(**kw):
        s = tw.TileShading(0.1, None, None, None, None, None)
        for k, v in kw.items():
            setattr(s, k, C.cast(v, C.c_void_p) if v is not None else None)
        return s

    def launch(h, s):
        return L.tw_create_tiles_launch_ex(h, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs), C.byref(s))
    assert launch(None, shading(ao=ao)) == tw.TW_ERR_ARG
    import torch
    if not torch.cuda.is_available():
        return
    ctx = tw.Context(0)
    try:
        h = ctx._h
        assert launch(h, shading(weights=w, tile_params=tp)) == tw.TW_ERR_ARG                       # no wp
        assert launch(h, shading(weights=w, wp=C.pointer(wp))) == tw.TW_ERR_ARG                     # no tile_params
        assert launch(h, shading(ao=ao, has_any_grass=f)) == tw.TW_ERR_ARG                          # has_any_grass without weights
        bad = _weight_params(tw)
        bad.tex_class[4] = 0                                                                        # class 0 twice
        assert launch(h, shading(weights=w, wp=C.pointer(bad), tile_params=tp)) == tw.TW_ERR_ARG
        bad = _weight_params(tw)
        bad.zmax = bad.zmin
        assert launch(h, shading(weights=w, wp=C.pointer(bad), tile_params=tp)) == tw.TW_ERR_ARG
        assert launch(h, shading(weights=w, wp=C.pointer(wp), tile_params=tp)) == tw.TW_ERR_STATE     # tw_set_sine_params has not been called
        assert L.tw_create_tiles_poll(h, 0) == tw.TW_OK                                            # nothing pending
    finally:
        ctx.close()


def test_tile_shading_mirror_matches_the_header(tw, tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in tw.TileShading._fields_]
    src.write_text("#include <tw3d.h>\n#include <stdio.h>\n#include <stddef.h>\nint main(void) {printf(\"%zu\", sizeof(tw_tile_shading));" +
                   "".join('printf(" %%zu", offsetof(tw_tile_shading, %s));' % f for f in fields) + "return 0;}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    nums = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    assert nums[0] == C.sizeof(tw.TileShading)
    assert nums[1:] == [getattr(tw.TileShading, f).offset for f in fields]


def test_adapter_shading_overload_compiles(tw, tmp_path):
    from test_cpp_tiles_shading import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
