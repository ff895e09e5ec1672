"""CPU: the asynchronous tile entry points on the host side - exported, their argument checks return TW_ERR_ARG instead of crashing, the ctypes
mirror of tw_tile_outputs matches the header, and the C++ adapter's create_tiles_async compiles against the library."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_async_tile_symbols_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for sym in ("tw_create_tiles_launch", "tw_create_tiles_poll"):
        assert " T %s\n" % sym in out, sym
        assert sym in tw.ABI_SYMBOLS


def test_null_and_empty_arguments(tw):
    L = tw.lib
    hp, ep = tw.HeightParams(), tw.ErosionParams()
    org = (C.c_int32 * 2)(0, 0)
    z = (C.c_float * 64)()
    outs = tw.TileOutputs(C.cast(z, C.c_void_p), None, None, None, None)
    assert L.tw_create_tiles_launch(None, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs)) == tw.TW_ERR_ARG
    assert L.tw_create_tiles_poll(None, 0) == tw.TW_ERR_ARG
    assert L.tw_create_tiles_poll(None, 1) == tw.TW_ERR_ARG
    import torch
    if not torch.cuda.is_available():
        return
    ctx = tw.Context(0)
    try:
        h = ctx._h
        assert L.tw_create_tiles_launch(h, None, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs)) == tw.TW_ERR_ARG
        assert L.tw_create_tiles_launch(h, org, 0, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs)) == tw.TW_ERR_ARG
        assert L.tw_create_tiles_launch(h, org, 1, 16, 16, 0.1, 0.1, 8, None, 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs)) == tw.TW_ERR_ARG
        assert L.tw_create_tiles_launch(h, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, None) == tw.TW_ERR_ARG
        no_z = tw.TileOutputs(None, None, None, None, None)
        assert L.tw_create_tiles_launch(h, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(no_z)) == tw.TW_ERR_ARG
        mnz = (C.c_float * 1)()
        mnz_only = tw.TileOutputs(C.cast(z, C.c_void_p), None, None, None, C.cast(mnz, C.c_void_p))   # min_normal_z comes with the normal map
        assert L.tw_create_tiles_launch(h, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(mnz_only)) == tw.TW_ERR_ARG
        bnd = (tw.TileBounds * 1)()
        bad_size = tw.TileOutputs(C.cast(z, C.c_void_p), None, C.cast(bnd, C.c_void_p), None, None)   # zvsize 8: the last sub-block would end at cell 8
        assert L.tw_create_tiles_launch(h, org, 1, 16, 16, 0.1, 0.1, 8, C.byref(hp), 0, C.byref(ep), 0.0, 0.0, 16, C.byref(bad_size)) == tw.TW_ERR_ARG
        assert L.tw_create_tiles_poll(h, 0) == tw.TW_OK     # nothing pending
    finally:
        ctx.close()


def test_tile_outputs_mirror_matches_the_header(tw, tmp_path):
    src = tmp_path / "layout.c"
    fields = [f for f, _ in tw.TileOutputs._fields_]
    src.write_text("#include <tw3d.h>\n#include <stdio.h>\n#include <stddef.h>\nint main(void) {printf(\"%zu\", sizeof(tw_tile_outputs));" +
                   "".join('printf(" %%zu", offsetof(tw_tile_outputs, %s));' % f for f in fields) + "return 0;}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    nums = [int(v) for v in subprocess.check_output([exe], text=True).split()]
    assert nums[0] == C.sizeof(tw.TileOutputs)
    assert nums[1:] == [getattr(tw.TileOutputs, f).offset for f in fields]


def test_adapter_async_tiles_compiles(tw, tmp_path):
    from test_cpp_tiles_async import build_exe
    exe = build_exe(tw, tmp_path)
    out = subprocess.run([exe, "probe"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
