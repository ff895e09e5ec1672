"""CPU: the heightmap-texture tile job on the host side - tw_set_heightmap and tw_create_tiles_launch_hmap are exported and listed in ABI_SYMBOLS, a null
context or missing argument is refused, and the C++ adapter's heightmap overload compiles against the library."""
import ctypes as C
import os
import subprocess


def test_new_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ("tw_set_heightmap", "tw_create_tiles_launch_hmap"):
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


def test_null_context_and_arguments(tw):
    L = tw.lib
    img = (C.c_uint8 * 8)()
    assert L.tw_set_heightmap(None, C.cast(img, C.c_void_p), 2, 2) == tw.TW_ERR_ARG
    assert L.tw_set_heightmap(None, None, 0, 0) == tw.TW_ERR_ARG
    hs = tw.HmapSampler(2, 2, 2, 1.0, 0.0008, 1.0, 0.0, 1.0)
    org = (C.c_int32 * 2)(0, 0)
    z = (C.c_float * 16)()
    outs = tw.TileOutputs(C.cast(z, C.c_void_p), None, None, None, None)
    assert L.tw_create_tiles_launch_hmap(None, C.byref(hs), org, 1, 16, 16, 0.1, 0.1, 4, None, 0, None, 0.0, 0.0, 16, C.byref(outs), None, None) == tw.TW_ERR_ARG
    assert L.tw_create_tiles_launch_hmap(None, None, None, 0, 16, 16, 0.1, 0.1, 4, None, 0, None, 0.0, 0.0, 16, None, None, None) == tw.TW_ERR_ARG


def test_adapter_heightmap_overload_compiles(tw, tmp_path):
    from test_cpp_tiles_hmap import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
