"""CPU: the asynchronous heightmap job on the host side - tw_proc_gen_heightmap_launch is exported and listed in ABI_SYMBOLS, the ctypes mirror of
tw_heightmap_outputs matches the header, NULL arguments are refused without a device, and the C++ adapter's proc_gen_heightmap_async compiles."""
import ctypes as C
import os
import subprocess

from test_tile_set_host import _layout


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_proc_gen_heightmap_launch\n" in out
    assert "tw_proc_gen_heightmap_launch" in tw.ABI_SYMBOLS


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_heightmap_outputs", tw.HeightmapOutputs)
    _layout(tmp_path, "tw_heightmap_info", tw.HeightmapInfo)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    hp, ep = tw.HeightParams(), tw.ErosionParams()
    img = (C.c_uint8 * 32)()
    o = tw.HeightmapOutputs(C.cast(img, C.c_void_p), None, None, 0)
    assert L.tw_proc_gen_heightmap_launch(None, 4, 4, 1.0, 1.0, C.byref(hp), 0, C.byref(ep), C.byref(o)) == tw.TW_ERR_ARG
    assert L.tw_proc_gen_heightmap_launch(None, 4, 4, 1.0, 1.0, None, 0, None, None) == tw.TW_ERR_ARG


def test_adapter_proc_gen_heightmap_async_compiles(tw, tmp_path):
    from test_cpp_heightmap_job import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
