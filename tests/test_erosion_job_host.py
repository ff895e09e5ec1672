"""CPU: the asynchronous erosion job on the host side - tw_erode_launch is exported and listed in ABI_SYMBOLS, the ctypes mirror of tw_erosion_job matches
the header, NULL arguments are refused without a device, and the C++ adapter's apply_erosion_async / erode_heightmap_async compile."""
import ctypes as C
import os
import subprocess

from test_tile_set_host import _layout


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_erode_launch\n" in out
    assert "tw_erode_launch" in tw.ABI_SYMBOLS


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_erosion_job", tw.ErosionJobArgs)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    ep = tw.ErosionParams()
    m = (C.c_float * 16)()
    j = tw.ErosionJobArgs(C.cast(m, C.c_void_p), 4, 4, 0.0, 0.0, 0.0, 10, C.cast(C.pointer(ep), C.c_void_p), tw.TW_EROSION_SERIAL, 0, None)
    assert L.tw_erode_launch(None, C.byref(j)) == tw.TW_ERR_ARG
    assert L.tw_erode_launch(None, None) == tw.TW_ERR_ARG


def test_adapter_erosion_async_compiles(tw, tmp_path):
    from test_cpp_erosion_job import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
