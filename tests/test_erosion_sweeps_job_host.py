"""CPU: the sweeps erosion job on the host side - tw_erode_launch_ex is exported and listed in ABI_SYMBOLS, the ABI version and tw_erosion_job's layout
are unchanged, the ctypes mirror of tw_sweep_params matches the header, the mode / tw_sweep_params checks of the Python layer and NULL arguments are
refused without a device, and the C++ adapter's sweeps jobs compile."""
import ctypes as C
import os
import subprocess

import pytest

from test_tile_set_host import _layout


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_erode_launch_ex\n" in out
    assert "tw_erode_launch_ex" in tw.ABI_SYMBOLS


def test_abi_and_job_layout_unchanged(tw, tmp_path):
    assert tw.lib.tw_abi_version() == 1
    assert C.sizeof(tw.ErosionJobArgs) == 56     # 8 + 4*2 + 4*3 + 4 + 8 + 4 + 4 + 8, as before the sweeps mode
    _layout(tmp_path, "tw_erosion_job", tw.ErosionJobArgs)
    _layout(tmp_path, "tw_sweep_params", tw.SweepParams)
    assert tw.TW_EROSION_SWEEPS == 2


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    ep = tw.ErosionParams()
    m = (C.c_float * 16)()
    j = tw.ErosionJobArgs(C.cast(m, C.c_void_p), 4, 4, 0.0, 0.0, 0.0, 10, C.cast(C.pointer(ep), C.c_void_p), tw.TW_EROSION_SWEEPS, 0, None)
    sw = tw.SweepParams(64, 44)
    assert L.tw_erode_launch_ex(None, C.byref(j), C.byref(sw)) == tw.TW_ERR_ARG
    assert L.tw_erode_launch_ex(None, None, None) == tw.TW_ERR_ARG


def test_python_needs_sweep_and_halo_together(tw):
    c = object.__new__(tw.Context)      # no device: the check comes before the library call
    with pytest.raises(ValueError):
        c.erode_launch(__import__("numpy").zeros((4, 4), "f4"), 0.0, 10, tw.ErosionParams(), sweep=64)
    with pytest.raises(ValueError):
        c.erode_image_launch(1.0, 0.0, 10, tw.ErosionParams(), halo=44)


def test_adapter_erosion_sweeps_async_compiles(tw, tmp_path):
    from test_cpp_erosion_sweeps_job import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
