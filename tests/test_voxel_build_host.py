"""CPU: the asynchronous voxel build on the host side - tw_voxel_build_launch is exported and listed in ABI_SYMBOLS, the ctypes mirror of tw_voxel_build
matches the header, a NULL context or struct is refused without a device, and the C++ adapter's voxel_build_async compiles."""
import ctypes as C
import os
import subprocess

from test_tile_set_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_voxel_build_launch\n" in out
    assert "tw_voxel_build_launch" in tw.ABI_SYMBOLS


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_voxel_build", tw.VoxelBuild)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    p = tw.VoxelPostParams()
    p.nx = p.ny = p.nz = 4
    vals = (C.c_float * 64)()
    b = tw.VoxelBuild(None, None, C.cast(C.pointer(p), C.c_void_p), None, None, None, None, C.cast(vals, C.c_void_p), None, None, 0, None, None)
    assert L.tw_voxel_build_launch(None, C.byref(b)) == tw.TW_ERR_ARG
    assert L.tw_voxel_build_launch(None, None) == tw.TW_ERR_ARG


def test_adapter_voxel_build_async_compiles(tw, tmp_path):
    from test_cpp_voxel_build import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
