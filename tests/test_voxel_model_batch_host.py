"""CPU: the host side of the voxel model batch (tw_voxel_model_build_batch_launch / tw_voxel_model_edit_batch_launch) - both entry points are exported and
listed in ABI_SYMBOLS, the ctypes mirrors match the header, NULL contexts and arrays are refused without a device, and the batch's own kernels are the
sm_90a module tw_voxel_model_batch.cubin beside the library, holding exactly those kernels, none of them in the library, and none spilling."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from test_mesh_shadows_host import kernel_sass
from test_tile_set_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("tw_voxel_model_build_batch_launch", "tw_voxel_model_edit_batch_launch")
MODULE_KERNELS = {"tw_vmb_copy_kernel", "tw_vmb_box_scatter_kernel", "tw_vmb_diff_kernel", "tw_vmb_change_list_kernel", "tw_vmb_list_marked_kernel",
                  "tw_vmb_mesh_count_kernel", "tw_vmb_mesh_scan_kernel", "tw_vmb_mesh_emit_kernel"}


def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ENTRY_POINTS:
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    assert tw.lib.tw_abi_version() == 1


def test_mirrors_match_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_voxel_model_build", tw.VoxelModelBuild)
    _layout(tmp_path, "tw_voxel_model_edit", tw.VoxelModelEdit)


def test_null_arguments_without_a_device(tw):
    b, e = (tw.VoxelModelBuild * 1)(), (tw.VoxelModelEdit * 1)()
    for fn, arr in ((tw.lib.tw_voxel_model_build_batch_launch, b), (tw.lib.tw_voxel_model_edit_batch_launch, e)):
        assert fn(None, arr, 1) == tw.TW_ERR_ARG
        assert fn(None, None, 0) == tw.TW_ERR_ARG
        assert fn(None, None, 1) == tw.TW_ERR_ARG


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit not installed")
def test_module_holds_the_model_batch_kernels_for_sm_90a(tw):
    module = os.path.join(os.path.dirname(tw.LIB_PATH), "tw_voxel_model_batch.cubin")
    assert os.path.exists(module)
    assert set(kernel_sass(module)) == MODULE_KERNELS
    assert "code for sm_90a" in subprocess.run(["cuobjdump", "-sass", module], capture_output=True, text=True, check=True).stdout
    assert not MODULE_KERNELS & set(kernel_sass(tw.LIB_PATH))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_module_kernels_do_not_spill(tw, tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("tw_build", os.path.join(ROOT, "3dworld_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    flags = [f for f in b.NVCC_FLAGS if f != "--use_fast_math=false"]
    out = subprocess.run([b.nvcc()] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(b.CSRC, "tw_voxel_model_batch.cu"), "-o", str(tmp_path / "m.cubin")],
                         capture_output=True, text=True, check=True).stderr
    spills = dict(re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+ bytes spill stores, \d+ bytes spill loads)", out))
    assert set(spills) == MODULE_KERNELS
    assert all(v == "0 bytes spill stores, 0 bytes spill loads" for v in spills.values()), spills
