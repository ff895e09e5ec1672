"""CPU: the host side of the voxel batch (tw_voxel_build_batch_launch) - the entry point is exported and listed in ABI_SYMBOLS, NULL contexts and arrays are
refused without a device, and the batch's kernels are the sm_90a module tw_voxel_batch.cubin beside the library, holding exactly those kernels (the
library's own kernels keep their SASS: tests/test_voxel_changes_host.py)."""
import shutil
import subprocess
import os

import pytest

from test_mesh_shadows_host import kernel_sass

MODULE_KERNELS = {"tw_vbatch_tables_kernel", "tw_vbatch_fill_kernel", "tw_vbatch_flood_kernel", "tw_vbatch_mesh_count_kernel", "tw_vbatch_mesh_scan_kernel",
                  "tw_vbatch_mesh_emit_kernel"}


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_voxel_build_batch_launch\n" in out
    assert "tw_voxel_build_batch_launch" in tw.ABI_SYMBOLS and hasattr(tw.lib, "tw_voxel_build_batch_launch")
    assert tw.lib.tw_abi_version() == 1


def test_null_arguments_without_a_device(tw):
    b, m = (tw.VoxelBuild * 1)(), (tw.VoxelMesh * 1)()
    assert tw.lib.tw_voxel_build_batch_launch(None, b, m, 1) == tw.TW_ERR_ARG
    assert tw.lib.tw_voxel_build_batch_launch(None, None, None, 0) == tw.TW_ERR_ARG
    assert tw.lib.tw_voxel_build_batch_launch(None, None, m, 1) == tw.TW_ERR_ARG


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit not installed")
def test_module_holds_the_batch_kernels_for_sm_90a(tw):
    module = os.path.join(os.path.dirname(tw.LIB_PATH), "tw_voxel_batch.cubin")
    assert os.path.exists(module)
    assert set(kernel_sass(module)) == MODULE_KERNELS
    assert "code for sm_90a" in subprocess.run(["cuobjdump", "-sass", module], capture_output=True, text=True, check=True).stdout
    assert not MODULE_KERNELS & set(kernel_sass(tw.LIB_PATH))

