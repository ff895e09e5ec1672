"""CPU: the host side of a voxel model edit's change list - tw_voxel_model_edit_launch_ex is exported and listed in ABI_SYMBOLS, the ctypes mirror of
tw_voxel_changes matches the header, NULL models are refused without a device; the library's kernels are exactly those of the build before the change
list, each keeping its SASS (tests/golden/sass_before_voxel_changes.json), and the change list's kernels are the sm_90a module beside the library."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import pytest

from test_mesh_shadows_host import SASS_CUDA, kernel_sass
from test_tile_set_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_voxel_model_edit_launch_ex\n" in out
    assert "tw_voxel_model_edit_launch_ex" in tw.ABI_SYMBOLS and hasattr(tw.lib, "tw_voxel_model_edit_launch_ex")
    assert tw.lib.tw_abi_version() == 1


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_voxel_changes", tw.VoxelChanges)


def test_null_arguments_without_a_device(tw):
    n = C.c_uint64(0)
    ch = tw.VoxelChanges(None, None, None, 0, C.cast(C.pointer(n), C.c_void_p))
    out = tw.VoxelBlocksOut()
    assert tw.lib.tw_voxel_model_edit_launch_ex(None, None, 0, None, None, None) == tw.TW_ERR_ARG
    assert tw.lib.tw_voxel_model_edit_launch_ex(None, None, 0, None, C.byref(out), C.byref(ch)) == tw.TW_ERR_ARG
    assert n.value == 0


MODULE_KERNELS = {"tw_box_scatter_bits_kernel", "tw_diff_bits_kernel", "tw_change_count_kernel", "tw_change_emit_kernel"}


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_library_kernels_keep_their_sass_and_the_module_holds_the_list(tw):
    """The library's kernels are exactly the parent build's, each with its SASS - among them box_scatter_kernel and diff_kernel, which an edit without a
    change list still runs, every kernel of the mesh-shadow pass and the headline's noise kernels. The change list's kernels are in the sm_90a module
    beside the library, and only there."""
    release = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != SASS_CUDA:
        pytest.skip("the digests are those of CUDA %s" % SASS_CUDA)
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_voxel_changes.json")) as f:
        parent = json.load(f)
    assert kernel_sass(tw.LIB_PATH) == parent
    module = os.path.join(os.path.dirname(tw.LIB_PATH), "tw_voxel_changes.cubin")
    assert set(kernel_sass(module)) == MODULE_KERNELS
    assert "code for sm_90a" in subprocess.run(["cuobjdump", "-sass", module], capture_output=True, text=True, check=True).stdout
