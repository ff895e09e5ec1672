"""CPU: the host side of the heightmap-tile AO job (tw_hmap_tile_ao_launch / tw_hmap_tile_ao) - both entry points are exported and listed in ABI_SYMBOLS,
the ctypes mirror of tw_hmap_ao_job matches the header, NULL contexts and jobs are refused without a device, and the job's kernel is the sm_90a module
tw_hmap_ao.cubin beside the library, not spilling and not in the library, whose kernels keep the golden digests of tests/golden."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import pytest

from test_mesh_shadows_host import NEW_KERNELS, SASS_CUDA, kernel_sass
from test_tile_set_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("tw_hmap_tile_ao_launch", "tw_hmap_tile_ao")
MODULE_KERNELS = {"tw_hmap_ao_kernel"}


def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ENTRY_POINTS:
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    assert tw.lib.tw_abi_version() == 1


def test_job_layout(tw, tmp_path):
    _layout(tmp_path, "tw_hmap_ao_job", tw.HmapAoJobArgs)


def test_null_context_and_job_are_refused(tw):
    hs = tw.HmapSampler(8, 8, 0, 1.0, 1.0, 1.0, 0.0, 1.0)
    j = tw.HmapAoJobArgs(C.cast(C.pointer(hs), C.c_void_p), None, 0, 5, 0.03125, None, None, None, None)
    for fn in (tw.lib.tw_hmap_tile_ao_launch, tw.lib.tw_hmap_tile_ao):
        assert fn(None, C.byref(j)) == tw.TW_ERR_ARG
        assert fn(None, None) == tw.TW_ERR_ARG


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit not installed")
def test_module_holds_the_ao_kernel_for_sm_90a(tw):
    module = os.path.join(os.path.dirname(tw.LIB_PATH), "tw_hmap_ao.cubin")
    assert os.path.exists(module)
    assert set(kernel_sass(module)) == MODULE_KERNELS
    assert "code for sm_90a" in subprocess.run(["cuobjdump", "-sass", module], capture_output=True, text=True, check=True).stdout


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_library_kernels_are_unchanged(tw):
    release = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != SASS_CUDA:
        pytest.skip("the digests are those of CUDA %s" % SASS_CUDA)
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_mesh_shadows.json")) as f:
        parent = json.load(f)
    got = kernel_sass(tw.LIB_PATH)
    assert {k: got.get(k) for k in parent} == parent and set(got) == set(parent) | NEW_KERNELS


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_module_kernel_does_not_spill(tw, tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("tw_build", os.path.join(ROOT, "3dworld_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    flags = [f for f in b.NVCC_FLAGS if f != "--use_fast_math=false"]
    out = subprocess.run([b.nvcc()] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(b.CSRC, "tw_hmap_ao.cu"), "-o", str(tmp_path / "m.cubin")],
                         capture_output=True, text=True, check=True).stderr
    spills = dict(re.findall(r"Function properties for (\w+)\n\s*\d+ bytes stack frame, (\d+ bytes spill stores, \d+ bytes spill loads)", out))
    assert set(spills) == MODULE_KERNELS
    assert all(v == "0 bytes spill stores, 0 bytes spill loads" for v in spills.values()), spills
