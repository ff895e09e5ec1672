"""CPU: shared contexts on the host side - tw_create_shared is exported and listed in ABI_SYMBOLS, a NULL parent is refused without a device, and the C++
adapter's set_deferred_gens / tile_job_pool compile against the library."""
import ctypes as C
import os
import subprocess


def test_create_shared_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_create_shared\n" in out
    assert "tw_create_shared" in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


def test_null_parent_is_refused(tw):
    h = C.c_void_p(1234)
    assert tw.lib.tw_create_shared(None, C.byref(h)) == tw.TW_ERR_ARG
    assert h.value is None                                    # *out is cleared
    assert tw.lib.tw_create_shared(None, None) == tw.TW_ERR_ARG


def test_adapter_uses_the_shared_context_api(tw, tmp_path):
    from test_cpp_deferred_gens import ROOT, build_exe
    src = open(os.path.join(ROOT, "tests", "cpp", "test_deferred_gens.cpp")).read()
    assert "set_deferred_gens" in src and "tile_job_pool" in src
    hdr = open(os.path.join(ROOT, "3dworld_b200", "host", "tw3d_adapter.h")).read()
    assert "tw_create_shared" in hdr
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
