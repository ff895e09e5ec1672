"""CPU: tw_cancel on the host side - it is exported and listed in ABI_SYMBOLS, TW_ERR_CANCELED has the header's value in the binding, TwCanceled is a
TwError, a NULL context is refused without a device, and the C++ adapter's tiles_job::cancel() / cancelled() compile."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entry_point_is_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    assert " T tw_cancel\n" in out
    assert "tw_cancel" in tw.ABI_SYMBOLS


def test_status_code(tw):
    with open(os.path.join(ROOT, "include", "tw3d.h")) as f:
        m = re.search(r"TW_ERR_CANCELED\s*=\s*(-?\d+)", f.read())
    assert m and int(m.group(1)) == tw.TW_ERR_CANCELED == -6
    assert issubclass(tw.TwCanceled, tw.TwError)


def test_null_context_without_a_device(tw):
    assert tw.lib.tw_cancel(None) == tw.TW_ERR_ARG


def test_adapter_cancel_compiles(tw, tmp_path):
    exe = os.path.join(str(tmp_path), "test_cancel")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "3dworld_b200", "host"), "-I", "/usr/local/cuda/include",
                           os.path.join(ROOT, "tests", "cpp", "test_cancel.cpp"), "-L" + os.path.join(ROOT, "3dworld_b200"), "-l3dworld_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "3dworld_b200"), "-L/usr/local/cuda/lib64", "-lcudart", "-o", exe])
    assert os.access(exe, os.X_OK)
