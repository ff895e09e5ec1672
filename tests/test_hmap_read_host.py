"""CPU: the heightmap read on the host side - tw_read_heightmap_launch and tw_read_heightmap are exported and listed in ABI_SYMBOLS, the ctypes mirror of
tw_hmap_read matches the header, NULL contexts are refused. The read adds no kernel (it runs tw_update_heightmap's hmap_scatter_kernel the other way):
tests/test_mesh_shadows_host.py holds the library's kernels and their SASS."""
import ctypes as C
import os
import subprocess


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("tw_read_heightmap_launch", "tw_read_heightmap")


def test_entry_points_are_exported(tw):
    for name in ENTRY_POINTS:
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    assert tw.lib.tw_abi_version() == 1


def test_read_layout(tw, tmp_path):
    fields = [f for f, _ in tw.HmapReadArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tw3d.h"\nint main(void) {printf("%zu", sizeof(tw_hmap_read)); '
                   + "".join('printf(" %%zu", offsetof(tw_hmap_read, %s)); ' % f for f in fields) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(tw.HmapReadArgs)] + [getattr(tw.HmapReadArgs, f).offset for f in fields]


def test_null_context_is_refused(tw):
    arr, n = tw._rects([(0, 0, 1, 1)])
    buf = (C.c_uint8 * 2)()
    r = tw.HmapReadArgs(C.cast(arr, C.c_void_p), n, C.cast(buf, C.c_void_p), 2)
    for fn in (tw.lib.tw_read_heightmap_launch, tw.lib.tw_read_heightmap):
        assert fn(None, C.byref(r)) == tw.TW_ERR_ARG
        assert fn(None, None) == tw.TW_ERR_ARG
