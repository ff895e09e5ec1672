"""CPU: the host side of voxel model jobs on any context of the model's family - tw_voxel_model_build_launch_on, tw_voxel_model_edit_launch_on and
tw_voxel_model_read_launch are exported and listed in ABI_SYMBOLS with the ABI version unchanged, and a NULL context or model is refused with
TW_ERR_ARG without a device."""
import ctypes as C
import subprocess

NEW = ("tw_voxel_model_build_launch_on", "tw_voxel_model_edit_launch_on", "tw_voxel_model_read_launch")


def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in NEW:
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    assert tw.lib.tw_abi_version() == 1


def test_null_context_or_model_without_a_device(tw):
    L = tw.lib
    n = C.c_uint64(0)
    ch = tw.VoxelChanges(None, None, None, 0, C.cast(C.pointer(n), C.c_void_p))
    out = tw.VoxelBlocksOut()
    box = (tw.VoxelBox * 1)(tw.VoxelBox(0, 0, 0, 1, 1, 1))
    vals = (C.c_float * 1)()
    fake = C.c_void_p(0x1000)           # never dereferenced: the NULL partner is refused first
    for ctx, m in ((None, None), (None, fake), (fake, None)):
        assert L.tw_voxel_model_build_launch_on(ctx, m, None, None, None, C.byref(out)) == tw.TW_ERR_ARG
        assert L.tw_voxel_model_edit_launch_on(ctx, m, C.cast(box, C.c_void_p), 1, C.cast(vals, C.c_void_p), C.byref(out), C.byref(ch)) == tw.TW_ERR_ARG
        assert L.tw_voxel_model_read_launch(ctx, m, None, 0, C.cast(vals, C.c_void_p), None, None) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_build_launch(None, None, None, None, C.byref(out)) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_read(None, None, None, None) == tw.TW_ERR_ARG
    assert n.value == 0
