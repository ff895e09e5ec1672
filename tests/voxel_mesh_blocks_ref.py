"""The per-block welded-mesh reference of tests/voxel_mesh_blocks_ref.c, compiled on first use into a temporary directory (the tree may be read-only)
and loaded with ctypes. voxel_mesh_blocks(vals, outside, params, tables, bx, by) welds every block of bx x by cube columns on its own and returns
(verts [nv, 3] float32, indices [nt, 3] uint32 local to each block, table [nblocks, 5] uint64 = (block, voff, nverts, toff, ntris)); params: any ctypes
mirror of tw_voxel_post_params (the product's or the oracle's)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="voxel_mesh_blocks_ref_"), "libvoxel_mesh_blocks_ref.so")
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall", "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "voxel_mesh_blocks_ref.c"), "-o", out, "-lm"])
        L = C.CDLL(out)
        vp = C.c_void_p
        L.ref_voxel_mesh_blocks.argtypes = [vp] * 6 + [C.c_uint, C.c_uint, vp, C.c_ulonglong, vp, C.c_ulonglong, vp, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
        L.ref_voxel_mesh_blocks.restype = None
        _lib = L
    return _lib


def num_blocks(nx, ny, bx, by):
    """(nbx, nby): blocks of bx x by cubes over the (nx - 1) x (ny - 1) cube columns."""
    return (max(nx - 1, 0) + bx - 1) // bx, (max(ny - 1, 0) + by - 1) // by


def voxel_mesh_blocks(vals, outside, params, tables, bx, by):
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    vals = np.ascontiguousarray(vals, np.float32)
    outside = np.ascontiguousarray(outside, np.uint8)
    e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
    assert C.sizeof(params) == 64 and vals.size == outside.size == int(params.nx) * int(params.ny) * int(params.nz)
    nbx, nby = num_blocks(int(params.nx), int(params.ny), bx, by)
    table = np.zeros((nbx * nby, 5), np.uint64)
    nv, nt = C.c_ulonglong(), C.c_ulonglong()
    args = [p(vals), p(outside), C.cast(C.pointer(params), C.c_void_p), p(e), p(t), p(v), int(bx), int(by)]
    lib().ref_voxel_mesh_blocks(*args, None, 0, None, 0, None, C.byref(nv), C.byref(nt))
    verts, indices = np.empty((nv.value, 3), np.float32), np.empty((nt.value, 3), np.uint32)
    lib().ref_voxel_mesh_blocks(*args, p(verts), nv.value, p(indices), nt.value, p(table), C.byref(nv), C.byref(nt))
    return verts, indices, table
