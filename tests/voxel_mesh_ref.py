"""The sequential welded-mesh reference of tests/voxel_mesh_ref.c, compiled on first use into a temporary directory (the tree may be read-only) and
loaded with ctypes. voxel_mesh(vals, outside, params, tables) -> (verts [nv, 3] float32, indices [nt, 3] uint32); params: any ctypes mirror of
tw_voxel_post_params (the product's or the oracle's)."""
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
        out = os.path.join(tempfile.mkdtemp(prefix="voxel_mesh_ref_"), "libvoxel_mesh_ref.so")
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall", "-I", os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "voxel_mesh_ref.c"), "-o", out, "-lm"])
        L = C.CDLL(out)
        vp = C.c_void_p
        L.ref_voxel_mesh.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_ulonglong, vp, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
        L.ref_voxel_mesh.restype = None
        _lib = L
    return _lib


def voxel_mesh(vals, outside, params, tables):
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    vals = np.ascontiguousarray(vals, np.float32)
    outside = np.ascontiguousarray(outside, np.uint8)
    e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
    assert C.sizeof(params) == 64 and vals.size == outside.size == int(params.nx) * int(params.ny) * int(params.nz)
    nv, nt = C.c_ulonglong(), C.c_ulonglong()
    args = [p(vals), p(outside), C.cast(C.pointer(params), C.c_void_p), p(e), p(t), p(v)]
    lib().ref_voxel_mesh(*args, None, 0, None, 0, C.byref(nv), C.byref(nt))
    verts, indices = np.empty((nv.value, 3), np.float32), np.empty((nt.value, 3), np.uint32)
    lib().ref_voxel_mesh(*args, p(verts), nv.value, p(indices), nt.value, C.byref(nv), C.byref(nt))
    return verts, indices
