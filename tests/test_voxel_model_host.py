"""CPU: the per-block welded meshes of a voxel model in the sequential reference (tests/voxel_mesh_blocks_ref.c welds every block with a cache of its own), the
blocks an edit marks, and the host side of the voxel model's bindings.

- One block covering the grid is the whole-grid mesh, bit for bit.
- Each block's mesh is the whole-grid mesh of the block cut out of the grid (its cubes and the voxels they read): the same indices and vertex count,
  positions within float rounding (the cut-out grid's coordinates start at another origin).
- marked_blocks (the set an edit job re-meshes) holds every block whose mesh changes between two fields."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from test_tile_set_host import _layout
from test_voxel_mesh_host import CASES, make_case
from voxel_mesh_blocks_ref import num_blocks, voxel_mesh_blocks as welded_blocks
from voxel_mesh_ref import voxel_mesh as welded


@pytest.fixture(scope="module")
def tables():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def marked_blocks(old_vals, old_out, new_vals, new_out, nx, ny, bx, by):
    """The blocks whose cubes read a voxel whose value (bitwise) or flags differ: cubes x-1 and x, y-1 and y of the voxel's column."""
    old_vals, new_vals = np.ascontiguousarray(old_vals, np.float32), np.ascontiguousarray(new_vals, np.float32)
    diff = (old_vals.view(np.uint32) != new_vals.view(np.uint32)) | (np.asarray(old_out) != np.asarray(new_out))
    col = diff.reshape(ny, nx, -1).any(2)
    nbx, _ = num_blocks(nx, ny, bx, by)
    out = set()
    for y, x in zip(*np.nonzero(col)):
        for cy in (y - 1, y):
            for cx in (x - 1, x):
                if 0 <= cy < ny - 1 and 0 <= cx < nx - 1:
                    out.add(int((cy // by) * nbx + cx // bx))
    return out


def split_blocks(verts, indices, table):
    """{block: (verts, indices)} of a per-block mesh and its table rows (block, voff, nverts, toff, ntris)."""
    return {int(b): (verts[int(vo):int(vo) + int(nv)], indices[int(to):int(to) + int(nt)]) for b, vo, nv, to, nt in np.asarray(table, np.uint64)}


@pytest.mark.parametrize("case", CASES)
def test_one_block_is_the_whole_mesh(oracle, tables, case):
    vals, outside, p = make_case(oracle, oracle.VoxelPostParams, case)
    ev, ei = welded(vals, outside, p, tables)
    for bx, by in ((int(p.nx) - 1, int(p.ny) - 1), (10 ** 6, 10 ** 6)):
        gv, gi, t = welded_blocks(vals, outside, p, tables, bx, by)
        assert np.array_equal(gv.view(np.uint32), ev.view(np.uint32)) and np.array_equal(gi, ei)
        assert t.tolist() == [[0, 0, len(ev), 0, len(ei)]]


def _cut(vals, outside, p, cls, x0, x1, y0, y1):
    """The block's voxels [x0, x1] x [y0, y1] as a grid of their own, with the origin moved to voxel (x0, y0)."""
    q = cls()
    q.nx, q.ny, q.nz = x1 - x0 + 1, y1 - y0 + 1, p.nz
    for d in range(3):
        q.lo_pos[d], q.vsz[d] = p.lo_pos[d], p.vsz[d]
    q.lo_pos[0] = float(np.float32(x0) * np.float32(p.vsz[0]) + np.float32(p.lo_pos[0]))
    q.lo_pos[1] = float(np.float32(y0) * np.float32(p.vsz[1]) + np.float32(p.lo_pos[1]))
    q.isolevel, q.invert, q.make_closed_surface, q.skip_under_mesh = p.isolevel, p.invert, p.make_closed_surface, p.skip_under_mesh
    sl = (slice(y0, y1 + 1), slice(x0, x1 + 1), slice(None))
    ny, nx, nz = int(p.ny), int(p.nx), int(p.nz)
    return np.ascontiguousarray(vals.reshape(ny, nx, nz)[sl]), np.ascontiguousarray(outside.reshape(ny, nx, nz)[sl]), q


@pytest.mark.parametrize("case,bs", [(("golden", "mesh"), (7, 5)), (("random", 0), (8, 8)), (("random", 3), (1, 1)), (("random", 2), (5, 64)),
                                     (("golden", "sine"), (16, 3)), (("open", 0), (3, 100))])
def test_blocks_are_cut_out_grids(oracle, tables, case, bs):
    vals, outside, p = make_case(oracle, oracle.VoxelPostParams, case)
    bx, by = bs
    nx, ny = int(p.nx), int(p.ny)
    gv, gi, table = welded_blocks(vals, outside, p, tables, bx, by)
    nbx, nby = num_blocks(nx, ny, bx, by)
    assert len(table) == nbx * nby and table[:, 0].tolist() == list(range(nbx * nby))
    assert int(table[-1, 1] + table[-1, 2]) == len(gv) and int(table[-1, 3] + table[-1, 4]) == len(gi)
    assert (table[1:, 1] == table[:-1, 1] + table[:-1, 2]).all() and (table[1:, 3] == table[:-1, 3] + table[:-1, 4]).all()
    blocks = split_blocks(gv, gi, table)
    for b, (bv, bi) in blocks.items():
        x0, y0 = (b % nbx) * bx, (b // nbx) * by
        x1, y1 = min(x0 + bx, nx - 1), min(y0 + by, ny - 1)
        cv, co, q = _cut(vals, outside, p, oracle.VoxelPostParams, x0, x1, y0, y1)
        ev, ei = welded(cv, co, q, tables)
        assert len(bv) == len(ev) and np.array_equal(bi, ei), b
        assert np.allclose(bv, ev, rtol=0, atol=1e-4), b
    # a block face's vertices appear in both blocks: more vertices than the whole-grid mesh unless every face is empty
    assert len(gv) >= len(welded(vals, outside, p, tables)[0])


def test_marked_blocks_hold_every_changed_mesh(oracle, tables):
    """Random box edits of small fields through the oracle's flags and remove_unconnected: every block whose reference mesh changes is marked."""
    from test_voxel_flood_reference import post_params, random_field
    rng = np.random.default_rng(3)
    for dims, kw, (bx, by) in (((23, 19, 13), dict(remove_unconnected=1), (4, 5)), ((18, 20, 11), dict(remove_unconnected=0, make_closed_surface=0), (3, 3)),
                               ((21, 17, 15), dict(remove_unconnected=3, invert=1, isolevel=0.2), (6, 2))):
        raw, _ = random_field(dims, 5, 1)
        p = post_params(oracle.VoxelPostParams, dims, **kw)
        v0, o0, _ = oracle.voxel_remove_unconnected(raw, oracle.voxel_outside(raw, p), p)
        m0 = split_blocks(*welded_blocks(v0, o0, p, tables, bx, by))
        for _ in range(8):
            x, y, z = (int(rng.integers(0, n)) for n in dims)
            w, h, d = (int(rng.integers(1, n - c + 1)) for n, c in zip(dims, (x, y, z)))
            raw = raw.copy()
            raw[y:y + h, x:x + w, z:z + d] = rng.choice(np.array([-2.0, 2.0], np.float32))
            v1, o1, _ = oracle.voxel_remove_unconnected(raw, oracle.voxel_outside(raw, p), p)
            m1 = split_blocks(*welded_blocks(v1, o1, p, tables, bx, by))
            changed = {b for b in m0 if not (np.array_equal(m0[b][0].view(np.uint32), m1[b][0].view(np.uint32)) and np.array_equal(m0[b][1], m1[b][1]))}
            assert changed <= marked_blocks(v0, o0, v1, o1, dims[0], dims[1], bx, by)
            v0, o0, m0 = v1, o1, m1


# ---- bindings ----
def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ("tw_voxel_model_create", "tw_voxel_model_destroy", "tw_voxel_model_build_launch", "tw_voxel_model_edit_launch", "tw_voxel_model_read"):
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS
    assert tw.lib.tw_abi_version() == 1


@pytest.mark.parametrize("c_name,py_name", [("tw_voxel_block_mesh", "VoxelBlockMesh"), ("tw_voxel_blocks_out", "VoxelBlocksOut"), ("tw_voxel_box", "VoxelBox")])
def test_mirrors_match_the_header(tw, tmp_path, c_name, py_name):
    _layout(tmp_path, c_name, getattr(tw, py_name))


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    p = tw.VoxelPostParams()
    p.nx = p.ny = p.nz = 4
    e, t, v = (C.c_uint32 * 256)(), (C.c_int32 * 4096)(), (C.c_uint32 * 24)()
    h = C.c_void_p()
    assert L.tw_voxel_model_create(None, C.byref(p), C.cast(e, C.c_void_p), C.cast(t, C.c_void_p), C.cast(v, C.c_void_p), None, 8, 8, C.byref(h)) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_build_launch(None, None, None, None, None) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_edit_launch(None, None, 0, None, None) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_read(None, None, None, None) == tw.TW_ERR_ARG
    L.tw_voxel_model_destroy(None)
