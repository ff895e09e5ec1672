"""CPU: the welded marching-cubes mesh (create_block's shared vertex cache) in the sequential reference of tests/voxel_mesh_ref.c, and the host side of its
bindings.

voxel_mesh_ref fills an explicit per-edge cache cube by cube, as the reference does. It is held to the reference's welded triangles where oracle/_ref is
built, and everywhere to the plain-C oracle's unwelded soup: one vertex per crossing edge of a non-skipped cube, each on a distinct grid edge, indices
below the vertex count, and - where no triangle is degenerate - the soup's triangles within two ulps of the edge's endpoint coordinate (the two ends' interpolations
round independently; the largest difference on these fields is 1.5 ulps of |coordinate| + vsz). Two constructed fields pin what the
welding changes: a shared edge that its owner and a later cube interpolate to different floats, and make_closed_surface fields where welded and unwelded
degeneracy differ."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_tile_set_host import _layout
from test_voxel_flood_reference import RANDOM_FIELDS, post_params, random_field
from voxel_mesh_ref import voxel_mesh as welded

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
UNDER_MESH = 0x08
TOLERANCE = np.float32(1.0e-12)


@pytest.fixture(scope="module")
def tables():
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def golden_case(cls, name):
    """(vals2, outside2, params of class cls) of a golden case: the field and flags after remove_unconnected."""
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    a = g[name + "_params"]
    p = cls()
    p.nx, p.ny, p.nz = int(a[0]), int(a[1]), int(a[2])
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = float(a[3 + d]), float(a[6 + d])
    p.isolevel, p.invert, p.make_closed_surface, p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = (
        float(a[9]), int(a[10]), int(a[11]), int(a[12]), int(a[13]), int(a[14]), int(a[15]))
    return g[name + "_vals2"], g[name + "_outside2"], p


def random_case(oracle, cls, dims, seed, kw):
    """A smoothed random field of RANDOM_FIELDS through the oracle's outside flags and remove_unconnected: (vals, outside, params of class cls)."""
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    po = post_params(oracle.VoxelPostParams, dims, **kw)
    v2, o2, _ = oracle.voxel_remove_unconnected(vals, oracle.voxel_outside(vals, po, zix), po)
    return v2, o2, post_params(cls, dims, **kw)


def crossing_edges(outside, p):
    """Number of grid edges whose corner flags differ (outside or on edge vs inside) and that some non-skipped cube contains."""
    ny, nx, nz = int(p.ny), int(p.nx), int(p.nz)
    o = np.asarray(outside).reshape(ny, nx, nz)
    f = (o & 7) != 0
    vc = np.ones((max(ny - 1, 0), max(nx - 1, 0), max(nz - 1, 0)), bool)
    if p.skip_under_mesh:
        um = (o & UNDER_MESH) != 0
        vc &= ~(um[:-1, :-1, :-1] & um[:-1, 1:, :-1] & um[1:, :-1, :-1] & um[1:, 1:, :-1])
    vp = np.zeros((ny + 1, nx + 1, nz + 1), bool)
    vp[1:ny, 1:nx, 1:nz] = vc
    n = 0
    for ax in range(3):      # axis 0 = y, 1 = x, 2 = z of the [ny, nx, nz] arrays
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        cross = f[tuple(lo)] != f[tuple(hi)]
        has = np.zeros(cross.shape, bool)
        dims = (ny, nx, nz)
        for d1 in (0, 1):
            for d2 in (0, 1):
                sl, k = [], 0
                for a in range(3):
                    if a == ax:
                        sl.append(slice(1, dims[a]))
                    else:
                        d = (d1, d2)[k]
                        k += 1
                        sl.append(slice(1 - d, 1 - d + dims[a]))
                has |= vp[tuple(sl)]
        n += int((cross & has).sum())
    return n


def grid_coords(p):
    """The float32 coordinate of every grid line per axis (x, y, z), as the device and the reference compute them: float(i)*vsz + lo."""
    return [np.arange(n, dtype=np.float32) * np.float32(p.vsz[d]) + np.float32(p.lo_pos[d]) for d, n in enumerate((p.nx, p.ny, p.nz))]


def check_mesh(verts, indices, soup, outside, p):
    """The structural checks of the welded mesh against the flags and the unwelded soup of the same grid."""
    verts, indices, soup = np.asarray(verts, np.float32), np.asarray(indices, np.uint32), np.asarray(soup, np.float32)
    assert len(verts) == crossing_edges(outside, p)
    assert indices.size == 0 or int(indices.max()) < len(verts)
    g = grid_coords(p)
    on = np.stack([np.isin(verts[:, d], g[d]) for d in range(3)], 1)
    assert (on.sum(1) >= 2).all()                  # two coordinates on grid lines: on an edge, or on a grid point when interpolate_pt snaps
    inner = on.sum(1) == 2
    axis = np.argmin(on[inner], 1)
    keys = []
    for d in range(3):
        keys.append(np.where(axis == d, np.searchsorted(g[d], verts[inner, d]), np.searchsorted(g[d], verts[inner, d])))
    key = np.stack([axis] + keys, 1)
    assert len(np.unique(key, axis=0)) == len(key)  # distinct grid edges
    flat = verts[indices.astype(np.int64)] if len(indices) else np.empty((0, 3, 3), np.float32)
    return flat


def within_two_ulps(flat, soup, p):
    """|welded - soup| <= 2 ulps of |coordinate| + vsz, which bounds the edge's larger endpoint coordinate."""
    vsz = np.abs(np.array([p.vsz[0], p.vsz[1], p.vsz[2]], np.float32))
    a, b = flat.astype(np.float64), soup.astype(np.float64)
    bound = 2 * np.spacing((np.maximum(np.abs(flat), np.abs(soup)) + vsz).astype(np.float32)).astype(np.float64)
    return bool((np.abs(a - b) <= bound).all())


# the golden cases, the random fields, and the random fields without make_closed_surface ("open": no ON_EDGE corner, nothing degenerate)
CASES = [("golden", n) for n in ("sine", "inv", "mesh")] + [("random", i) for i in range(len(RANDOM_FIELDS))] + [("open", i) for i in (0, 2, 3)]


def make_case(oracle, cls, case):
    kind, k = case
    if kind == "golden":
        return golden_case(cls, k)
    dims, seed, kw = RANDOM_FIELDS[k]
    return random_case(oracle, cls, dims, seed, dict(kw, make_closed_surface=0) if kind == "open" else kw)


@pytest.mark.parametrize("case", CASES)
def test_welded_mesh_vs_the_soup(oracle, tables, case):
    vals, outside, p = make_case(oracle, oracle.VoxelPostParams, case)
    verts, indices = welded(vals, outside, p, tables)
    soup = oracle.voxel_triangles(vals, outside, p, tables)
    flat = check_mesh(verts, indices, soup, outside, p)
    assert len(verts) > 100 and len(indices) > 100
    if not p.make_closed_surface:                  # no triangle is degenerate, so the triangles pair up one to one
        assert len(flat) == len(soup) and within_two_ulps(flat, soup, p)


def _interp(iso, p1, p2, v1, v2):
    """interpolate_pt in float32 with separate roundings (the device's -fmad=false, the oracle's -ffp-contract=off)."""
    f = np.float32
    if abs(f(iso) - f(v1)) < TOLERANCE:
        return np.array(p1, f)
    if abs(f(iso) - f(v2)) < TOLERANCE:
        return np.array(p2, f)
    if abs(f(v1) - f(v2)) < TOLERANCE:
        return np.array(p1, f)
    mu = f(max(f(0.0), min(f(1.0), f((f(iso) - f(v1)) / (f(v2) - f(v1))))))
    p1, p2 = np.array(p1, f), np.array(p2, f)
    return (p1 + mu * (p2 - p1)).astype(f)


def _local_edge(tables, axis_xyz, offs):
    """The local edge along axis (0 x, 1 y, 2 z) whose low corner is at offs (x, y, z) in the cube, and its corners in edge_to_vals order."""
    for i in range(12):
        c = []
        for e in tables[2][i]:
            yhi = (int(e) & 2) >> 1
            c.append((yhi ^ (int(e) & 1), yhi, int(e) >> 2))
        d = [k for k in range(3) if c[0][k] != c[1][k]]
        lo = tuple(min(c[0][k], c[1][k]) for k in range(3))
        if d == [axis_xyz] and lo == tuple(offs):
            return i, c
    raise AssertionError("no such edge")


def orientation_case(cls, tables):
    """A 2x3x3 grid, outside everywhere except corner a = (x 0, y 1, z 1): the x-edge from a to b = (1, 1, 1) is in all four cubes. Its owner, cube
    (0, 0, 0), walks it from one end and the last cube, (0, 1, 1), from the other; the field values are searched until the two interpolations differ.
    Returns (vals, outside, params, the owner's position, the last cube's position)."""
    p = post_params(cls, (2, 3, 3), make_closed_surface=0, remove_unconnected=0)
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = (-0.13, -0.21, -0.17)[d], (0.1, 0.07, 0.06)[d]
    g = grid_coords(p)
    pos = lambda c: (g[0][c[0]], g[1][c[1]], g[2][c[2]])
    _, c_own = _local_edge(tables, 0, (0, 1, 1))      # in cube (0, 0, 0)
    _, c_last = _local_edge(tables, 0, (0, 0, 0))     # in cube (0, 1, 1)
    rng = np.random.default_rng(11)
    for _ in range(10000):
        va, vb = np.float32(rng.uniform(0.01, 1.0)), np.float32(rng.uniform(-1.0, -0.01))
        val = lambda x: va if x == 0 else vb        # corners on the edge: x decides a or b
        own = _interp(0.0, pos(c_own[0]), pos(c_own[1]), val(c_own[0][0]), val(c_own[1][0]))
        last = _interp(0.0, pos((c_last[0][0], 1 + c_last[0][1], 1 + c_last[0][2])), pos((c_last[1][0], 1 + c_last[1][1], 1 + c_last[1][2])),
                       val(c_last[0][0]), val(c_last[1][0]))
        if not np.array_equal(own.view(np.uint32), last.view(np.uint32)):
            break
    else:
        raise AssertionError("no field found")
    vals = np.full((3, 2, 3), -1.0, np.float32)
    vals[1, 0, 1], vals[1, 1, 1] = va, vb
    outside = np.where(vals < 0, 1, 0).astype(np.uint8)
    return vals, outside, p, own, last


def _has_point(pts, q):
    return bool((np.asarray(pts, np.float32).reshape(-1, 3).view(np.uint32) == np.asarray(q, np.float32).view(np.uint32)).all(1).any())


def test_orientation_case(oracle, tables):
    vals, outside, p, own, last = orientation_case(oracle.VoxelPostParams, tables)
    assert np.array_equal(oracle.voxel_outside(vals, p), outside)
    verts, indices = welded(vals, outside, p, tables)
    soup = oracle.voxel_triangles(vals, outside, p, tables)
    assert len(verts) == 5 and len(indices) == 4 and len(soup) == 4   # the +x, +-y and +-z edges of a; one triangle per cube
    assert _has_point(verts, own) and not _has_point(verts, last)
    assert _has_point(soup[-1], last) and not _has_point(soup[-1], own)   # the last cube's own interpolation
    assert _has_point(verts[indices[-1].astype(np.int64)], own)           # welded: the owner's


def degenerate_case(cls, oracle, tables, max_seeds=50):
    """A make_closed_surface field whose welded triangle count differs from the soup's: values near the isolevel make interpolate_pt land on a
    corner from one end of an edge but an ulp away from the other, so a triangle can collapse in one mesh and not in the other. Returns
    (vals, outside, params of class cls, seed)."""
    dims = (6, 5, 7)
    for seed in range(max_seeds):
        rng = np.random.default_rng(seed)
        vals = rng.choice(np.array([-1, 1, 2e-12, -2e-12, -0.5, 0.5], np.float32), (dims[1], dims[0], dims[2])).astype(np.float32)
        po = post_params(oracle.VoxelPostParams, dims, make_closed_surface=1, remove_unconnected=0)
        for d in range(3):
            po.lo_pos[d], po.vsz[d] = (-0.13, -0.21, -0.17)[d], (0.1, 0.07, 0.06)[d]
        o = oracle.voxel_outside(vals, po)
        if len(welded(vals, o, po, tables)[1]) != len(oracle.voxel_triangles(vals, o, po, tables)):
            p = post_params(cls, dims, make_closed_surface=1, remove_unconnected=0)
            for d in range(3):
                p.lo_pos[d], p.vsz[d] = po.lo_pos[d], po.vsz[d]
            return vals, o, p, seed
    raise AssertionError("no degenerate case in %d seeds" % max_seeds)


def _normals(tris):
    t = np.asarray(tris, np.float32)
    a, b = (t[:, 1] - t[:, 0]).astype(np.float32), (t[:, 2] - t[:, 1]).astype(np.float32)
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1).astype(np.float32)


def test_degenerate_case(oracle, tables):
    vals, outside, p, _ = degenerate_case(oracle.VoxelPostParams, oracle, tables)
    verts, indices = welded(vals, outside, p, tables)
    soup = oracle.voxel_triangles(vals, outside, p, tables)
    flat = check_mesh(verts, indices, soup, outside, p)
    assert len(flat) != len(soup)
    assert (_normals(flat) != 0).any(1).all()        # no welded triangle has a zero normal in its welded positions
    assert (_normals(soup) != 0).any(1).all()


# ---- against the reference's own welded create_block cache (oracle/_ref) ----
def test_welded_mesh_against_reference(oracle, ref, beq):
    """refapi.Vox.triangles(welded=True) flattens the reference's shared cache; voxel_mesh_ref's mesh flattened the same way must equal it bit for bit."""
    from test_oracle_vs_reference import _need_vox, _vox_case
    _need_vox(ref)
    tables = ref.mc_tables()
    rng = np.random.default_rng(5)
    cases = [dict(dims=(24, 20, 16), gen=0, kw=dict(remove_unconnected=3)),
             dict(dims=(18, 22, 30), gen=1, kw=dict(remove_unconnected=3, invert=1, isolevel=0.1)),
             dict(dims=(16, 16, 16), gen=2, kw=dict(remove_unconnected=1, make_closed_surface=0, keep_at_scene_edge=1)),
             dict(dims=(12, 10, 9), gen=-1, kw=dict(remove_unconnected=3)),
             dict(dims=(13, 11, 17), gen=-1, kw=dict(remove_unconnected=1, make_closed_surface=0))]
    for c in cases:
        dims, kw = c["dims"], c["kw"]
        V, vpp, _ = _vox_case(oracle, ref, dims, (0.15, 0.12, 0.1), (0.0, 0.0, 0.3), max(c["gen"], 0), **kw)
        if c["gen"] >= 0:
            V.create_procedural(1.0, 1.3, (0.2, 0.1, -0.3), 1, 123, 456, c["gen"])
        else:
            V.set_vals(rng.uniform(-1, 1, (dims[1], dims[0], dims[2])).astype(np.float32))
        V.determine_outside()
        V.remove_unconnected()
        if kw["remove_unconnected"] > 2:
            V.remove_interior_holes()
        tr, _ = V.triangles(welded=True)
        verts, indices = welded(V.vals(), V.outside(), vpp, tables)
        flat = verts[indices.astype(np.int64)]
        assert flat.shape == tr.shape and beq(flat, tr) == 0, c


# ---- bindings ----
def test_entry_points_are_exported(tw):
    out = subprocess.check_output(["nm", "-D", "--defined-only", tw.LIB_PATH], text=True)
    for name in ("tw_voxel_mesh_welded", "tw_voxel_build_launch_ex"):
        assert " T %s\n" % name in out
        assert name in tw.ABI_SYMBOLS


def test_mirror_matches_the_header(tw, tmp_path):
    _layout(tmp_path, "tw_voxel_mesh", tw.VoxelMesh)


def test_null_arguments_without_a_device(tw):
    L = tw.lib
    p = tw.VoxelPostParams()
    p.nx = p.ny = p.nz = 4
    vals, flags = (C.c_float * 64)(), (C.c_uint8 * 64)()
    e, t, v = (C.c_uint32 * 256)(), (C.c_int32 * 4096)(), (C.c_uint32 * 24)()
    nv, nt = C.c_uint64(), C.c_uint64()
    m = tw.VoxelMesh(None, 0, None, 0, C.cast(C.pointer(nv), C.c_void_p), C.cast(C.pointer(nt), C.c_void_p))
    args = [C.cast(vals, C.c_void_p), C.cast(flags, C.c_void_p), C.byref(p), C.cast(e, C.c_void_p), C.cast(t, C.c_void_p), C.cast(v, C.c_void_p), C.byref(m)]
    assert L.tw_voxel_mesh_welded(None, *args) == tw.TW_ERR_ARG
    b = tw.VoxelBuild(None, None, C.cast(C.pointer(p), C.c_void_p), None, None, None, None, C.cast(vals, C.c_void_p), None, None, 0, None, None)
    assert L.tw_voxel_build_launch_ex(None, C.byref(b), C.byref(m)) == tw.TW_ERR_ARG
    assert L.tw_voxel_build_launch_ex(None, None, None) == tw.TW_ERR_ARG


def test_adapter_voxel_mesh_compiles(tw, tmp_path):
    from test_cpp_voxel_mesh import build_exe
    assert os.access(build_exe(tw, tmp_path), os.X_OK)
