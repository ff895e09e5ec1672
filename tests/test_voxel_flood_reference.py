"""An independent reference for remove_unconnected (remove_unconnected_outside + remove_interior_holes), written with numpy and scipy.ndimage.label
(6-connectivity) instead of a depth-first fill, and pinned here against the plain-C oracle (terrain_oracle.c, to_voxel_remove_unconnected) on smoothed
random fields and on constructed grids whose answer is known by construction. tests/test_gpu_voxel_shapes.py holds the device fills to it.

Semantics:
  pass 0   seeds: the centre voxel, or every voxel whose flag is exactly UNDER_MESH; with keep_at_edge also every voxel of the x/y edge columns whose flag
           is not 1. The fill spreads from the seeds through voxels whose flag is exactly 0. Every 0 it does not reach becomes 1 with val = isolevel -+ 1e-12.
  pass 1   (remove_unconnected > 2) seeds: the top plane (z = nz-1) where the flag is not 0. The fill spreads through flags of exactly 1; every 1 it does not
           reach becomes 0 with val = isolevel +- 1e-12 (the signs swap when invert is set)."""
import numpy as np
import pytest

from cases import convert

UNDER_MESH = 0x08
TOLERANCE = np.float32(1.0e-12)


def reached(passable, seeds):
    """Voxels of `passable` that a 6-connected fill from `seeds` reaches: the components of `passable` that hold a seed or touch one."""
    from scipy import ndimage
    labels, _ = ndimage.label(passable, structure=ndimage.generate_binary_structure(3, 1))
    touch = seeds.copy()
    for ax in range(3):
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        touch[tuple(lo)] |= seeds[tuple(hi)]
        touch[tuple(hi)] |= seeds[tuple(lo)]
    keep = np.zeros(int(labels.max()) + 1, bool)
    keep[labels[touch & passable]] = True
    keep[0] = False
    return keep[labels]


def remove_unconnected_ref(vals, outside, p):
    """Returns (vals, outside, changed) like oracle.voxel_remove_unconnected; vals / outside are [ny, nx, nz] arrays, p a VoxelPostParams."""
    ny, nx, nz = int(p.ny), int(p.nx), int(p.nz)
    v = np.array(vals, np.float32, copy=True).reshape(ny, nx, nz)
    o = np.array(outside, np.uint8, copy=True).reshape(ny, nx, nz)
    if p.remove_unconnected <= 0:
        return v, o, 0
    iso = np.float32(p.isolevel)
    tol = -TOLERANCE if p.invert else TOLERANCE
    if p.centre_seed:
        seeds = np.zeros(o.shape, bool)
        seeds[ny // 2, nx // 2, nz // 2] = True
    else:
        seeds = (o == UNDER_MESH)
    if p.keep_at_edge:
        edge = np.zeros((ny, nx), bool)
        edge[0, :] = edge[-1, :] = edge[:, 0] = edge[:, -1] = True
        seeds |= edge[:, :, None] & (o != 1)
    lost = (o == 0) & ~reached(o == 0, seeds)
    o[lost] = 1
    v[lost] = iso - tol
    changed = int(lost.sum())
    if p.remove_unconnected > 2:
        seeds = np.zeros(o.shape, bool)
        seeds[:, :, nz - 1] = o[:, :, nz - 1] != 0
        if seeds.any():
            lost = (o == 1) & ~reached(o == 1, seeds)
            o[lost] = 0
            v[lost] = iso + tol
            changed += int(lost.sum())
    return v, o, changed


# ---- cases shared with tests/test_gpu_voxel_shapes.py ----
def post_params(cls, dims, **kw):
    """A VoxelPostParams of the given ctypes class (product or oracle); kw: isolevel, invert, make_closed_surface, remove_unconnected, keep_at_edge,
    centre_seed, skip_under_mesh."""
    p = cls()
    p.nx, p.ny, p.nz = (int(d) for d in dims)
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = (-1.0, 0.5, 0.25)[d], (0.05, 0.07, 0.04)[d]
    p.isolevel, p.invert, p.make_closed_surface = kw.get("isolevel", 0.0), kw.get("invert", 0), kw.get("make_closed_surface", 1)
    p.remove_unconnected, p.keep_at_edge = kw.get("remove_unconnected", 1), kw.get("keep_at_edge", 0)
    p.centre_seed, p.skip_under_mesh = kw.get("centre_seed", 1), kw.get("skip_under_mesh", 0)
    return p


# the smoothed random fields of tests/test_gpu_voxel_post.py (many components, pockets, long thin connections)
RANDOM_FIELDS = [((40, 33, 29), 1, dict(remove_unconnected=3)), ((64, 64, 64), 2, dict(remove_unconnected=3, invert=1, isolevel=0.2, make_closed_surface=0)),
                 ((130, 70, 50), 3, dict(remove_unconnected=1, keep_at_edge=1, centre_seed=0)), ((17, 19, 23), 4, dict(remove_unconnected=3, centre_seed=0, skip_under_mesh=1))]


def random_field(dims, seed, centre_seed):
    """(vals [ny, nx, nz], zix [ny, nx] or None) as tests/test_gpu_voxel_post.py builds them."""
    nx, ny, nz = dims
    rng = np.random.default_rng(seed)
    f = rng.standard_normal((ny, nx, nz)).astype(np.float32)
    for ax in range(3):
        f = (f + np.roll(f, 1, ax) + np.roll(f, -1, ax)) / 3
    vals = np.ascontiguousarray(f * 3, np.float32)
    zix = None if centre_seed else rng.integers(0, nz // 2, (ny, nx)).astype(np.uint32)
    return vals, zix


def column_case(nz):
    """A 3x3xnz column with make_closed_surface: the inside is the one-voxel line x = y = 1, z = 1..nz-2, seeded at its centre voxel z = nz//2, so the
    fill runs max(nz//2 - 1, nz - 2 - nz//2) generations and reaches all of it: nothing changes. Returns (vals, kw)."""
    return np.ones((3, 3, nz), np.float32), dict(make_closed_surface=1, remove_unconnected=1, centre_seed=1)


def column_generations(nz):
    return max(nz // 2 - 1, nz - 2 - nz // 2)


def serpentine(nx, nz):
    """Cells (x, z) of a serpentine in the x-z plane in path order: rows z = 1, 3, ... run x = 1..nx-2 alternately right and left, joined at the row ends."""
    cells = []
    rows = list(range(1, nz - 1, 2))
    for r, z in enumerate(rows):
        xs = range(1, nx - 1) if r % 2 == 0 else range(nx - 2, 0, -1)
        cells += [(x, z) for x in xs]
        if r + 1 < len(rows):
            cells.append((xs[-1], z + 1))
    return cells


def serpentine_case(nx=64, nz=63, cut=900):
    """Pass 0: an inside serpentine corridor at y = 1 of an all-outside nx x 3 x nz grid, entered from the x = 0 edge column (keep_at_edge seeds it) and
    cut at path position `cut`: the part before the cut stays, the part after it becomes outside. Returns (vals, kw, expected outside, expected vals)."""
    cells = [(0, 1)] + serpentine(nx, nz)
    vals = np.full((3, nx, nz), -1.0, np.float32)
    for x, z in cells:
        vals[1, x, z] = 1.0
    vals[1, cells[cut][0], cells[cut][1]] = -1.0
    exp_o = (vals < 0).astype(np.uint8)
    exp_v = vals.copy()
    for x, z in cells[cut + 1:]:
        exp_o[1, x, z], exp_v[1, x, z] = 1, np.float32(0.0) - TOLERANCE
    return vals, dict(make_closed_surface=0, remove_unconnected=1, keep_at_edge=1, centre_seed=0), exp_o, exp_v


def corridor_case(nx=64, nz=63, cut=1500):
    """Pass 1: an all-inside nx x 4 x nz grid holding an outside corridor at y = 1 that enters from the top plane at x = 1 and winds down as a serpentine,
    cut at path position `cut`, plus a detached outside pocket. Pass 0 changes nothing (the centre voxel sits in the inside at y = 2); pass 1 turns the
    corridor beyond the cut and the pocket inside. Returns (vals, kw, expected outside, expected vals)."""
    rows = list(range(nz - 3, 0, -2))
    path = [(1, z) for z in range(nz - 1, rows[0], -1)]
    for r, z in enumerate(rows):
        xs = range(1, nx - 1) if r % 2 == 0 else range(nx - 2, 0, -1)
        path += [(x, z) for x in xs]
        if r + 1 < len(rows):
            path.append((xs[-1], z - 1))
    vals = np.ones((4, nx, nz), np.float32)
    for x, z in path:
        vals[1, x, z] = -1.0
    vals[1, path[cut][0], path[cut][1]] = 1.0
    pocket = [(2, nx // 2 + d, 5) for d in range(3)]
    for y, x, z in pocket:
        vals[y, x, z] = -1.0
    exp_o = (vals < 0).astype(np.uint8)
    exp_v = vals.copy()
    for y, x, z in [(1, x, z) for x, z in path[cut + 1:]] + pocket:
        exp_o[y, x, z], exp_v[y, x, z] = 0, np.float32(0.0) + TOLERANCE
    return vals, dict(make_closed_surface=0, remove_unconnected=3, centre_seed=1), exp_o, exp_v


# ---- the reference against the oracle (CPU) ----
@pytest.fixture(scope="module")
def scipy_ndimage():
    return pytest.importorskip("scipy.ndimage")


def _both(oracle, vals, p, zix=None):
    outside = oracle.voxel_outside(vals, p, zix)
    return outside, oracle.voxel_remove_unconnected(vals, outside, p), remove_unconnected_ref(vals, outside, p)


def _same(a, b, beq):
    assert np.array_equal(a[1], b[1]) and beq(a[0], b[0]) == 0 and a[2] == b[2]


@pytest.mark.parametrize("dims,seed,kw", RANDOM_FIELDS)
def test_reference_matches_oracle_random_fields(oracle, beq, scipy_ndimage, dims, seed, kw):
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    _, o, r = _both(oracle, vals, post_params(oracle.VoxelPostParams, dims, **kw), zix)
    _same(r, o, beq)
    assert o[2] > 0


@pytest.mark.parametrize("mode", [1, 3])
@pytest.mark.parametrize("keep_at_edge", [0, 1])
@pytest.mark.parametrize("mesh", [0, 1])
@pytest.mark.parametrize("invert", [0, 1])
def test_reference_matches_oracle_options(oracle, beq, scipy_ndimage, mode, keep_at_edge, mesh, invert):
    """Every combination of the options that pick the seeds and the two passes, on one odd-sized field."""
    dims = (31, 27, 23)
    vals, zix = random_field(dims, 11, centre_seed=not mesh)
    p = post_params(oracle.VoxelPostParams, dims, remove_unconnected=mode, keep_at_edge=keep_at_edge, centre_seed=int(not mesh), invert=invert,
                    isolevel=0.1, make_closed_surface=int(not keep_at_edge))
    outside, o, r = _both(oracle, vals, p, zix)
    _same(r, o, beq)
    assert o[2] > 0


@pytest.mark.parametrize("nz", [16, 18, 20, 32, 34, 36, 40002])
def test_reference_matches_oracle_column(oracle, beq, scipy_ndimage, nz):
    vals, kw = column_case(nz)
    outside, o, r = _both(oracle, vals, post_params(oracle.VoxelPostParams, (3, 3, nz), **kw))
    _same(r, o, beq)
    assert o[2] == 0 and np.array_equal(o[1], outside) and beq(o[0], vals) == 0


def test_column_generations():
    """The column lengths of the deep-fill tests end the fill at 7, 8, 9, 15, 16, 17 and 20000 generations (the GPU checks its frontier every 8)."""
    assert [column_generations(nz) for nz in (16, 18, 20, 32, 34, 36, 40002)] == [7, 8, 9, 15, 16, 17, 20000]


@pytest.mark.parametrize("case", [serpentine_case, corridor_case])
def test_reference_matches_oracle_corridors(oracle, beq, scipy_ndimage, case):
    vals, kw, exp_o, exp_v = case()
    ny, nx, nz = vals.shape
    _, o, r = _both(oracle, vals, post_params(oracle.VoxelPostParams, (nx, ny, nz), **kw))
    _same(r, o, beq)
    assert np.array_equal(o[1], exp_o) and beq(o[0], exp_v) == 0 and o[2] == int((exp_o != (vals < 0)).sum()) > 100
