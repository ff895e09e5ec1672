"""GPU: resident voxel models (tw_voxel_model_*, Context.voxel_model) - per-block welded meshes, in-place edits, and re-meshing of the blocks an edit
changes.

- The build job with one block equals tw_voxel_mesh_welded bit for bit; with many blocks it equals the per-block sequential reference of
  tests/voxel_mesh_blocks_ref.c on the golden cases, random fields with every option, block sizes that do not divide the grid, one-column blocks, a block larger
  than the grid, odd and tiny grids.
- Edit sequences of random boxes (block faces, grid edges, overlaps, an edit that changes nothing, an edit that cuts a region off so remove_unconnected
  flips voxels far from the box): after each, the raw field is the caller's copy, the field and flags are tw_voxel_outside -> tw_voxel_remove_unconnected
  on it, every block's latest mesh equals a fresh per-block build, and the listed blocks are exactly the blocks that read a changed voxel - which holds
  every block whose mesh changed.
- 256^3 and 512^3 GLM fills with device and page-locked outputs; capacities, refusals, tw_cancel, destroy with a job pending, other jobs afterwards."""
import os

import numpy as np
import pytest

from test_gpu_voxel_build import _post_for, _scfg
from test_gpu_voxel_mesh import _mesh_bufs, _np, _same_mesh, _untouched
from test_voxel_flood_reference import post_params, random_field
from test_voxel_mesh_host import CASES, make_case
from test_voxel_model_host import marked_blocks, split_blocks
from voxel_mesh_blocks_ref import voxel_mesh_blocks as welded_blocks

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def tables():
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _rows(job):
    b = job.blocks
    return np.stack([b["block"], b["voff"], b["nverts"], b["toff"], b["ntris"]], 1).astype(np.uint64) if len(b) else np.zeros((0, 5), np.uint64)


def _run(ctx, launch, nv, nt, kind="device"):
    """A model job into buffers of nv, nt rows plus sentinels: (job, verts, indices) with the counts' rows."""
    v, i = _mesh_bufs(kind, nv, nt)
    job = launch(v[:nv], i[:nt])
    assert ctx.create_tiles_poll(wait=True)
    assert job.nverts <= nv and job.ntris <= nt and _untouched(v, i, nv, nt)
    return job, np.array(_np(v)[:job.nverts]), np.asarray(_np(i)).view(np.uint32)[:job.ntris].copy()


def _chain(ctx, raw, p, zix):
    o = ctx.voxel_outside(raw, p, zix)
    v = raw.copy()
    ctx.voxel_remove_unconnected(v, o, p)
    return v, o


# ---- the build ----
@pytest.mark.parametrize("case", CASES)
def test_one_block_is_the_welded_mesh(tw, oracle, ctx, tables, case):
    vals, outside, p = make_case(oracle, tw.VoxelPostParams, case)
    p.remove_unconnected = 0      # the field is already post-processed: its flags are its outside flags
    exp = ctx.voxel_mesh(vals, ctx.voxel_outside(vals, p), p, tables)
    m = ctx.voxel_model(p, tables, bx=int(p.nx), by=int(p.ny))
    job, gv, gi = _run(ctx, lambda v, i: m.build_launch(vals=vals, verts=v, indices=i), len(exp[0]) + 5, len(exp[1]) + 5)
    _same_mesh((gv, gi), exp)
    assert _rows(job).tolist() == [[0, 0, len(exp[0]), 0, len(exp[1])]]
    m.close()


BLOCK_SHAPES = [((40, 33, 29), 1, dict(remove_unconnected=3), (7, 5)), ((64, 64, 64), 2, dict(remove_unconnected=3, invert=1, isolevel=0.2, make_closed_surface=0), (16, 16)),
                ((130, 70, 50), 3, dict(remove_unconnected=1, keep_at_edge=1, centre_seed=0), (1, 1)),
                ((17, 19, 23), 4, dict(remove_unconnected=3, centre_seed=0, skip_under_mesh=1), (100, 3)),
                ((33, 17, 65), 5, dict(remove_unconnected=3, invert=1, isolevel=0.1), (32, 16)), ((2, 2, 2), 6, dict(remove_unconnected=0, make_closed_surface=0), (1, 1)),
                ((5, 7, 9), 7, dict(remove_unconnected=1), (3, 4)), ((1, 9, 9), 8, dict(remove_unconnected=0), (4, 4)),
                ((70, 3, 200), 9, dict(remove_unconnected=1, make_closed_surface=0), (9, 1)), ((64, 40, 48), 10, dict(remove_unconnected=3, centre_seed=0, skip_under_mesh=1), (13, 11))]


@pytest.mark.parametrize("dims,seed,kw,bs", BLOCK_SHAPES)
def test_blocks_vs_reference(tw, ctx, tables, dims, seed, kw, bs):
    raw, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    p = post_params(tw.VoxelPostParams, dims, **kw)
    v2, o2 = _chain(ctx, raw, p, zix)
    ev, ei, et = welded_blocks(v2, o2, p, tables, *bs)
    m = ctx.voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
    job, gv, gi = _run(ctx, lambda v, i: m.build_launch(vals=raw, verts=v, indices=i), len(ev) + 2, len(ei) + 2, "pinned")
    _same_mesh((gv, gi), (ev, ei))
    assert np.array_equal(_rows(job), et) and job.nverts == len(ev) and job.ntris == len(ei)
    r, v, o = m.read()
    assert np.array_equal(r.view(np.uint32), raw.view(np.uint32)) and np.array_equal(v.view(np.uint32), v2.view(np.uint32)) and np.array_equal(o, o2)


def test_golden_cases_in_blocks(tw, oracle, ctx, tables):
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    for name in ("sine", "inv", "mesh"):
        _, _, p = make_case(oracle, tw.VoxelPostParams, ("golden", name))
        raw = g[name + "_vals"]
        zix = g[name + "_zix"] if name + "_zix" in g else None
        v2, o2 = _chain(ctx, raw, p, zix)
        assert np.array_equal(v2.view(np.uint32), g[name + "_vals2"].view(np.uint32)) and np.array_equal(o2, g[name + "_outside2"])
        for bs in ((5, 6), (int(p.nx), 1)):
            ev, ei, et = welded_blocks(v2, o2, p, tables, *bs)
            m = ctx.voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
            job, gv, gi = _run(ctx, lambda v, i: m.build_launch(vals=raw, verts=v, indices=i), len(ev), len(ei))
            _same_mesh((gv, gi), (ev, ei))
            assert np.array_equal(_rows(job), et)
            m.close()


# ---- edits ----
def _dumbbell():
    """Two inside blobs joined by a one-voxel bar along x; the centre seed sits in blob A. Cutting the bar at x = 30 disconnects the bar's far part and
    blob B (x ~ 42), which remove_unconnected turns outside."""
    nx, ny, nz = 48, 20, 20
    y, x, z = np.meshgrid(np.arange(ny), np.arange(nx), np.arange(nz), indexing="ij")
    vals = np.full((ny, nx, nz), -1.0, np.float32)
    vals[(x - 24) ** 2 + (y - 10) ** 2 + (z - 10) ** 2 <= 16] = 1.0
    vals[((x - 42) ** 2 + (y - 10) ** 2 + (z - 10) ** 2 <= 9)] = 1.0
    vals[10, 24:43, 10] = 1.0
    return vals, (nx, ny, nz)


def _edit_sequence(tw, ctx, tables, raw, zix, p, bs, boxes_fn, steps, kind="device"):
    dims = (int(p.nx), int(p.ny), int(p.nz))
    m = ctx.voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
    v0, o0 = _chain(ctx, raw, p, zix)
    ev, ei, et = welded_blocks(v0, o0, p, tables, *bs)
    cap_v, cap_i = 2 * len(ev) + 1000, 2 * len(ei) + 1000
    job, gv, gi = _run(ctx, lambda v, i: m.build_launch(vals=raw, verts=v, indices=i), cap_v, cap_i, kind)
    latest = split_blocks(gv, gi, _rows(job))
    raw = raw.copy()
    listed = []
    for step in range(steps):
        boxes, values = boxes_fn(step, raw)
        for (x, y, z, w, h, d), val in zip(boxes, values):
            raw[y:y + h, x:x + w, z:z + d] = val.reshape(h, w, d)
        packed = np.concatenate([np.ascontiguousarray(val, np.float32).ravel() for val in values]) if boxes else np.zeros(0, np.float32)
        job, gv, gi = _run(ctx, lambda v, i: m.edit_launch(boxes, packed, verts=v, indices=i), cap_v, cap_i, kind)
        rows = _rows(job)
        v1, o1 = _chain(ctx, raw, p, zix)
        r, gv1, go1 = m.read()
        assert np.array_equal(r.view(np.uint32), raw.view(np.uint32)), step
        assert np.array_equal(gv1.view(np.uint32), v1.view(np.uint32)) and np.array_equal(go1, o1), step
        fresh = split_blocks(*welded_blocks(v1, o1, p, tables, *bs))
        marked = marked_blocks(v0, o0, v1, o1, dims[0], dims[1], *bs)
        assert sorted(int(b) for b in rows[:, 0]) == sorted(marked) and list(rows[:, 0]) == sorted(rows[:, 0]), step
        assert job.nverts == int(rows[:, 2].sum()) and job.ntris == int(rows[:, 4].sum())
        changed = {b for b in fresh if not (np.array_equal(fresh[b][0].view(np.uint32), latest[b][0].view(np.uint32)) and np.array_equal(fresh[b][1], latest[b][1]))}
        assert changed <= marked, step
        latest.update(split_blocks(gv, gi, rows))
        for b in fresh:
            assert np.array_equal(latest[b][0].view(np.uint32), fresh[b][0].view(np.uint32)) and np.array_equal(latest[b][1], fresh[b][1]), (step, b)
        listed.append(len(rows))
        v0, o0 = v1, o1
    m.close()
    return listed


def _random_boxes(rng, dims, bs, n=3):
    """Up to n boxes per edit: on block faces, at the grid's edges, overlapping, or anywhere; values from a few levels around the isolevel."""
    def boxes_fn(step, raw):
        nx, ny, nz = dims
        boxes, values = [], []
        for _ in range(int(rng.integers(1, n + 1))):
            kind = rng.integers(0, 4)
            w, h, d = int(rng.integers(1, 6)), int(rng.integers(1, 6)), int(rng.integers(1, 8))
            w, h, d = min(w, nx), min(h, ny), min(d, nz)
            if kind == 0:      # straddling a block face
                x = max(0, min(nx - w, bs[0] * int(rng.integers(0, max(1, nx // bs[0]) + 1)) - w // 2))
                y = max(0, min(ny - h, bs[1] * int(rng.integers(0, max(1, ny // bs[1]) + 1)) - h // 2))
            elif kind == 1:    # at the grid's edge
                x, y = (0 if rng.integers(0, 2) else nx - w), (0 if rng.integers(0, 2) else ny - h)
            else:
                x, y = int(rng.integers(0, nx - w + 1)), int(rng.integers(0, ny - h + 1))
            z = int(rng.integers(0, nz - d + 1))
            boxes.append((x, y, z, w, h, d))
            values.append(rng.choice(np.array([-2.0, -0.3, 0.0, 0.4, 2.5], np.float32), (h, w, d)))
        return boxes, values
    return boxes_fn


@pytest.mark.parametrize("rm", [0, 1, 3])
@pytest.mark.parametrize("kind", ["device", "pinned"])
def test_random_edit_sequences(tw, ctx, tables, rm, kind):
    dims, bs = (40, 33, 29), (8, 5)
    kw = dict(remove_unconnected=rm, centre_seed=0, skip_under_mesh=1, keep_at_edge=1) if rm == 1 else dict(remove_unconnected=rm, invert=int(rm == 3))
    raw, zix = random_field(dims, 11 + rm, kw.get("centre_seed", 1))
    p = post_params(tw.VoxelPostParams, dims, **kw)
    listed = _edit_sequence(tw, ctx, tables, raw, zix, p, bs, _random_boxes(np.random.default_rng(rm), dims, bs), 22, kind)
    assert max(listed) > 0


def test_edit_that_changes_nothing_and_empty_edits(tw, ctx, tables):
    dims, bs = (21, 17, 15), (4, 4)
    for kw in (dict(remove_unconnected=0), dict(remove_unconnected=3)):
        raw, _ = random_field(dims, 2, 1)
        p = post_params(tw.VoxelPostParams, dims, **kw)
        same = lambda step, r: ([(3, 4, 2, 6, 5, 7), (0, 0, 0, 21, 1, 15)], [r[4:9, 3:9, 2:9].copy(), r[0:1, 0:21, 0:15].copy()])  # noqa: E731
        empty = lambda step, r: ([], [])  # noqa: E731
        assert _edit_sequence(tw, ctx, tables, raw, None, p, bs, same, 2) == [0, 0]
        assert _edit_sequence(tw, ctx, tables, raw, None, p, bs, empty, 1) == [0]


def test_edit_that_cuts_a_region_off(tw, ctx, tables):
    raw, dims = _dumbbell()
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=1, make_closed_surface=0, centre_seed=1)
    bs = (8, 4)
    m = ctx.voxel_model(p, tables, bx=bs[0], by=bs[1])
    big = (200000, 200000)
    _run(ctx, lambda v, i: m.build_launch(vals=raw, verts=v, indices=i), *big)
    _, v_before, _ = m.read()
    assert v_before[10, 42, 10] > 0                    # blob B is connected
    job, _, _ = _run(ctx, lambda v, i: m.edit_launch([(30, 10, 10, 1, 1, 1)], np.float32([-1.0]), verts=v, indices=i), *big)
    _, v_after, o_after = m.read()
    assert v_after[10, 42, 10] < 0 and o_after[10, 42, 10] == 1 and job.changed > 0
    listed = set(int(b) for b in job.blocks["block"])
    nbx = (dims[0] - 1 + bs[0] - 1) // bs[0]
    assert {2 * nbx + 3, 2 * nbx + 5} <= listed        # the box's block (cubes x 24..31, y 8..11) and blob B's (x 40..46), far from it
    m.close()
    # the same edit through the sequence checks
    _edit_sequence(tw, ctx, tables, raw, None, p, bs, lambda s, r: ([(30, 10, 10, 1, 1, 1)], [np.float32([[[-1.0]]])]), 1)


# ---- big fills ----
@pytest.mark.parametrize("n,kind", [(256, "device"), (512, "pinned")])
def test_glm_fill(tw, scene, ctx, tables, n, kind):
    vp = scene.voxel_landscape_params(_scfg(scene, 1), n, n, n, z_gradient=-2.0)
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=3, centre_seed=0, skip_under_mesh=1)
    zix = np.random.default_rng(7).integers(n // 16, n // 4, (n, n)).astype(np.uint32)
    m = ctx.voxel_model(p, tables, zix_xy=zix, bx=32, by=32)
    probe = m.build_launch(fill=vp)
    assert ctx.create_tiles_poll(wait=True)
    raw, v2, o2 = m.read()
    ev, ei, et = welded_blocks(v2, o2, p, tables, 32, 32)
    assert (probe.nverts, probe.ntris) == (len(ev), len(ei)) and len(ei) > 10000 and np.array_equal(_rows(probe), et)
    job, gv, gi = _run(ctx, lambda v, i: m.build_launch(fill=vp, verts=v, indices=i), len(ev), len(ei), kind)
    _same_mesh((gv, gi), (ev, ei))
    # one brush stroke: a ball of radius 6 voxels set inside around a surface point
    c = np.array([n // 2, n // 2, int(np.argmax(o2[n // 2, n // 2] == 1))])
    x0, y0, z0 = (max(0, int(k) - 6) for k in c)
    w, h, d = min(13, n - x0), min(13, n - y0), min(13, n - z0)
    box = raw[y0:y0 + h, x0:x0 + w, z0:z0 + d].copy()
    yy, xx, zz = np.meshgrid(np.arange(y0, y0 + h), np.arange(x0, x0 + w), np.arange(z0, z0 + d), indexing="ij")
    box[(xx - c[0]) ** 2 + (yy - c[1]) ** 2 + (zz - c[2]) ** 2 <= 36] = 1.0
    ejob, gv, gi = _run(ctx, lambda v, i: m.edit_launch([(x0, y0, z0, w, h, d)], box, verts=v, indices=i), len(ev), len(ei), kind)
    raw[y0:y0 + h, x0:x0 + w, z0:z0 + d] = box
    r, v3, o3 = m.read()
    assert np.array_equal(r.view(np.uint32), raw.view(np.uint32))
    ev3, eo3 = _chain(ctx, raw, p, zix)
    assert np.array_equal(v3.view(np.uint32), ev3.view(np.uint32)) and np.array_equal(o3, eo3)
    fresh = split_blocks(*welded_blocks(v3, o3, p, tables, 32, 32))
    rows = _rows(ejob)
    assert len(rows) >= 1 and sorted(rows[:, 0]) == sorted(marked_blocks(v2, o2, v3, o3, n, n, 32, 32))
    for b, (bv, bi) in split_blocks(gv, gi, rows).items():
        assert np.array_equal(bv.view(np.uint32), fresh[b][0].view(np.uint32)) and np.array_equal(bi, fresh[b][1])
    m.close()


# ---- rules ----
def test_capacities(tw, ctx, tables):
    dims, bs = (40, 33, 29), (8, 5)
    raw, _ = random_field(dims, 1, 1)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=3)
    v2, o2 = _chain(ctx, raw, p, None)
    ev, ei, et = welded_blocks(v2, o2, p, tables, *bs)
    m = ctx.voxel_model(p, tables, bx=bs[0], by=bs[1])
    for cv, ct in ((0, 0), (len(ev) // 2, len(ei) // 3), (17, 5)):
        v, i = _mesh_bufs("device", cv, ct)
        job = m.build_launch(vals=raw, verts=v[:cv] if cv else None, indices=i[:ct] if ct else None)
        assert ctx.create_tiles_poll(wait=True)
        assert (job.nverts, job.ntris) == (len(ev), len(ei)) and np.array_equal(_rows(job), et) and _untouched(v, i, cv, ct)
        assert np.array_equal(_np(v)[:cv].view(np.uint32), ev[:cv].view(np.uint32)) and np.array_equal(np.asarray(_np(i)).view(np.uint32)[:ct], ei[:ct])


def test_refusals(tw, ctx, tables):
    import ctypes as C
    p = post_params(tw.VoxelPostParams, (12, 10, 8), remove_unconnected=1)
    with pytest.raises(tw.TwError):
        ctx.voxel_model(p, tables, bx=0, by=4)
    with pytest.raises(tw.TwError):
        ctx.voxel_model(post_params(tw.VoxelPostParams, (1200, 1200, 1000)), tables, bx=2000, by=2000)     # 3*(block's voxels) >= 2^32
    m = ctx.voxel_model(p, tables, bx=4, by=4)
    raw = np.ones((10, 12, 8), np.float32)
    with pytest.raises(tw.TwError) as e:
        m.edit_launch([(0, 0, 0, 1, 1, 1)], np.zeros(1, np.float32))      # before the first build
    assert e.value.status == tw.TW_ERR_STATE
    with pytest.raises(tw.TwError) as e:
        m.read()
    assert e.value.status == tw.TW_ERR_STATE
    with pytest.raises(tw.TwError):
        m.build_launch(vals=raw, verts=np.zeros((8, 3), np.float32))     # pageable verts
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    for boxes in ([(0, 0, 0, 0, 1, 1)], [(11, 0, 0, 2, 1, 1)], [(0, 9, 0, 1, 2, 1)], [(0, 0, 7, 1, 1, 2)], [(12, 0, 0, 1, 1, 1)]):
        with pytest.raises(tw.TwError) as e:
            m.edit_launch(boxes, np.zeros(8, np.float32))
        assert e.value.status == tw.TW_ERR_ARG
    L, h = tw.lib, m._h
    out = tw.VoxelBlocksOut(None, 4, None, 0, None, None, None, None, None)
    assert L.tw_voxel_model_edit_launch(h, None, 0, None, C.byref(out)) == tw.TW_ERR_ARG      # no table / counts; a capacity without its buffer
    assert L.tw_voxel_model_build_launch(h, None, None, None, C.byref(out)) == tw.TW_ERR_ARG
    assert ctx.create_tiles_poll(wait=True)                 # nothing was enqueued
    m.close()


def test_cancel_destroy_and_other_jobs(tw, oracle, ctx, tables):
    dims, bs = (64, 64, 64), (16, 16)
    raw, _ = random_field(dims, 2, 1)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=3)
    c = tw.Context(0)
    try:
        m = c.voxel_model(p, tables, bx=bs[0], by=bs[1])
        m.build_launch(vals=raw)
        with pytest.raises(tw.TwError) as e:
            c.cancel()
        assert e.value.status == tw.TW_ERR_STATE
        assert c.create_tiles_poll(wait=True)
        m.edit_launch([(10, 10, 10, 4, 4, 4)], np.full(64, 3.0, np.float32))
        with pytest.raises(tw.TwError) as e:
            c.cancel()
        assert e.value.status == tw.TW_ERR_STATE
        m.close()                                           # destroys with the edit pending
        # other jobs on the context afterwards: the welded mesh and the voxel build job, bit for bit
        vals, outside, q = make_case(oracle, tw.VoxelPostParams, ("random", 0))
        from voxel_mesh_ref import voxel_mesh as welded
        _same_mesh(c.voxel_mesh(vals, outside, q, tables), welded(vals, outside, q, tables))
        m2 = c.voxel_model(p, tables, bx=bs[0], by=bs[1])
        m2.build_launch(vals=raw)                           # pending when the context closes
    finally:
        c.close()
