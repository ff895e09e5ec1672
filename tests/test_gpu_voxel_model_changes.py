"""GPU: the change list of a voxel model edit (tw_voxel_model_edit_launch_ex, VoxelModel.edit_launch(changes=...)).

For every edit, tw_voxel_model_read before and after gives the voxels whose value after remove_unconnected (bitwise) or flags differ. The list must be
exactly those, ascending, with their new values (bitwise) and flags; the first min(capacity, count) entries are written and nothing past them; a copy of
the read before the edit patched with the list equals the read after it; and the re-meshed blocks are exactly the readers of the listed voxels.
Covered: random edit sequences with remove_unconnected 0 and 3 on random, sine and GLM fields with overlapping boxes; an edit that cuts a region off a
256^3 grid, so millions of voxels far from the box change over thousands of scan chunks; no-op and empty edits; a grid whose voxel count is not a
multiple of 32 with changes straddling bitmask words; capacities 0 (no index), count - 1, count and more; device and page-locked outputs; every
refusal; and the list beside an overflowing mesh capacity."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_voxel_build import _post_for, _scfg
from test_gpu_voxel_mesh import _mesh_bufs, _np
from test_voxel_flood_reference import post_params, random_field
from test_voxel_model_host import marked_blocks

pytestmark = pytest.mark.gpu
SENT_I, SENT_O = 0xDEADBEEF, 0xAB
EXTRA = 3


@pytest.fixture(scope="module")
def tables():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _list_bufs(kind, cap):
    """index / vals / outside buffers of cap + EXTRA entries filled with sentinels: 'device' CUDA tensors or 'pinned' page-locked torch tensors."""
    import torch
    dev = "cuda" if kind == "device" else "cpu"
    i = torch.full((cap + EXTRA,), SENT_I - (1 << 32), dtype=torch.int32, device=dev)
    v = torch.full((cap + EXTRA,), float("nan"), dtype=torch.float32, device=dev)
    o = torch.full((cap + EXTRA,), SENT_O, dtype=torch.uint8, device=dev)
    if kind == "pinned":
        i, v, o = i.pin_memory(), v.pin_memory(), o.pin_memory()
    torch.cuda.synchronize()
    return i, v, o


def _rows(job):
    return sorted(int(b) for b in job.blocks["block"])


def _readers(index, shape, bx, by):
    """The blocks whose cubes read the listed voxels (marked_blocks of a field that differs exactly there)."""
    ny, nx, nz = shape
    mask = np.zeros(ny * nx * nz, np.float32)
    mask[index] = 1.0
    zero = np.zeros(ny * nx * nz, np.uint8)
    return marked_blocks(np.zeros_like(mask), zero, mask, zero, nx, ny, bx, by)


def _checked_edit(ctx, m, boxes, values, cap=None, kind="device", with_vals=True, with_outside=True, mesh=None):
    """One edit with a change list of capacity cap (None: the grid's voxel count; 0: no index) against the reads before and after it. Returns
    (count, job)."""
    shape = (int(m.vpp.ny), int(m.vpp.nx), int(m.vpp.nz))
    n = int(np.prod(shape))
    _, v0, o0 = m.read()
    cap = n if cap is None else cap
    i, v, o = _list_bufs(kind, cap)
    bufs = (i[:cap] if cap else None, v[:cap] if cap and with_vals else None, o[:cap] if cap and with_outside else None)
    packed = np.concatenate([np.ascontiguousarray(x, np.float32).ravel() for x in values]) if boxes else np.zeros(0, np.float32)
    mv, mi = mesh if mesh is not None else (None, None)
    job = m.edit_launch(boxes, packed, verts=mv, indices=mi, changes=bufs)
    assert ctx.create_tiles_poll(wait=True)
    _, v1, o1 = m.read()
    diff = (v0.view(np.uint32) != v1.view(np.uint32)) | (o0 != o1)
    exp = np.flatnonzero(diff.ravel())
    assert job.nchanged == len(exp)
    k = min(cap, len(exp))
    gi, gv, go = np.asarray(_np(i)).view(np.uint32), _np(v), _np(o)
    assert np.array_equal(gi[:k], exp[:k]) and (gi[k:] == SENT_I).all()
    if with_vals:
        assert np.array_equal(gv[:k].view(np.uint32), v1.ravel()[exp[:k]].view(np.uint32)) and np.isnan(gv[k:]).all()
    else:
        assert np.isnan(gv).all()
    if with_outside:
        assert np.array_equal(go[:k], o1.ravel()[exp[:k]]) and (go[k:] == SENT_O).all()
    else:
        assert (go == SENT_O).all()
    got = job.changes
    assert (got[0] is None) if not cap else len(got[0]) == k
    if k == len(exp) and with_vals and with_outside:       # the list patches the read before the edit into the read after it
        pv, po = v0.ravel().copy(), o0.ravel().copy()
        pv[gi[:k]], po[gi[:k]] = gv[:k], go[:k]
        assert np.array_equal(pv.view(np.uint32), v1.ravel().view(np.uint32)) and np.array_equal(po, o1.ravel())
    nx, ny = shape[1], shape[0]
    assert _rows(job) == sorted(marked_blocks(v0, o0, v1, o1, nx, ny, m.bx, m.by)) == sorted(_readers(exp, shape, m.bx, m.by))
    return len(exp), job


def _boxes(rng, dims, n=3):
    """Up to n random boxes, the last overlapping the first, with values from a few levels around the isolevel."""
    nx, ny, nz = dims
    boxes, values = [], []
    for _ in range(int(rng.integers(1, n + 1))):
        w, h, d = min(int(rng.integers(1, 7)), nx), min(int(rng.integers(1, 7)), ny), min(int(rng.integers(1, 9)), nz)
        boxes.append((int(rng.integers(0, nx - w + 1)), int(rng.integers(0, ny - h + 1)), int(rng.integers(0, nz - d + 1)), w, h, d))
    x, y, z, w, h, d = boxes[0]
    boxes.append((x + w // 2, y + h // 2, z + d // 2, min(w, nx - x - w // 2), min(h, ny - y - h // 2), min(d, nz - z - d // 2)))
    for (_, _, _, w, h, d) in boxes:
        values.append(rng.choice(np.array([-2.0, -0.3, 0.0, 0.4, 2.5], np.float32), (h, w, d)))
    return boxes, values


# ---- edit sequences ----
@pytest.mark.parametrize("rm", [0, 3])
@pytest.mark.parametrize("kind", ["device", "pinned"])
def test_random_edit_sequences(tw, ctx, tables, rm, kind):
    dims = (40, 33, 29)
    raw, zix = random_field(dims, 21 + rm, 1)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=rm, invert=int(rm == 3))
    m = ctx.voxel_model(p, tables, zix_xy=zix, bx=8, by=5)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    rng = np.random.default_rng(100 + rm)
    counts = [_checked_edit(ctx, m, *_boxes(rng, dims), kind=kind)[0] for _ in range(16)]
    assert max(counts) > 0
    m.close()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("rm", [0, 3])
def test_fills(tw, scene, ctx, tables, mode, rm):
    """The sine (mode 0) and GLM (mode 1) fills of a 96 x 80 x 64 grid, edited with overlapping boxes and with brush balls."""
    vp = scene.voxel_landscape_params(_scfg(scene, mode), 96, 80, 64, z_gradient=-2.0)
    assert vp.gen_mode == mode      # TW_MGEN_SINE, TW_MGEN_SIMPLEX (the GLM noise)
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=rm, centre_seed=0, skip_under_mesh=1)
    zix = np.random.default_rng(5).integers(2, 16, (80, 96)).astype(np.uint32)
    m = ctx.voxel_model(p, tables, zix_xy=zix, bx=16, by=16)
    m.build_launch(fill=vp)
    assert ctx.create_tiles_poll(wait=True)
    rng = np.random.default_rng(7 + mode + rm)
    for step in range(10):
        if step % 2:
            raw, _, o = m.read()
            c = np.array([int(rng.integers(8, 88)), int(rng.integers(8, 72)), 0])
            c[2] = int(np.argmax(o[c[1], c[0]] == 1))
            x0, y0, z0 = (max(0, int(k) - 6) for k in c)
            w, h, d = min(13, 96 - x0), min(13, 80 - y0), min(13, 64 - z0)
            box = raw[y0:y0 + h, x0:x0 + w, z0:z0 + d].copy()
            yy, xx, zz = np.meshgrid(np.arange(y0, y0 + h), np.arange(x0, x0 + w), np.arange(z0, z0 + d), indexing="ij")
            box[(xx - c[0]) ** 2 + (yy - c[1]) ** 2 + (zz - c[2]) ** 2 <= 36] = 1.0 if step % 4 == 1 else -3.0
            _checked_edit(ctx, m, [(x0, y0, z0, w, h, d)], [box], kind="pinned")
        else:
            _checked_edit(ctx, m, *_boxes(rng, (96, 80, 64)))
    m.close()


def _cut_field(n):
    """An n^3 field: a ball around the centre seed, joined by a one-voxel bar along x to a slab that fills x >= 5n/8 - millions of voxels, which
    remove_unconnected turns outside once the bar is cut."""
    c = n // 2
    y, x, z = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij", sparse=True)
    vals = np.full((n, n, n), -1.0, np.float32)
    vals[((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2 <= (n // 16) ** 2).nonzero()] = 1.0
    vals[:, 5 * n // 8:, 4:n - 4] = 1.0
    vals[c, c:5 * n // 8, c] = 1.0
    return vals


def test_edit_that_cuts_a_region_off_256(tw, ctx, tables):
    n = 256
    raw = _cut_field(n)
    p = post_params(tw.VoxelPostParams, (n, n, n), remove_unconnected=1, make_closed_surface=0, centre_seed=1)
    m = ctx.voxel_model(p, tables, bx=32, by=32)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    cut, mend = (([(5 * n // 8 - 8, n // 2, n // 2, 1, 1, 1)], [np.float32([[[v]]])]) for v in (-1.0, 1.0))
    count, job = _checked_edit(ctx, m, cut[0], cut[1])
    assert count > 5 * 10 ** 6 and (n ** 3 + 31) // 32 // 256 >= 2048       # the slab, over more scan chunks than one pass of the scan's block
    listed = _rows(job)
    assert len(listed) > 20                                                 # far from the box's own blocks
    # the same edit and its undo with capacities count - 1, count and more, on device and page-locked outputs
    for cap, kind in ((count - 1, "device"), (count, "pinned"), (count + 1000, "device"), (0, "pinned")):
        assert _checked_edit(ctx, m, mend[0], mend[1], cap=cap, kind=kind)[0] == count
        assert _checked_edit(ctx, m, cut[0], cut[1], cap=cap, kind=kind)[0] == count
    m.close()


def test_no_op_and_empty_edits(tw, ctx, tables):
    dims = (21, 17, 15)
    for rm in (0, 3):
        raw, _ = random_field(dims, 2, 1)
        p = post_params(tw.VoxelPostParams, dims, remove_unconnected=rm)
        m = ctx.voxel_model(p, tables, bx=4, by=4)
        m.build_launch(vals=raw)
        assert ctx.create_tiles_poll(wait=True)
        assert _checked_edit(ctx, m, [(3, 4, 2, 6, 5, 7), (0, 0, 0, 21, 1, 15)], [raw[4:9, 3:9, 2:9], raw[0:1, 0:21, 0:15]])[0] == 0
        for cap in (None, 0):
            count, job = _checked_edit(ctx, m, [], [], cap=cap)
            assert count == 0 and job.nchanged == 0 and not len(job.blocks)
        m.close()


@pytest.mark.parametrize("rm", [0, 3])
def test_odd_voxel_count_and_word_boundaries(tw, ctx, tables, rm):
    """5 x 7 x 9 = 315 voxels (9 words and 27 bits): boxes whose voxels straddle words 0 / 1 and run into the last, partial word."""
    dims = (5, 7, 9)
    raw, _ = random_field(dims, 9, 1)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=rm, make_closed_surface=0)
    m = ctx.voxel_model(p, tables, bx=2, by=3)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    for step, (box, val) in enumerate((((3, 0, 2, 2, 1, 7), 2.0), ((3, 0, 0, 2, 1, 9), -2.0), ((0, 6, 0, 5, 1, 9), 3.0), ((4, 6, 5, 1, 1, 4), -3.0),
                                       ((0, 0, 0, 5, 7, 9), 1.5))):
        x, y, z, w, h, d = box
        count, _ = _checked_edit(ctx, m, [box], [np.full((h, w, d), val, np.float32)], kind=("device", "pinned")[step % 2])
        assert count > 0
    for k, cap in enumerate((1, 31, 32, 33)):
        assert _checked_edit(ctx, m, [(0, 0, 0, 5, 7, 9)], [np.full((7, 5, 9), (-1.5, 2.5)[k % 2], np.float32)], cap=cap)[0] == 315
    m.close()


def test_list_without_vals_or_outside(tw, ctx, tables):
    dims = (24, 20, 16)
    raw, _ = random_field(dims, 4, 1)
    m = ctx.voxel_model(post_params(tw.VoxelPostParams, dims, remove_unconnected=3), tables, bx=8, by=8)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    rng = np.random.default_rng(12)
    _checked_edit(ctx, m, *_boxes(rng, dims), with_vals=False)
    _checked_edit(ctx, m, *_boxes(rng, dims), with_outside=False, kind="pinned")
    _checked_edit(ctx, m, *_boxes(rng, dims), with_vals=False, with_outside=False)
    m.close()


def test_list_with_an_overflowing_mesh(tw, ctx, tables):
    dims = (40, 33, 29)
    raw, _ = random_field(dims, 6, 1)
    m = ctx.voxel_model(post_params(tw.VoxelPostParams, dims, remove_unconnected=3), tables, bx=8, by=5)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    rng = np.random.default_rng(13)
    for kind in ("device", "pinned"):
        v, i = _mesh_bufs(kind, 5, 2)
        count, job = _checked_edit(ctx, m, [(10, 10, 5, 12, 12, 15)], [rng.choice(np.float32([-2.0, 2.5]), (12, 12, 15))], kind=kind, mesh=(v[:5], i[:2]))
        assert count > 0 and job.nverts > 5 and job.ntris > 2
        assert np.isnan(_np(v)[5:]).all()
    m.close()


# ---- refusals ----
def test_refusals(tw, ctx, tables):
    import torch
    dims = (12, 10, 8)
    raw, _ = random_field(dims, 3, 1)
    m = ctx.voxel_model(post_params(tw.VoxelPostParams, dims, remove_unconnected=1), tables, bx=4, by=4)
    m.build_launch(vals=raw)
    assert ctx.create_tiles_poll(wait=True)
    before = m.read()
    L = tw.lib
    box = (tw.VoxelBox * 1)(tw.VoxelBox(0, 0, 0, 2, 2, 2))
    vals = np.full(8, 5.0, np.float32)
    job = tw.VoxelModelJob(m.nblocks)
    out = job._out(None, None)
    n = C.c_uint64(77)
    pn = C.cast(C.pointer(n), C.c_void_p)
    di = torch.zeros(16, dtype=torch.int32, device="cuda")
    dv = torch.zeros(16, dtype=torch.float32, device="cuda")
    do = torch.zeros(16, dtype=torch.uint8, device="cuda")
    hi, hv, ho = np.zeros(16, np.uint32), np.zeros(16, np.float32), np.zeros(16, np.uint8)
    p = tw._ptr
    bad = [tw.VoxelChanges(p(di), p(dv), p(do), 16, None),           # no nchanged
           tw.VoxelChanges(None, None, None, 16, pn),                # a capacity without index
           tw.VoxelChanges(None, p(dv), None, 0, pn),                # vals without index
           tw.VoxelChanges(None, None, p(do), 0, pn),                # outside without index
           tw.VoxelChanges(p(hi), p(dv), p(do), 16, pn),             # pageable index
           tw.VoxelChanges(p(di), p(hv), p(do), 16, pn),             # pageable vals
           tw.VoxelChanges(p(di), p(dv), p(ho), 16, pn)]             # pageable outside
    for ch in bad:
        assert L.tw_voxel_model_edit_launch_ex(m._h, C.cast(box, C.c_void_p), 1, p(vals), C.byref(out), C.byref(ch)) == tw.TW_ERR_ARG
        assert ctx.create_tiles_poll(wait=True)              # nothing was enqueued
        assert n.value == 77
    after = m.read()
    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, after))
    # the edit's own refusals come first; a model job stays non-cancellable with a list
    ok = tw.VoxelChanges(p(di), p(dv), p(do), 16, pn)
    assert L.tw_voxel_model_edit_launch_ex(m._h, None, 1, p(vals), C.byref(out), C.byref(ok)) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_edit_launch_ex(m._h, C.cast(box, C.c_void_p), 1, p(vals), C.byref(out), C.byref(ok)) == tw.TW_OK
    with pytest.raises(tw.TwError) as e:
        ctx.cancel()
    assert e.value.status == tw.TW_ERR_STATE
    assert ctx.create_tiles_poll(wait=True) and n.value > 0
    m.close()
