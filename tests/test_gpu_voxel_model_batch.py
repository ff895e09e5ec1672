"""GPU: tw_voxel_model_build_batch_launch / tw_voxel_model_edit_batch_launch (Context.voxel_model_build_batch_launch / voxel_model_edit_batch_launch) -
many small voxel models built and edited in one job each.

Every batched model has a twin: a model created with the same arguments and driven by the single-model calls (build_launch / edit_launch with ctx=) on the
same context. After every job both are compared bit for bit: tw_voxel_model_read (raw field, field and flags), the block tables, the vertex and index
buffers with sentinels past their capacities, the counts, changed, and the change lists (capacities above and below their counts) with nchanged.
Covered: 64^3, 8x8x4096, 512x512x1, odd and 2x2x2 grids; remove_unconnected 0 / 1 / 3, keep_at_edge, centre_seed, invert, make_closed_surface,
skip_under_mesh with zix_xy; block sizes 1x1, odd and one block for the grid; every fill mode, host and device input fields; boxes at faces and corners,
overlapping boxes, a box that cuts ground off, entries without boxes; batches of 1, 7 and 300; ten random brush frames; batches on two shared contexts
interleaved with single-model edits and reads on a third; equal launch counts for 1 and 64 models; every refusal and tw_cancel."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_voxel_batch import _fill_spec
from test_voxel_flood_reference import post_params, random_field

pytestmark = pytest.mark.gpu
SENT = 0xDEADBEEF
EXTRA = 3


@pytest.fixture(scope="module")
def tables():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _field_spec(tw, dims, seed, kind="host", zix=False, **kw):
    vals, z = random_field(dims, seed, kw.get("centre_seed", 0))
    return {"vpp": post_params(tw.VoxelPostParams, dims, **kw), "vals": vals, "kind": kind, "zix": z if zix else None}


def _pair(ctx, spec, tables, bx=4, by=3):
    """(batched model, twin) of one spec, both on ctx."""
    z = spec.get("zix")
    return tuple(ctx.voxel_model(spec["vpp"], tables, zix_xy=z, bx=spec.get("bx", bx), by=spec.get("by", by)) for _ in range(2))


def _mesh(cap):
    """verts / indices buffers of cap + EXTRA rows filled with sentinels; the job gets the first cap rows (None for 0)."""
    import torch
    vc, tc = cap
    v = torch.full((vc + EXTRA, 3), float("nan"), dtype=torch.float32, device="cuda")
    i = torch.full((tc + EXTRA, 3), SENT - (1 << 32), dtype=torch.int32, device="cuda")
    return v, i, (v[:vc] if vc else None), (i[:tc] if tc else None)


def _list(cap, n):
    import torch
    i = torch.full((cap + EXTRA,), SENT - (1 << 32), dtype=torch.int32, device="cuda")
    v = torch.full((cap + EXTRA,), float("nan"), dtype=torch.float32, device="cuda")
    o = torch.full((cap + EXTRA,), 0xAB, dtype=torch.uint8, device="cuda")
    return (i, v, o), ((i[:cap], v[:cap], o[:cap]) if cap else (None, None, None))


def _vals(spec):
    import torch
    if spec.get("vals") is None:
        return None
    v = spec["vals"].copy()
    return torch.from_numpy(v).cuda() if spec.get("kind") == "device" else v


def _snap(m, job, bufs, lists):
    """Everything a job and its model give, as host arrays and ints."""
    raw, vals, outside = m.read()
    out = [raw.view(np.uint32), vals.view(np.uint32), outside, job.blocks.tobytes(), job.nverts, job.ntris, job.changed,
           bufs[0].cpu().numpy().view(np.uint32), bufs[1].cpu().numpy().view(np.uint32)]
    if lists is not None:
        out += [job.nchanged] + [b.cpu().numpy().view(np.uint8) for b in lists]
    return out


def _same(got, exp, what):
    for k, (a, b) in enumerate(zip(got, exp)):
        if isinstance(a, np.ndarray):
            assert a.shape == b.shape and np.array_equal(a, b), "%s: output %d differs" % (what, k)
        else:
            assert a == b, "%s: output %d differs (%r != %r)" % (what, k, a, b)


class Fleet:
    """Batched models and their twins on ctx, with per-model capacities; build() and edit() run a batch and the twins' single calls, then compare."""

    def __init__(self, ctx, specs, tables, caps=None):
        self.ctx, self.specs = ctx, specs
        self.pairs = [_pair(ctx, s, tables) for s in specs]
        self.caps = caps or [s.get("cap", (4000, 4000)) for s in specs]

    def build(self, batch_ctx=None):
        bc = batch_ctx or self.ctx
        runs = []
        for (a, b), s, cap in zip(self.pairs, self.specs, self.caps):
            runs.append([_mesh(cap) for _ in range(2)])
        builds = [{"model": a, "fill": s.get("fill"), "vals": _vals(s), "rdata": s.get("rdata"), "verts": r[0][2], "indices": r[0][3]}
                  for (a, _), s, r in zip(self.pairs, self.specs, runs)]
        jobs = bc.voxel_model_build_batch_launch(builds)
        assert bc.create_tiles_poll(wait=True)
        for i, ((a, b), s, r) in enumerate(zip(self.pairs, self.specs, runs)):
            tj = b.build_launch(fill=s.get("fill"), vals=_vals(s), rdata=s.get("rdata"), verts=r[1][2], indices=r[1][3], ctx=self.ctx)
            assert self.ctx.create_tiles_poll(wait=True)
            _same(_snap(a, jobs[i], r[0], None), _snap(b, tj, r[1], None), "build of model %d" % i)
        return jobs

    def edit(self, per_model, list_caps=None, batch_ctx=None):
        """per_model[i] = (boxes, values) or None (no boxes); list_caps[i] = None (no change list) or a capacity ('n': the voxel count)."""
        bc = batch_ctx or self.ctx
        list_caps = list_caps or [None] * len(self.pairs)
        runs, edits, lists = [], [], []
        for (a, b), e, cap, lc in zip(self.pairs, per_model, self.caps, list_caps):
            r = [_mesh(cap) for _ in range(2)]
            n = int(a.vpp.nx) * int(a.vpp.ny) * int(a.vpp.nz)
            ls = None if lc is None else [_list(n if lc == "n" else lc, n) for _ in range(2)]
            boxes, values = e if e is not None else ([], np.zeros(0, np.float32))
            edits.append({"model": a, "boxes": boxes, "values": values, "verts": r[0][2], "indices": r[0][3], "changes": None if ls is None else ls[0][1]})
            runs.append((r, boxes, values))
            lists.append(ls)
        jobs = bc.voxel_model_edit_batch_launch(edits)
        assert bc.create_tiles_poll(wait=True)
        for i, ((a, b), (r, boxes, values), ls) in enumerate(zip(self.pairs, runs, lists)):
            tj = b.edit_launch(boxes, values, verts=r[1][2], indices=r[1][3], changes=None if ls is None else ls[1][1], ctx=self.ctx)
            assert self.ctx.create_tiles_poll(wait=True)
            _same(_snap(a, jobs[i], r[0], None if ls is None else ls[0][0]), _snap(b, tj, r[1], None if ls is None else ls[1][0]), "edit of model %d" % i)
        return jobs


def _ball(rng, m, r=4, value=None):
    """A radius-r sphere brush at a random voxel of model m, clipped to the grid: ([box], values)."""
    dims = (int(m.vpp.nx), int(m.vpp.ny), int(m.vpp.nz))
    c = [int(rng.integers(0, d)) for d in dims]
    lo = [max(c[k] - r, 0) for k in range(3)]
    hi = [min(c[k] + r + 1, dims[k]) for k in range(3)]
    w, h, d = hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]
    raw, _, _ = m.read()
    vals = raw[lo[1]:hi[1], lo[0]:hi[0], lo[2]:hi[2]].copy()
    yy, xx, zz = np.meshgrid(np.arange(lo[1], hi[1]) - c[1], np.arange(lo[0], hi[0]) - c[0], np.arange(lo[2], hi[2]) - c[2], indexing="ij")
    v = value if value is not None else (1.0 if rng.random() < 0.5 else -2.0)
    vals[xx ** 2 + yy ** 2 + zz ** 2 <= r * r] = v
    return [(lo[0], lo[1], lo[2], w, h, d)], vals.ravel()


def _random_boxes(rng, m, k):
    dims = (int(m.vpp.nx), int(m.vpp.ny), int(m.vpp.nz))
    boxes = []
    for _ in range(k):
        lo = [int(rng.integers(0, d)) for d in dims]
        size = [int(rng.integers(1, max(2, min(d - l, 6)) + 1)) for d, l in zip(dims, lo)]
        size = [min(s, d - l) for s, d, l in zip(size, dims, lo)]
        boxes.append((lo[0], lo[1], lo[2], size[0], size[1], size[2]))
    vals = np.concatenate([rng.standard_normal(b[3] * b[4] * b[5]).astype(np.float32) for b in boxes])
    return boxes, vals


def _face_boxes(m):
    """Boxes at the grid's faces and corners, overlapping each other, with values that flip their voxels."""
    nx, ny, nz = int(m.vpp.nx), int(m.vpp.ny), int(m.vpp.nz)
    boxes = [(0, 0, 0, min(nx, 3), min(ny, 3), min(nz, 3)), (nx - min(nx, 2), ny - min(ny, 2), nz - min(nz, 2), min(nx, 2), min(ny, 2), min(nz, 2)),
             (0, 0, 0, nx, 1, nz), (0, 0, nz - 1, nx, ny, 1), (0, 0, 0, min(nx, 2), min(ny, 2), min(nz, 2))]
    vals = np.concatenate([np.linspace(-1.5, 1.5, b[3] * b[4] * b[5], dtype=np.float32) for b in boxes])
    return boxes, vals


def test_shapes_options_and_edits(tw, scene, ctx, tables):
    """The shapes of the 2^18-voxel limit and odd ones with every fill mode and option, built, edited at faces and corners with overlapping boxes and
    change lists above and below their counts, then three random brush frames."""
    specs = [_fill_spec(tw, scene, 1, (64, 64, 64)), _fill_spec(tw, scene, 2, (8, 8, 4096)), _fill_spec(tw, scene, 0, (512, 512, 1), remove_unconnected=1),
             _fill_spec(tw, scene, 0, (37, 23, 61), remove_unconnected=0), _fill_spec(tw, scene, 2, (2, 2, 2))]
    specs[0]["bx"], specs[0]["by"] = 64, 64                     # one block for the whole grid
    specs[3]["bx"], specs[3]["by"] = 1, 1
    specs[4]["bx"], specs[4]["by"] = 5, 7
    seed = 0
    for rm in (0, 1, 3):
        for cs, kae, sk, inv, mcs in ((1, 0, 0, 0, 0), (0, 1, 1, 1, 1), (0, 0, 1, 0, 1)):
            seed += 1
            specs.append(dict(_field_spec(tw, (13 + seed % 5, 11, 19 + seed % 7), seed, kind="device" if seed % 2 else "host", zix=bool(sk),
                                          remove_unconnected=rm, centre_seed=cs, keep_at_edge=kae, skip_under_mesh=sk, invert=inv, make_closed_surface=mcs),
                              bx=1 + seed % 5, by=2 + seed % 3))
    caps = [(4000, 4000) if k % 3 else (7, 5) for k in range(len(specs))]
    caps[1] = (0, 0)
    f = Fleet(ctx, specs, tables, caps)
    f.build()
    models = [a for a, _ in f.pairs]
    f.edit([_face_boxes(m) if k % 4 != 3 else None for k, m in enumerate(models)], list_caps=[["n", 5, None, 0][k % 4] for k in range(len(models))])
    rng = np.random.default_rng(5)
    for frame in range(3):
        f.edit([_ball(rng, m) for m in models], list_caps=["n" if frame % 2 == 0 else 3] * len(models))


def test_a_cut_that_floods_far(tw, ctx, tables):
    """A slab of inside ground on a thin stalk: a box that cuts the stalk turns the whole slab outside, far from the box."""
    nx, ny, nz = 20, 20, 24
    vals = np.full((ny, nx, nz), -1.0, np.float32)
    vals[:, :, 0:3] = 1.0                  # ground at the bottom (the centre seed's column reaches it through the stalk)
    vals[9:11, 9:11, 0:13] = 1.0           # stalk up to the centre voxel
    vals[:, :, 12:16] = 1.0                # slab around the centre
    vals[1:19, 1:19, 12:16] = 1.0
    spec = {"vpp": post_params(tw.VoxelPostParams, (nx, ny, nz), isolevel=0.0, remove_unconnected=3, centre_seed=1), "vals": vals, "kind": "host"}
    f = Fleet(ctx, [spec, dict(spec, kind="device")], tables)
    f.build()
    # the boxes as a numpy array of two rows, as VoxelModel.edit_launch takes them; the second overlaps the first
    cut = (np.array([(0, 0, 12, nx, ny, 4), (0, 0, 13, nx, ny, 2)], np.uint32), np.full(nx * ny * 6, -1.0, np.float32))
    jobs = f.edit([cut, cut], list_caps=["n", 10])
    assert jobs[0].nchanged > 100


@pytest.mark.parametrize("n", [1, 7, 300])
def test_batch_sizes(tw, scene, ctx, tables, n):
    specs = []
    for k in range(n):
        if k % 3 == 2:
            specs.append(_fill_spec(tw, scene, k % 3, (9 + k % 4, 10, 11 + k % 9), atten=k % 6))
        else:
            specs.append(_field_spec(tw, (6 + k % 5, 5 + k % 3, 7 + k % 11), k, kind="device" if k % 2 else "host", remove_unconnected=(0, 1, 3)[k % 3],
                                     centre_seed=1))
    f = Fleet(ctx, specs, tables)
    f.build()
    rng = np.random.default_rng(n)
    f.edit([_random_boxes(rng, a, 1 + k % 3) if k % 5 else None for k, (a, _) in enumerate(f.pairs)], list_caps=["n" if k % 2 else None for k in range(n)])


def test_ten_brush_frames(tw, scene, ctx, tables):
    """GLM rocks of 32^3 hit by random boxes for ten frames; a quarter of them hit in the odd frames."""
    specs = [_fill_spec(tw, scene, 1 + k % 2, (32, 32, 32)) for k in range(8)]
    f = Fleet(ctx, specs, tables)
    f.build()
    rng = np.random.default_rng(11)
    for frame in range(10):
        hit = [frame % 2 == 0 or k % 4 == 0 for k in range(len(specs))]
        f.edit([_random_boxes(rng, a, 1 + frame % 3) if h else None for (a, _), h in zip(f.pairs, hit)], list_caps=["n" if frame % 3 else 4] * len(specs))


def test_shared_contexts_interleaved(tw, scene, tables):
    """Batches on two shared contexts and single-model edits and reads on a third, on the same models, each launched while the others run (a launch
    completes only its own context's earlier job): the models' events order them. The twins run the same sequence one job at a time on the parent."""
    P = tw.Context(0)
    S = [P.shared() for _ in range(3)]
    specs = [_fill_spec(tw, scene, 1, (24, 20, 28)) for _ in range(3)]
    pairs = [_pair(P, s, tables) for s in specs]
    A, B = [a for a, _ in pairs], [b for _, b in pairs]
    keep = []
    big = lambda: _mesh((20000, 20000))  # noqa: E731
    bufs = [big() for _ in range(3)]
    keep.append(S[0].voxel_model_build_batch_launch([{"model": a, "fill": s["fill"], "verts": m[2], "indices": m[3]} for a, s, m in zip(A, specs, bufs)]))
    rng = np.random.default_rng(3)
    steps = [[_random_boxes(rng, A[0], 2) for _ in A] for _ in range(3)]
    single = _random_boxes(rng, A[1], 1)
    b1 = [big() for _ in A]
    keep.append(S[1].voxel_model_edit_batch_launch([{"model": a, "boxes": e[0], "values": e[1], "verts": m[2], "indices": m[3]} for a, e, m in zip(A, steps[0], b1)]))
    m2 = big()
    keep.append(A[1].edit_launch(single[0], single[1], verts=m2[2], indices=m2[3], ctx=S[2]))
    read_mid = A[1].read_launch(ctx=S[2])
    b2 = [big() for _ in A]
    keep.append(S[0].voxel_model_edit_batch_launch([{"model": a, "boxes": e[0], "values": e[1], "verts": m[2], "indices": m[3]} for a, e, m in zip(A, steps[1], b2)]))
    got_mid = read_mid.poll(wait=True)
    for c in (S[1], S[0]):
        assert c.create_tiles_poll(wait=True)
    # the twins, one job at a time on the parent
    for b, s in zip(B, specs):
        b.build_launch(fill=s["fill"], ctx=P)
        assert P.create_tiles_poll(wait=True)
    for k, (b, e) in enumerate(zip(B, steps[0])):
        b.edit_launch(e[0], e[1], ctx=P)
        assert P.create_tiles_poll(wait=True)
    B[1].edit_launch(single[0], single[1], ctx=P)
    assert P.create_tiles_poll(wait=True)
    mid = B[1].read()
    for g, e in zip(got_mid, mid):
        assert np.array_equal(np.asarray(g).view(np.uint8), e.view(np.uint8))
    tj = []
    for b, e in zip(B, steps[1]):
        m = big()
        tj.append((b.edit_launch(e[0], e[1], verts=m[2], indices=m[3], ctx=P), m))
        assert P.create_tiles_poll(wait=True)
    for a, b, j, (t, m), bb in zip(A, B, keep[3], tj, b2):
        _same(_snap(a, j, bb, None), _snap(b, t, m, None), "interleaved")
    P.close()


def test_launch_count_does_not_depend_on_n(tw, scene, ctx, tables):
    """The same options in every model (input fields, remove_unconnected 3, boxes in every edit), so both batches take the same steps."""
    mix = lambda k: _field_spec(tw, (9, 8, 10), k, kind="device" if k % 2 else "host", remove_unconnected=3, centre_seed=1)  # noqa: E731
    deltas = []
    for n in (1, 64):
        specs = [mix(k) for k in range(n)]
        models = [ctx.voxel_model(s["vpp"], tables, bx=3, by=3) for s in specs]
        c0 = ctx.launch_count
        ctx.voxel_model_build_batch_launch([{"model": m, "vals": _vals(s)} for m, s in zip(models, specs)])
        assert ctx.create_tiles_poll(wait=True)
        c1 = ctx.launch_count
        rng = np.random.default_rng(n)
        ctx.voxel_model_edit_batch_launch([dict(zip(("model", "boxes", "values"), (m,) + _random_boxes(rng, m, 2))) for m in models])
        assert ctx.create_tiles_poll(wait=True)
        deltas.append((c1 - c0, ctx.launch_count - c1))
        for m in models:
            m.close()
    assert deltas[0] == deltas[1], deltas


def test_refusals_leave_models_unchanged(tw, scene, ctx, tables):
    small = _field_spec(tw, (9, 8, 10), 1, remove_unconnected=3, centre_seed=1)
    a, b = _pair(ctx, small, tables)
    big = ctx.voxel_model(post_params(tw.VoxelPostParams, (65, 64, 64)), tables)
    never = ctx.voxel_model(small["vpp"], tables)
    other = tw.Context(0)
    foreign = other.voxel_model(small["vpp"], tables)
    ctx.voxel_model_build_batch_launch([{"model": a, "vals": small["vals"]}, {"model": b, "vals": small["vals"]}])
    assert ctx.create_tiles_poll(wait=True)
    before = [x.read() for x in (a, b)]
    L = tw.lib
    box = ([(0, 0, 0, 2, 2, 2)], np.zeros(8, np.float32))

    def edit(entries, status=tw.TW_ERR_ARG):
        with pytest.raises(tw.TwError) as ei:
            ctx.voxel_model_edit_batch_launch(entries)
        assert ei.value.status == status and "model %d" % (len(entries) - 1) in str(ei.value)

    def build(entries):
        with pytest.raises(tw.TwError) as ei:
            ctx.voxel_model_build_batch_launch(entries)
        assert ei.value.status == tw.TW_ERR_ARG and "model %d" % (len(entries) - 1) in str(ei.value)

    e = lambda m, bx=box: {"model": m, "boxes": bx[0], "values": bx[1]}  # noqa: E731
    build([{"model": a, "vals": small["vals"]}, {"model": big, "vals": np.zeros((64, 65, 64), np.float32)}])
    build([{"model": a, "vals": small["vals"]}, {"model": a, "vals": small["vals"]}])
    build([{"model": a, "vals": small["vals"]}, {"model": foreign, "vals": small["vals"]}])
    build([{"model": a, "vals": small["vals"], "fill": _fill_spec(tw, scene, 1, (9, 8, 10))["fill"]}])
    build([{"model": a}])
    build([{"model": a, "fill": _fill_spec(tw, scene, 1, (9, 8, 11))["fill"]}])
    edit([e(a), e(never)], tw.TW_ERR_STATE)
    edit([e(a), e(b), e(a)])
    edit([e(a), e(foreign)])
    edit([e(a), e(b, ([(8, 0, 0, 2, 1, 1)], np.zeros(2, np.float32)))])
    edit([e(a), e(b, ([(0, 0, 0, 0, 1, 1)], np.zeros(0, np.float32)))])
    edit([e(a), e(big)])
    # NULL arrays, n == 0, NULL outputs and a capacity without a buffer, through the C ABI
    assert L.tw_voxel_model_build_batch_launch(ctx._h, None, 1) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_edit_batch_launch(ctx._h, None, 1) == tw.TW_ERR_ARG
    assert L.tw_voxel_model_edit_batch_launch(ctx._h, (tw.VoxelModelEdit * 1)(), 0) == tw.TW_ERR_ARG
    es = (tw.VoxelModelEdit * 1)(tw.VoxelModelEdit(a._h, None, 0, None, None, None))
    assert L.tw_voxel_model_edit_batch_launch(ctx._h, es, 1) == tw.TW_ERR_ARG
    assert b"model 0" in L.tw_last_error(ctx._h)
    n = C.c_uint64(0)
    ch = tw.VoxelChanges(None, None, None, 5, C.cast(C.pointer(n), C.c_void_p))
    job = tw.VoxelModelJob(a.nblocks)
    out = job._out(None, None)
    es = (tw.VoxelModelEdit * 2)(tw.VoxelModelEdit(a._h, None, 0, None, C.cast(C.pointer(out), C.c_void_p), None),
                                 tw.VoxelModelEdit(b._h, None, 0, None, C.cast(C.pointer(out), C.c_void_p), C.cast(C.pointer(ch), C.c_void_p)))
    assert L.tw_voxel_model_edit_batch_launch(ctx._h, es, 2) == tw.TW_ERR_ARG
    assert b"model 1" in L.tw_last_error(ctx._h)
    es = (tw.VoxelModelEdit * 1)(tw.VoxelModelEdit(never._h, None, 0, None, C.cast(C.pointer(out), C.c_void_p), None))
    assert L.tw_voxel_model_edit_batch_launch(ctx._h, es, 1) == tw.TW_ERR_STATE
    for x, r in zip((a, b), before):
        for g, w in zip(x.read(), r):
            assert np.array_equal(g.view(np.uint8), w.view(np.uint8))
    # a batch job cannot be cancelled
    ctx.voxel_model_edit_batch_launch([e(a), e(b)])
    assert L.tw_cancel(ctx._h) == tw.TW_ERR_STATE
    assert ctx.create_tiles_poll(wait=True)
    other.close()
