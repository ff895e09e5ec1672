"""GPU: voxel model jobs on any context of the model's family (tw_voxel_model_build_launch_on / edit_launch_on / read_launch; VoxelModel's ctx=).

A script of a build, brush edits (with change lists of capacities above and below their counts) and reads runs on a model through its own context alone,
then on fresh models of the same grid spread round-robin over the parent and three shared contexts: one job at a time; four jobs on four contexts before
any poll, polled newest first; and with a tile frame launched on the next context after every model job, so the frames complete model jobs and the model
jobs complete frames. Every block table, count, vertex, index, change list and read must equal the owner-only script's, bit for bit, on 128^3 and 256^3
GLM terrains with several block sizes and remove_unconnected 0 and 3. Also: a read between two edits sees the first only; box reads equal slices of
tw_voxel_model_read, into device, page-locked and pageable memory; a change list that overflows followed by read_launch restores the host mirror;
tw_voxel_model_destroy, tw_destroy(shared) and tw_destroy(parent) with model jobs in flight on other contexts; refusals."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_shared_ctx import _cfg
from test_gpu_tiles_shading import ZV, ITERS, _host, _origins
from test_gpu_voxel_build import _post_for, _scfg

pytestmark = pytest.mark.gpu
R = 6


@pytest.fixture(scope="module")
def tables():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _family(tw, scene, nshared=3):
    """A parent Context with the tile frames' sine params, and nshared shared Contexts of it."""
    P = tw.Context(0)
    P.set_sine_params(_cfg(scene, 0).sine_params())
    return P, [P.shared() for _ in range(nshared)]


def _grid(tw, scene, n, rm):
    vp = scene.voxel_landscape_params(_scfg(scene, 1), n, n, n, z_gradient=-2.0)
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=rm, centre_seed=0, skip_under_mesh=1)
    zix = np.random.default_rng(7).integers(n // 16, n // 4, (n, n)).astype(np.uint32)
    return vp, p, zix


def _brush(rng, raw, flags, k):
    """A ball of radius R around the first outside voxel of a random column, +1 (inside) for even k, -2 (outside) for odd k: (box, values)."""
    n = raw.shape[0]
    x, y = (int(v) for v in rng.integers(R, n - R, 2))
    col = flags[y, x]
    z = min(max(int(np.argmax(col == 1)) if (col == 1).any() else n // 2, R), n - R - 1)
    box = raw[y - R:y + R + 1, x - R:x + R + 1, z - R:z + R + 1].copy()
    yy, xx, zz = np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="ij")
    box[xx ** 2 + yy ** 2 + zz ** 2 <= R * R] = 1.0 if k % 2 == 0 else -2.0
    return (x - R, y - R, z - R, 2 * R + 1, 2 * R + 1, 2 * R + 1), box


def _script(raw, flags, nedits, seed):
    """[("build",), ("edit", boxes, values, capacity), ("read", boxes, kind)...]: capacities alternate between the grid's voxels and 5; a read of the
    whole grid after the second edit, box reads after the fourth and at the end, and a whole read at the end."""
    rng = np.random.default_rng(seed)
    steps = [("build",)]
    for k in range(nedits):
        box, vals = _brush(rng, raw, flags, k)
        boxes, values = [box], [vals]
        if k == 2:                                                    # two boxes, the second overlapping the first
            x, y, z, w, h, d = box
            boxes.append((x + 3, y + 3, z + 3, 4, 4, 4))
            values.append(np.full((4, 4, 4), -1.5, np.float32))
        steps.append(("edit", boxes, np.concatenate([v.ravel() for v in values]), None if k % 2 == 0 else 5))
        if k == 1:
            steps.append(("read", None, "pageable"))
        if k == 3:
            steps.append(("read", [box, (0, 0, 0, 3, 2, raw.shape[2])], "device"))
    steps.append(("read", [steps[1][1][0]], "pinned"))
    steps.append(("read", None, "device"))
    return steps


def _buf(kind, shape, dt):
    import torch
    if kind == "device":
        return torch.empty(shape, dtype=dt, device="cuda")
    t = torch.empty(shape, dtype=dt)
    return t.pin_memory() if kind == "pinned" else t.numpy()


class _Launch:
    """One step launched on c; result() (after its job completed) is everything it produced, as bytes."""

    def __init__(self, tw, m, c, step, vp, caps):
        import torch
        self.step, n = step, int(m.vpp.nx) * int(m.vpp.ny) * int(m.vpp.nz)
        if step[0] in ("build", "edit"):
            self.v = torch.full((caps[0], 3), float("nan"), device="cuda")
            self.i = torch.full((caps[1], 3), -1, dtype=torch.int32, device="cuda")
        if step[0] == "build":
            self.job = m.build_launch(fill=vp, verts=self.v, indices=self.i, ctx=c)
        elif step[0] == "edit":
            cap = n if step[3] is None else step[3]
            self.ch = (torch.full((cap,), -1, dtype=torch.int32, device="cuda"), torch.full((cap,), float("nan"), device="cuda"),
                       torch.full((cap,), 0xAB, dtype=torch.uint8, device="cuda"))
            self.job = m.edit_launch(step[1], step[2], verts=self.v, indices=self.i, changes=self.ch, ctx=c)
        else:
            boxes, kind = step[1], step[2]
            size = (int(m.vpp.ny), int(m.vpp.nx), int(m.vpp.nz)) if boxes is None else (sum(b[3] * b[4] * b[5] for b in boxes),)
            self.out = (_buf(kind, size, torch.float32), _buf(kind, size, torch.float32), _buf(kind, size, torch.uint8))
            self.job = m.read_launch(boxes, *self.out, ctx=c)

    def result(self):
        j = self.job
        if self.step[0] == "read":
            return [np.ascontiguousarray(_host(a)).tobytes() for a in self.out]
        r = [j.blocks.tobytes(), j.nverts, j.ntris, j.changed, _host(self.v)[:j.nverts].tobytes(), _host(self.i)[:j.ntris].tobytes()]
        if self.step[0] == "edit":
            k = min(j.nchanged, int(self.ch[0].numel())) + 16                     # the listed entries and a few untouched ones past them
            r += [j.nchanged] + [np.ascontiguousarray(_host(a[:k])).tobytes() for a in self.ch]
        return r


def _frame(tw, cfg, c):
    """A 4-tile frame (tw_create_tiles_launch_ex) on c: (zvals, mm) once it completes."""
    import torch
    hp, ep = cfg.height_params(), cfg.erosion_params()
    z, mm = torch.empty((4, ZV, ZV), device="cuda"), np.empty((4, 2), np.float32)
    c.create_tiles_launch(_origins(2), cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), ZV, hp, ITERS, ep, ep.zmin, z, mm=mm)
    return z, mm


def _run(tw, scene, m, ctxs, steps, vp, caps, group=1, frames=False):
    """The steps launched on ctxs round-robin, group launches at a time, each group's contexts then polled newest first. With frames, a tile frame is
    launched on each context right after its model job, so the frame's launch completes the model job and the context's next model launch completes the
    frame; every frame's output must equal the first's."""
    out, pend, fr, done = [None] * len(steps), [], {}, []
    cfg = _cfg(scene, 0)
    for k, st in enumerate(steps):
        c = ctxs[k % len(ctxs)]
        L = _Launch(tw, m, c, st, vp, caps)
        if frames:
            if id(c) in fr:
                done.append(fr.pop(id(c)))
            fr[id(c)] = _frame(tw, cfg, c)
            out[k] = L.result()
            continue
        pend.append((k, c, L))
        if len(pend) == group:
            for j, cc, LL in reversed(pend):
                assert cc.create_tiles_poll(wait=True)
                out[j] = LL.result()
            pend = []
    for j, cc, LL in reversed(pend):
        assert cc.create_tiles_poll(wait=True)
        out[j] = LL.result()
    for cc in ctxs:
        assert cc.create_tiles_poll(wait=True)
    snaps = [(_host(z).tobytes(), mm.tobytes()) for z, mm in done + list(fr.values())]
    assert all(x == snaps[0] for x in snaps)
    return out


def _prepare(tw, scene, P, tables, n, rm, bs):
    """The grid, a probe build's mesh capacities, and the script (its brushes placed on the built field)."""
    vp, p, zix = _grid(tw, scene, n, rm)
    m = P.voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
    probe = m.build_launch(fill=vp)
    assert P.create_tiles_poll(wait=True)
    raw, _, flags = m.read()
    m.close()
    return vp, p, zix, (probe.nverts + 16, probe.ntris + 16), _script(raw, flags, 5, n + rm)


CASES = [(128, 0, (16, 16)), (128, 3, (32, 8)), (128, 3, (127, 127)), (256, 0, (32, 32)), (256, 3, (64, 16))]


@pytest.mark.parametrize("n,rm,bs", CASES)
def test_scripts_across_the_family(tw, scene, tables, n, rm, bs):
    P, shared = _family(tw, scene)
    try:
        vp, p, zix, caps, steps = _prepare(tw, scene, P, tables, n, rm, bs)
        fam = [P] + shared

        def run(ctxs, **kw):
            m = P.voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
            r = _run(tw, scene, m, ctxs, steps, vp, caps, **kw)
            m.close()
            return r

        exp = run([P])
        edits = [r for s, r in zip(steps, exp) if s[0] == "edit"]
        assert any(r[6] > 5 for r in edits) and all(r[6] > 0 for r in edits)     # some lists overflow capacity 5; the others hold everything
        for kw in ({}, {"group": 4}, {"frames": True}):
            got = run(fam, **kw)
            for s, a, b in zip(steps, exp, got):
                assert a == b, (s[0], kw)
        # a model created on a shared context, driven from the parent and the other shared contexts
        m = shared[1].voxel_model(p, tables, zix_xy=zix, bx=bs[0], by=bs[1])
        got = _run(tw, scene, m, [shared[1], P, shared[0], shared[2]], steps, vp, caps, group=4)
        assert got == exp
        m.close()
    finally:
        P.close()


def test_reads_see_exactly_the_jobs_before_them(tw, scene, tables):
    import torch
    P, shared = _family(tw, scene)
    try:
        vp, p, zix = _grid(tw, scene, 128, 3)
        m = P.voxel_model(p, tables, zix_xy=zix, bx=32, by=32)
        m.build_launch(fill=vp, ctx=shared[0])
        raw0, v0, o0 = m.read_launch(ctx=shared[1]).poll(wait=True)
        rng = np.random.default_rng(3)
        n, expect = v0.size, raw0.copy()
        for k in range(4):
            box, vals = _brush(rng, raw0, o0, k)
            box2, vals2 = _brush(rng, raw0, o0, k + 1)
            c1, c2, c3 = shared[k % 3], shared[(k + 1) % 3], P
            m.edit_launch([box], vals, ctx=c1)                                       # edit k
            rd = m.read_launch(ctx=c2)                                               # between edits k and k + 1
            small = (torch.empty(4, dtype=torch.int32).pin_memory(), None, None)
            ej = m.edit_launch([box2], vals2, changes=small, ctx=c3)                 # edit k + 1, a list of capacity 4
            assert c3.create_tiles_poll(wait=True) and c1.create_tiles_poll(wait=True)
            a_raw, a_v, a_o = rd.poll(wait=True)
            r1, v1, o1 = m.read()
            # the read has edit k and not edit k + 1
            for (x, y, z, w, h, d), vv, seen in ((box, vals, a_raw), (box2, vals2, r1)):
                expect[y:y + h, x:x + w, z:z + d] = vv
                assert np.array_equal(seen.view(np.uint32), expect.view(np.uint32))
            # box reads equal slices of tw_voxel_model_read, into each kind of memory
            for kind in ("device", "pinned", "pageable"):
                t = sum(b[3] * b[4] * b[5] for b in (box, box2))
                bufs = (_buf(kind, (t,), torch.float32), _buf(kind, (t,), torch.float32), _buf(kind, (t,), torch.uint8))
                br, bv, bo = (np.ascontiguousarray(_host(a)) for a in m.read_launch([box, box2], *bufs, ctx=shared[2]).poll(wait=True))
                exp = [np.concatenate([a[b[1]:b[1] + b[4], b[0]:b[0] + b[3], b[2]:b[2] + b[5]].ravel() for b in (box, box2)]) for a in (r1, v1, o1)]
                assert np.array_equal(br.view(np.uint32), exp[0].view(np.uint32)) and np.array_equal(bv.view(np.uint32), exp[1].view(np.uint32))
                assert np.array_equal(bo, exp[2])
            # the host mirror: edit k + 1 overflowed its list, so read_launch replaces it
            assert ej.nchanged > 4
            _, mirror_v, mirror_o = m.read_launch(raw=False, ctx=shared[(k + 2) % 3]).poll(wait=True)
            assert np.array_equal(mirror_v.view(np.uint32), v1.view(np.uint32)) and np.array_equal(mirror_o, o1) and mirror_v.size == n
            raw0 = r1
        m.close()
    finally:
        P.close()


def _snapshot(m):
    r, v, o = m.read()
    return r.tobytes(), v.tobytes(), o.tobytes()


def _scrub(nbytes):
    """Fresh device memory of nbytes filled with NaN bits: after a model is freed it is likely to take the model's pages, so a job still reading them
    would read NaN."""
    import torch
    t = torch.full((nbytes // 4,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("what", ["model", "shared", "parent"])
def test_destroy_with_model_jobs_in_flight(tw, scene, tables, what):
    """Edits and device reads in flight on shared contexts, none on the model's own context, when the model, a shared context or the parent is
    destroyed: the destroy must wait for their device work on the model, so every read still holds the field with all the edits."""
    import torch
    P, shared = _family(tw, scene, 5)
    n = 256
    vp, p, zix = _grid(tw, scene, n, 3)
    rng = np.random.default_rng(5)
    m = P.voxel_model(p, tables, zix_xy=zix, bx=32, by=32)
    m.build_launch(fill=vp)
    raw, _, flags = m.read()                                      # the owner context has nothing pending from here on
    expect = raw.copy()
    for k in range(3):
        (x, y, z, w, h, d), vals = _brush(rng, raw, flags, k)
        m.edit_launch([(x, y, z, w, h, d)], vals, ctx=shared[k])
        expect[y:y + h, x:x + w, z:z + d] = vals
    reads = [m.read_launch(raw=torch.empty(raw.shape, device="cuda"), vals=False, outside=False, ctx=c) for c in shared[3:]]

    def check_reads():
        for r in reads:
            assert np.array_equal(_host(r.out[0]).view(np.uint32), expect.view(np.uint32))

    if what == "model":
        m.close()                                                 # returns once the edits and reads on the shared contexts are done with the model
        scrub = _scrub(15 * n ** 3)
        check_reads()
        for c in [P] + shared:
            assert c.create_tiles_poll(wait=True)
        del scrub
        # a fresh model on the same contexts still matches the owner-only script
        vp2, p2, zix2, caps, steps = _prepare(tw, scene, P, tables, 128, 3, (16, 16))
        m1 = P.voxel_model(p2, tables, zix_xy=zix2, bx=16, by=16)
        exp = _run(tw, scene, m1, [P], steps, vp2, caps)
        m1.close()
        m2 = P.voxel_model(p2, tables, zix_xy=zix2, bx=16, by=16)
        assert _run(tw, scene, m2, [P] + shared[:3], steps, vp2, caps, group=4) == exp
        m2.close()
        P.close()
    elif what == "shared":
        shared[3].close()                                         # completes its read, which waited for the three edits
        assert np.array_equal(_host(reads[0].out[0]).view(np.uint32), expect.view(np.uint32))
        for c in [P] + shared[:3] + shared[4:]:
            assert c.create_tiles_poll(wait=True)
        check_reads()
        box, vals = _brush(rng, raw, flags, 3)
        m.edit_launch([box], vals, ctx=shared[2])                 # the model and the other contexts still work
        assert shared[2].create_tiles_poll(wait=True)
        x, y, z, w, h, d = box
        assert np.array_equal(m.read()[0][y:y + h, x:x + w, z:z + d].view(np.uint32), vals.view(np.uint32))
        P.close()
    else:
        P.close()                                                 # destroys the model, then the shared contexts
        scrub = _scrub(15 * n ** 3)
        check_reads()
        del scrub


def test_refusals(tw, scene, tables):
    P, shared = _family(tw, scene, 1)
    Q = tw.Context(0)
    try:
        vp, p, zix = _grid(tw, scene, 128, 0)
        m = P.voxel_model(p, tables, zix_xy=zix, bx=32, by=32)
        with pytest.raises(tw.TwError) as e:
            m.read_launch(ctx=shared[0])                          # before the first build
        assert e.value.status == tw.TW_ERR_STATE
        with pytest.raises(tw.TwError) as e:
            m.edit_launch([(0, 0, 0, 1, 1, 1)], np.zeros(1, np.float32), ctx=shared[0])
        assert e.value.status == tw.TW_ERR_STATE
        m.build_launch(fill=vp, ctx=shared[0])
        with pytest.raises(tw.TwError) as e:
            shared[0].cancel()
        assert e.value.status == tw.TW_ERR_STATE
        assert shared[0].create_tiles_poll(wait=True)
        before = _snapshot(m)
        Q2 = Q.shared()
        for c in (Q, Q2):                                         # another family: refused, nothing changes
            for launch in (lambda: m.build_launch(fill=vp, ctx=c), lambda: m.edit_launch([(0, 0, 0, 2, 2, 2)], np.full(8, 5.0, np.float32), ctx=c),
                           lambda: m.read_launch(ctx=c)):
                with pytest.raises(tw.TwError) as e:
                    launch()
                assert e.value.status == tw.TW_ERR_ARG
            assert c.create_tiles_poll(wait=True)
        assert _snapshot(m) == before
        for boxes in ([(0, 0, 0, 0, 1, 1)], [(127, 0, 0, 2, 1, 1)], [(0, 0, 127, 1, 1, 2)]):
            with pytest.raises(tw.TwError) as e:
                m.read_launch(boxes, ctx=shared[0])
            assert e.value.status == tw.TW_ERR_ARG
        L, f = tw.lib, C.c_float(0)
        assert L.tw_voxel_model_read_launch(shared[0]._h, m._h, None, 1, C.byref(f), None, None) == tw.TW_ERR_ARG
        job = m.read_launch([(1, 2, 3, 1, 1, 1)], ctx=shared[0])
        with pytest.raises(tw.TwError) as e:
            shared[0].cancel()
        assert e.value.status == tw.TW_ERR_STATE
        r, v, o = job.poll(wait=True)
        rr, vv, oo = m.read()
        assert r[0] == rr[2, 1, 3] and v[0] == vv[2, 1, 3] and o[0] == oo[2, 1, 3]
        m.close()
    finally:
        Q.close()
        P.close()
