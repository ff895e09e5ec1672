"""GPU: frame launches into a tile set (tw_tile_set_create_tiles_launch). Every scenario runs the new launch on one set and, on a second set in the same state,
the sequence it replaces - tw_tile_set_remove, the tile job (tw_create_tiles_launch_ex / _hmap), a completing poll, tw_tile_set_put of the job's zvals,
tw_tile_set_shadows_launch and its poll - and requires every output of the job and of the relight, the recomputed flags, tw_last_erosion_steps() and the sets'
later behaviour (stale, follow-up relights with the sun moved and not moved) to agree bit for bit; the final relights are also checked against
tw_tile_shadows_batch_ex over all resident tiles, the set's own contract."""
import ctypes as C

import numpy as np
import pytest

from cases import HM_CFG
from test_weights_host import weight_cases

pytestmark = pytest.mark.gpu

S, ZV = 32, 34
SUN, SUN2, MOON = (3.0, 2.0, 0.15), (2.0, 3.5, 0.2), (-2.0, -3.0, 0.2)   # the sun lights from +x / +y: new rows at larger y are on its side
CASES = {"m0": (0, False, False), "m1": (1, False, False), "m1_ao": (1, True, False), "m4": (4, False, False), "m4_ao": (4, True, False),
         "hmap": (4, False, True)}


class Job:
    """One scene: the job's arguments without the tiles."""

    def __init__(self, tw, scene, ctx, case, iters):
        mode, self.ao, self.hmap = CASES[case]
        self.cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1),
                                     scene_size=(0.5, 0.5, 4.0))
        ctx.set_sine_params(self.cfg.sine_params())               # the weights texture's jitter noise
        self.hp, self.ep, self.iters = self.cfg.height_params(), self.cfg.erosion_params(), iters
        self.dx, self.dy = float(self.cfg.dx_val), float(self.cfg.dy_val)
        self.wp = weight_cases(tw.WeightParams, np.random.default_rng(7), -1.0, 1.5, S, self.dx, self.dy)[3]
        self.hs = tw.HmapSampler(257, 300, 2, 1.0, 0.0012, 1.7, -0.3, 0.8) if self.hmap else None
        self.tw = tw

    def light(self, lp):
        sp = self.tw.ShadowParams()
        sp.x_scene_size = sp.y_scene_size = 0.5
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = self.dx, self.dy, 1.0 / np.float32(self.dx), 1.0 / np.float32(self.dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, float(self.ep.zmin), float(self.ep.zmax), 0
        sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp
        return sp


def _alloc(where, shape, dtype):
    import torch
    t = {"u1": torch.uint8, "f4": torch.float32}[dtype]
    if where == "host":
        return np.empty(shape, {"u1": np.uint8, "f4": np.float32}[dtype])
    if where == "pinned":
        return torch.empty(shape, dtype=t).pin_memory()
    return torch.empty(shape, dtype=t, device="cuda")


def _host(a):
    if a is None:
        return None
    if hasattr(a, "cpu"):
        return a.cpu().numpy().copy()
    if isinstance(a, np.ndarray):
        return a.copy()
    return np.frombuffer(bytes(a), np.uint8).copy()                # ctypes arrays (tile bounds)


def _bytes_equal(a, b):
    return a is None and b is None or (a is not None and b is not None and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                                                         np.ascontiguousarray(b).view(np.uint8)))


def _outputs(tw, job, nt, where, zvals=True):
    w = "host" if where == "host" else ("pinned" if where == "pinned" else "device")
    o = {"zvals": _alloc(w, (nt, ZV, ZV), "f4") if zvals else None, "mm": np.empty((nt, 2), np.float32), "bounds": (tw.TileBounds * nt)(),
         "normals": _alloc(w, (nt, ZV - 1, ZV - 1, 4), "u1"), "min_normal_z": np.empty(nt, np.float32),
         "weights": _alloc(w, (nt, ZV - 1, ZV - 1, 4), "u1"), "has_any_grass": np.empty(nt, np.uint8)}
    if job.ao:
        o["ao"] = _alloc(w, (nt, ZV - 1, ZV - 1), "u1")
    return o


def _kw(job, o, nt):
    tp = np.random.default_rng(nt).uniform(-0.2, 1.3, (nt, 8)).astype(np.float32)
    return dict(o, wpz_max=0.1, size=S, half_dxy=0.0625 if job.ao else None, wp=job.wp, tile_params=tp, hmap=job.hs)


def _origins(keys, shift=0):
    return [(x * S + shift, y * S + 9000) for x, y in keys]


def _lights(tw, job, lps, n, where):
    w = "device" if where == "nozvals" else where
    return [tw.Light(job.light(lp), _alloc(w, (n, ZV, ZV), "u1"), _alloc(w, (n, ZV), "f4"), _alloc(w, (n, ZV), "f4")) for lp in lps]


def _louts(lights):
    return [(_host(L.smask), _host(L.sh_out_x), _host(L.sh_out_y)) for L in lights]


def sequence(tw, ctx, ts, job, keys, origins, remove, relight, lps, where):
    """The calls a frame launch replaces, on ts's own context: (job outputs, erosion steps, recomputed, relight outputs)."""
    if remove:
        ts.remove(remove)
    o = _outputs(tw, job, len(keys), "pinned" if where == "nozvals" else where)
    ctx.create_tiles_launch(origins, job.cfg.mesh_size, job.dx, job.dy, ZV, job.hp, job.iters, job.ep, job.ep.zmin, **_kw(job, o, len(keys)))
    assert ctx.create_tiles_poll(wait=True)
    steps = ctx.last_erosion_steps
    ts.put(keys, o["zvals"])
    rec, louts = None, None
    if relight:
        lights = _lights(tw, job, lps, len(relight), where)
        rec = ts.shadows_launch(np.array(relight, np.int32), lights)
        assert ctx.create_tiles_poll(wait=True)
        louts = _louts(lights)
    return {k: _host(v) for k, v in o.items()}, steps, rec, louts


def frame_launch(tw, lctx, ts, job, keys, origins, remove, relight, lps, where):
    """The frame launch on lctx, not polled: (outputs, lights, recomputed)."""
    o = _outputs(tw, job, len(keys), where, zvals=(where != "nozvals"))
    lights = _lights(tw, job, lps, len(relight), where) if relight else None
    rec = ts.create_tiles_launch(origins, job.cfg.mesh_size, job.dx, job.dy, job.hp, job.iters, job.ep, job.ep.zmin, keys, remove_xy=remove or None,
                                 relight_xy=relight or None, lights=lights, ctx=lctx, **_kw(job, o, len(keys)))
    return o, lights, rec


def check_frame(got, want):
    (o, lights, rec, steps), (wo, wsteps, wrec, wlouts) = got, want
    for k, v in o.items():
        if v is None:
            continue
        assert _bytes_equal(_host(v), wo[k]), k
    assert steps == wsteps
    assert (rec is None) == (wrec is None)
    if rec is not None:
        assert np.array_equal(rec, wrec)
        for a, b in zip(_louts(lights), wlouts):
            assert all(_bytes_equal(x, y) for x, y in zip(a, b))


def full(tw, ctx, ts_keys_z, sp):
    keys = sorted(ts_keys_z)
    z = np.ascontiguousarray(np.stack([ts_keys_z[k] for k in keys]))
    txy = np.array(keys, np.int32)
    nt = len(keys)
    m, ox, oy = np.empty((nt, ZV, ZV), np.uint8), np.empty((nt, ZV), np.float32), np.empty((nt, ZV), np.float32)
    ctx._check(tw.lib.tw_tile_shadows_batch_ex(ctx._h, tw._ptr(z), tw._ptr(txy), nt, ZV, C.byref(sp), None, None, tw._ptr(m), tw._ptr(ox), tw._ptr(oy)))
    return {k: (m[i], ox[i], oy[i]) for i, k in enumerate(keys)}


def follow_ups(tw, ctx, job, sets, resident_z, check_full):
    """After the frames: stale agrees, and relights of every resident tile with the lights unchanged and with the sun moved agree on both sets."""
    keys = sorted(resident_z)
    for lps in ((SUN, MOON), (SUN2, MOON)):
        sps = [job.light(lp) for lp in lps]
        stales = [ts.stale(sps) for ts in sets]
        assert np.array_equal(stales[0], stales[1])
        res = []
        for ts in sets:
            lights = _lights(tw, job, lps, len(keys), "pinned")
            rec = ts.shadows_launch(np.array(keys, np.int32), lights)
            assert ts.ctx.create_tiles_poll(wait=True)
            res.append((rec, _louts(lights)))
        assert np.array_equal(res[0][0], res[1][0])
        for a, b in zip(res[0][1], res[1][1]):
            assert all(_bytes_equal(x, y) for x, y in zip(a, b))
        if check_full:
            for sp, (m, ox, oy) in zip(sps, res[0][1]):
                ref = full(tw, ctx, resident_z, sp)
                for i, k in enumerate(keys):
                    assert np.array_equal(m[i], ref[k][0]) and _bytes_equal(ox[i], ref[k][1]) and _bytes_equal(oy[i], ref[k][2]), k
    return res


@pytest.fixture
def heightmap(ctx):
    img = np.random.default_rng(257).integers(0, 256, (300, 257, 2), dtype=np.uint8)
    ctx.set_heightmap(img)
    yield
    ctx.set_heightmap(None)


def _rows(y0, y1, x0=0, x1=4):
    return [(x, y) for y in range(y0, y1) for x in range(x0, x1)]


@pytest.mark.parametrize("where", ["host", "pinned", "device", "nozvals"])
@pytest.mark.parametrize("iters", [100, 0])
@pytest.mark.parametrize("case", list(CASES))
def test_frames_equal_the_sequence(tw, scene, ctx, heightmap, case, iters, where):
    """Four frames: the first into an empty set (4 x 4 tiles), a row on the sun's side (its downstream closure relit, slab growth inside the launch), an evicted
    far row plus a new light-side row relit with one light of two slots, then the far row back plus a re-put of a resident tile with other heights."""
    job = Job(tw, scene, ctx, case, iters)
    ts_new, ts_ref = ctx.tile_set(ZV, 2), ctx.tile_set(ZV, 2)
    resident = {}
    try:
        frames = [(_rows(0, 4), [], "all", (SUN, MOON)), (_rows(4, 5), [], "after", (SUN, MOON)), (_rows(5, 6), _rows(0, 1), "after", (SUN,)),
                  (_rows(0, 1) + [(1, 2)], [], "after", (SUN, MOON))]
        for keys, remove, which, lps in frames:
            origins = _origins(keys[:4]) + _origins(keys[4:], shift=17 * S)      # the re-put tile gets other heights
            sps = [job.light(lp) for lp in lps]
            relight = sorted(set(resident) - set(remove) | set(keys)) if which == "all" else [tuple(t) for t in ts_ref.stale_after(sps, remove, keys)]
            assert [tuple(t) for t in ts_new.stale_after(sps, remove, keys)] == [tuple(t) for t in ts_ref.stale_after(sps, remove, keys)]
            assert set(keys) <= set(relight)
            want = sequence(tw, ctx, ts_ref, job, keys, origins, remove, relight, lps, where)
            o, lights, rec = frame_launch(tw, ctx, ts_new, job, keys, origins, remove, relight, lps, where)
            assert ctx.create_tiles_poll(wait=True)
            check_frame((o, lights, rec, ctx.last_erosion_steps), want)
            for k in remove:
                del resident[k]
            resident.update(zip(keys, want[0]["zvals"]))
            assert np.array_equal(ts_new.stale([job.light(lp) for lp in (SUN, MOON)]), ts_ref.stale([job.light(lp) for lp in (SUN, MOON)]))
        follow_ups(tw, ctx, job, (ts_new, ts_ref), resident, check_full=(where == "pinned"))
    finally:
        ts_new.close()
        ts_ref.close()


def test_strip_takes_the_graph_path(tw, scene, ctx):
    """40 tiles in a row along the sun's direction: 40 dependency waves per light (more than 32: the relight's CUDA graph path) in one frame."""
    job = Job(tw, scene, ctx, "m4", 100)
    keys = [(0, y) for y in range(40)]
    sets = (ctx.tile_set(ZV, 2), ctx.tile_set(ZV, 2))
    try:
        want = sequence(tw, ctx, sets[1], job, keys, _origins(keys), [], keys, (SUN, MOON), "device")
        o, lights, rec = frame_launch(tw, ctx, sets[0], job, keys, _origins(keys), [], keys, (SUN, MOON), "device")
        assert ctx.create_tiles_poll(wait=True)
        check_frame((o, lights, rec, ctx.last_erosion_steps), want)
        assert rec.all()
        follow_ups(tw, ctx, job, sets, dict(zip(keys, want[0]["zvals"])), check_full=True)
    finally:
        for ts in sets:
            ts.close()


def test_poll_reports_not_ready_then_completes(tw, scene, ctx):
    job = Job(tw, scene, ctx, "m4", 2000)
    keys = [(x, y) for y in range(8) for x in range(8)]
    sets = (ctx.tile_set(ZV, 1), ctx.tile_set(ZV, 1))
    try:
        want = sequence(tw, ctx, sets[1], job, keys, _origins(keys), [], keys, (SUN,), "pinned")
        o, lights, rec = frame_launch(tw, ctx, sets[0], job, keys, _origins(keys), [], keys, (SUN,), "pinned")
        rc = tw.lib.tw_create_tiles_poll(ctx._h, 0)
        assert rc == tw.TW_ERR_NOT_READY
        while not ctx.create_tiles_poll(wait=False):
            pass
        check_frame((o, lights, rec, ctx.last_erosion_steps), want)
    finally:
        for ts in sets:
            ts.close()


def test_frames_on_a_pool_equal_frames_on_one_context(tw, scene, ctx):
    """K = 6 frames of a row of 8 tiles, each on its own shared context of a pool, all launched back to back with no poll and no other work in between; only
    then the same 6 frames as the separate calls, one after the other, on a second set on the parent context; then every frame is polled and compared. The
    frames alternate 4000 and 20 droplets per tile, so a light frame's generation and erosion end long before the heavy frame launched just before it: its
    set tail must wait for that frame's tail on the set's event (a relight that ran early would read tiles not yet in the slabs). Frame 2 grows the slabs
    while frame 0 is in flight, and frames 3 to 5 evict the rows of frames 0 to 2. Relight requests come from stale_after at launch time, when the host
    state of the earlier frames is already committed."""
    jobs = [Job(tw, scene, ctx, "m4", 4000), Job(tw, scene, ctx, "m4", 20)]   # tables first: setting them on the parent completes the pool's jobs
    K = 6
    pool = [ctx.shared() for _ in range(K)]
    sets = (ctx.tile_set(ZV, 2), ctx.tile_set(ZV, 2))
    lps = (SUN, MOON)
    sps = [jobs[0].light(lp) for lp in lps]
    try:
        plan = [(_rows(f, f + 1, 0, 8), _rows(f - 3, f - 2, 0, 8) if f >= 3 else []) for f in range(K)]
        launched = []
        for f, (keys, remove) in enumerate(plan):
            relight = [tuple(t) for t in sets[0].stale_after(sps, remove, keys)]
            assert set(keys) <= set(relight)
            launched.append(frame_launch(tw, pool[f], sets[0], jobs[f % 2], keys, _origins(keys), remove, relight, lps, "device") + (relight,))
        in_flight = sum(tw.lib.tw_create_tiles_poll(c._h, 0) == tw.TW_ERR_NOT_READY for c in pool)
        print("%d of %d frames still in flight after the last launch" % (in_flight, K))
        assert in_flight >= 1
        wants, resident = [], {}
        for f, ((keys, remove), (_, _, _, relight)) in enumerate(zip(plan, launched)):
            wants.append(sequence(tw, ctx, sets[1], jobs[f % 2], keys, _origins(keys), remove, relight, lps, "device"))
            for k in remove:
                del resident[k]
            resident.update(zip(keys, wants[f][0]["zvals"]))
        for f, c in enumerate(pool):
            assert c.create_tiles_poll(wait=True)
            o, lights, rec, _ = launched[f]
            check_frame((o, lights, rec, c.last_erosion_steps), wants[f])
        assert wants[0][1] > 10 * wants[1][1] > 0                    # the heavy frames are heavy
        follow_ups(tw, ctx, jobs[0], sets, resident, check_full=True)
    finally:
        for ts in sets:
            ts.close()
        for c in pool:
            c.close()


def test_argument_errors_leave_the_set_unchanged(tw, scene, ctx, heightmap):
    import torch
    L = tw.lib
    job = Job(tw, scene, ctx, "m4", 50)
    keys = _rows(0, 3)
    ts = ctx.tile_set(ZV, 2)
    other = tw.Context(0)
    try:
        sequence(tw, ctx, ts, job, keys, _origins(keys), [], keys[:5], (SUN, MOON), "pinned")
        sps = [job.light(SUN), job.light(MOON)]
        before = ts.stale(sps)
        nt = 2
        org = np.array(_origins([(0, 5), (1, 5)]), np.int32)
        o = _outputs(tw, job, nt, "pinned")
        outs = tw.TileOutputs(tw._ptr(o["zvals"]), tw._ptr(o["mm"]), None, None, None)
        m = np.empty((2, ZV, ZV), np.uint8)
        dm = torch.empty(2 * ZV * ZV + 4, dtype=torch.uint8, device="cuda")
        rec = np.zeros(2, np.uint8)
        ao = np.empty((nt, ZV - 1, ZV - 1), np.uint8)

        def xy(*ks):
            return np.array(ks, np.int32).reshape(-1, 2)

        def launch(tile_xy, remove=None, relight=None, lights=None, nl=None, c=ctx, hs=None, shading=None, n=nt, origins=org, p=job.hp):
            arr = (tw.TileSetLight * max(1, len(lights or [])))(*(lights or []))
            req = None
            if relight is not None:
                req = tw.TileSetRequest(tw._ptr(relight), len(relight), len(lights) if nl is None else nl, C.cast(arr, C.c_void_p) if lights else None, tw._ptr(rec))
            fr = tw.TileSetFrame(tw._ptr(remove), 0 if remove is None else len(remove), tw._ptr(tile_xy), C.cast(C.pointer(hs), C.c_void_p) if hs else None,
                                 C.cast(C.pointer(req), C.c_void_p) if req is not None else None)
            return L.tw_tile_set_create_tiles_launch(c._h, ts._h, tw._ptr(origins), n, S, S, job.dx, job.dy, C.byref(p) if p is not None else None, job.iters,
                                                     C.byref(job.ep), job.ep.zmin, 0.1, S, C.byref(outs), C.byref(shading) if shading else None, C.byref(fr))
        good = tw.TileSetLight(sps[0], tw._ptr(m), None, None)
        new = xy((0, 5), (1, 5))
        refused = [
            ("no tile_xy", launch(None)),
            ("tile_xy twice", launch(xy((0, 5), (0, 5)))),
            ("ntiles 0", launch(new, n=0)),
            ("no p", launch(new, p=None)),
            ("remove not resident", launch(new, remove=xy((7, 7)))),
            ("remove twice", launch(new, remove=xy((0, 0), (0, 0)))),
            ("removed and put", launch(xy((0, 0), (1, 5)), remove=xy((0, 0)))),
            ("relight names a removed tile", launch(new, remove=xy((1, 1)), relight=xy((1, 1), (0, 5)), lights=[good])),
            ("relight not resident", launch(new, relight=xy((0, 5), (3, 3), (7, 7)), lights=[good])),
            ("relight twice", launch(new, relight=xy((0, 5), (0, 5)), lights=[good])),
            ("relight no lights", launch(new, relight=xy((0, 5), (1, 5)), lights=[])),
            ("relight 3 lights", launch(new, relight=xy((0, 5), (1, 5)), lights=[good, good, good])),
            ("relight no smask", launch(new, relight=xy((0, 5), (1, 5)), lights=[tw.TileSetLight(sps[0], None, None, None)])),
            ("relight misaligned smask", launch(new, relight=xy((0, 5), (1, 5)), lights=[tw.TileSetLight(sps[0], dm.data_ptr() + 1, None, None)])),
            ("ctx of another family", launch(new, c=other)),
            ("hs with ao", launch(new, hs=job.hs or tw.HmapSampler(257, 300, 2, 1.0, 0.0012, 1.7, -0.3, 0.8),
                                  shading=tw.TileShading(0.0625, None, None, tw._ptr(ao), None, None))),
            ("hs of another size", launch(new, hs=tw.HmapSampler(256, 300, 2, 1.0, 0.0012, 1.7, -0.3, 0.8))),
        ]
        k = C.c_uint32()
        arr2 = (tw.ShadowParams * 2)(*sps)
        refused.append(("stale_after removed and put", L.tw_tile_set_stale_after(ts._h, C.cast(arr2, C.c_void_p), 2, tw._ptr(xy((0, 0))), 1, tw._ptr(xy((0, 0))), 1,
                                                                                 None, 0, C.byref(k))))
        refused.append(("stale_after not resident", L.tw_tile_set_stale_after(ts._h, C.cast(arr2, C.c_void_p), 2, tw._ptr(xy((9, 9))), 1, None, 0, None, 0, C.byref(k))))
        for what, rc in refused:
            assert rc == tw.TW_ERR_ARG, what
        assert ctx.create_tiles_poll(wait=False) and other.create_tiles_poll(wait=False)    # nothing was enqueued
        assert not rec.any()
        assert np.array_equal(ts.stale(sps), before)                                       # the set is as it was
        ref = ctx.tile_set(ZV, 2)
        try:
            z = sequence(tw, ctx, ref, job, keys, _origins(keys), [], keys[:5], (SUN, MOON), "pinned")[0]["zvals"]
            follow_ups(tw, ctx, job, (ts, ref), dict(zip(keys, z)), check_full=True)
        finally:
            ref.close()
    finally:
        ts.close()
        other.close()
