"""GPU: tile sets (tw_tile_set_*). Every relight output must equal, bit for bit, tw_tile_shadows_batch_ex over ALL tiles resident at launch time with no caller
rows; the cache may only skip tiles whose result cannot have changed, and its counts are checked against the closure rule computed here in Python. The terrain
is BASELINE's (mode 4, 8-octave domain warp, droplet erosion) from tw_create_zvals_batch."""
import ctypes as C

import numpy as np
import pytest

from cases import HM_CFG

pytestmark = pytest.mark.gpu

ITERS = 100
GRID = 8                                       # the terrain pool: GRID x GRID tile coordinates, two height variants each (for replacing puts)
LIGHTS = {"q++": (3.0, 2.0, 0.15), "q-+": (-3.0, 1.5, 0.2), "q+-": (2.5, -3.0, 0.15), "q--": (-2.0, -4.0, 0.2), "overhead": (0.0, 0.0, 5.0),
          "below": (2.0, 1.0, None), "no_shadow": (3.0, 2.0, 0.3)}


@pytest.fixture(scope="module")
def terrain(tw, scene, ctx):
    """zv -> (light factory, {(tx, ty): [variant 0 zvals, variant 1 zvals]})."""
    out = {}
    for zv in (34, 130):
        size = zv - 2
        cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(size, size, 1))
        hp, ep = cfg.height_params(), cfg.erosion_params()
        dx, dy = float(cfg.dx_val), float(cfg.dy_val)
        keys = [(tx, ty) for ty in range(GRID) for tx in range(GRID)]
        tiles = {}
        for v in range(2):
            origins = [(tx * size * 9 - 3000, ty * size * 9 + 500 + 7000 * v) for tx, ty in keys]   # spread out: ocean and mountain tiles
            z = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, ITERS, ep, ep.zmin)
            for k, zt in zip(keys, z):
                tiles.setdefault(k, []).append(zt.copy())

        def light(name, lp=None, ep=ep, dx=dx, dy=dy, size=size):
            lp = lp if lp is not None else LIGHTS[name]
            sp = tw.ShadowParams()
            sp.x_scene_size = sp.y_scene_size = 0.5
            sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
            sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * size, float(ep.zmin), float(ep.zmax), int(name == "no_shadow")
            sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp[0], lp[1], float(ep.zmin) - 1.0 if lp[2] is None else lp[2]
            return sp
        out[zv] = (light, tiles)
    return out


def _full(tw, ctx, resident, sp):
    """tw_tile_shadows_batch_ex over every resident tile, no caller rows: {key: (smask, sh_out_x, sh_out_y)}."""
    keys = sorted(resident)
    z = np.ascontiguousarray(np.stack([resident[k] for k in keys]))
    txy = np.array(keys, np.int32)
    nt, zv = z.shape[0], z.shape[1]
    m, ox, oy = np.empty((nt, zv, zv), np.uint8), np.empty((nt, zv), np.float32), np.empty((nt, zv), np.float32)
    ctx._check(tw.lib.tw_tile_shadows_batch_ex(ctx._h, tw._ptr(z), tw._ptr(txy), nt, zv, C.byref(sp), None, None, tw._ptr(m), tw._ptr(ox), tw._ptr(oy)))
    return {k: (m[i], ox[i], oy[i]) for i, k in enumerate(keys)}


def _alloc(where, shape, dtype):
    import torch
    t = {"u1": torch.uint8, "f4": torch.float32}[dtype]
    if where == "host":
        return np.empty(shape, {"u1": np.uint8, "f4": np.float32}[dtype])
    if where == "pinned":
        return torch.empty(shape, dtype=t).pin_memory()
    return torch.empty(shape, dtype=t, device="cuda")


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


def _relight(tw, ctx, ts, req, sps, where="pinned"):
    n, zv = len(req), ts.zvsize
    lights = [tw.Light(sp, _alloc(where, (n, zv, zv), "u1"), _alloc(where, (n, zv), "f4"), _alloc(where, (n, zv), "f4")) for sp in sps]
    rec = ts.shadows_launch(np.array(req, np.int32).reshape(-1, 2), lights)
    assert ctx.create_tiles_poll(wait=True)
    return rec, [(_host(L.smask).copy(), _host(L.sh_out_x).copy(), _host(L.sh_out_y).copy()) for L in lights]


def _assert_full(tw, ctx, resident, req, sps, outs, beq):
    for sp, (m, ox, oy) in zip(sps, outs):
        ref = _full(tw, ctx, resident, sp)
        for i, k in enumerate(req):
            em, ex, ey = ref[tuple(k)]
            assert np.array_equal(m[i], em), k
            assert beq(ox[i], ex) == 0 and beq(oy[i], ey) == 0, k


def _sign(v):
    return -1 if v < 0 else 1


def _downstream(keys, seeds, sp):
    """The resident tiles whose incoming rows come from the seeds, transitively, the resident seeds included."""
    sx, sy = _sign(sp.lpos[0]), _sign(sp.lpos[1])
    out, todo = set(), list(seeds)
    while todo:
        k = todo.pop()
        if k in keys and k not in out:
            out.add(k)
            todo += [(k[0] - sx, k[1]), (k[0], k[1] - sy)]
    return out


SHAPES = {
    "square": [(x, y) for y in range(1, 7) for x in range(1, 7)],
    "L_with_holes": [k for k in [(x, y) for y in range(2) for x in range(7)] + [(x, y) for y in range(2, 8) for x in range(2)] if k not in ((3, 0), (1, 4), (5, 1))],
    "strip": [(3, y) for y in range(8)],
    "single": [(2, 3)],
}


@pytest.mark.parametrize("where", ["host", "pinned", "device"])
@pytest.mark.parametrize("zv", [34, 130])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_full_relight_equals_batch_ex(tw, ctx, terrain, beq, shape, zv, where):
    """Every light of LIGHTS, two per request on one set (each request changes both slots' params, so everything is recomputed)."""
    import torch
    light, tiles = terrain[zv]
    keys = SHAPES[shape]
    resident = {k: tiles[k][0] for k in keys}
    ts = ctx.tile_set(zv, 2)
    try:
        z = np.stack([resident[k] for k in keys])
        ts.put(keys, torch.from_numpy(z).cuda() if where == "device" else z)
        names = list(LIGHTS)
        shadowed = 0
        for a, b in zip(names[0::2], names[1::2] + ["q++"]):
            sps = [light(a), light(b)]
            rec, outs = _relight(tw, ctx, ts, keys, sps, where)
            assert rec.all()
            _assert_full(tw, ctx, resident, keys, sps, outs, beq)
            shadowed += int((outs[0][0] == 2).sum())
            if b == "below":
                assert (outs[1][0] == 2).all()
            if a in ("no_shadow", "overhead"):
                assert not outs[0][0].any()
        print("%s, %d^2: %d cells in shadow" % (shape, zv, shadowed))
        assert shadowed > 0 or len(keys) < 10
    finally:
        ts.close()


def test_random_sequence(tw, ctx, terrain, beq):
    """About 60 seeded steps of put (new and replacing), remove, light change and relight of a random subset; after every relight each requested tile's
    outputs equal a fresh tw_tile_shadows_batch_ex over the whole current set."""
    rng = np.random.default_rng(2024)
    light, tiles = terrain[34]
    pool = sorted(tiles)
    resident = {}
    names = [n for n in LIGHTS if n not in ("overhead", "no_shadow")]
    sps = [light("q++"), light("q--")]
    ts = ctx.tile_set(34, 2)
    relights = recomputed = 0
    try:
        for step in range(60):
            op = rng.choice(["put", "put", "remove", "light", "relight", "relight"]) if resident else "put"
            if op == "put":
                ks = [pool[int(i)] for i in rng.choice(len(pool), int(rng.integers(1, 7)), replace=False)]
                z = [tiles[k][int(rng.integers(0, 2))] for k in ks]
                ts.put(ks, np.stack(z))
                resident.update(zip(ks, z))
            elif op == "remove":
                ks = [sorted(resident)[int(i)] for i in rng.choice(len(resident), min(len(resident), int(rng.integers(1, 4))), replace=False)]
                ts.remove(ks)
                for k in ks:
                    del resident[k]
            elif op == "light":
                li = int(rng.integers(0, 2))
                if rng.random() < 0.5:
                    sps[li] = light(names[int(rng.integers(0, len(names)))])
                else:
                    sps[li] = light("q++", (float(rng.uniform(-4, 4)), float(rng.uniform(-4, 4)), float(rng.uniform(0.1, 0.4))))
            else:
                keys = sorted(resident)
                req = [keys[int(i)] for i in rng.choice(len(keys), int(rng.integers(1, len(keys) + 1)), replace=False)]
                use = sps[:int(rng.integers(1, 3))]
                rec, outs = _relight(tw, ctx, ts, req, use, "pinned" if step % 2 else "device")
                _assert_full(tw, ctx, resident, req, use, outs, beq)
                relights += 1
                recomputed += int(rec.sum())
        print("%d relights, %d tiles recomputed, %d resident at the end" % (relights, recomputed, len(resident)))
        assert relights >= 10
    finally:
        ts.close()


def test_cache_counts(tw, ctx, terrain, beq):
    light, tiles = terrain[34]
    keys = [(x, y) for y in range(GRID) for x in range(GRID) if (x, y) not in ((2, 2), (5, 6))]
    resident = {k: tiles[k][0] for k in keys}
    ts = ctx.tile_set(34, 2)
    try:
        ts.put(keys, np.stack([resident[k] for k in keys]))
        sps = [light("q++"), light("q--")]
        assert len(ts.stale(sps)) == len(keys)
        rec, outs = _relight(tw, ctx, ts, keys, sps)
        assert rec.all()
        _assert_full(tw, ctx, resident, keys, sps, outs, beq)
        # a repeated identical request recomputes nothing and gives the same bytes
        assert len(ts.stale(sps)) == 0
        rec2, outs2 = _relight(tw, ctx, ts, keys, sps)
        assert not rec2.any()
        for a, b in zip(outs, outs2):
            assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
        # changing one light's params recomputes every requested tile
        sps[1] = light("q-+")
        req = keys[30:]                                           # rows 3..7: rows 0..2 are not upstream of them for a light from -x / +y
        rec, outs = _relight(tw, ctx, ts, req, sps)
        assert rec.all()
        _assert_full(tw, ctx, resident, req, sps, outs, beq)
        left = {tuple(t) for t in ts.stale(sps)}                  # slot 1 outside req and its upstream closure
        assert left and not left & set(req)
        rec, _ = _relight(tw, ctx, ts, keys, sps)                 # so that both slots are valid everywhere
        assert {kk for kk, r in zip(keys, rec) if r} == left
        # putting one tile (replacing, then new) recomputes exactly it and its resident downstream closure
        for k, v in (((4, 3), 1), ((2, 2), 0)):
            resident[k] = tiles[k][v]
            ts.put([k], tiles[k][v][None])
            expect = set().union(*[_downstream(set(resident), [k], sp) for sp in sps])
            allk = sorted(resident)
            stale = {tuple(t) for t in ts.stale(sps)}
            assert stale == expect
            rec, outs = _relight(tw, ctx, ts, allk, sps)
            assert {kk for kk, r in zip(allk, rec) if r} == expect == stale
            _assert_full(tw, ctx, resident, allk, sps, outs, beq)
            print("put %s: %d of %d tiles recomputed" % (k, len(expect), len(allk)))
            assert 1 <= len(expect) < len(allk)
        # removing a tile: stale lists its downstream closure, and the next request recomputes exactly that
        k = (3, 4)
        ts.remove([k])
        del resident[k]
        expect = set().union(*[_downstream(set(resident), [(k[0] - _sign(sp.lpos[0]), k[1]), (k[0], k[1] - _sign(sp.lpos[1]))], sp) for sp in sps])
        allk = sorted(resident)
        assert {tuple(t) for t in ts.stale(sps)} == expect
        rec, outs = _relight(tw, ctx, ts, allk, sps)
        assert {kk for kk, r in zip(allk, rec) if r} == expect
        _assert_full(tw, ctx, resident, allk, sps, outs, beq)
        # one light only: stale and the recompute ask about the first slot alone
        sps1 = [light("q+-")]
        assert len(ts.stale(sps1)) == len(allk)
        rec, outs = _relight(tw, ctx, ts, allk, sps1)
        assert rec.all() and len(ts.stale(sps1)) == 0
    finally:
        ts.close()


def test_relight_returns_before_the_work_is_done(tw, ctx, terrain, beq):
    """32 x 32 tiles of 130^2 (63 dependency waves per light, the graph path), two lights into device memory: the launch returns while the device works."""
    import time
    import torch
    light, tiles = terrain[130]
    keys = [(x, y) for y in range(32) for x in range(32)]
    resident = {k: tiles[(k[0] % GRID, k[1] % GRID)][(k[0] // GRID + k[1] // GRID) % 2] for k in keys}
    ts = ctx.tile_set(130, 2)
    try:
        ts.put(keys, torch.from_numpy(np.stack([resident[k] for k in keys])).cuda())
        sps = [light("q++"), light("q--")]
        n = len(keys)
        lights = [tw.Light(sp, torch.empty((n, 130, 130), dtype=torch.uint8, device="cuda"), torch.empty((n, 130), device="cuda"),
                           torch.empty((n, 130), device="cuda")) for sp in sps]
        t0 = time.perf_counter()
        rec = ts.shadows_launch(np.array(keys, np.int32), lights)
        t_launch = time.perf_counter() - t0
        ready_at_once = ctx.create_tiles_poll(wait=False)
        while not ctx.create_tiles_poll(wait=False):
            pass
        print("launch blocked the host for %.3f ms; ready after %.2f ms" % (1e3 * t_launch, 1e3 * (time.perf_counter() - t0)))
        assert not ready_at_once and rec.all()
        outs = [(L.smask.cpu().numpy(), L.sh_out_x.cpu().numpy(), L.sh_out_y.cpu().numpy()) for L in lights]
        _assert_full(tw, ctx, resident, keys, sps, outs, beq)
    finally:
        ts.close()


def test_calls_complete_a_pending_job_first(tw, scene, ctx, terrain, beq):
    """put, remove and a new relight complete a pending tile job (its outputs are then final) before they change anything."""
    import torch
    light, tiles = terrain[34]
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(32, 32, 1))
    hp, ep = cfg.height_params(), cfg.erosion_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    origins = [((t % 8) * 32, (t // 8 + 90) * 32) for t in range(64)]
    expect = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, 34, hp, 2000, ep, ep.zmin)
    keys = [(x, y) for y in range(4) for x in range(4)]
    ts = ctx.tile_set(34, 1)
    try:
        ts.put(keys, np.stack([tiles[k][0] for k in keys]))
        sps = [light("q++")]
        for what in ("put", "remove", "relight"):
            z = torch.empty((64, 34, 34), dtype=torch.float32).pin_memory()
            ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, 34, hp, 2000, ep, ep.zmin, z)
            if what == "put":
                ts.put([(7, 7)], tiles[(7, 7)][0][None])
            elif what == "remove":
                ts.remove([(7, 7)])
            else:
                lt = tw.Light(sps[0], torch.empty((16, 34, 34), dtype=torch.uint8).pin_memory(), None, None)
                ts.shadows_launch(np.array(keys, np.int32), [lt])
            assert beq(z.numpy(), expect) == 0, what            # the tile job was complete when the call returned
            assert ctx.create_tiles_poll(wait=True)
    finally:
        ts.close()


def test_shared_context_and_destroy(tw, ctx, terrain, beq):
    """A set on a shared context gives the parent's results; tw_destroy of a context with live sets (and a pending relight) is clean."""
    light, tiles = terrain[34]
    keys = SHAPES["L_with_holes"]
    z = np.stack([tiles[k][1] for k in keys])
    sps = [light("q-+"), light("q+-")]
    res = []
    parent = tw.Context(0)
    try:
        shared = parent.shared()
        for c in (parent, shared):
            ts = c.tile_set(34, 2)
            ts.put(keys, z)
            res.append(_relight(tw, c, ts, keys, sps))
        for (ra, oa), (rb, ob) in zip(res[:1], res[1:]):
            assert np.array_equal(ra, rb)
            for a, b in zip(oa, ob):
                assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
        _assert_full(tw, ctx, {k: zt for k, zt in zip(keys, z)}, keys, sps, res[0][1], beq)
        extra = parent.tile_set(34, 1)                         # a pending relight on a live set when the parent goes
        extra.put(keys, z)
        m = np.empty((len(keys), 34, 34), np.uint8)
        extra.shadows_launch(np.array(keys, np.int32), [(sps[0], m, None, None)])
    finally:
        parent.close()                                         # destroys the shared context and every set
    assert all(s._h is None for s in (extra,) + tuple(parent._sets))
    extra.close()                                              # its handle is gone: a no-op


def test_argument_errors_leave_the_set_unchanged(tw, ctx, terrain, beq):
    import torch
    L = tw.lib
    light, tiles = terrain[34]
    keys = [(x, y) for y in range(3) for x in range(3)]
    resident = {k: tiles[k][0] for k in keys}
    h = C.c_void_p()
    assert L.tw_tile_set_create(ctx._h, 1, 1, C.byref(h)) == tw.TW_ERR_ARG and not h.value
    assert L.tw_tile_set_create(ctx._h, 34, 0, C.byref(h)) == tw.TW_ERR_ARG and not h.value
    assert L.tw_tile_set_create(ctx._h, 34, 1, None) == tw.TW_ERR_ARG
    ts = ctx.tile_set(34, 2)
    try:
        ts.put(keys, np.stack([resident[k] for k in keys]))
        sps = [light("q++"), light("q--")]
        _relight(tw, ctx, ts, keys[:4], sps)
        before = ts.stale(sps)
        z2 = np.stack([tiles[(5, 5)][0], tiles[(5, 5)][0]])

        def xy(*ks):
            return np.array(ks, np.int32)
        refused = []
        a = xy((5, 5), (5, 5))
        refused.append(("put duplicate", L.tw_tile_set_put(ts._h, tw._ptr(a), 2, tw._ptr(z2))))
        refused.append(("put empty", L.tw_tile_set_put(ts._h, tw._ptr(a), 0, tw._ptr(z2))))
        refused.append(("put no zvals", L.tw_tile_set_put(ts._h, tw._ptr(a), 1, None)))
        b = xy((0, 0), (6, 6))
        refused.append(("remove not resident", L.tw_tile_set_remove(ts._h, tw._ptr(b), 2)))
        c = xy((0, 0), (0, 0))
        refused.append(("remove duplicate", L.tw_tile_set_remove(ts._h, tw._ptr(c), 2)))
        k = C.c_uint32()
        arr3 = (tw.ShadowParams * 3)(*(sps + sps[:1]))
        refused.append(("stale 3 lights", L.tw_tile_set_stale(ts._h, C.cast(arr3, C.c_void_p), 3, None, 0, C.byref(k))))
        refused.append(("stale 0 lights", L.tw_tile_set_stale(ts._h, C.cast(arr3, C.c_void_p), 0, None, 0, C.byref(k))))
        refused.append(("stale no out", L.tw_tile_set_stale(ts._h, C.cast(arr3, C.c_void_p), 2, None, 4, C.byref(k))))
        n = 2
        m = np.empty((n, 34, 34), np.uint8)
        dm = torch.empty(n * 34 * 34 + 4, dtype=torch.uint8, device="cuda")
        rec = np.zeros(n, np.uint8)

        def launch(txy, nn, lights, nl=None):
            arr = (tw.TileSetLight * max(1, len(lights)))(*lights)
            req = tw.TileSetRequest(tw._ptr(txy), nn, len(lights) if nl is None else nl, C.cast(arr, C.c_void_p) if lights else None, tw._ptr(rec))
            rc = L.tw_tile_set_shadows_launch(ts._h, C.byref(req))
            return rc
        good = tw.TileSetLight(sps[0], tw._ptr(m), None, None)
        ok = xy((0, 0), (1, 0))
        refused.append(("launch n = 0", launch(ok, 0, [good])))
        refused.append(("launch not resident", launch(xy((0, 0), (7, 7)), 2, [good])))
        refused.append(("launch duplicate", launch(xy((1, 1), (1, 1)), 2, [good])))
        refused.append(("launch no lights", launch(ok, 2, [])))
        refused.append(("launch 0 lights", launch(ok, 2, [good], 0)))
        refused.append(("launch 3 lights", launch(ok, 2, [good, good, good])))
        refused.append(("launch no smask", launch(ok, 2, [tw.TileSetLight(sps[0], None, None, None)])))
        refused.append(("launch misaligned smask", launch(ok, 2, [tw.TileSetLight(sps[0], dm.data_ptr() + 1, None, None)])))
        refused.append(("launch no tile_xy", launch(None, 2, [good])))
        for what, rc in refused:
            assert rc == tw.TW_ERR_ARG, what
        assert L.tw_last_error(ctx._h)
        assert ctx.create_tiles_poll(wait=False)                   # nothing was enqueued
        assert not rec.any()
        assert np.array_equal(ts.stale(sps), before)               # the cache is as it was
        rec, outs = _relight(tw, ctx, ts, keys, sps)
        assert rec.sum() == len(before)
        _assert_full(tw, ctx, resident, keys, sps, outs, beq)
    finally:
        ts.close()
