"""GPU: the mesh-shadow tracer (shadow_rays_kernel and its plan) on non-square cells, unequal scene sizes, axis, signed-zero and exactly diagonal lights, and
grazing and steep suns, in the three paths that run it: tw_tile_shadows_batch(_ex), the tile job's shadow pass (procedural and heightmap-image heights) and a
tile set's relight. Every comparison is bit for bit. The batch is checked against the CPU oracle (pinned against the reference on a 32 x 48 mesh) and the
spike tiles of tests/test_shadows_geometry_host.py against their analytic shadow as well, so a geometry mistake the oracle shared would still show."""
import ctypes as C

import numpy as np
import pytest

from cases import convert, HM_CFG
from test_gpu_tile_set import _downstream, _full, _relight
from test_shadows_geometry_host import GEOMS, LIGHTS, ZV, check_spike, geometry, shadow_params, spike_tile, trace_spike
from test_shadows_in_oracle import MIN_Z, tile_shadows_batch_in

pytestmark = pytest.mark.gpu

BATCH_LIGHTS = dict(LIGHTS, **{"-0x": (-0.0, 3.0, 1.0), "-0y": (2.0, -0.0, 1.0)})     # signed zeros: the plan's neighbour signs take -0.0 as +
LAYOUTS = {
    "single": [(2, -1)],
    "block4x3": [(tx - 1, ty + 3) for ty in range(3) for tx in range(4)],
    "L_holes": [k for k in [(x, y) for y in range(2) for x in range(5)] + [(x, y) for y in range(2, 5) for x in range(2)] if k not in ((2, 0), (1, 3))],
}
# (geometry, zvsize, layout): every geometry of the host test, tile sizes 40 (the reference pin's), 19 (odd: a tile's mask starts mid-word), 258 and 1026
# (4104 rays in 33 blocks per tile, walks of about 1000 steps), a single tile, a chained 4 x 3 block and an L with holes
CASES = [("dx>dy", 40, "block4x3"), ("dx<dy_xs!=ys", 40, "L_holes"), ("sq_xs!=ys", 19, "block4x3"), ("dx>dy_xs!=ys", 19, "L_holes"), ("dx>dy", 19, "single"),
         ("dx<dy", 258, "block4x3"), ("sq", 258, "single"), ("dx>dy_xs!=ys", 1026, "block4x3"), ("dx<dy_xs!=ys", 1026, "single")]


def _relief(lp):
    """Height scale of the terrain for light lp: a steep sun only casts shadows on steep terrain."""
    return np.float32(10.0 * max(1.0, lp[2] / np.hypot(lp[0], lp[1]) / 0.3))


def _terrain(scene, ctx, gname, zv, txy):
    """heightgen_tiles terrain of geometry gname around 0 (the rays run at z = 0 and are clipped against [zmin, zmax])."""
    mesh, size, dx, dy = geometry(scene, gname)
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.0, mesh_size=mesh, scene_size=size)
    S = zv - 2
    z = ctx.heightgen_tiles([(tx * S, ty * S) for tx, ty in txy], mesh, dx, dy, zv, cfg.height_params())
    z += np.random.default_rng(zv).normal(0.0, 0.01, z.shape).astype(np.float32)       # some roughness: every light finds an edge to cast from
    return (z - np.float32(z.mean())).astype(np.float32)


def _hands_over(lp):
    """Whether shadows can leave a tile in general: a ray leaves toward -x (-y) at index 0, its last cell, which writes sh_out; toward +x and +y it leaves at
    index zvsize, outside the tile, so a light with lpos.x < 0 and lpos.y < 0 hands over only what a ray's last row or column inside the tile carries."""
    return not (lp[0] < 0.0 and lp[1] < 0.0)


def _rows(rng, nt, zv, zlo, zhi):
    """Caller rows: heights inside the terrain's range, 30 % of them "none" (MESH_MIN_Z)."""
    r = rng.uniform(zlo, zhi, (nt, zv)).astype(np.float32)
    r[rng.random((nt, zv)) < 0.3] = MIN_Z
    return r


@pytest.mark.parametrize("gname,zv,layout", CASES)
def test_batch_equals_oracle(tw, scene, oracle, ctx, beq, gname, zv, layout):
    """Every light on the terrain; caller rows (tw_tile_shadows_batch_ex) for every other light, device zvals and mask for the first. Each light casts a
    partial shadow, and on the block layouts some shadow leaves a tile through sh_out."""
    import torch
    txy = LAYOUTS[layout]
    base = _terrain(scene, ctx, gname, zv, txy)
    nt = len(txy)
    rng = np.random.default_rng(zv)
    for li, (lname, lp) in enumerate(BATCH_LIGHTS.items()):
        z = (base * _relief(lp)).astype(np.float32)
        zlo, zhi = float(z.min()) - 0.5, float(z.max()) + 0.5
        assert zlo < 0.0 < zhi
        sp = shadow_params(tw.ShadowParams, scene, gname, lp, zlo, zhi)
        sp.xy_sum_size = 2 * zv                                         # rays long enough to cross the tile
        spo = convert(sp, oracle.ShadowParams)
        ix = iy = None
        if li % 2:
            ix, iy = _rows(rng, nt, zv, zlo, zhi), _rows(rng, nt, zv, zlo, zhi)
            mo, oxo, oyo = tile_shadows_batch_in(oracle, z, txy, spo, ix, iy)
        else:
            mo, oxo, oyo = oracle.tile_shadows_batch(z, txy, spo)
        if li == 0:
            dm = torch.empty((nt, zv, zv), dtype=torch.uint8, device="cuda")
            _, ox, oy = ctx.tile_shadows(torch.from_numpy(z).cuda(), txy, sp, out=dm)
            m = dm.cpu().numpy()
        else:
            m, ox, oy = ctx.tile_shadows(z, txy, sp, sh_in_x=ix, sh_in_y=iy)
        assert np.array_equal(m, mo), (lname, int((m != mo).sum()))
        assert beq(ox, oxo) == 0 and beq(oy, oyo) == 0, lname
        assert 0 < (mo == 2).sum() < mo.size, lname
        if layout != "single" and _hands_over(lp):
            assert (oxo > MIN_Z).any() or (oyo > MIN_Z).any(), lname


@pytest.mark.parametrize("gname", list(GEOMS))
def test_spike_shadows(tw, scene, oracle, ctx, beq, gname):
    """The spike tiles of the host test: the GPU's mask and edges equal the oracle's, and obey the analytic shadow on their own."""
    for lname, lp in LIGHTS.items():
        h, k, at, mo, oxo, oyo = trace_spike(oracle, scene, gname, lname)
        sp = shadow_params(tw.ShadowParams, scene, gname, lp, -1.0, h + 1.0)
        m, ox, oy = ctx.tile_shadows(spike_tile(h, at)[None], [(0, 0)], sp)
        assert np.array_equal(m[0], mo) and beq(ox[0], oxo) == 0 and beq(oy[0], oyo) == 0, lname
        check_spike(scene, gname, lname, h, k, at, m[0], ox[0], oy[0])


def _batch_ex(tw, ctx, z, txy, sp, ix=None, iy=None):
    """tw_tile_shadows_batch_ex on host arrays: (smask, sh_out_x, sh_out_y)."""
    z = np.ascontiguousarray(z, np.float32)
    txy = np.ascontiguousarray(txy, np.int32)
    nt, zv = z.shape[0], z.shape[1]
    m, ox, oy = np.empty((nt, zv, zv), np.uint8), np.empty((nt, zv), np.float32), np.empty((nt, zv), np.float32)
    ctx._check(tw.lib.tw_tile_shadows_batch_ex(ctx._h, tw._ptr(z), tw._ptr(txy), nt, zv, C.byref(sp), tw._ptr(ix), tw._ptr(iy), tw._ptr(m), tw._ptr(ox),
                                               tw._ptr(oy)))
    return m, ox, oy


@pytest.mark.parametrize("hmap", [False, True], ids=["procedural", "hmap"])
def test_tile_job_on_non_square_cells(tw, scene, oracle, ctx, beq, hmap):
    """The tile job on a 32 x 48 mesh's cells with unequal scene sizes, two lights per job (an axis sun and an exact diagonal, one with caller rows):
    the masks and edges equal tw_tile_shadows_batch_ex on the job's own zvals, and the oracle's."""
    import torch
    gname, zv = "dx>dy_xs!=ys", 40
    mesh, size, dx, dy = geometry(scene, gname)
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=mesh, scene_size=size)
    hp, ep = cfg.height_params(), cfg.erosion_params()
    txy = np.array([(tx, ty) for ty in range(3) for tx in range(4)], np.int32)
    origins = [(int(tx) * (zv - 2) - 60, int(ty) * (zv - 2) + 20) for tx, ty in txy]
    nt = len(origins)
    rng = np.random.default_rng(7)
    if hmap:
        img = rng.integers(0, 256, (300, 257, 2), dtype=np.uint8)
        img[..., 1] //= 8                                               # 16-bit heights of at most 8191: steep enough for shadows, not a wall
        ctx.set_heightmap(img)
        hs = tw.HmapSampler(257, 300, 2, 1.0, 0.0012, 1.0, -0.3, 1.0)
        lps = [(-0.0, -3.0, 0.5), (2.0, -2.0, 0.4)]
    else:
        hs = None
        lps = [(0.0, 3.0, 0.02), (-2.0, -2.0, 0.02)]
    zlo, zhi = (-200.0, 200.0) if hmap else (float(ep.zmin), float(ep.zmax))
    ix = _rows(rng, nt, zv, -0.2, 0.2)
    lights = []
    for i, lp in enumerate(lps):
        sp = shadow_params(tw.ShadowParams, scene, gname, lp, zlo, zhi)
        sp.xy_sum_size = 2 * zv
        lights.append(tw.Light(sp, torch.empty((nt, zv, zv), dtype=torch.uint8, device="cuda"), torch.empty((nt, zv), device="cuda"),
                               torch.empty((nt, zv), device="cuda"), ix if i == 0 else None, None))
    z = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
    try:
        if hmap:
            ctx.create_tiles_launch(origins, mesh, dx, dy, zv, None, 0, None, 0.0, z, tile_xy=txy, lights=lights, hmap=hs)
        else:
            ctx.create_tiles_launch(origins, mesh, dx, dy, zv, hp, 0, ep, ep.zmin, z, tile_xy=txy, lights=lights)
        assert ctx.create_tiles_poll(wait=True)
    finally:
        if hmap:
            ctx.set_heightmap(None)
    zh = z.cpu().numpy()
    assert zlo < float(zh.min()) and float(zh.max()) < zhi
    for L in lights:
        m, ox, oy = L.smask.cpu().numpy(), L.sh_out_x.cpu().numpy(), L.sh_out_y.cpu().numpy()
        em, eox, eoy = _batch_ex(tw, ctx, zh, txy, L.sp, L.sh_in_x, None)
        assert np.array_equal(m, em) and beq(ox, eox) == 0 and beq(oy, eoy) == 0, tuple(L.sp.lpos)
        om, oox, ooy = tile_shadows_batch_in(oracle, zh, txy, convert(L.sp, oracle.ShadowParams), L.sh_in_x, None)
        assert np.array_equal(m, om) and beq(ox, oox) == 0 and beq(oy, ooy) == 0, tuple(L.sp.lpos)
        assert 0 < (m == 2).sum() < m.size, tuple(L.sp.lpos)
        assert (ox > MIN_Z).any() or (oy > MIN_Z).any() or not _hands_over(L.sp.lpos), tuple(L.sp.lpos)


def test_tile_set_relight_through_axis_and_zero_lights(tw, scene, ctx, beq):
    """A tile set of 32 x 48-mesh cells, filled by a frame launch (tw_tile_set_create_tiles_launch) and puts, relit while two lights move through
    +axis -> +0.0 -> -0.0 -> -axis -> a diagonal -> a steep sun (slot 0 along x, slot 1 along y). After each move every output equals
    tw_tile_shadows_batch_ex over all resident tiles; under the zero lights a put and a remove make stale() name exactly the downstream tiles, with
    -0.0 taking the sign +1 as the plan does."""
    import torch
    gname, zv = "dx<dy_xs!=ys", 40
    mesh, size, dx, dy = geometry(scene, gname)
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=mesh, scene_size=size)
    hp, ep = cfg.height_params(), cfg.erosion_params()
    keys = [(x, y) for y in range(5) for x in range(5) if (x, y) not in ((2, 2), (4, 1))]
    z = _terrain(scene, ctx, gname, zv, keys + [(2, 2)])
    z[:, 17, 23] += np.float32(2000.0)                                   # one tall cell per tile: shadows under the steep sun
    resident = {k: z[i] for i, k in enumerate(keys)}
    zlo, zhi = float(z.min()) - 0.5, float(z.max()) + 0.5

    def light(lp):
        sp = shadow_params(tw.ShadowParams, scene, gname, lp, zlo, zhi)
        sp.xy_sum_size = 2 * zv
        return sp
    ts = ctx.tile_set(zv, 2)
    try:
        first, rest = keys[:3], keys[3:]
        ts.put(rest, np.stack([resident[k] for k in rest]))
        sps = [light((3.0, 1.0, 0.3)), light((1.0, 3.0, 0.3))]
        zf = torch.empty((len(first), zv, zv), dtype=torch.float32, device="cuda")
        n = len(keys)
        lights = [tw.Light(sp, torch.empty((n, zv, zv), dtype=torch.uint8, device="cuda"), torch.empty((n, zv), device="cuda"),
                           torch.empty((n, zv), device="cuda")) for sp in sps]
        rec = ts.create_tiles_launch([(x * 38, y * 38) for x, y in first], mesh, dx, dy, hp, 0, ep, ep.zmin, first, zvals=zf, relight_xy=keys, lights=lights)
        assert ctx.create_tiles_poll(wait=True)
        assert np.asarray(rec).all()
        resident.update(zip(first, zf.cpu().numpy()))
        outs = [(L.smask.cpu().numpy(), L.sh_out_x.cpu().numpy(), L.sh_out_y.cpu().numpy()) for L in lights]
        _check_all(tw, ctx, beq, resident, keys, sps, outs)
        moves = [((0.0, 1.0, 0.3), (1.0, 0.0, 0.3)), ((-0.0, 1.0, 0.3), (1.0, -0.0, 0.3)), ((-3.0, 1.0, 0.3), (1.0, -3.0, 0.3)),
                 ((-2.0, 2.0, 0.3), (2.0, 2.0, 0.3)), ((8.0e-4, -6.0e-4, 5.0), (-6.0e-4, 8.0e-4, 5.0))]
        for step, (a, b) in enumerate(moves):
            sps = [light(a), light(b)]
            allk = sorted(resident)
            assert len(ts.stale(sps)) == len(allk)
            rec, outs = _relight(tw, ctx, ts, allk, sps, "device")
            assert rec.all()
            _check_all(tw, ctx, beq, resident, allk, sps, outs)
            if step < 2:                                                # the zero lights: put, then remove, and what stale() names
                for op, k in (("put", (2, 2)), ("remove", (1, 3))):
                    if op == "put":
                        resident[k] = z[len(keys)] if k not in resident else resident[k]
                        ts.put([k], resident[k][None])
                        seeds = {s: [k] for s in range(2)}
                    else:
                        ts.remove([k])
                        del resident[k]
                        seeds = {s: [(k[0] - _sign(sp.lpos[0]), k[1]), (k[0], k[1] - _sign(sp.lpos[1]))] for s, sp in enumerate(sps)}
                    expect = set().union(*[_downstream(set(resident), seeds[s], sp) for s, sp in enumerate(sps)])
                    assert {tuple(t) for t in ts.stale(sps)} == expect, (op, step)
                    assert 1 <= len(expect) < len(resident)
                    allk = sorted(resident)
                    rec, outs = _relight(tw, ctx, ts, allk, sps, "device")
                    assert {kk for kk, r in zip(allk, rec) if r} == expect
                    _check_all(tw, ctx, beq, resident, allk, sps, outs)
                ts.put([(1, 3)], z[keys.index((1, 3))][None])                # back to the full set
                resident[(1, 3)] = z[keys.index((1, 3))]
    finally:
        ts.close()


def _sign(v):
    """twts::light_sign: -0.0 is not below 0."""
    return -1 if v < 0.0 else 1


def _check_all(tw, ctx, beq, resident, req, sps, outs):
    for sp, (m, ox, oy) in zip(sps, outs):
        ref = _full(tw, ctx, resident, sp)
        shadowed = 0
        for i, k in enumerate(req):
            em, ex, ey = ref[tuple(k)]
            assert np.array_equal(m[i], em), (k, tuple(sp.lpos))
            assert beq(ox[i], ex) == 0 and beq(oy[i], ey) == 0, (k, tuple(sp.lpos))
            shadowed += int((m[i] == 2).sum())
        assert shadowed > 0, tuple(sp.lpos)
