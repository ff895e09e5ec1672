"""GPU: tw_create_tiles_launch_shadows - the asynchronous tile job with the mesh shadows of its tiles. Every light's mask and outgoing edges must equal, bit
for bit, tw_tile_shadows_batch_ex on the job's own zvals with the same tile_xy, light and incoming rows; every other output and the erosion step count must
equal the same job without shadows."""
import time

import numpy as np
import pytest

from cases import HM_CFG
from test_gpu_tiles_shading import S, ZV, ITERS, _host, _origins, _scene
from test_shadows_in_oracle import MIN_Z, gather_edges

pytestmark = pytest.mark.gpu


def _light(tw, ep, dx, dy, lp, size=S, no_shadow=0):
    sp = tw.ShadowParams()
    sp.x_scene_size = sp.y_scene_size = 0.5
    sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * size, float(ep.zmin), float(ep.zmax), no_shadow
    for d in range(3):
        sp.lpos[d] = lp[d]
    return sp


SUN, MOON = (3.0, 2.0, 0.15), (-2.0, -4.0, 0.2)


def _grid(side):
    return np.array([(tx, ty) for ty in range(side) for tx in range(side)], np.int32)


def _outs(buf, nt, zv, ao):
    return dict(zvals=buf((nt, zv, zv), "f4"), normals=buf((nt, zv - 1, zv - 1, 4), "u1"), ao=buf((nt, zv - 1, zv - 1), "u1") if ao else None)


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("side,mode,ao", [(3, 0, False), (3, 1, False), (3, 4, False), (3, 4, True), (70, 0, False), (70, 1, False), (70, 4, False), (70, 4, True)])
def test_launch_shadows_equals_batch_ex(tw, scene, ctx, beq, side, mode, ao, where):
    """Two lights; 70x70 = 4900 tiles is the chunked, heaviest-first path. The moon takes incoming rows for the tiles on the block's light side."""
    import torch
    cfg, hp, ep, dx, dy = _scene(scene, ctx, mode)
    origins = _origins(side)
    nt, hd, wpz_max = len(origins), 0.5 * (dx + dy), float(ep.water_plane_z)
    txy = _grid(side)
    dt = {"f4": torch.float32, "u1": torch.uint8}

    def buf(shape, t):
        return torch.empty(shape, dtype=dt[t], device="cuda") if where == "device" else torch.empty(shape, dtype=dt[t]).pin_memory()

    def run(lights):
        o = _outs(buf, nt, ZV, ao)
        mm, b, mnz = np.empty((nt, 2), np.float32), (tw.TileBounds * nt)(), np.empty(nt, np.float32)
        ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, o["zvals"], mm=mm, bounds=b, normals=o["normals"], min_normal_z=mnz,
                                wpz_max=wpz_max, size=S, ao=o["ao"], half_dxy=hd if ao else None,
                                tile_xy=txy if lights else None, lights=lights)
        assert ctx.create_tiles_poll(wait=True)
        return o, mm, b, mnz, ctx.last_erosion_steps
    o0, mm0, b0, mnz0, steps0 = run(None)
    rng = np.random.default_rng(side + 10 * mode)
    moon_sp = _light(tw, ep, dx, dy, MOON)
    in_x = rng.uniform(float(ep.zmin), float(ep.zmax), (nt, ZV)).astype(np.float32)
    in_x[rng.random((nt, ZV)) < 0.3] = MIN_Z
    in_y = np.full((nt, ZV), MIN_Z, np.float32)
    in_y[:, ::2] = 0.25
    lights = []
    for sp, six, siy in ((_light(tw, ep, dx, dy, SUN), None, None), (moon_sp, in_x, in_y)):
        lights.append(tw.Light(sp, buf((nt, ZV, ZV), "u1"), buf((nt, ZV), "f4"), buf((nt, ZV), "f4"),
                               six if (six is None or where == "pinned") else torch.from_numpy(six).cuda(), siy))
    o1, mm1, b1, mnz1, steps1 = run(lights)
    assert steps1 == steps0
    for k in ("zvals", "normals", "ao"):
        if o0[k] is not None:
            assert np.array_equal(_host(o0[k]).view(np.uint8), _host(o1[k]).view(np.uint8)), k
    assert beq(mm0, mm1) == 0 and beq(mnz0, mnz1) == 0 and all(bytes(x) == bytes(y) for x, y in zip(b0, b1))
    z = _host(o1["zvals"])
    shadowed = 0
    for L in lights:
        m, ox, oy = ctx.tile_shadows(z, txy, L.sp, sh_in_x=None if L.sh_in_x is None else _host(L.sh_in_x), sh_in_y=L.sh_in_y)
        assert np.array_equal(_host(L.smask), m)
        assert beq(_host(L.sh_out_x), ox) == 0 and beq(_host(L.sh_out_y), oy) == 0
        shadowed += int((m == 2).sum())
    assert shadowed > 0


@pytest.mark.parametrize("mode", [1, 4])
def test_special_lights_and_rows_from_an_earlier_job(tw, scene, ctx, beq, mode):
    """Two jobs over one 4x6 block, the half nearer the sun first: the second takes its incoming rows from the first job's sh_out, and its results are the
    whole block's. Also a no_shadow light, a light below zmin (all shadowed) and a light straight overhead (no rays)."""
    cfg, hp, ep, dx, dy = _scene(scene, ctx, mode)
    side = 4
    sun = _light(tw, ep, dx, dy, (1.0, 4.0, 0.12))                       # toward +y: the rows y = 3..5 are nearer the light than y = 0..2
    txy_all = np.array([(tx, ty) for ty in range(6) for tx in range(side)], np.int32)
    origins_all = [(tx * S * 40 - 3000, ty * S * 40 + 500) for tx, ty in txy_all]
    nt_all = len(origins_all)
    a, b = np.arange(nt_all) >= 12, np.arange(nt_all) < 12
    z_all = np.empty((nt_all, ZV, ZV), np.float32)
    outs = {}
    for part, rows in (("a", a), ("b", b)):
        idx = np.nonzero(rows)[0]
        nt = len(idx)
        z = np.empty((nt, ZV, ZV), np.float32)
        m, ox, oy = np.empty((nt, ZV, ZV), np.uint8), np.empty((nt, ZV), np.float32), np.empty((nt, ZV), np.float32)
        ix = iy = None
        if part == "b":
            ix, iy = gather_edges(sun, txy_all[idx], txy_all[a], outs["a"][1], outs["a"][2], ZV)
            print("incoming heights across the cut: %d" % int((ix > MIN_Z).sum()))
        specials = [tw.Light(_light(tw, ep, dx, dy, (3.0, 2.0, 0.3), no_shadow=1), np.empty((nt, ZV, ZV), np.uint8), np.empty((nt, ZV), np.float32), None),
                    tw.Light(_light(tw, ep, dx, dy, (2.0, 1.0, float(ep.zmin) - 1.0)), np.empty((nt, ZV, ZV), np.uint8), None, np.empty((nt, ZV), np.float32)),
                    tw.Light(_light(tw, ep, dx, dy, (0.0, 0.0, 5.0)), np.empty((nt, ZV, ZV), np.uint8), np.empty((nt, ZV), np.float32), np.empty((nt, ZV), np.float32))]
        ctx.create_tiles_launch([origins_all[i] for i in idx], cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, tile_xy=txy_all[idx],
                                lights=[(sun, m, ox, oy, ix, iy)] + specials)
        assert ctx.create_tiles_poll(wait=True)
        z_all[idx] = z
        outs[part] = (m, ox, oy)
        em, eox, eoy = ctx.tile_shadows(z, txy_all[idx], sun, sh_in_x=ix, sh_in_y=iy)
        assert np.array_equal(m, em) and beq(ox, eox) == 0 and beq(oy, eoy) == 0
        for L in specials:
            em, eox, eoy = ctx.tile_shadows(z, txy_all[idx], L.sp)
            assert np.array_equal(L.smask, em)
            assert (L.sh_out_x is None or beq(L.sh_out_x, eox) == 0) and (L.sh_out_y is None or beq(L.sh_out_y, eoy) == 0)
        assert not specials[0].smask.any() and (specials[0].sh_out_x == MIN_Z).all()                  # no_shadow
        assert (specials[1].smask == 2).all()                                                          # below zmin: everything in shadow
        assert not specials[2].smask.any() and (specials[2].sh_out_x == MIN_Z).all() and (specials[2].sh_out_y == MIN_Z).all()   # no rays
    wm, wox, woy = ctx.tile_shadows(z_all, txy_all, sun)                 # the whole block in one batch
    assert np.array_equal(outs["a"][0], wm[a]) and np.array_equal(outs["b"][0], wm[b])
    assert beq(outs["b"][1], wox[b]) == 0 and beq(outs["b"][2], woy[b]) == 0
    assert (wm == 2).any()


def test_launch_shadows_returns_before_the_work_is_done(tw, scene, ctx, beq):
    """4096 tiles of 258^2, 1000 droplets each, AO and two lights into device memory: the launch returns while the device works; tile_xy, the lights
    array handed to the library and the host sh_in rows are overwritten right after it, and the result still equals tw_tile_shadows_batch_ex's."""
    import torch
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(256, 256, 1))
    hp, ep = cfg.height_params(), cfg.erosion_params()
    nt, zv = 4096, 258
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    origins = np.array([((t % 64) * 256, (t // 64) * 256) for t in range(nt)], np.int32)
    txy = np.ascontiguousarray(origins // 256)
    rng = np.random.default_rng(3)
    in_y = rng.uniform(float(ep.zmin), float(ep.zmax), (nt, zv)).astype(np.float32)
    in_y[rng.random((nt, zv)) < 0.5] = MIN_Z
    in_y_copy, txy_copy = in_y.copy(), txy.copy()
    sps = [_light(tw, ep, dx, dy, SUN, 256), _light(tw, ep, dx, dy, MOON, 256)]
    z = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
    ao = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8, device="cuda")
    lights = [tw.Light(sp, torch.empty((nt, zv, zv), dtype=torch.uint8, device="cuda"), torch.empty((nt, zv), device="cuda"), torch.empty((nt, zv), device="cuda"),
                       None, in_y if i == 1 else None) for i, sp in enumerate(sps)]
    t0 = time.perf_counter()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, ao=ao, half_dxy=0.5 * (dx + dy), tile_xy=txy, lights=lights)
    t_launch = time.perf_counter() - t0
    txy[:] = 7                                                # all copied during the launch
    in_y[:] = 1.0e3
    arr = ctx._tiles_job[12][-1]                              # the tw_tile_light array the library was given
    for i in range(len(arr)):
        arr[i].sp.lpos[0], arr[i].sp.lpos[1] = -arr[i].sp.lpos[0], 0.0
    ready_at_once = ctx.create_tiles_poll(wait=False)
    while not ctx.create_tiles_poll(wait=False):
        pass
    print("launch blocked the host for %.3f ms; ready after %.1f ms" % (1e3 * t_launch, 1e3 * (time.perf_counter() - t0)))
    assert not ready_at_once
    shadowed = 0
    for i, (sp, L) in enumerate(zip(sps, lights)):
        m = torch.empty_like(L.smask)
        _, ox, oy = ctx.tile_shadows(z, txy_copy, sp, out=m, sh_in_y=in_y_copy if i == 1 else None)
        assert torch.equal(L.smask, m)
        assert beq(L.sh_out_x.cpu().numpy(), ox) == 0 and beq(L.sh_out_y.cpu().numpy(), oy) == 0
        shadowed += int((m == 2).sum())
    assert shadowed > 0

