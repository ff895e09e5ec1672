"""GPU: tw_set_heightmap + tw_create_tiles_launch_hmap - the asynchronous tile job with heights from the context's heightmap image. Every output must equal,
bit for bit, the synchronous chain it replaces: tw_heightmap_sample_tiles, tw_erode_tiles(min_zval_all = min_zval), per-tile min/max, tw_tile_bounds_batch,
tw_tile_normals_batch, tw_tile_weights_batch and tw_tile_shadows_batch_ex per light."""
import ctypes as C
import time

import numpy as np
import pytest

from cases import convert, HM_CFG
from test_gpu_tiles_shading import S, ZV, ITERS, _host, _weights_case
from test_gpu_tiles_shadows import SUN, MOON, _light
from test_shadows_in_oracle import MIN_Z

pytestmark = pytest.mark.gpu


def _terrain(tw, scene, ctx, n=1024):
    """A 16-bit terrain image of n^2 texels from tw_proc_gen_heightmap and a mirror-edge sampler scaled from its tw_heightmap_info: the sampled heights are
    the terrain's, so the erosion parameters' water level lies inside their range."""
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1), scene_size=(0.5, 0.5, 4.0))
    ctx.set_sine_params(cfg.sine_params())           # the weights texture's jitter noise
    hp, ep = cfg.height_params(), cfg.erosion_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    data16, info, _ = ctx.proc_gen_heightmap(n, n, dx, dy, hp, 0, ep)
    hs = tw.HmapSampler(n, n, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), info.mesh_file_scale, info.mesh_file_tz, hp.mesh_scale_z_inv)
    return cfg, hp, ep, dx, dy, data16.reshape(n, n, 2), hs


def _expected(ctx, img, hs, origins, zv, iters, ep):
    raw = ctx.heightmap_sample_tiles(img, hs, origins, zv)
    z = raw.copy()
    ctx.erode_tiles(z, iters, ep, min_zval_all=ep.zmin)
    return raw, z, ctx.last_erosion_steps


@pytest.mark.parametrize("where", ["host", "pinned", "device"])
@pytest.mark.parametrize("zv", [34, 130])
def test_zvals_equal_the_oracle(tw, oracle, ctx, beq, zv, where):
    """No erosion: every edge mode and both sampling branches (nearest texel, bilinear below mesh_scale 1), origins inside and outside the image."""
    import torch
    rng = np.random.default_rng(zv)
    img = rng.integers(0, 256, (300, 257, 2), dtype=np.uint8)
    origins = [(int(x), int(y)) for x, y in rng.integers(-900, 900, (40, 2))] + [(-10, -20), (100, 130)]
    nt = len(origins)
    ctx.set_heightmap(img)
    for edge in (0, 1, 2):
        for ms in (1.0, 0.45, 2.2):
            hs = tw.HmapSampler(257, 300, edge, ms, 0.0012, 1.7, -0.3, 0.8)
            exp = oracle.hmap_sample_tiles(img, convert(hs, oracle.HmapSampler), origins, zv)
            if where == "device":
                z = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
            else:
                z = torch.empty((nt, zv, zv), dtype=torch.float32).pin_memory() if where == "pinned" else np.empty((nt, zv, zv), np.float32)
            mm = np.empty((nt, 2), np.float32)
            ctx.create_tiles_launch(origins, (S, S), 0.0625, 0.0625, zv, None, 0, None, 0.0, z, mm=mm, hmap=hs)
            assert ctx.create_tiles_poll(wait=True)
            assert ctx.last_erosion_steps == 0
            zh = _host(z)
            assert beq(zh, exp) == 0, (edge, ms)
            assert beq(mm, np.stack([exp.reshape(nt, -1).min(1), exp.reshape(nt, -1).max(1)], 1)) == 0


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("side", [3, 70])
def test_job_equals_synchronous_chain(tw, scene, oracle, ctx, beq, side, where):
    """Erosion, z range, bounds, normals, weights and two lights' shadows; 70x70 = 4900 tiles is the chunked, heaviest-first path whose coarse pre-pass
    samples the image. The sun takes host sh_in rows, the moon device rows."""
    import torch
    cfg, hp, ep, dx, dy, img, hs = _terrain(tw, scene, ctx)
    step = 300 if side == 3 else S
    txy = np.array([(tx, ty) for ty in range(side) for tx in range(side)], np.int32)
    origins = [(int(tx) * step - side * step // 2, int(ty) * step - side * step // 2 - 40) for tx, ty in txy]
    nt, wpz_max = len(origins), float(ep.water_plane_z)
    raw, exp_z, steps = _expected(ctx, img, hs, origins, ZV, ITERS, ep)
    print("sampled heights %.3f .. %.3f, water at %.3f; %d droplet steps" % (raw.min(), raw.max(), wpz_max, steps))
    assert raw.min() < wpz_max < raw.max() and steps > 0 and beq(raw, exp_z) > 0
    wp, corners = _weights_case(tw, exp_z, S, dx, dy, nt)
    exp_b = ctx.tile_bounds(exp_z, wpz_max, dx, dy, S)
    exp_n, exp_mnz = ctx.tile_normals(exp_z, dx, dy)
    exp_w, exp_f = ctx.tile_weights(exp_z, origins, cfg.mesh_size, dx, dy, hp, wp, corners)
    rng = np.random.default_rng(side)
    in_x = rng.uniform(float(ep.zmin), float(ep.zmax), (nt, ZV)).astype(np.float32)
    in_x[rng.random((nt, ZV)) < 0.3] = MIN_Z
    in_y = np.full((nt, ZV), MIN_Z, np.float32)
    in_y[:, ::2] = 0.25

    def buf(shape, dt):
        return torch.empty(shape, dtype=dt, device="cuda") if where == "device" else torch.empty(shape, dtype=dt).pin_memory()
    lights = [tw.Light(_light(tw, ep, dx, dy, SUN), buf((nt, ZV, ZV), torch.uint8), buf((nt, ZV), torch.float32), buf((nt, ZV), torch.float32), in_x, None),
              tw.Light(_light(tw, ep, dx, dy, MOON), buf((nt, ZV, ZV), torch.uint8), buf((nt, ZV), torch.float32), buf((nt, ZV), torch.float32), None,
                       torch.from_numpy(in_y).cuda())]
    z, n = buf((nt, ZV, ZV), torch.float32), buf((nt, ZV - 1, ZV - 1, 4), torch.uint8)
    w, f = buf((nt, ZV - 1, ZV - 1, 4), torch.uint8), buf((nt,), torch.uint8)
    mm, b, mnz = np.empty((nt, 2), np.float32), (tw.TileBounds * nt)(), np.empty(nt, np.float32)
    ctx.set_heightmap(img)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, mm=mm, bounds=b, normals=n, min_normal_z=mnz, wpz_max=wpz_max, size=S,
                            weights=w, has_any_grass=f, wp=wp, tile_params=corners, tile_xy=txy, lights=lights, hmap=hs)
    assert ctx.create_tiles_poll(wait=True)
    assert ctx.last_erosion_steps == steps
    zh = _host(z)
    assert beq(zh, exp_z) == 0
    assert beq(mm, np.stack([exp_z.reshape(nt, -1).min(1), exp_z.reshape(nt, -1).max(1)], 1)) == 0
    assert all(bytes(g) == bytes(e) for g, e in zip(b, exp_b))
    assert np.array_equal(_host(n), exp_n) and beq(mnz, exp_mnz) == 0
    assert np.array_equal(_host(w), exp_w) and np.array_equal(_host(f), exp_f)
    shadowed = 0
    for L, ix, iy in zip(lights, (in_x, None), (None, in_y)):
        m, ox, oy = ctx.tile_shadows(exp_z, txy, L.sp, sh_in_x=ix, sh_in_y=iy)
        assert np.array_equal(_host(L.smask), m)
        assert beq(_host(L.sh_out_x), ox) == 0 and beq(_host(L.sh_out_y), oy) == 0
        shadowed += int((m == 2).sum())
    assert shadowed > 0
    ep_o = convert(ep, oracle.ErosionParams)
    for t in (0, nt // 2, nt - 1):
        zc, _ = oracle.apply_erosion(raw[t], ep.zmin, ITERS, ep_o)
        assert beq(zh[t], zc) == 0


def test_image_from_host_and_device_pointers(tw, scene, ctx, beq):
    import torch
    cfg, hp, ep, dx, dy, img, hs = _terrain(tw, scene, ctx)
    origins = [(tx * 200 - 500, ty * 200 - 450) for ty in range(4) for tx in range(4)]
    outs = []
    for src in (img, torch.from_numpy(img).cuda()):
        ctx.set_heightmap(src)
        z, n = np.empty((16, ZV, ZV), np.float32), np.empty((16, ZV - 1, ZV - 1, 4), np.uint8)
        ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, normals=n, hmap=hs)
        assert ctx.create_tiles_poll(wait=True)
        outs.append((z, n, ctx.last_erosion_steps))
    assert beq(outs[0][0], outs[1][0]) == 0 and np.array_equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
    _, exp_z, steps = _expected(ctx, img, hs, origins, ZV, ITERS, ep)
    assert beq(outs[0][0], exp_z) == 0 and outs[0][2] == steps


def test_set_heightmap_completes_the_pending_job(tw, scene, ctx, beq):
    """A new image set while a job runs: the job completes first, on the old image; the next job samples the new one."""
    import torch
    cfg, hp, ep, dx, dy, img_a, hs = _terrain(tw, scene, ctx)
    img_b = np.ascontiguousarray(img_a[::-1])               # the same terrain upside down
    origins = [(tx * 130 - 600, ty * 130 - 500) for ty in range(8) for tx in range(8)]
    zv, nt = 130, 64
    _, exp_a, steps_a = _expected(ctx, img_a, hs, origins, zv, 1000, ep)
    _, exp_b, steps_b = _expected(ctx, img_b, hs, origins, zv, 1000, ep)
    assert beq(exp_a, exp_b) > 0
    ctx.set_heightmap(img_a)
    z = torch.empty((nt, zv, zv), dtype=torch.float32).pin_memory()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, hmap=hs)
    ctx.set_heightmap(img_b)
    assert tw.lib.tw_create_tiles_poll(ctx._h, 0) == tw.TW_OK                  # nothing pending any more
    assert beq(_host(z), exp_a) == 0 and ctx.last_erosion_steps == steps_a
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, hmap=hs)
    assert ctx.create_tiles_poll(wait=True)
    assert beq(_host(z), exp_b) == 0 and ctx.last_erosion_steps == steps_b


def test_launch_hmap_returns_before_the_work_is_done(tw, scene, ctx, beq):
    """16384 tiles of 258^2, 1000 droplets each, into device memory: the launch returns while the device works, and origins overwritten right after it
    do not change the result."""
    import torch
    cfg, hp, ep, dx, dy, img, hs = _terrain(tw, scene, ctx, n=2048)
    nt, zv = 16384, 258
    origins = np.array([((t % 128) * 256 - 16384, (t // 128) * 256 - 16384) for t in range(nt)], np.int32)
    exp_z = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
    ctx.heightmap_sample_tiles(img, hs, origins, zv, out=exp_z)
    ctx.erode_tiles(exp_z, 1000, ep, min_zval_all=ep.zmin)
    steps = ctx.last_erosion_steps
    ctx.set_heightmap(img)
    z = torch.empty_like(exp_z)
    mm = np.empty((nt, 2), np.float32)
    t0 = time.perf_counter()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, mm=mm, hmap=hs)
    t_launch = time.perf_counter() - t0
    origins[:] = -12345
    ready_at_once = ctx.create_tiles_poll(wait=False)
    while not ctx.create_tiles_poll(wait=False):
        pass
    print("launch blocked the host for %.3f ms; ready after %.1f ms" % (1e3 * t_launch, 1e3 * (time.perf_counter() - t0)))
    assert not ready_at_once
    assert ctx.last_erosion_steps == steps
    assert torch.equal(z.view(torch.int32), exp_z.view(torch.int32))
    assert np.array_equal(mm[:, 0], exp_z.amin(dim=(1, 2)).cpu().numpy()) and np.array_equal(mm[:, 1], exp_z.amax(dim=(1, 2)).cpu().numpy())


def test_argument_errors(tw, ctx):
    """Each refusal returns its status with nothing enqueued: the next poll reports no pending job."""
    L, h = tw.lib, ctx._h
    hp, ep = tw.HeightParams(), tw.ErosionParams()
    hp.gen_mode = 1
    nt, zv = 2, 18
    org = np.array([[0, 0], [16, 0]], np.int32)
    z = np.empty((nt, zv, zv), np.float32)
    nrm = np.empty((nt, zv - 1, zv - 1, 4), np.uint8)
    img = np.zeros((40, 30, 2), np.uint8)
    hs = tw.HmapSampler(30, 40, 2, 1.0, 0.0008, 1.0, 0.0, 1.0)
    wp = tw.WeightParams()
    for i in range(5):
        wp.tex_class[i] = i
    wp.zmin, wp.zmax = -1.0, 1.0

    def launch(sampler, outs, shading=None, p=hp, zvsize=zv):
        return L.tw_create_tiles_launch_hmap(h, C.byref(sampler) if sampler is not None else None, tw._ptr(org), nt, 16, 16, 0.0625, 0.0625, zvsize,
                                             C.byref(p) if p is not None else None, 0, C.byref(ep), 0.0, 0.0, 16, C.byref(outs),
                                             C.byref(shading) if shading is not None else None, None)

    def refused(status, *args, **kw):
        assert launch(*args, **kw) == status
        assert L.tw_last_error(h)
        assert L.tw_create_tiles_poll(h, 0) == tw.TW_OK
    outs = tw.TileOutputs(tw._ptr(z), None, None, None, None)
    ctx.set_heightmap(None)
    refused(tw.TW_ERR_STATE, hs, outs)                                                          # no image
    assert L.tw_set_heightmap(h, tw._ptr(img), 0, 40) == tw.TW_ERR_ARG
    assert L.tw_set_heightmap(h, tw._ptr(img), 30, -1) == tw.TW_ERR_ARG
    ctx.set_heightmap(img)
    refused(tw.TW_ERR_ARG, None, outs)                                                          # no sampler
    refused(tw.TW_ERR_ARG, tw.HmapSampler(31, 40, 2, 1.0, 0.0008, 1.0, 0.0, 1.0), outs)        # sized unlike the image
    refused(tw.TW_ERR_ARG, tw.HmapSampler(30, 41, 2, 1.0, 0.0008, 1.0, 0.0, 1.0), outs)
    refused(tw.TW_ERR_ARG, tw.HmapSampler(30, 40, 3, 1.0, 0.0008, 1.0, 0.0, 1.0), outs)        # edge_mode
    refused(tw.TW_ERR_ARG, tw.HmapSampler(30, 40, -1, 1.0, 0.0008, 1.0, 0.0, 1.0), outs)
    ao = np.empty((nt, zv - 1, zv - 1), np.uint8)
    refused(tw.TW_ERR_ARG, hs, outs, tw.TileShading(0.0625, None, None, tw._ptr(ao), None, None))                     # AO
    w, tp = np.empty((nt, zv - 1, zv - 1, 4), np.uint8), np.zeros((nt, 8), np.float32)
    refused(tw.TW_ERR_ARG, hs, outs, tw.TileShading(0.0, C.cast(C.pointer(wp), C.c_void_p), tw._ptr(tp), None, tw._ptr(w), None), p=None)  # weights without p
    refused(tw.TW_ERR_ARG, hs, tw.TileOutputs(tw._ptr(z), None, None, None, tw._ptr(np.empty(nt, np.float32))))        # min_normal_z without normals
    refused(tw.TW_ERR_ARG, hs, tw.TileOutputs(None, None, None, tw._ptr(nrm), None))                                    # no zvals
    refused(tw.TW_ERR_ARG, hs, outs, zvsize=0)
    assert launch(hs, outs, p=None) == tw.TW_OK                                                 # heights only: p is not needed
    assert ctx.create_tiles_poll(wait=True)
    ctx.set_heightmap(None)
