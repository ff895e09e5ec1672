"""GPU: tw_create_tiles_launch_ex - the asynchronous tile job with the AO map and the terrain weights texture. Every output must equal, bit for bit,
separate synchronous calls that do not go through the tile job: tw_create_zvals_batch (CPU gen modes) or the context grids of tw_heightgen_tiles cut
to their interior and eroded with tw_erode_tiles (GPU gen modes, where AO makes the zvals those of the context), then tw_tile_ao_batch,
tw_tile_weights_batch, tw_tile_bounds_batch and tw_tile_normals_batch on those zvals."""
import time

import numpy as np
import pytest

from cases import convert, HM_CFG
from test_weights_host import weight_cases

pytestmark = pytest.mark.gpu

S, ZV, ITERS = 16, 18, 60


def _scene(scene, ctx, mode, S=S):
    cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1), scene_size=(0.5, 0.5, 4.0))
    ctx.set_sine_params(cfg.sine_params())           # the weights texture's jitter noise is sine mode whatever the gen mode
    return cfg, cfg.height_params(), cfg.erosion_params(), float(cfg.dx_val), float(cfg.dy_val)


def _origins(side, S=S):
    return [(tx * S * 40 - 3000, ty * S * 40 + 500) for ty in range(side) for tx in range(side)]   # spread out: ocean and mountain tiles


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


def _weights_case(tw, z, S, dx, dy, nt):
    rng = np.random.default_rng(nt)
    wp = weight_cases(tw.WeightParams, rng, float(z.min()), float(z.max()), S, dx, dy)[3]      # a permuted texture order
    return wp, rng.uniform(-0.2, 1.3, (nt, 8)).astype(np.float32)


def _expected(ctx, cfg, hp, ep, dx, dy, mode, origins, zv, iters):
    """zvals and step count from synchronous calls outside the tile job."""
    if mode >= 3:
        corg = [(x - 36, y - 36) for x, y in origins]
        ctxs = ctx.heightgen_tiles(corg, cfg.mesh_size, dx, dy, zv - 1 + 72, hp)
        z = np.ascontiguousarray(ctxs[:, 36:36 + zv, 36:36 + zv])
        ctx.erode_tiles(z, iters, ep, min_zval_all=ep.zmin)
        return z, ctx.last_erosion_steps
    z = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin)
    return z, ctx.last_erosion_steps


def _expected_ctx_device(ctx, cfg, hp, ep, dx, dy, origins, zv, iters):
    """_expected's GPU-gen-mode zvals for batches that live on the device: context grids of tw_heightgen_tiles cut to their interior, tw_erode_tiles."""
    import torch
    csz = zv - 1 + 72
    ctxs = torch.empty((len(origins), csz, csz), dtype=torch.float32, device="cuda")
    ctx.heightgen_tiles(np.asarray(origins, np.int32) - 36, cfg.mesh_size, dx, dy, csz, hp, out=ctxs)
    z = ctxs[:, 36:36 + zv, 36:36 + zv].contiguous()
    torch.cuda.synchronize()                              # the copy runs on torch's stream, the erosion below on the library's
    del ctxs
    ctx.erode_tiles(z, iters, ep, min_zval_all=ep.zmin)
    return z, ctx.last_erosion_steps


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("side,mode", [(3, 0), (3, 1), (3, 2), (3, 3), (3, 4), (70, 0), (70, 1), (70, 2), (70, 3), (70, 4)])
def test_launch_ex_equals_synchronous_calls(tw, scene, oracle, ctx, beq, side, mode, where):
    """70x70 = 4900 tiles is the chunked, heaviest-first path (four chunks, one context buffer each)."""
    import torch
    cfg, hp, ep, dx, dy = _scene(scene, ctx, mode)
    origins = _origins(side)
    nt = len(origins)
    wpz_max, hd = float(ep.water_plane_z), 0.5 * (dx + dy)
    exp_z, steps = _expected(ctx, cfg, hp, ep, dx, dy, mode, origins, ZV, ITERS)
    wp, corners = _weights_case(tw, exp_z, S, dx, dy, nt)
    exp_ao = ctx.tile_ao(exp_z, origins, cfg.mesh_size, dx, dy, hp, hd)
    exp_w, exp_f = ctx.tile_weights(exp_z, origins, cfg.mesh_size, dx, dy, hp, wp, corners)
    exp_b = ctx.tile_bounds(exp_z, wpz_max, dx, dy, S)
    exp_n, exp_mnz = ctx.tile_normals(exp_z, dx, dy)
    if mode < 3:
        assert beq(exp_z, ctx.create_zvals_ao_batch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, hd)[0]) == 0

    def buf(shape, dt):
        return torch.empty(shape, dtype=dt, device="cuda") if where == "device" else torch.empty(shape, dtype=dt).pin_memory()
    z, n = buf((nt, ZV, ZV), torch.float32), buf((nt, ZV - 1, ZV - 1, 4), torch.uint8)
    ao, w, f = buf((nt, ZV - 1, ZV - 1), torch.uint8), buf((nt, ZV - 1, ZV - 1, 4), torch.uint8), buf((nt,), torch.uint8)
    mm, b, mnz = np.empty((nt, 2), np.float32), (tw.TileBounds * nt)(), np.empty(nt, np.float32)
    tp = torch.from_numpy(corners).cuda() if where == "device" else corners
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, mm=mm, bounds=b, normals=n, min_normal_z=mnz, wpz_max=wpz_max, size=S,
                            ao=ao, weights=w, has_any_grass=f, half_dxy=hd, wp=wp, tile_params=tp)
    assert ctx.create_tiles_poll(wait=True)
    assert ctx.last_erosion_steps == steps
    zh = _host(z)
    assert beq(zh, exp_z) == 0
    assert beq(mm, np.stack([exp_z.reshape(nt, -1).min(1), exp_z.reshape(nt, -1).max(1)], 1)) == 0
    assert all(bytes(g) == bytes(e) for g, e in zip(b, exp_b))
    assert np.array_equal(_host(n), exp_n) and beq(mnz, exp_mnz) == 0
    assert np.array_equal(_host(ao), exp_ao) and ao.min() < 255
    assert np.array_equal(_host(w), exp_w) and np.array_equal(_host(f), exp_f)
    # three tiles against the oracle: the reference's AO flows and the weights texture
    hp_o = convert(hp, oracle.HeightParams)
    for t in (0, nt // 2, nt - 1):
        x1, y1 = origins[t]
        csz = ZV - 1 + 72
        c = oracle.heightgen_2d(oracle.Grid2D(x1 - 36 - S // 2, y1 - 36 - S // 2, dx, dy, csz, csz), hp_o, cfg.sine_params() if mode == 0 else None, 1, 0)
        assert np.array_equal(_host(ao)[t], oracle.tile_ao(zh[t:t + 1], c[None], hd, use_ao_zvals=(mode >= 3))[0])
        rand = oracle.weights_noise(hp_o, cfg.sine_params(), [origins[t]], cfg.mesh_size[:2], dx, dy, S + 1)
        ow, of = oracle.tile_weights(zh[t:t + 1], rand, corners[t:t + 1], convert(wp, oracle.WeightParams))
        assert np.array_equal(_host(w)[t], ow[0]) and int(_host(f)[t]) == int(of[0])


@pytest.mark.parametrize("mode", [1, 4])
def test_partial_requests(tw, scene, ctx, beq, mode):
    """AO only, then weights only (where the GPU gen modes keep tw_create_zvals_batch's zvals)."""
    cfg, hp, ep, dx, dy = _scene(scene, ctx, mode)
    origins = _origins(4)
    nt, hd = len(origins), 0.5 * (dx + dy)
    exp_z, steps = _expected(ctx, cfg, hp, ep, dx, dy, mode, origins, ZV, ITERS)
    z, ao = np.empty_like(exp_z), np.empty((nt, ZV - 1, ZV - 1), np.uint8)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, ao=ao, half_dxy=hd)
    assert ctx.create_tiles_poll(wait=True)
    assert beq(z, exp_z) == 0 and ctx.last_erosion_steps == steps
    assert np.array_equal(ao, ctx.tile_ao(exp_z, origins, cfg.mesh_size, dx, dy, hp, hd))
    plain_z = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin)
    wp, corners = _weights_case(tw, plain_z, S, dx, dy, nt)
    exp_w, _ = ctx.tile_weights(plain_z, origins, cfg.mesh_size, dx, dy, hp, wp, corners)
    w = np.empty_like(exp_w)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, weights=w, wp=wp, tile_params=corners)
    assert ctx.create_tiles_poll(wait=True)
    assert beq(z, plain_z) == 0 and np.array_equal(w, exp_w)


def test_launch_ex_returns_before_the_work_is_done(tw, scene, ctx, beq):
    """4096 tiles of 258^2, 1000 droplets each, with AO and weights: the launch returns while the device works, the origins and tile_params may be
    overwritten right after it, and the result equals the synchronous calls'."""
    import torch
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(256, 256, 1))
    ctx.set_sine_params(cfg.sine_params())
    hp, ep = cfg.height_params(), cfg.erosion_params()
    nt, zv = 4096, 258
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    hd = 0.5 * (dx + dy)
    origins = np.array([((t % 64) * 256, (t // 64) * 256) for t in range(nt)], np.int32)
    exp_z, steps = _expected_ctx_device(ctx, cfg, hp, ep, dx, dy, origins, zv, 1000)
    exp_ao = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8, device="cuda")
    ctx.tile_ao(exp_z, origins, cfg.mesh_size, dx, dy, hp, hd, out=exp_ao)
    wp, corners = _weights_case(tw, exp_z[:16].cpu().numpy(), 256, dx, dy, nt)
    exp_w = torch.empty((nt, zv - 1, zv - 1, 4), dtype=torch.uint8, device="cuda")
    _, exp_f = ctx.tile_weights(exp_z, origins, cfg.mesh_size, dx, dy, hp, wp, corners, out=exp_w)
    z, ao, w = torch.empty_like(exp_z), torch.empty_like(exp_ao), torch.empty_like(exp_w)
    f = np.empty(nt, np.uint8)
    t0 = time.perf_counter()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, ao=ao, weights=w, has_any_grass=f, half_dxy=hd, wp=wp, tile_params=corners)
    t_launch = time.perf_counter() - t0
    origins[:] = -12345                                   # both were copied during the launch
    corners[:] = -7.0
    ready_at_once = ctx.create_tiles_poll(wait=False)
    while not ctx.create_tiles_poll(wait=False):
        pass
    print("launch blocked the host for %.3f ms; ready after %.1f ms" % (1e3 * t_launch, 1e3 * (time.perf_counter() - t0)))
    assert not ready_at_once
    assert ctx.last_erosion_steps == steps
    assert torch.equal(z.view(torch.int32), exp_z.view(torch.int32)) and torch.equal(ao, exp_ao)
    assert torch.equal(w, exp_w) and np.array_equal(f, exp_f)


@pytest.mark.parametrize("mode", [1, 4])
def test_context_buffers_taking_turns(tw, scene, ctx, mode):
    """450 tiles of 1026^2: 4.8 MB of AO context per tile bound a chunk to 149 tiles, so the job runs four chunks on three context buffers: chunk 0
    keeps its own, and the fourth chunk's contexts overwrite the second chunk's once its stream has read them. Device outputs, equal to the synchronous
    calls."""
    import torch
    S, zv, nt, iters = 1024, 1026, 450, 20
    cfg, hp, ep, dx, dy = _scene(scene, ctx, mode, S)
    origins = np.array([((t % 30) * S - 15 * S, (t // 30) * S - 7 * S) for t in range(nt)], np.int32)
    hd = 0.5 * (dx + dy)
    if mode >= 3:
        exp_z, steps = _expected_ctx_device(ctx, cfg, hp, ep, dx, dy, origins, zv, iters)
    else:
        exp_z = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
        ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, out=exp_z)
        steps = ctx.last_erosion_steps
    wp, corners = _weights_case(tw, exp_z[:4].cpu().numpy(), S, dx, dy, nt)
    exp_ao = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8, device="cuda")
    ctx.tile_ao(exp_z, origins, cfg.mesh_size, dx, dy, hp, hd, out=exp_ao)
    exp_w = torch.empty((nt, zv - 1, zv - 1, 4), dtype=torch.uint8, device="cuda")
    _, exp_f = ctx.tile_weights(exp_z, origins, cfg.mesh_size, dx, dy, hp, wp, corners, out=exp_w)
    z, ao, w, f = torch.empty_like(exp_z), torch.empty_like(exp_ao), torch.empty_like(exp_w), np.empty(nt, np.uint8)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, z, ao=ao, weights=w, has_any_grass=f, half_dxy=hd, wp=wp, tile_params=corners)
    assert ctx.create_tiles_poll(wait=True)
    assert ctx.last_erosion_steps == steps
    assert torch.equal(z.view(torch.int32), exp_z.view(torch.int32)) and torch.equal(ao, exp_ao)
    assert torch.equal(w, exp_w) and np.array_equal(f, exp_f)
