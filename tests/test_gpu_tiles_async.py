"""GPU: tw_create_tiles_launch / tw_create_tiles_poll - a frame's new tiles (heights, erosion, z range, sub-block bounds, normal map) enqueued without
waiting for the device. Every output must equal tw_create_zvals_batch + tw_tile_bounds_batch + tw_tile_normals_batch bit for bit; the launch must
return before the work is done; a pending job must complete before any other call reuses the context."""
import time

import numpy as np
import pytest

from cases import convert, HM_CFG

pytestmark = pytest.mark.gpu

S, ZV = 16, 18


def _scene(tw, scene, ctx, mode):
    cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1), scene_size=(0.5, 0.5, 4.0))
    if mode == 0:
        ctx.set_sine_params(cfg.sine_params())
    return cfg, cfg.height_params(), cfg.erosion_params(), float(cfg.dx_val), float(cfg.dy_val)


def _origins(side):
    return [(tx * S * 40 - 3000, ty * S * 40 + 500) for ty in range(side) for tx in range(side)]   # spread out: ocean and mountain tiles


def _outputs(tw, nt, where):
    """zvals / normal maps in device memory or in pinned host memory; mm, bounds and min_normal_z are host arrays."""
    import torch
    if where == "device":
        z = torch.empty((nt, ZV, ZV), dtype=torch.float32, device="cuda")
        n = torch.empty((nt, ZV - 1, ZV - 1, 4), dtype=torch.uint8, device="cuda")
    else:
        z = torch.empty((nt, ZV, ZV), dtype=torch.float32).pin_memory()
        n = torch.empty((nt, ZV - 1, ZV - 1, 4), dtype=torch.uint8).pin_memory()
    return z, n, np.empty((nt, 2), np.float32), (tw.TileBounds * nt)(), np.empty(nt, np.float32)


def _assert_bounds_equal(tw, beq, g, e, t):
    for f, typ in tw.TileBounds._fields_:
        if typ is tw.C.c_int32:
            assert getattr(g, f) == getattr(e, f), (t, f)
        else:
            assert beq(np.array(getattr(g, f), np.float32), np.array(getattr(e, f), np.float32)) == 0, (t, f)


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("side,mode", [(3, 1), (3, 0), (3, 4), (70, 1), (70, 4), (70, 0)])
def test_launch_poll_equals_synchronous_calls(tw, scene, oracle, ctx, beq, side, mode, where):
    """70x70 = 4900 tiles is the chunked, heaviest-first path (modes 1 and 4; sine mode generates the batch up front)."""
    cfg, hp, ep, dx, dy = _scene(tw, scene, ctx, mode)
    origins = _origins(side)
    nt = len(origins)
    wpz_max = float(ep.water_plane_z)
    exp_z, exp_mm = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, ZV, hp, 60, ep, ep.zmin, want_minmax=True)
    steps = ctx.last_erosion_steps
    exp_b = ctx.tile_bounds(exp_z, wpz_max, dx, dy, S)
    exp_n, exp_mnz = ctx.tile_normals(exp_z, dx, dy)

    z, n, mm, b, mnz = _outputs(tw, nt, where)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 60, ep, ep.zmin, z, mm=mm, bounds=b, normals=n, min_normal_z=mnz, wpz_max=wpz_max, size=S)
    assert ctx.create_tiles_poll(wait=True)
    assert ctx.last_erosion_steps == steps
    assert beq(_host(z), exp_z) == 0
    assert beq(mm, exp_mm) == 0
    assert np.array_equal(_host(n), exp_n) and beq(mnz, exp_mnz) == 0
    for t, (g, e) in enumerate(zip(b, exp_b)):
        _assert_bounds_equal(tw, beq, g, e, t)
    # three tiles against the oracle: the reference's apply_erosion, tile bounds and normal map of the un-eroded heights
    raw = ctx.heightgen_tiles(origins, cfg.mesh_size, dx, dy, ZV, hp)
    zh = _host(z)
    for t in (0, nt // 2, nt - 1):
        zc, _ = oracle.apply_erosion(raw[t], ep.zmin, 60, convert(ep, oracle.ErosionParams))
        assert beq(zh[t], zc) == 0
        assert bytes(b[t]) == bytes(oracle.tile_bounds(zc[None], wpz_max, dx, dy, S)[0])
        on, om = oracle.tile_normals(zc[None], dx, dy)
        assert np.array_equal(_host(n)[t], on[0]) and beq(mnz[t:t + 1], om) == 0


@pytest.mark.parametrize("mode", [1, 0])
def test_partial_outputs_and_no_erosion(tw, scene, ctx, beq, mode):
    """Only the requested outputs are produced; erosion_iters == 0 is the height fill of tw_heightgen_tiles."""
    cfg, hp, ep, dx, dy = _scene(tw, scene, ctx, mode)
    origins = _origins(4)
    raw, raw_mm = ctx.heightgen_tiles(origins, cfg.mesh_size, dx, dy, ZV, hp, want_minmax=True)
    z = np.empty_like(raw)
    mm = np.empty((len(origins), 2), np.float32)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 0, ep, ep.zmin, z, mm=mm)
    assert ctx.create_tiles_poll(wait=True)
    assert beq(z, raw) == 0 and beq(mm, raw_mm) == 0 and ctx.last_erosion_steps == 0
    exp_n, _ = ctx.tile_normals(raw, dx, dy)
    n = np.empty_like(exp_n)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 0, None, 0.0, z, normals=n)
    ctx.create_tiles_poll(wait=True)
    assert np.array_equal(n, exp_n)


def test_launch_returns_before_the_work_is_done(tw, scene, ctx, beq):
    """16384 tiles of 258^2 with 1000 droplets each (BASELINE config 5 shape, a quarter of it): the launch returns while the device works, the
    origins may be overwritten right after it, and the result equals the synchronous call's."""
    import torch
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(256, 256, 1))
    hp, ep = cfg.height_params(), cfg.erosion_params()
    nt, zv = 16384, 258
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    origins = np.array([((t % 128) * 256, (t // 128) * 256) for t in range(nt)], np.int32)
    exp = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
    _, exp_mm = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, out=exp, want_minmax=True)
    steps = ctx.last_erosion_steps
    got = torch.empty_like(exp)
    mm = np.empty((nt, 2), np.float32)
    t0 = time.perf_counter()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, got, mm=mm)
    t_launch = time.perf_counter() - t0
    origins[:] = -12345                                   # the library copied them during the launch
    ready_at_once = ctx.create_tiles_poll(wait=False)
    polls = 1
    while not ctx.create_tiles_poll(wait=False):
        polls += 1
    t_ready = time.perf_counter() - t0
    print("launch blocked the host for %.3f ms; ready after %.1f ms (%d polls)" % (1e3 * t_launch, 1e3 * t_ready, polls))
    assert not ready_at_once
    assert ctx.last_erosion_steps == steps
    assert torch.equal(got.view(torch.int32), exp.view(torch.int32)) and beq(mm, exp_mm) == 0


def test_pending_job_completes_before_other_calls(tw, scene, ctx, beq):
    """One job per context: tw_minmax_f32 after a tile launch, and a tile launch after tw_heightgen_2d_launch, both see the earlier job finished."""
    cfg, hp, ep, dx, dy = _scene(tw, scene, ctx, 1)
    origins = _origins(30)
    exp_z, exp_mm = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, ZV, hp, 200, ep, ep.zmin, want_minmax=True)
    steps = ctx.last_erosion_steps
    import torch
    z = torch.empty((len(origins), ZV, ZV), dtype=torch.float32, device="cuda")
    mm = np.empty((len(origins), 2), np.float32)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 200, ep, ep.zmin, z, mm=mm)
    lo, hi = ctx.minmax(z)                                 # completes the tile job first, then reads its output
    assert (lo, hi) == (float(exp_z.min()), float(exp_z.max()))
    assert beq(mm, exp_mm) == 0 and ctx.last_erosion_steps == steps
    assert ctx.create_tiles_poll(wait=False)              # nothing pending any more
    assert beq(z.cpu().numpy(), exp_z) == 0
    # a pending 2-D grid, then a tile launch
    g = cfg.heightmap_grid(1024, 768)
    exp_grid, exp_gmm = ctx.heightgen_2d(g, hp, want_minmax=True)
    grid = torch.empty((768, 1024), dtype=torch.float32).pin_memory()
    gmm = tw.MinMax()
    ctx.heightgen_2d_launch(g, hp, 1, 0, grid, gmm)
    z2 = np.empty_like(exp_z)
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 200, ep, ep.zmin, z2)
    assert beq(grid.numpy(), exp_grid) == 0 and (gmm.zmin, gmm.zmax) == exp_gmm   # collected by the tile launch
    assert ctx.create_tiles_poll(wait=True)
    assert beq(z2, exp_z) == 0 and ctx.last_erosion_steps == steps
