"""GPU: tw_update_heightmap (edits of the context's heightmap image that complete no job) and re-creating the tiles tw_hmap_tiles_touched names.
The image is read back exactly by sampling tiles that cover it with mesh_scale 1, clamp edges and unit scales: each cell is then hi + lo/256 of one texel."""
import time

import numpy as np
import pytest

from cases import HM_CFG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ectx(tw):
    c = tw.Context(0)
    yield c
    c.close()


def readback(tw, c, W, H, zv=128):
    """The context's image, decoded from a heightmap tile job on c (uint8 [H, W, 2])."""
    hs = tw.HmapSampler(W, H, 0, 1.0, 1.0, 1.0, 0.0, 1.0)
    nx, ny = -(-W // zv), -(-H // zv)
    org = np.array([(tx * zv - W // 2, ty * zv - H // 2) for ty in range(ny) for tx in range(nx)], np.int32)
    z = np.empty((len(org), zv, zv), np.float32)
    c.create_tiles_launch(org, (zv, zv), 1.0, 1.0, zv, None, 0, None, 0.0, z, hmap=hs)
    assert c.create_tiles_poll(wait=True)
    full = z.reshape(ny, nx, zv, zv).transpose(0, 2, 1, 3).reshape(ny * zv, nx * zv)[:H, :W]
    v = (full.astype(np.float64) * 256).astype(np.uint32)
    return np.stack([(v & 255).astype(np.uint8), (v >> 8).astype(np.uint8)], axis=2)


def edit(rng, img, rects, lo=0, hi=256):
    for x, y, w, h in rects:
        img[y:y + h, x:x + w] = rng.integers(lo, hi, (h, w, 2), dtype=np.uint8)


def test_edits_equal_the_host_image(tw, ectx):
    rng = np.random.default_rng(1)
    W, H = 7168, 640
    img = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
    ectx.set_heightmap(img)
    batches = [[(0, 0, 1, 1)], [(W - 1, H - 1, 1, 1)], [(0, 17, W, 1), (0, H - 1, W, 1)], [(5, 0, 1, H), (W - 1, 0, 1, H)],
               [(0, 0, 3, 2), (W - 3, 0, 3, 2), (0, H - 2, 3, 2), (W - 3, H - 2, 3, 2)],
               [(x, int(rng.integers(0, H - 40)), 7085, 33) for x in (0, 1, 7, 8, 13, 83)],
               [(int(rng.integers(0, W - 300)), int(rng.integers(0, H - 200)), int(rng.integers(1, 300)), int(rng.integers(1, 200))) for _ in range(20)]]
    for rects in batches:
        edit(rng, img, rects)
        ectx.update_heightmap(img, rects)
        assert np.array_equal(readback(tw, ectx, W, H), img), rects
    edit(rng, img, [(0, 0, W, H)])
    ectx.update_heightmap(img, [(0, 0, W, H)])
    ectx.update_heightmap(img, [])                                        # nothing to do
    assert np.array_equal(readback(tw, ectx, W, H), img)
    for _ in range(1000):                                                 # staging reuse: the host image changes right after each call
        w, h = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        r = [(int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h)]
        edit(rng, img, r)
        ectx.update_heightmap(img, r)
    assert np.array_equal(readback(tw, ectx, W, H), img)
    sub = np.ascontiguousarray(img[:, :4000])                             # a source pitch narrower than the image, covering only the rects
    edit(rng, sub, [(100, 50, 3900, 70)])
    ectx.update_heightmap(sub, [(100, 50, 3900, 70)])
    img[:, :4000] = sub
    assert np.array_equal(readback(tw, ectx, W, H), img)


def _terrain(tw, scene, c, n):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(32, 32, 1), scene_size=(0.5, 0.5, 4.0))
    c.set_sine_params(cfg.sine_params())
    hp, ep = cfg.height_params(), cfg.erosion_params()
    data16, info, _ = c.proc_gen_heightmap(n, n, float(cfg.dx_val), float(cfg.dy_val), hp, 0, ep)
    hs = tw.HmapSampler(n, n, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), info.mesh_file_scale, info.mesh_file_tz, hp.mesh_scale_z_inv)
    return cfg, hp, ep, data16.reshape(n, n, 2).copy(), hs, info


def _bump(img, rects, d=3):
    """A brush stroke: the high byte of the rects' texels raised by d (kept below 255)."""
    for x, y, w, h in rects:
        img[y:y + h, x:x + w, 1] = np.minimum(img[y:y + h, x:x + w, 1].astype(np.int32) + d, 254).astype(np.uint8)


def _tiles(tw, c, cfg, ep, hs, org, zv, iters):
    """One heightmap tile job on c, launched, not polled: its zvals buffer."""
    import torch
    z = torch.empty((len(org), zv, zv), dtype=torch.float32).pin_memory()
    c.create_tiles_launch(org, cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), zv, None, iters, ep, ep.zmin, z, hmap=hs)
    return z


def test_ordering_on_a_pool(tw, scene, ectx):
    """A long frame launched before the edit sees the old image and is still running when the edit returns; frames after it see the new one."""
    n, zv = 1024, 65
    cfg, hp, ep, img0, hs, _ = _terrain(tw, scene, ectx, n)
    pool = [ectx.shared() for _ in range(3)]
    org = np.array([(-100, -80)], np.int32)
    org2 = np.array([(-100, -80), (400, 300), (-480, 200)], np.int32)
    rects = [(n // 2 - 120, n // 2 - 100, 80, 90), (900, 500, 60, 60)]
    img1 = img0.copy()
    _bump(img1, rects)
    # A: 1e6 droplets with the water plane below the terrain, so that no droplet stops in the sea and the frame runs for seconds
    ep_a = tw.ErosionParams(*[getattr(ep, f) for f, _ in ep._fields_])
    ep_a.water_plane_z = float(ep.zmin) - 100.0
    # references: each job alone, after tw_set_heightmap of the image it must see
    ectx.set_heightmap(img0)
    t0 = time.perf_counter()
    ref_a = _tiles(tw, pool[0], cfg, ep_a, hs, org, zv, 1000000)
    assert pool[0].create_tiles_poll(wait=True)
    assert time.perf_counter() - t0 > 0.5
    ectx.set_heightmap(img1)
    ref_b = _tiles(tw, pool[1], cfg, ep, hs, org2, zv, 200)
    ref_r = _tiles(tw, ectx, cfg, ep, hs, org2, zv, 200)                  # also sizes the root's scratch, so the launch below reallocates nothing
    assert pool[1].create_tiles_poll(wait=True) and ectx.create_tiles_poll(wait=True)
    assert np.array_equal(ref_r.numpy(), ref_b.numpy())
    # the same jobs around one edit
    ectx.set_heightmap(img0)
    a = _tiles(tw, pool[0], cfg, ep_a, hs, org, zv, 1000000)
    img = img0.copy()
    _bump(img, rects)
    ectx.update_heightmap(img, rects)
    img[:] = 0                                                            # the call copied what it needs
    assert not pool[0].create_tiles_poll(wait=False)                      # the edit completed nothing
    b = _tiles(tw, pool[1], cfg, ep, hs, org2, zv, 200)
    r = _tiles(tw, ectx, cfg, ep, hs, org2, zv, 200)
    assert pool[1].create_tiles_poll(wait=True) and ectx.create_tiles_poll(wait=True) and pool[0].create_tiles_poll(wait=True)
    assert np.array_equal(a.numpy(), ref_a.numpy())
    assert np.array_equal(b.numpy(), ref_b.numpy()) and np.array_equal(r.numpy(), ref_b.numpy())
    ectx.set_heightmap(img0)
    old_b = _tiles(tw, pool[2], cfg, ep, hs, org2, zv, 200)
    assert pool[2].create_tiles_poll(wait=True)
    assert not np.array_equal(old_b.numpy(), ref_b.numpy())              # the edit is visible in those tiles
    for s in pool:
        s.close()


def test_cancel_lets_the_edit_land(tw, scene, ectx):
    n, zv = 1024, 65
    cfg, hp, ep, img0, hs, _ = _terrain(tw, scene, ectx, n)
    s1, s2 = ectx.shared(), ectx.shared()
    org = np.array([(-100, -80)], np.int32)
    rects = [(400, 400, 100, 100)]
    img1 = img0.copy()
    _bump(img1, rects)
    ectx.set_heightmap(img1)
    ref = _tiles(tw, s2, cfg, ep, hs, org, zv, 0)
    assert s2.create_tiles_poll(wait=True)
    ectx.set_heightmap(img0)
    ep_a = tw.ErosionParams(*[getattr(ep, f) for f, _ in ep._fields_])
    ep_a.water_plane_z = float(ep.zmin) - 100.0                          # no droplet stops in the sea: the job runs for seconds
    _tiles(tw, s1, cfg, ep_a, hs, org, zv, 1000000)
    ectx.update_heightmap(img1, rects)
    s1.cancel()
    b = _tiles(tw, s2, cfg, ep, hs, org, zv, 0)
    assert s2.create_tiles_poll(wait=True)
    with pytest.raises(tw.TwCanceled):
        s1.create_tiles_poll(wait=True)
    assert np.array_equal(b.numpy(), ref.numpy())
    assert np.array_equal(readback(tw, ectx, n, n), img1)
    s1.close()
    s2.close()


def test_image_erosion_after_edits(tw, scene, ectx):
    n = 512
    cfg, hp, ep, img0, hs, info = _terrain(tw, scene, ectx, n)
    rng = np.random.default_rng(5)
    rects = [(10, 20, 200, 100), (300, 300, 150, 150), (0, 0, n, 3)]
    img1 = img0.copy()
    _bump(img1, rects)
    iters = 20000
    ectx.set_heightmap(img1)                                              # the chain on the edited image
    ectx.erode_image_launch(info.val_mult, info.val_add, iters, ep)
    assert ectx.create_tiles_poll(wait=True)
    want_steps = ectx.last_erosion_steps
    want = readback(tw, ectx, n, n)
    ectx.set_heightmap(img0)
    ectx.update_heightmap(img1, rects[:2])
    ectx.update_heightmap(img1, rects[2:])
    ectx.erode_image_launch(info.val_mult, info.val_add, iters, ep)
    with pytest.raises(tw.TwError) as e:                                  # no image while the job runs
        ectx.update_heightmap(img0, rects)
    assert e.value.status == tw.TW_ERR_STATE
    assert ectx.create_tiles_poll(wait=True)
    assert ectx.last_erosion_steps == want_steps > 0
    assert np.array_equal(readback(tw, ectx, n, n), want)
    job = ectx.proc_gen_heightmap_launch(n, n, float(cfg.dx_val), float(cfg.dy_val), hp, 0, ep, set_image=True)
    with pytest.raises(tw.TwError) as e:
        ectx.update_heightmap(img0, rects)
    assert e.value.status == tw.TW_ERR_STATE
    assert ectx.create_tiles_poll(wait=True)
    assert np.array_equal(readback(tw, ectx, n, n), img0)                 # the generated image, unchanged by the refused edit
    del job, rng


def test_refusals_enqueue_nothing(tw, ectx):
    import ctypes as C
    import torch
    W, H = 64, 48
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
    ectx.set_heightmap(None)
    with pytest.raises(tw.TwError) as e:
        ectx.update_heightmap(img, [(0, 0, 1, 1)])
    assert e.value.status == tw.TW_ERR_STATE
    ectx.set_heightmap(img)
    s = ectx.shared()
    other = img.copy()
    edit(rng, other, [(0, 0, W, H)])
    L, R = tw.lib, tw.HmapRect
    one = (R * 1)(R(0, 0, 1, 1))
    base = ectx.launch_count
    refused = [
        (s._h, tw._ptr(other), 2 * W, one, 1),                               # a shared context
        (ectx._h, None, 2 * W, one, 1),                                       # NULL src16
        (ectx._h, tw._ptr(other), 2 * W, None, 1),                            # NULL rects
        (ectx._h, tw._ptr(other), 2 * W, (R * 1)(R(0, 0, 0, 3)), 1),          # w <= 0
        (ectx._h, tw._ptr(other), 2 * W, (R * 1)(R(0, 0, 3, -1)), 1),         # h <= 0
        (ectx._h, tw._ptr(other), 2 * W, (R * 1)(R(W - 2, 0, 3, 1)), 1),      # past the right edge
        (ectx._h, tw._ptr(other), 2 * W, (R * 1)(R(0, H - 1, 1, 2)), 1),      # past the bottom edge
        (ectx._h, tw._ptr(other), 2 * W, (R * 1)(R(-1, 0, 2, 1)), 1),         # negative x
        (ectx._h, tw._ptr(other), 2 * W, (R * 2)(R(0, 0, 1, 1), R(0, -1, 1, 1)), 2),   # one bad rect among good ones
        (ectx._h, tw._ptr(other), 2 * 10 - 1, (R * 1)(R(5, 0, 5, 1)), 1),     # src_pitch < 2*(x + w)
    ]
    for args in refused:
        assert L.tw_update_heightmap(*args) == tw.TW_ERR_ARG
    dev = torch.from_numpy(other).cuda()
    assert L.tw_update_heightmap(ectx._h, C.c_void_p(dev.data_ptr()), 2 * W, one, 1) == tw.TW_ERR_ARG
    assert L.tw_update_heightmap(None, tw._ptr(other), 2 * W, one, 1) == tw.TW_ERR_ARG
    assert L.tw_update_heightmap(ectx._h, None, 0, None, 0) == tw.TW_OK
    assert ectx.launch_count == base
    assert np.array_equal(readback(tw, s, W, H), img)
    s.close()


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ms", [0.5, 2.0])
def test_tile_set_round_trip(tw, scene, ectx, mode, ms):
    """16 x 16 heightmap tiles in a set relit for sun and moon; an edit, hmap_tiles_touched, one frame that re-creates the touched tiles and relights what
    that makes stale: every resident tile equals a fresh set built from the edited image and fully relit."""
    S, ZV, n = 32, 34, 300
    cfg, hp, ep, img0, hs0, _ = _terrain(tw, scene, ectx, n)
    hs = tw.HmapSampler(n, n, mode, ms, hs0.h_scale, hs0.mesh_file_scale, hs0.mesh_file_tz, hs0.mesh_scale_z_inv)
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    keys = [(x, y) for y in range(-8, 8) for x in range(-8, 8)]
    org = np.array([(x * S, y * S) for x, y in keys], np.int32)

    def light(lp):
        sp = tw.ShadowParams()
        sp.x_scene_size = sp.y_scene_size = 0.5
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, float(ep.zmin), float(ep.zmax), 0
        sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp
        return sp
    sps = [light((3.0, 2.0, 0.15)), light((-2.0, -3.0, 0.2))]

    def lights(k):
        return [tw.Light(sp, np.empty((k, ZV, ZV), np.uint8), np.empty((k, ZV), np.float32), np.empty((k, ZV), np.float32)) for sp in sps]

    def build(c):
        ts = c.tile_set(ZV, 2)
        ts.create_tiles_launch(org, cfg.mesh_size, dx, dy, None, 0, ep, ep.zmin, np.array(keys, np.int32), relight_xy=np.array(keys, np.int32),
                               lights=lights(len(keys)), hmap=hs)
        assert c.create_tiles_poll(wait=True)
        return ts

    def relight_all(ts):
        ls = lights(len(keys))
        ts.shadows_launch(np.array(keys, np.int32), ls)
        assert ts.ctx.create_tiles_poll(wait=True)
        return [(L.smask.copy(), L.sh_out_x.copy(), L.sh_out_y.copy()) for L in ls]

    ectx.set_heightmap(img0)
    ts = build(ectx)
    rects = [(n // 2 - 40, n // 2 - 30, 50, 40), (0, n - 7, 9, 7)]
    img1 = img0.copy()
    _bump(img1, rects, 9)
    ectx.update_heightmap(img1, rects)
    touched = tw.hmap_tiles_touched(hs, org, ZV, rects)
    assert 0 < touched.sum() < len(keys)
    txy = np.array(keys, np.int32)[touched == 1]
    stale = ts.stale_after(sps, put_xy=txy)
    z = np.empty((len(txy), ZV, ZV), np.float32)
    ts.create_tiles_launch(org[touched == 1], cfg.mesh_size, dx, dy, None, 0, ep, ep.zmin, txy, zvals=z, relight_xy=stale, lights=lights(len(stale)), hmap=hs)
    assert ectx.create_tiles_poll(wait=True)
    assert np.array_equal(z, ectx.heightmap_sample_tiles(img1, hs, org[touched == 1], ZV))
    untouched = org[touched == 0]                                         # what hmap_tiles_touched left alone did not change
    assert np.array_equal(ectx.heightmap_sample_tiles(img0, hs, untouched, ZV).view(np.uint32), ectx.heightmap_sample_tiles(img1, hs, untouched, ZV).view(np.uint32))
    fresh_ctx = tw.Context(0)
    fresh_ctx.set_heightmap(img1)
    fresh = build(fresh_ctx)
    got, want = relight_all(ts), relight_all(fresh)
    for a, b in zip(got, want):
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    ts.close()
    fresh_ctx.close()
