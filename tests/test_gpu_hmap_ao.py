"""GPU: tw_hmap_tile_ao_launch - the AO map of heightmap-texture tiles from their final zvals and the context's image. Every AO byte must equal the
composition of two pinned oracle functions: oracle.tile_ao(zvals, oracle.hmap_sample_tiles(image, hs, origins - 36, stride + 72), half_dxy)."""
import ctypes as C

import numpy as np
import pytest

from cases import convert
from test_gpu_tiles_hmap import _terrain
from test_gpu_tiles_shading import S, ZV, ITERS, _host

pytestmark = pytest.mark.gpu

HALF_DXY = 0.03125
W, H = 257, 300


def _expected(oracle, img, hs, origins, zvals, half_dxy=HALF_DXY):
    org = np.asarray(origins, np.int32).reshape(-1, 2)
    zv = zvals.shape[1]
    czv = oracle.hmap_sample_tiles(img, convert(hs, oracle.HmapSampler), org - 36, zv - 1 + 72)
    return oracle.tile_ao(zvals, czv, half_dxy)


def _image(seed):
    """Rough 16-bit terrain: smooth hills plus texel noise, so rays hit at every distance."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    v = 128.0 + 90.0 * np.sin(0.07 * x) * np.cos(0.05 * y) + rng.uniform(-8, 8, (H, W))
    v = np.clip(v, 0, 255.99)
    img = np.empty((H, W, 2), np.uint8)
    img[..., 1] = np.floor(v).astype(np.uint8)
    img[..., 0] = ((v - np.floor(v)) * 256).astype(np.uint8)
    return img


def _origins(stride, ms, seed):
    """Tiles whose windows cross every image edge and corner (for the sampler's scale ms), tiles inside, and tiles entirely off the image."""
    hw, hh = int(W / 2 / ms), int(H / 2 / ms)
    out = [(ox, oy) for ox in (-hw - stride // 2, -stride // 2, hw - stride // 2) for oy in (-hh - stride // 2, -stride // 2, hh - stride // 2)]
    out += [(5000, -7000), (-9000, 300)]
    rng = np.random.default_rng(seed)
    out += [(int(x), int(y)) for x, y in rng.integers(-2 * hw, 2 * hw, (4, 2))]
    return np.array(out, np.int32)


def _zvals(ctx, img, hs, origins, zv, seed):
    """Final zvals: the image's samples with a perturbation, as erosion would leave them (the rays start at the zval and read it inside the tile)."""
    z = ctx.heightmap_sample_tiles(img, hs, origins, zv)
    return (z + np.random.default_rng(seed).uniform(-0.02, 0.02, z.shape).astype(np.float32)).astype(np.float32)


@pytest.mark.parametrize("zv", [2, 3, 17, 130, 200, 258])
def test_ao_equals_oracle(tw, oracle, ctx, beq, zv):
    """Every edge mode, nearest (mesh_scale 1, 2) and bilinear (0.5) sampling; 200 and 258 cut into sub-squares that do not divide the tile."""
    img = _image(zv)
    ctx.set_heightmap(img)
    for edge in (0, 1, 2):
        for ms in (0.5, 1.0, 2.0):
            hs = tw.HmapSampler(W, H, edge, ms, 0.0012, 1.7, -0.3, 0.8)
            origins = _origins(zv - 1, ms, zv + edge)
            z = _zvals(ctx, img, hs, origins, zv, edge)
            exp = _expected(oracle, img, hs, origins, z)
            got = ctx.hmap_tile_ao(hs, origins, z, HALF_DXY)
            assert got.shape == exp.shape and beq(got, exp) == 0, (edge, ms)
            if zv > 3:
                assert len(np.unique(exp)) > 3   # the rays hit at many distances


@pytest.mark.parametrize("where", ["host", "pinned", "device"])
def test_eroded_zvals_in_every_memory(tw, scene, oracle, ctx, beq, where):
    """zvals of an eroding heightmap tile job, passed and returned as host, pinned and device memory."""
    import torch
    cfg, hp, ep, dx, dy, img, hs = _terrain(tw, scene, ctx, n=512)
    ctx.set_heightmap(img)
    origins = np.array([(tx * S - 300, ty * S - 260) for ty in range(6) for tx in range(7)], np.int32)
    nt = len(origins)
    z = np.empty((nt, ZV, ZV), np.float32)
    ctx.create_tiles_launch(origins, (S, S), dx, dy, ZV, None, ITERS, ep, ep.zmin, z, hmap=hs)
    assert ctx.create_tiles_poll(wait=True) and ctx.last_erosion_steps > 0
    exp = _expected(oracle, img, hs, origins, z)
    if where == "device":
        zin, out = torch.from_numpy(z).cuda(), torch.empty((nt, ZV - 1, ZV - 1), dtype=torch.uint8, device="cuda")
    elif where == "pinned":
        zin, out = torch.from_numpy(z).pin_memory(), torch.empty((nt, ZV - 1, ZV - 1), dtype=torch.uint8).pin_memory()
    else:
        zin, out = z, np.empty((nt, ZV - 1, ZV - 1), np.uint8)
    job = ctx.hmap_tile_ao_launch(hs, origins, zin, HALF_DXY, out=out)
    got = _host(job.poll(wait=True))
    assert beq(got, exp) == 0
    assert len(np.unique(exp)) > 3


def test_set_sourced_after_frame_on_shared_contexts(tw, scene, oracle, ctx, beq):
    """A frame into a tile set with no zvals output, then the AO of its tiles from the set on another shared context, launched with no poll in between."""
    cfg, hp, ep, dx, dy, img, hs = _terrain(tw, scene, ctx, n=512)
    ctx.set_heightmap(img)
    a, b = ctx.shared(), ctx.shared()
    ts = ctx.tile_set(ZV, 1)
    try:
        for rnd in range(2):   # the second frame replaces the tiles with others at the same keys
            txy = np.array([(tx, ty) for ty in range(5) for tx in range(6)], np.int32)
            origins = txy * S - np.array([200 + 37 * rnd, 150 - 53 * rnd], np.int32)
            nt = len(origins)
            ts.create_tiles_launch(origins, (S, S), dx, dy, None, ITERS, ep, ep.zmin, txy, hmap=hs, ctx=a)
            job = ts.hmap_ao_launch(txy[::-1], origins[::-1], hs, HALF_DXY, ctx=b)
            got = job.poll(wait=True)
            assert a.create_tiles_poll(wait=True)
            z = np.empty((nt, ZV, ZV), np.float32)
            ctx.create_tiles_launch(origins, (S, S), dx, dy, ZV, None, ITERS, ep, ep.zmin, z, hmap=hs)
            assert ctx.create_tiles_poll(wait=True)
            assert beq(got, ctx.hmap_tile_ao(hs, origins[::-1], z[::-1].copy(), HALF_DXY)) == 0
            assert beq(got, _expected(oracle, img, hs, origins[::-1], z[::-1].copy())) == 0
    finally:
        ts.close()
        a.close()
        b.close()


def test_edits_order_and_touched_tiles(tw, oracle, ctx, beq):
    """A job launched before tw_update_heightmap sees the old image, one launched after it the new one; every tile whose AO the edit changed is flagged
    by the window form of tw_hmap_tiles_touched, and every unflagged tile's AO is unchanged."""
    img = _image(7)
    ctx.set_heightmap(img)
    sh = ctx.shared()
    try:
        for edge, ms in ((2, 1.0), (0, 0.5), (1, 2.0)):
            hs = tw.HmapSampler(W, H, edge, ms, 0.0012, 1.7, -0.3, 0.8)
            stride = 24
            origins = np.array([(tx * stride - 200, ty * stride - 200) for ty in range(16) for tx in range(16)], np.int32)
            z = _zvals(ctx, img, hs, origins, stride + 1, 3)
            new = img.copy()
            rect = (100, 120, 9, 7)
            new[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2], 1] ^= 0x5a
            before = sh.hmap_tile_ao_launch(hs, origins, z, HALF_DXY)
            ctx.update_heightmap(new, [rect])
            after = ctx.hmap_tile_ao_launch(hs, origins, z, HALF_DXY)
            old_ao, new_ao = before.poll(wait=True), after.poll(wait=True)
            assert beq(old_ao, _expected(oracle, img, hs, origins, z)) == 0
            assert beq(new_ao, _expected(oracle, new, hs, origins, z)) == 0
            changed = (old_ao != new_ao).reshape(len(origins), -1).any(1)
            flagged = tw.hmap_tiles_touched(hs, origins - 36, stride + 72, [rect]).astype(bool)
            assert changed.any() and not (changed & ~flagged).any(), (edge, ms)
            assert (flagged & ~tw.hmap_tiles_touched(hs, origins, stride + 1, [rect]).astype(bool)).any()   # tiles re-shaded whose heights stay
            img = new
    finally:
        sh.close()
        ctx.set_heightmap(None)


def _job(tw, hs, origins, nt, zv, zvals=None, tset=None, tile_xy=None, ao=None):
    return tw.HmapAoJobArgs(C.cast(C.pointer(hs), C.c_void_p) if hs is not None else None, tw._ptr(origins), nt, zv, HALF_DXY, tw._ptr(zvals),
                            tset, tw._ptr(tile_xy), tw._ptr(ao))


def test_refusals_cancel_and_empty(tw, ctx):
    img = _image(1)
    hs = tw.HmapSampler(W, H, 0, 1.0, 0.0012, 1.7, -0.3, 0.8)
    org = np.zeros((2, 2), np.int32)
    z = np.zeros((2, 5, 5), np.float32)
    ao = np.zeros((2, 4, 4), np.uint8)
    fresh = tw.Context(0)
    try:   # no image
        assert tw.lib.tw_hmap_tile_ao_launch(fresh._h, C.byref(_job(tw, hs, org, 2, 5, z, ao=ao))) == tw.TW_ERR_STATE
        assert tw.lib.tw_hmap_tile_ao_launch(fresh._h, C.byref(_job(tw, hs, org, 0, 5, z, ao=ao))) == tw.TW_OK
    finally:
        fresh.close()
    ctx.set_heightmap(img)
    ts = ctx.tile_set(5, 1)
    other = tw.Context(0)
    try:
        ok = _job(tw, hs, org, 2, 5, z, ao=ao)
        assert tw.lib.tw_hmap_tile_ao(ctx._h, C.byref(ok)) == tw.TW_OK
        bad_edge = tw.HmapSampler(W, H, 3, 1.0, 0.0012, 1.7, -0.3, 0.8)
        bad_size = tw.HmapSampler(W + 1, H, 0, 1.0, 0.0012, 1.7, -0.3, 0.8)
        txy = np.array([[0, 0], [1, 0]], np.int32)
        ts.put(txy, z)
        for j in (_job(tw, None, org, 2, 5, z, ao=ao), _job(tw, bad_edge, org, 2, 5, z, ao=ao), _job(tw, bad_size, org, 2, 5, z, ao=ao),
                  _job(tw, hs, org, 2, 1, z, ao=ao), _job(tw, hs, org, 2, 5, ao=ao), _job(tw, hs, org, 2, 5, z, ts._h, txy, ao),
                  _job(tw, hs, org, 2, 5, z), _job(tw, hs, None, 2, 5, z, ao=ao), _job(tw, hs, org, 2, 5, None, ts._h, None, ao),
                  _job(tw, hs, org, 2, 5, None, ts._h, np.array([[0, 0], [0, 0]], np.int32), ao),
                  _job(tw, hs, org, 2, 5, None, ts._h, np.array([[0, 0], [2, 0]], np.int32), ao),
                  _job(tw, hs, org, 2, 6, None, ts._h, txy, ao)):
            assert tw.lib.tw_hmap_tile_ao_launch(ctx._h, C.byref(j)) == tw.TW_ERR_ARG
        assert tw.lib.tw_hmap_tile_ao_launch(None, C.byref(ok)) == tw.TW_ERR_ARG
        assert tw.lib.tw_hmap_tile_ao_launch(ctx._h, None) == tw.TW_ERR_ARG
        other.set_heightmap(img)   # a context of another family, with an image of the same size
        assert tw.lib.tw_hmap_tile_ao_launch(other._h, C.byref(_job(tw, hs, org, 2, 5, None, ts._h, txy, ao))) == tw.TW_ERR_ARG
        assert tw.lib.tw_hmap_tile_ao_launch(ctx._h, C.byref(_job(tw, hs, None, 0, 5, z, ao=ao))) == tw.TW_OK
        # set-sourced from the set's own context, then cancel: no cancellation point
        exp = ctx.hmap_tile_ao(hs, org, z, HALF_DXY)
        got = np.zeros_like(ao)
        assert tw.lib.tw_hmap_tile_ao_launch(ctx._h, C.byref(_job(tw, hs, org, 2, 5, None, ts._h, txy, got))) == tw.TW_OK
        assert tw.lib.tw_cancel(ctx._h) == tw.TW_ERR_STATE
        assert ctx.create_tiles_poll(wait=True)
        assert (got == exp).all()
    finally:
        other.close()
        ts.close()
        ctx.set_heightmap(None)
