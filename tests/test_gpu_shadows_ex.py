"""GPU: tw_tile_shadows_batch_ex - mesh shadows of a batch of tiles with incoming heights from tiles outside the batch. Bit for bit against the chained oracle
with caller rows (tests/test_shadows_in_oracle.py), against the reference's own chained 3x3 block split in two, and against tw_tile_shadows_batch where the
caller rows must not matter."""
import os

import numpy as np
import pytest

from cases import convert, HM_CFG
from test_gpu_shadows import _params
from test_shadows_in_oracle import MIN_Z, gather_edges, splits_by_light, tile_shadows_batch_in

pytestmark = pytest.mark.gpu

LIGHTS = ((3.0, 2.0, 0.4), (-4.0, 1.0, 0.3), (1.0, -5.0, 0.5), (-2.0, -3.0, 2.0), (0.2, 6.0, 0.15), (5.0, 0.0, 1.0), (0.0, 0.0, 5.0))


def _case(scene, ctx, S, side):
    zv = S + 2
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.0, mesh_size=(S, S, 1))
    txy = [(tx - 1, ty + 3) for ty in range(side) for tx in range(side)]
    if side == 5:
        txy = [t for i, t in enumerate(txy) if i % 4 != 1]
    tiles = ctx.heightgen_tiles([(tx * S, ty * S) for tx, ty in txy], cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), zv, cfg.height_params())
    tiles = ((tiles - np.float32(tiles.mean())) * np.float32(3.0)).astype(np.float32)
    return cfg, txy, tiles, float(tiles.min()) - 0.5, float(tiles.max()) + 0.5


def _random_edges(rng, nt, zv, zlo, zhi):
    """Caller rows: heights across the clip range, a third of them 'no incoming height' (MESH_MIN_Z or below)."""
    e = rng.uniform(zlo, zhi, (nt, zv)).astype(np.float32)
    e[rng.random((nt, zv)) < 0.2] = MIN_Z
    e[rng.random((nt, zv)) < 0.1] = np.float32(-3.0e6)
    return e


@pytest.mark.parametrize("S,side", [(64, 1), (32, 4), (128, 3), (17, 5)])
def test_tile_shadows_ex_vs_oracle(tw, scene, oracle, ctx, beq, S, side):
    import torch
    cfg, txy, tiles, zlo, zhi = _case(scene, ctx, S, side)
    rng = np.random.default_rng(S * 10 + side)
    nt, zv = tiles.shape[0], tiles.shape[1]
    for k, lp in enumerate(LIGHTS + ((2.0, 1.0, zlo - 1.0),)):
        sp = _params(tw, cfg, S, zlo, zhi, lp)
        spo = convert(sp, oracle.ShadowParams)
        ix, iy = _random_edges(rng, nt, zv, zlo, zhi), _random_edges(rng, nt, zv, zlo, zhi)
        for six, siy in ((ix, iy), (ix, None), (None, iy)):
            mo, oxo, oyo = tile_shadows_batch_in(oracle, tiles, txy, spo, six, siy)
            m, ox, oy = ctx.tile_shadows(tiles, txy, sp, sh_in_x=six, sh_in_y=siy)
            assert np.array_equal(m, mo), (lp, int((m != mo).sum()))
            assert beq(ox, oxo) == 0 and beq(oy, oyo) == 0, lp
        if k == 0:                                              # device zvals, mask and caller rows
            mo, oxo, oyo = tile_shadows_batch_in(oracle, tiles, txy, spo, ix, iy)
            assert (mo == 2).any()
            dm = torch.empty(tiles.shape, dtype=torch.uint8, device="cuda")
            _, ox, oy = ctx.tile_shadows(torch.from_numpy(tiles).cuda(), txy, sp, out=dm, sh_in_x=torch.from_numpy(ix).cuda(), sh_in_y=torch.from_numpy(iy).cuda())
            assert np.array_equal(dm.cpu().numpy(), mo) and beq(ox, oxo) == 0 and beq(oy, oyo) == 0


def test_golden_block_split_in_two(tw, ctx, beq):
    """tests/golden/shadows.npz (the reference's own chained 3x3 block) at every cut across each light: the light-side part alone, then the rest with sh_in
    from the first part's sh_out, give the reference's masks and edges."""
    from test_oracle_golden import shadow_params
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shadows.npz"))
    txy = [tuple(int(v) for v in t) for t in g["tile_xy"]]
    tiles = g["tiles"]
    crossed = 0
    for li, lp in enumerate(g["lights"]):
        sp = shadow_params(tw.ShadowParams, g["params"], lp)
        gm, gx, gy = g["smask_%d" % li], g["sh_out_x_%d" % li], g["sh_out_y_%d" % li]
        for a, b in splits_by_light(sp, txy):
            ta, tb = [txy[i] for i in a], [txy[i] for i in b]
            ma, oxa, oya = ctx.tile_shadows(np.ascontiguousarray(tiles[a]), ta, sp)
            ix, iy = gather_edges(sp, tb, ta, oxa, oya, tiles.shape[1])
            crossed += int((ix > MIN_Z).sum() + (iy > MIN_Z).sum())
            mb, oxb, oyb = ctx.tile_shadows(np.ascontiguousarray(tiles[b]), tb, sp, sh_in_x=ix, sh_in_y=iy)
            assert np.array_equal(ma, gm[a]) and beq(oxa, gx[a]) == 0 and beq(oya, gy[a]) == 0, li
            assert np.array_equal(mb, gm[b]) and beq(oxb, gx[b]) == 0 and beq(oyb, gy[b]) == 0, li
    assert crossed > 0


def test_in_batch_neighbours_win(tw, scene, ctx, beq):
    """Garbage caller rows for tiles whose neighbour toward the light is in the batch change nothing."""
    S, side = 32, 4
    cfg, txy, tiles, zlo, zhi = _case(scene, ctx, S, side)
    nt, zv = tiles.shape[0], tiles.shape[1]
    for lp in LIGHTS[:5]:
        sp = _params(tw, cfg, S, zlo, zhi, lp)
        sx, sy = (-1 if lp[0] < 0 else 1), (-1 if lp[1] < 0 else 1)
        have = set(txy)
        ix, iy = np.full((nt, zv), MIN_Z, np.float32), np.full((nt, zv), MIN_Z, np.float32)
        for t, (x, y) in enumerate(txy):
            if (x, y + sy) in have:
                ix[t] = np.float32(1.0e3)                   # would shadow the tile's whole edge
            if (x + sx, y) in have:
                iy[t] = np.float32(1.0e3)
        assert (ix > MIN_Z).any() and (iy > MIN_Z).any()
        m, ox, oy = ctx.tile_shadows(tiles, txy, sp)
        m2, ox2, oy2 = ctx.tile_shadows(tiles, txy, sp, sh_in_x=ix, sh_in_y=iy)
        assert np.array_equal(m, m2) and beq(ox, ox2) == 0 and beq(oy, oy2) == 0, lp


def test_more_tiles_than_one_launch_takes(tw, scene, ctx, beq):
    """70000 tiles with no neighbours among them are one wave: it runs in pieces of at most 65535 tiles. Equal to two tw_tile_shadows_batch calls."""
    S, nt = 6, 70000
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.0, mesh_size=(S, S, 1))
    rng = np.random.default_rng(5)
    tiles = rng.uniform(-0.3, 0.3, (nt, S + 2, S + 2)).astype(np.float32)
    txy = np.stack([2 * np.arange(nt), np.zeros(nt, np.int64)], 1).astype(np.int32)      # every other column: no tile has a neighbour in the batch
    sp = _params(tw, cfg, S, -0.8, 0.8, (3.0, 2.0, 0.1))
    ix = _random_edges(rng, nt, S + 2, -0.8, 0.8)
    m, ox, oy = ctx.tile_shadows(tiles, txy, sp, sh_in_x=ix)
    assert (m == 2).any()
    # the same with the caller rows is tw_tile_shadows_batch_ex in two halves
    h = 35000
    m1, ox1, oy1 = ctx.tile_shadows(tiles[:h], txy[:h], sp, sh_in_x=ix[:h])
    m2, ox2, oy2 = ctx.tile_shadows(tiles[h:], txy[h:], sp, sh_in_x=ix[h:])
    assert np.array_equal(m, np.concatenate([m1, m2])) and beq(ox, np.concatenate([ox1, ox2])) == 0 and beq(oy, np.concatenate([oy1, oy2])) == 0
    with pytest.raises(tw.TwError):                         # tw_tile_shadows_batch keeps its limit
        ctx.tile_shadows(tiles, txy, sp)


def test_duplicate_tiles_are_refused(tw, ctx):
    import ctypes as C
    tiles = np.zeros((2, 8, 8), np.float32)
    txy = np.array([[0, 0], [0, 0]], np.int32)
    sp = tw.ShadowParams()
    sp.lpos[0], sp.lpos[1], sp.lpos[2] = 1.0, 1.0, 1.0
    sp.dx_val = sp.dy_val = 0.1
    ix = np.zeros((2, 8), np.float32)
    m = np.empty((2, 8, 8), np.uint8)
    rc = tw.lib.tw_tile_shadows_batch_ex(ctx._h, tw._ptr(tiles), tw._ptr(txy), 2, 8, C.byref(sp), tw._ptr(ix), None, tw._ptr(m), None, None)
    assert rc == tw.TW_ERR_ARG and b"twice" in tw.lib.tw_last_error(ctx._h)
    assert tw.lib.tw_tile_shadows_batch(ctx._h, tw._ptr(tiles), tw._ptr(txy), 2, 8, C.byref(sp), tw._ptr(m), None, None) == tw.TW_OK   # unchanged
