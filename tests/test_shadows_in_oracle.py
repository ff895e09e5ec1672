"""CPU: the chained mesh-shadow oracle with incoming heights from tiles outside the batch (what tw_tile_shadows_batch_ex and the tile job's shadow pass are
checked against). It is tile_t::calc_shadows_for_light over a batch, built on the oracle's calc_mesh_shadows (which takes sh_in): a tile whose neighbour toward
the light is in the batch starts from that neighbour's sh_out, any other tile from the caller's row. Pinned here against the oracle's own batch chain, and by
splitting a block in two: the tiles nearer the light first, then the rest with sh_in gathered from the first part, must give the one-batch result."""
import numpy as np
import pytest

from cases import convert, HM_CFG

MIN_Z = np.float32(-1.0e6)      # TW_MESH_MIN_Z


def light_signs(sp):
    return (-1 if sp.lpos[0] < 0.0 else 1), (-1 if sp.lpos[1] < 0.0 else 1)


def _coords(tile_xy):
    return [tuple(int(v) for v in t) for t in np.asarray(tile_xy).reshape(-1, 2)]


def gather_edges(sp, tile_xy, src_xy, src_ox, src_oy, zv):
    """sh_in_x / sh_in_y rows of the tiles tile_xy taken from the sh_out of the tiles src_xy: MESH_MIN_Z where the neighbour toward the light is not among them."""
    sx, sy = light_signs(sp)
    where = {t: i for i, t in enumerate(_coords(src_xy))}
    txy = _coords(tile_xy)
    ix, iy = np.full((len(txy), zv), MIN_Z, np.float32), np.full((len(txy), zv), MIN_Z, np.float32)
    for t, (x, y) in enumerate(txy):
        if (x, y + sy) in where:
            ix[t] = np.asarray(src_ox)[where[(x, y + sy)]]
        if (x + sx, y) in where:
            iy[t] = np.asarray(src_oy)[where[(x + sx, y)]]
    return ix, iy


def tile_shadows_batch_in(oracle, tiles, tile_xy, sp, sh_in_x=None, sh_in_y=None):
    """(smask [nt, zv, zv], sh_out_x [nt, zv], sh_out_y [nt, zv]) as tw_tile_shadows_batch_ex defines them; sp is an oracle.ShadowParams."""
    tiles = np.ascontiguousarray(tiles, np.float32)
    nt, zv = tiles.shape[0], tiles.shape[1]
    sx, sy = light_signs(sp)
    txy = _coords(tile_xy)
    where = {t: i for i, t in enumerate(txy)}
    assert len(where) == nt
    smask = np.empty((nt, zv, zv), np.uint8)
    ox, oy = np.full((nt, zv), MIN_Z, np.float32), np.full((nt, zv), MIN_Z, np.float32)
    for t in sorted(range(nt), key=lambda t: -(sx * txy[t][0] + sy * txy[t][1])):     # nearest the light first: its neighbours toward the light are done
        x, y = txy[t]
        nbx, nby = where.get((x + sx, y)), where.get((x, y + sy))
        six = ox[nby] if nby is not None else (None if sh_in_x is None else np.asarray(sh_in_x)[t])
        siy = oy[nbx] if nbx is not None else (None if sh_in_y is None else np.asarray(sh_in_y)[t])
        smask[t], ox[t], oy[t] = oracle.calc_mesh_shadows(sp, tiles[t], six, siy)
    return smask, ox, oy


def splits_by_light(sp, tile_xy):
    """Every cut of the batch across the light direction: (indices of the tiles nearer the light, indices of the rest). No tile of the first part has its
    neighbour toward the light in the second."""
    sx, sy = light_signs(sp)
    key = np.array([sx * x + sy * y for x, y in _coords(tile_xy)])
    return [(np.nonzero(key > c)[0], np.nonzero(key <= c)[0]) for c in range(int(key.min()), int(key.max()))]


LIGHTS = ((4.0, 1.0, 0.3), (-4.0, 1.0, 0.2), (1.0, -5.0, 0.3), (-6.0, -1.0, 0.1))     # one per quadrant, each with shadows that cross tile edges


def _block(tw, scene, oracle, side, S=32):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.0, mesh_size=(S, S, 1))
    hp_o, dx, dy, zv = convert(cfg.height_params(), oracle.HeightParams), float(cfg.dx_val), float(cfg.dy_val), S + 2
    txy = [(tx - 1, ty + 3) for ty in range(side) for tx in range(side)]
    tiles = np.stack([oracle.heightgen_2d(oracle.Grid2D(tx * S - S // 2, ty * S - S // 2, dx, dy, zv, zv), hp_o, None, 1, 0) for tx, ty in txy])
    tiles = ((tiles - np.float32(tiles.mean())) * np.float32(3.0)).astype(np.float32)
    zlo, zhi = float(tiles.min()) - 0.5, float(tiles.max()) + 0.5

    def params(lp):
        sp = oracle.ShadowParams()
        sp.x_scene_size, sp.y_scene_size = cfg.scene_size[0], cfg.scene_size[1]
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, zlo, zhi, 0
        for d in range(3):
            sp.lpos[d] = lp[d]
        return sp
    return tiles, txy, params


def test_without_incoming_rows_equals_the_batch_chain(tw, scene, oracle, beq):
    tiles, txy, params = _block(tw, scene, oracle, 3)
    for lp in LIGHTS + ((5.0, 0.0, 1.0), (0.0, 0.0, 5.0)):
        sp = params(lp)
        m, ox, oy = tile_shadows_batch_in(oracle, tiles, txy, sp)
        mo, oxo, oyo = oracle.tile_shadows_batch(tiles, txy, sp)
        assert np.array_equal(m, mo) and beq(ox, oxo) == 0 and beq(oy, oyo) == 0, lp
        none = np.full((len(txy), tiles.shape[1]), MIN_Z, np.float32)           # rows of "no incoming height" are no rows
        m2, ox2, oy2 = tile_shadows_batch_in(oracle, tiles, txy, sp, none, none)
        assert np.array_equal(m2, mo) and beq(ox2, oxo) == 0 and beq(oy2, oyo) == 0, lp


@pytest.mark.parametrize("lp", LIGHTS)
def test_split_equals_whole(tw, scene, oracle, beq, lp):
    """A 4x4 block in two batches, at every cut across the light: the tiles nearer the light, then the rest with sh_in gathered from the first batch's
    sh_out."""
    tiles, txy, params = _block(tw, scene, oracle, 4)
    sp = params(lp)
    mo, oxo, oyo = oracle.tile_shadows_batch(tiles, txy, sp)
    assert 0 < (mo == 2).mean() < 1
    lost = 0
    for a, b in splits_by_light(sp, txy):
        ta, tb = [txy[i] for i in a], [txy[i] for i in b]
        ma, oxa, oya = tile_shadows_batch_in(oracle, tiles[a], ta, sp)
        ix, iy = gather_edges(sp, tb, ta, oxa, oya, tiles.shape[1])
        mb, oxb, oyb = tile_shadows_batch_in(oracle, tiles[b], tb, sp, ix, iy)
        assert np.array_equal(ma, mo[a]) and beq(oxa, oxo[a]) == 0 and beq(oya, oyo[a]) == 0
        assert np.array_equal(mb, mo[b]) and beq(oxb, oxo[b]) == 0 and beq(oyb, oyo[b]) == 0
        mb0, _, _ = tile_shadows_batch_in(oracle, tiles[b], tb, sp)         # the second batch without the incoming rows
        lost += int((mb0 != mo[b]).sum())
    assert lost > 0                                                         # shadows do cross the cuts
