"""GPU parity of the domain-warp simplex kernel (mode 4) on the paths its octave loop takes: the unrolled 8-octave body (mesh_freq_filter 1,
shape 0), the rolled loop (9 and 7 octaves, and shapes 1 and 2 at 8), in tile batches, and on grids that cross the lattice range guard, where
cells of one launch run the unrolled body and others the scalar fallback. Bit for bit against the CPU oracle."""
import numpy as np
import pytest

from cases import convert, HM_CFG

pytestmark = pytest.mark.gpu


def _cfg(scene, ff, shape, **kw):
    return scene.SceneConfig(mesh_gen_mode=4, mesh_gen_shape=shape, mesh_freq_filter=ff, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, **kw)


@pytest.mark.parametrize("shape", [0, 1, 2])
@pytest.mark.parametrize("ff", [0, 1, 2])
def test_tile_batch_matches_oracle(tw, scene, oracle, ctx, beq, ff, shape):
    cfg = _cfg(scene, ff, shape, mesh_size=(32, 32, 1))
    hp = cfg.height_params()
    S, zv = 32, 34
    origins = [(tx * S - 3 * S, ty * S + 5 * S) for ty in range(2) for tx in range(2)] + [(40000 * S, -25000 * S)]
    tiles, mm = ctx.heightgen_tiles(origins, cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), zv, hp, want_minmax=True)
    for t, (x1, y1) in enumerate(origins):
        g = oracle.Grid2D(float(x1 - S // 2), float(y1 - S // 2), float(cfg.dx_val), float(cfg.dy_val), zv, zv)
        zc = oracle.heightgen_2d(g, convert(hp, oracle.HeightParams), None, 1, 0)
        assert beq(tiles[t], zc) == 0, (t, ff, shape)
        assert mm[t, 0] == zc.min() and mm[t, 1] == zc.max()


@pytest.mark.parametrize("shape", [0, 1, 2])
@pytest.mark.parametrize("ff", [0, 1, 2])
def test_grid_across_the_lattice_range_guard(tw, scene, oracle, ctx, beq, ff, shape):
    # cell x covers x * 2^19 grid units: |xv| runs from 0 to ~3.5e4, past the bound below which the paired kernel keeps every octave's lattice
    # coordinates under 2^22, so the right part of each row takes the scalar fallback with the literal division
    cfg = _cfg(scene, ff, shape)
    hp = cfg.height_params()
    g = tw.Grid2D(0.0, -3.0, float(cfg.dx_val) * 2 ** 19, float(cfg.dy_val), 97, 6)
    z = ctx.heightgen_2d(g, hp)
    zc = oracle.heightgen_2d(convert(g, oracle.Grid2D), convert(hp, oracle.HeightParams), None, 1, 0)
    assert np.isfinite(zc).all()
    assert beq(z, zc) == 0, (ff, shape)
