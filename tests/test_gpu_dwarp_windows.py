"""GPU: the windowed domain-warp kernel (single grids of mode 4 at 8 octaves and shape 0: tables indexed inside per-launch lattice windows, no mod 289
in the windowed octaves) against the reducing kernel, bit for bit. A batch of one tile keeps the reducing kernel, so it is the reference for square
grids; other grids are checked row by row against the CPU oracle. Covered: the 8192^2 headline to device memory and banded to host memory, odd sizes,
origins inside and beyond the windows' coordinate limit, and a grid too wide for the tables (both of which keep the reducing kernel)."""
import numpy as np
import pytest

from cases import convert, HM_CFG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup(scene):
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
    return cfg, cfg.height_params(), float(cfg.dx_val), float(cfg.dy_val)


def _one_tile(ctx, setup, x0, y0, n):
    """The n x n grid at integer origin (x0, y0) as a batch of one tile (mesh size 2: the tile's grid starts one cell before its origin)"""
    cfg, hp, dx, dy = setup
    return ctx.heightgen_tiles([(x0 + 1, y0 + 1)], (2, 2), dx, dy, n, hp)[0]


def _grid(tw, setup, x0, y0, nx, ny):
    return tw.Grid2D(float(x0), float(y0), setup[2], setup[3], nx, ny)


def _device(ctx, g, hp):
    import torch
    z = torch.full((g.ny, g.nx), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.heightgen_2d(g, hp, out=z)
    ctx.sync()
    return z.cpu().numpy()


def test_headline_grid_device_and_banded_host(tw, ctx, beq, setup):
    g = _grid(tw, setup, -4096, -4096, 8192, 8192)
    ref = _one_tile(ctx, setup, -4096, -4096, 8192)
    assert np.isfinite(ref).all()
    assert beq(_device(ctx, g, setup[1]), ref) == 0
    n0 = ctx.launch_count
    z = np.full((8192, 8192), np.nan, np.float32)                # 256 MiB to host memory: row bands, each with its own narrower y windows
    ctx.heightgen_2d(g, setup[1], out=z)
    assert ctx.launch_count - n0 > 1                             # the banded path
    assert beq(z, ref) == 0


@pytest.mark.parametrize("x0,y0,nx,ny", [(-37, 5000, 1001, 777), (3, -9, 1, 5), (-2049, 77, 4097, 3), (12345, -6789, 333, 2)])
def test_odd_grids_match_oracle(tw, ctx, oracle, beq, setup, x0, y0, nx, ny):
    cfg, hp, dx, dy = setup
    z = _device(ctx, _grid(tw, setup, x0, y0, nx, ny), hp)
    for r in sorted({0, ny // 2, ny - 1}):
        zc = oracle.heightgen_2d(oracle.Grid2D(float(x0), float(y0 + r), dx, dy, nx, 1), convert(hp, oracle.HeightParams), None, 1, 0)
        assert beq(z[r:r + 1], zc) == 0, (x0, y0, nx, ny, r)


@pytest.mark.parametrize("x0,y0,n", [(600000, -600000, 256),     # |lattice index| just below the windows' limit at octave 6: windowed
                                     (700000, 5, 256),           # beyond it: the reducing kernel
                                     (-4500, -4500, 9000)])      # windows wider than the tables: the reducing kernel
def test_origins_and_widths_at_the_limits(tw, ctx, beq, setup, x0, y0, n):
    ref = _one_tile(ctx, setup, x0, y0, n)
    assert beq(_device(ctx, _grid(tw, setup, x0, y0, n, n), setup[1]), ref) == 0
