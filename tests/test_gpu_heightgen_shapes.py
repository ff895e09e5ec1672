"""GPU: the 2-D height generator at launch shapes the parity cases never build - odd and one-cell widths, output 4 bytes off 8-byte alignment, grids of
several block waves, banded host output, tile batches past the 65535 gridDim.z limit and a grid of more than 2^32 cells. Every comparison is bit for bit
against the plain-C oracle, and every fused min/max must equal the min/max of the output.

At the default cell size (2^-4) and integer origins the noise modes (1-4) are pure functions of the global cell coordinate, so a large grid is checked
against oracle grids of a few of its rows. Sine mode (0) folds the origin into its tables and is compared whole."""
import numpy as np
import pytest

from cases import convert, HM_ALL, HM_CFG

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _cfg(scene, mode, shape=0, ff=1, hmap=HM_ALL, **kw):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_gen_shape=shape, mesh_freq_filter=ff, mesh_seed=1, hmap=hmap, zmax_est=2.3, **kw)


def _setup(scene, ctx, mode, **kw):
    cfg = _cfg(scene, mode, **kw)
    hp, sp = cfg.height_params(), cfg.sine_params()
    ctx.set_sine_params(sp)
    return cfg, hp, sp, float(cfg.dx_val), float(cfg.dy_val)


def _oracle_grid(oracle, hp, sp, x0, y0, dx, dy, nx, ny):
    return oracle.heightgen_2d(oracle.Grid2D(float(x0), float(y0), dx, dy, nx, ny), convert(hp, oracle.HeightParams), sp, 1, 0)


def _host(z):
    return z.cpu().numpy() if hasattr(z, "cpu") else z


def _check_rows(oracle, beq, z, g, hp, sp, rows):
    """Each run of consecutive rows of the grid z (numpy or CUDA tensor) equals the oracle grid of just those rows."""
    rows = sorted(set(r for r in rows if 0 <= r < g.ny))
    runs = []
    for r in rows:
        if runs and runs[-1][1] == r:
            runs[-1][1] = r + 1
        else:
            runs.append([r, r + 1])
    for r0, r1 in runs:
        zc = _oracle_grid(oracle, hp, sp, g.x0, g.y0 + r0, g.dx, g.dy, g.nx, r1 - r0)
        assert beq(_host(z[r0:r1]), zc) == 0, "rows %d..%d of %d x %d" % (r0, r1 - 1, g.nx, g.ny)


def _aminmax(t):
    import torch
    lo, hi = torch.aminmax(t)
    return lo.item(), hi.item()


def _nan_fill(t):
    """Fills a CUDA tensor with NaN, so cells a kernel never writes show, and waits for it: the context's stream does not wait for torch's."""
    import torch
    t.fill_(NAN)
    torch.cuda.synchronize()
    return t


# ---------------------------------------------------------------------------------------------------- A. odd and degenerate widths
ODD = ((1, 37), (3, 29), (65, 33), (257, 19))   # nx = 1: every cell pair crosses a row end; odd nx*ny: the last pair is half valid


@pytest.mark.parametrize("shape", [0, 1, 2])
@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_odd_widths_and_misaligned_output(tw, scene, oracle, ctx, beq, mode, shape):
    """The paired noise kernel deals cells out in pairs that cross row ends when nx is odd, and stores a pair as one float2 only at 8-byte alignment.
    Whole grids against the oracle, then the same grid into a device tensor that starts 4 bytes into its allocation (scalar stores for every pair)."""
    import torch
    cfg, hp, sp, dx, dy = _setup(scene, ctx, mode, shape=shape)
    for nx, ny in ODD:
        g = tw.Grid2D(-37.0, 11.0, dx, dy, nx, ny)
        z, mm = ctx.heightgen_2d(g, hp, want_minmax=True)
        zc = _oracle_grid(oracle, hp, sp, g.x0, g.y0, dx, dy, nx, ny)
        assert beq(z, zc) == 0, (nx, ny)
        assert mm == (zc.min(), zc.max())
        n = nx * ny
        buf = _nan_fill(torch.empty(n + 2, dtype=torch.float32, device="cuda"))
        out = buf[1:1 + n].view(ny, nx)
        assert out.data_ptr() % 8 == 4
        _, mm_dev = ctx.heightgen_2d(g, hp, out=out, want_minmax=True)
        assert beq(out.cpu().numpy(), z) == 0, (nx, ny)
        assert mm_dev == mm
        assert torch.isnan(buf[0]) and torch.isnan(buf[-1])     # nothing written outside the grid


@pytest.mark.parametrize("mode", [1, 4])
def test_tiles_odd_zvsize(tw, scene, oracle, ctx, beq, mode):
    """zvsize 33: every other tile of the batch starts at an odd cell of the output, so its pairs are never 8-byte aligned."""
    S, zv = 32, 33
    cfg, hp, sp, dx, dy = _setup(scene, ctx, mode)
    origins = [(tx * S - 5 * S, ty * S + 2 * S) for ty in range(2) for tx in range(3)]
    tiles, mm = ctx.heightgen_tiles(origins, (S, S), dx, dy, zv, hp, want_minmax=True)
    for t, (x1, y1) in enumerate(origins):
        zc = _oracle_grid(oracle, hp, sp, x1 - S // 2, y1 - S // 2, dx, dy, zv, zv)
        assert beq(tiles[t], zc) == 0, t
        assert mm[t, 0] == zc.min() and mm[t, 1] == zc.max()


# ---------------------------------------------------------------------------------------------------- B. several block waves
def _wave_cells():
    """Cells of one wave of the persistent noise grid: num_sms x TW_NOISE2_MIN_BLOCKS (2) resident blocks of TW_NOISE2_BLOCK_CELLS (2048) cells each
    (tw_heightgen.cu). A single grid launches at most one wave of blocks, which stride over the chunk groups."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 2 * 2048


WAVE_NX = 1001


@pytest.mark.parametrize("mode,shape,ff", [(1, 0, 1), (2, 0, 1), (3, 0, 1), (4, 0, 1), (2, 1, 1), (2, 2, 1), (4, 1, 1), (4, 2, 1), (4, 0, 2)],
                         ids=lambda v: str(v))
def test_several_block_waves(tw, scene, oracle, ctx, beq, mode, shape, ff):
    """Odd-width grids just below one wave (every block one chunk group), just above it (some blocks take a second group) and between two and three
    waves. The first two are compared whole; the third at the rows around each wave boundary and at its first and last rows. mesh_freq_filter 1
    runs the domain warp's unrolled 8-octave body, 2 the rolled loop."""
    import torch
    wave = _wave_cells()
    cfg, hp, sp, dx, dy = _setup(scene, ctx, mode, shape=shape, ff=ff)
    for ny, whole in ((wave // WAVE_NX, True), (wave // WAVE_NX + 3, True), (5 * wave // (2 * WAVE_NX), False)):
        n = WAVE_NX * ny
        assert (n < wave) if ny == wave // WAVE_NX else (n > wave)
        g = tw.Grid2D(-500.0, -300.0, dx, dy, WAVE_NX, ny)
        out = _nan_fill(torch.empty((ny, WAVE_NX), dtype=torch.float32, device="cuda"))
        _, mm = ctx.heightgen_2d(g, hp, out=out, want_minmax=True)
        assert mm == _aminmax(out), ny
        if whole:
            zc = _oracle_grid(oracle, hp, sp, g.x0, g.y0, dx, dy, WAVE_NX, ny)
            assert beq(out.cpu().numpy(), zc) == 0, ny
        else:
            assert 2 * wave < n < 3 * wave
            rows = [0, ny - 1]
            for k in (1, 2):
                r = k * wave // WAVE_NX
                rows += [r - 1, r, r + 1]
            _check_rows(oracle, beq, out, g, hp, sp, rows)


# ---------------------------------------------------------------------------------------------------- C. banded host output
def _band_rows(nx, ny):
    """band_rows_for (tw_heightgen.cu): a host-bound grid of 32 MiB or more is issued in at most 16 row bands of a multiple of 64 rows."""
    if nx * ny * 4 < (32 << 20):
        return ny
    return max(64, ((ny + 15) // 16 + 63) & ~63)


@pytest.mark.parametrize("mode", [0, 1, 4])
def test_banded_host_output(tw, scene, oracle, ctx, beq, mode):
    """2901 x 2897 to host memory: 16 bands of 192 rows, the last one 17 rows (an odd cell count), each copied to the host while the next computes.
    Before each host call a grid of the same size with other values goes through the same device staging buffer, and the host buffer is filled
    with NaN, so a copy that ran ahead of its band, a band never copied or a wrong band offset shows. The call must take the banded path: it issues
    band count - 1 more kernels than the same grid into device memory. Host buffers: pageable numpy, pinned torch, and pinned through
    heightgen_2d_launch + heightgen_2d_poll."""
    import torch
    nx, ny = 2901, 2897
    rows = _band_rows(nx, ny)
    nbands = -(-ny // rows)
    assert (rows, nbands) == (192, 16) and (ny - (nbands - 1) * rows) * nx % 2 == 1
    cfg, hp, sp, dx, dy = _setup(scene, ctx, mode, hmap=HM_CFG)
    g = tw.Grid2D(-1450.0, -1448.0, dx, dy, nx, ny)
    other = tw.Grid2D(3000.0, -7000.0, dx, dy, nx, ny)
    ctx.heightgen_2d(other, hp)                                 # also sets up the tables, so the launch counts below are the grid's own
    dev = torch.empty((ny, nx), dtype=torch.float32, device="cuda")
    n0 = ctx.launch_count
    _, mm = ctx.heightgen_2d(g, hp, out=dev, want_minmax=True)
    launches_dev = ctx.launch_count - n0
    assert mm == _aminmax(dev)
    ref = dev.cpu().numpy()
    if mode == 0:
        zc = _oracle_grid(oracle, hp, sp, g.x0, g.y0, dx, dy, nx, ny)
        assert beq(ref, zc) == 0
    else:
        bounds = [k * rows for k in range(1, nbands)]
        _check_rows(oracle, beq, ref, g, hp, sp, [0, ny - 1] + [r - 1 for r in bounds] + bounds)
    for where in ("numpy", "pinned", "launch"):
        stale = ctx.heightgen_2d(other, hp)
        assert beq(stale, ref) > 0
        out = np.full((ny, nx), NAN, np.float32) if where == "numpy" else torch.full((ny, nx), NAN, dtype=torch.float32).pin_memory()
        n0 = ctx.launch_count
        if where == "launch":
            m = tw.MinMax()
            ctx.heightgen_2d_launch(g, hp, 1, 0, out, m)
            while not ctx.heightgen_2d_poll(wait=False):
                pass
            mm_host = (m.zmin, m.zmax)
        else:
            _, mm_host = ctx.heightgen_2d(g, hp, out=out, want_minmax=True)
        assert ctx.launch_count - n0 - launches_dev == nbands - 1, where
        assert beq(_host(out), ref) == 0, where
        assert mm_host == mm, where


# ---------------------------------------------------------------------------------------------------- D. more than 65535 tiles
S_SMALL, ZV_SMALL = 32, 34


def _tile_grid(nt, cols, step):
    return np.array([((t % cols) * step - 4000, (t // cols) * step - 3000) for t in range(nt)], np.int32)


def _spots(nt):
    return sorted(set([0, 1, 300, nt // 2, 65534, 65535, 65536, nt - 2, nt - 1]))


@pytest.mark.parametrize("mode,cols,nt", [(1, 257, 65537), (0, 257, 257 * 256)], ids=["m1_65537", "m0_257x256"])
def test_tiles_past_65535(tw, scene, oracle, ctx, beq, mode, cols, nt):
    """tw_heightgen_tiles splits a batch at the 65535 gridDim.z limit; the sine tables need nux + nuy <= 65535, so mode 0 takes a 257 x 256 block."""
    cfg, hp, sp, dx, dy = _setup(scene, ctx, mode)
    origins = _tile_grid(nt, cols, S_SMALL)
    tiles, mm = ctx.heightgen_tiles(origins, (S_SMALL, S_SMALL), dx, dy, ZV_SMALL, hp, want_minmax=True)
    for t in _spots(nt):
        x1, y1 = origins[t]
        zc = _oracle_grid(oracle, hp, sp, x1 - S_SMALL // 2, y1 - S_SMALL // 2, dx, dy, ZV_SMALL, ZV_SMALL)
        assert beq(tiles[t], zc) == 0, t
        assert mm[t, 0] == zc.min() and mm[t, 1] == zc.max(), t


def test_create_zvals_batch_past_65535(tw, scene, oracle, ctx, beq):
    """tw_create_zvals_batch with 65537 tiles and 300 droplets per tile: at least two chunks, generated and eroded in the heaviest-first order that a
    coarse pre-pass over all tiles (issued in pieces of at most 65535 tiles) decides. Spot tiles: oracle heights, then oracle erosion."""
    nt, iters = 65537, 300
    cfg, hp, sp, dx, dy = _setup(scene, ctx, 1, hmap=HM_CFG, mesh_size=(S_SMALL, S_SMALL, 1), scene_size=(1.0, 1.0, 4.0))
    assert dx == 0.0625
    ep = cfg.erosion_params()
    origins = _tile_grid(nt, 257, 4 * S_SMALL)                  # spread out: ocean and mountain tiles
    z, mm = ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, ZV_SMALL, hp, iters, ep, ep.zmin, want_minmax=True)
    assert ctx.last_erosion_steps > 0
    ep_o = convert(ep, oracle.ErosionParams)
    eroded = 0
    for t in _spots(nt):
        x1, y1 = origins[t]
        raw = _oracle_grid(oracle, hp, sp, x1 - S_SMALL // 2, y1 - S_SMALL // 2, dx, dy, ZV_SMALL, ZV_SMALL)
        zc, _ = oracle.apply_erosion(raw, ep.zmin, iters, ep_o)
        eroded += beq(zc, raw) > 0
        assert beq(z[t], zc) == 0, t
        assert mm[t, 0] == zc.min() and mm[t, 1] == zc.max(), t
    assert eroded >= 2


def test_hmap_tiles_job_past_65535(tw, oracle, ctx, beq):
    """tw_create_tiles_launch_hmap with 65537 tiles sampled from a random 16-bit image and eroded: the coarse pre-pass samples all tiles in one
    internal call. Spot tiles: oracle samples, then oracle erosion."""
    import torch
    nt, iters = 65537, 300
    rng = np.random.default_rng(65537)
    img = rng.integers(0, 256, (300, 257, 2), dtype=np.uint8)
    hs = tw.HmapSampler(257, 300, 2, 1.0, 0.0012, 1.7, -0.3, 0.8)
    hs_o = convert(hs, oracle.HmapSampler)
    origins = _tile_grid(nt, 257, S_SMALL)
    spots = _spots(nt)
    raw = oracle.hmap_sample_tiles(img, hs_o, origins[spots], ZV_SMALL)
    lo, hi = float(raw.min()), float(raw.max())
    ep = tw.ErosionParams(1.0, float(np.median(raw)), 0.0625, lo - 0.1, hi + 0.1, 0.0, 0.5)
    ctx.set_heightmap(img)
    z = torch.empty((nt, ZV_SMALL, ZV_SMALL), dtype=torch.float32, device="cuda")
    mm = np.empty((nt, 2), np.float32)
    ctx.create_tiles_launch(origins, (S_SMALL, S_SMALL), 0.0625, 0.0625, ZV_SMALL, None, iters, ep, ep.zmin, z, mm=mm, hmap=hs)
    assert ctx.create_tiles_poll(wait=True)
    assert ctx.last_erosion_steps > 0
    ctx.set_heightmap(None)
    ep_o = convert(ep, oracle.ErosionParams)
    eroded = 0
    for i, t in enumerate(spots):
        zc, _ = oracle.apply_erosion(raw[i], ep.zmin, iters, ep_o)
        eroded += beq(zc, raw[i]) > 0
        assert beq(z[t].cpu().numpy(), zc) == 0, t
        assert mm[t, 0] == zc.min() and mm[t, 1] == zc.max(), t
    assert eroded >= 2


# ---------------------------------------------------------------------------------------------------- E. more than 2^32 cells
def test_more_than_2_32_cells(tw, scene, oracle, ctx, beq):
    """65537^2 cells into device memory: cell indices past 2^32 take the 64-bit division (row 65535 starts at cell 2^32 - 1). Rows on both sides of
    that boundary and a middle row against the oracle; the fused min/max against torch.aminmax of the whole grid."""
    import torch
    N = 65537
    free, _ = torch.cuda.mem_get_info()
    if free < (18 << 30):
        pytest.skip("a 65537^2 float32 grid needs 18 GiB of free device memory; %.1f GiB free" % (free / 2**30))
    out = torch.empty((N, N), dtype=torch.float32, device="cuda")
    try:
        for mode in (4, 1):
            cfg, hp, sp, dx, dy = _setup(scene, ctx, mode)
            g = tw.Grid2D(-32768.0, -32768.0, dx, dy, N, N)
            _nan_fill(out)
            _, mm = ctx.heightgen_2d(g, hp, out=out, want_minmax=True)
            assert mm == _aminmax(out), mode
            _check_rows(oracle, beq, out, g, hp, sp, [0, N // 2, 65534, 65535, 65536])
    finally:
        del out
        torch.cuda.empty_cache()
