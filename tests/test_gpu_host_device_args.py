"""Every synchronous entry point that takes its arrays as host or device memory gives the same bytes whichever it gets: the same seeded inputs with
all-host arrays, all-device arrays, and host inputs with device outputs. Arrays an entry point updates in place count as outputs."""
import os

import numpy as np
import pytest

from cases import HM_CFG
from test_weights_host import weight_cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODES = [("host", "host"), ("device", "device"), ("host", "device")]   # (inputs, outputs)


class Args:
    def __init__(self, mode):
        self.inp, self.out = mode

    @staticmethod
    def _dev(a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def i(self, a):
        """An input array."""
        return self._dev(a) if self.inp == "device" else np.ascontiguousarray(a).copy()

    def o(self, a):
        """An output (or in-place) array, starting with a's contents."""
        return self._dev(a) if self.out == "device" else np.ascontiguousarray(a).copy()


def _bytes(x):
    if hasattr(x, "cpu"):
        x = x.cpu().numpy()
    if isinstance(x, (tuple, list)):
        return [_bytes(v) for v in x]
    if isinstance(x, np.ndarray):
        return np.ascontiguousarray(x).tobytes()
    if isinstance(x, (float, int, np.floating, np.integer)):
        return np.float64(x).tobytes()
    return bytes(x)          # ctypes arrays (tile bounds)


def same_every_mode(run):
    """run(Args) returns the results; all three modes must agree byte for byte."""
    got = [_bytes(run(Args(m))) for m in MODES]
    for m, g in zip(MODES[1:], got[1:]):
        assert g == got[0], m


@pytest.fixture(scope="module")
def terrain(tw, scene, ctx):
    S, zv = 32, 34
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1))
    ctx.set_sine_params(cfg.sine_params())
    txy = [(tx - 1, ty + 2) for ty in range(3) for tx in range(3)]
    origins = [(tx * S, ty * S) for tx, ty in txy]
    tiles = ctx.heightgen_tiles(origins, cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), zv, cfg.height_params())
    return cfg, S, zv, txy, origins, tiles


def _erosion_params(tw, z):
    zmin, zmax = float(z.min()), float(z.max())
    return tw.ErosionParams(1.0, zmin + 0.2 * (zmax - zmin), 0.0625, zmin - 0.1, zmax + 0.1, 0.0, 0.5)


def test_height_and_tile_tails(tw, ctx, terrain):
    cfg, S, zv, txy, origins, tiles = terrain
    hp, dx, dy = cfg.height_params(), float(cfg.dx_val), float(cfg.dy_val)
    ctx.set_sine_params(cfg.sine_params())              # the weights' jitter noise is sine mode
    nt = len(origins)
    same_every_mode(lambda a: ctx.heightgen_tiles(origins, cfg.mesh_size, dx, dy, zv, hp, out=a.o(np.zeros((nt, zv, zv), np.float32)), want_minmax=True))
    same_every_mode(lambda a: ctx.tile_bounds(a.i(tiles), float(np.median(tiles)), dx, dy, S))
    same_every_mode(lambda a: ctx.tile_normals(a.i(tiles), dx, dy, out=a.o(np.zeros((nt, zv - 1, zv - 1, 4), np.uint8))))
    rng = np.random.default_rng(3)
    corners = rng.uniform(-0.2, 1.3, (nt, 8)).astype(np.float32)
    for wp in weight_cases(tw.WeightParams, rng, float(tiles.min()), float(tiles.max()), S, dx, dy, n=2):
        same_every_mode(lambda a: ctx.tile_weights(a.i(tiles), origins, cfg.mesh_size, dx, dy, hp, wp, a.i(corners),
                                                   out=a.o(np.zeros((nt, zv - 1, zv - 1, 4), np.uint8))))


def test_glaciate_mesh(tw, scene, ctx):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=2, hmap=HM_CFG, zmax_est=2.3)
    hp = cfg.height_params()
    MX, MY = 128, 96
    mesh = ctx.heightgen_2d(tw.Grid2D(float(37 - MX // 2), float(-50 - MY // 2), float(cfg.dx_val), float(cfg.dy_val), MX, MY), hp, enable_glaciate=0)

    def run(a):
        m = a.o(mesh)
        zr = ctx.glaciate_mesh(m, 37, -50, (MX, MY), hp)
        return m, zr
    same_every_mode(run)
    out, _ = run(Args(("host", "host")))
    assert not np.array_equal(out, mesh)


def test_erosion(tw, ctx, terrain):
    _, _, zv, _, _, tiles = terrain
    ep = _erosion_params(tw, tiles)

    def tiles_run(a):
        t = a.o(tiles)
        ctx.erode_tiles(t, 300, ep, min_zval_all=float(tiles.min()))
        return t, ctx.last_erosion_steps
    same_every_mode(tiles_run)

    def parallel_run(a):       # one droplet at a time: the serial order, reproducible run to run
        h = a.o(tiles[0])
        ctx.erode_parallel(h, float(tiles.min()), 300, ep, num_threads=1)
        return h, ctx.last_erosion_steps
    same_every_mode(parallel_run)


def test_heightmap_sampling_and_packing(tw, ctx):
    rng = np.random.default_rng(5)
    w, h, zv = 97, 80, 17
    img = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
    hs = tw.HmapSampler(w, h, 2, 1.0, 0.0008, 1.0, 0.0, 1.0)
    origins = [(-20, 5), (30, 40), (90, -10), (0, 70)]
    same_every_mode(lambda a: ctx.heightmap_sample_tiles(a.i(img), hs, origins, zv, out=a.o(np.zeros((len(origins), zv, zv), np.float32))))
    vals = rng.uniform(0.0, 1.0, 5000).astype(np.float32)
    same_every_mode(lambda a: ctx.from_floats_u16(a.i(vals), 0.005, -0.1, out=a.o(np.zeros(2 * vals.size, np.uint8))))
    data = rng.integers(0, 256, 2 * 5000, dtype=np.uint8)
    same_every_mode(lambda a: ctx.to_floats_u16(a.i(data), 0.003, -0.5, out=a.o(np.zeros(5000, np.float32))))
    same_every_mode(lambda a: ctx.minmax(a.i(vals)))


def test_points_and_voxel_fill(tw, scene, ctx):
    cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_freq_filter=1, mesh_seed=4, hmap={}, zmax_est=1.0)
    ctx.set_sine_params(cfg.sine_params())
    rng = np.random.default_rng(7)
    xy = rng.uniform(-300.0, 300.0, (4000, 2)).astype(np.float32)
    pq = tw.PointQuery(tw.PQ_SIN_TERMS_SCALED, 1.0, 128, 128, 4.0, 4.0, 0, 0, 0)
    same_every_mode(lambda a: ctx.eval_points(a.i(xy), cfg.height_params(), pq, out=a.o(np.zeros(len(xy), np.float32))))
    vp = scene.voxel_landscape_params(scene.SceneConfig(scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64)), 40, 24, 32)
    same_every_mode(lambda a: ctx.voxel_fill(vp, out=a.o(np.zeros((vp.ny, vp.nx, vp.nz), np.float32))))


def _shadow_params(tw, cfg, S, zlo, zhi, lp):
    sp = tw.ShadowParams()
    sp.x_scene_size, sp.y_scene_size = cfg.scene_size[0], cfg.scene_size[1]
    sp.dx_val, sp.dy_val = float(cfg.dx_val), float(cfg.dy_val)
    sp.dx_val_inv, sp.dy_val_inv = 1.0 / np.float32(cfg.dx_val), 1.0 / np.float32(cfg.dy_val)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, zlo, zhi, 0
    for d in range(3):
        sp.lpos[d] = lp[d]
    return sp


def test_shadows_and_tile_set_put(tw, ctx, terrain):
    cfg, S, zv, txy, _, tiles = terrain
    z = ((tiles - np.float32(tiles.mean())) * np.float32(3.0)).astype(np.float32)
    sp = _shadow_params(tw, cfg, S, float(z.min()) - 0.5, float(z.max()) + 0.5, (3.0, 2.0, 0.4))
    same_every_mode(lambda a: ctx.tile_shadows(a.i(z), txy, sp, out=a.o(np.zeros(z.shape, np.uint8))))
    m, _, _ = ctx.tile_shadows(z, txy, sp)
    assert m.any()                                      # some cells are shadowed

    def put_run(a):
        ts = ctx.tile_set(zv, 1)
        try:
            ts.put(txy, a.i(z))
            smask, ox, oy = np.zeros(z.shape, np.uint8), np.zeros((len(txy), zv), np.float32), np.zeros((len(txy), zv), np.float32)
            ts.shadows_launch(txy, [(sp, smask, ox, oy)])
            ctx.create_tiles_poll(wait=True)
            return smask, ox, oy
        finally:
            ts.close()
    same_every_mode(put_run)


def test_voxel_post(tw, scene, ctx):
    vp = scene.voxel_landscape_params(scene.SceneConfig(scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64)), 48, 40, 32)
    vals = ctx.voxel_fill(vp)
    vpp = tw.VoxelPostParams()
    vpp.nx, vpp.ny, vpp.nz = vp.nx, vp.ny, vp.nz
    for d in range(3):
        vpp.lo_pos[d], vpp.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    vpp.isolevel, vpp.make_closed_surface, vpp.remove_unconnected, vpp.centre_seed = 0.0, 1, 3, 1
    gold = np.load(os.path.join(GOLD, "voxel_post.npz"))
    tables = (gold["edge_table"], gold["tri_table"], gold["edge_to_vals"])
    zix = np.random.default_rng(9).integers(0, vp.nz // 2, vp.ny * vp.nx, dtype=np.uint32)
    shape = (vp.ny, vp.nx, vp.nz)
    same_every_mode(lambda a: ctx.voxel_outside(a.i(vals), vpp, zix_xy=a.i(zix), out=a.o(np.zeros(shape, np.uint8))))
    outside = ctx.voxel_outside(vals, vpp)

    def remove_run(a):
        v = a.o(vals)
        changed = ctx.voxel_remove_unconnected(v, outside.copy(), vpp)
        return v, changed
    same_every_mode(remove_run)
    v_rm = vals.copy()
    o_rm = outside.copy()
    ctx.voxel_remove_unconnected(v_rm, o_rm, vpp)
    ntris = ctx.voxel_triangles(v_rm, o_rm, vpp, tables).shape[0]
    assert ntris > 0

    def tris_run(a):
        out = ctx.voxel_triangles(a.i(v_rm), a.i(o_rm), vpp, tables, out=a.o(np.zeros((ntris, 3, 3), np.float32)))
        return out[0] if isinstance(out, tuple) else out
    same_every_mode(tris_run)
    verts, idx = ctx.voxel_mesh(v_rm, o_rm, vpp, tables)

    def mesh_run(a):
        return ctx.voxel_mesh(a.i(v_rm), a.i(o_rm), vpp, tables, verts=a.o(np.zeros(verts.shape, np.float32)), indices=a.o(np.zeros(idx.shape, np.uint32)))
    same_every_mode(mesh_run)
