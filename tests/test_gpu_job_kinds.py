"""GPU: the context's pending job across job kinds. Every launch first completes the job the context has in flight, so a launch of one kind completes a
job of another, and the completing call must unpack the first job's staging into the first job's outputs only. For every ordered pair (A, B) of six job
types, launching A, then B, then polling once must give, bit for bit, what A, poll, B, poll gives on a fresh context: every output of A and of B, the
context's heightmap image and tw_last_erosion_steps. A refused B returns TW_ERR_ARG, A still completes with TW_OK, and nothing is left pending."""
import os

import numpy as np
import pytest
import torch

from cases import HM_CFG
from test_voxel_flood_reference import RANDOM_FIELDS, post_params, random_field
from test_weights_host import weight_cases

pytestmark = pytest.mark.gpu
f32, u8 = np.float32, np.uint8
NAN = float("nan")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

G = 256                      # 2-D grid side
S, ZV, ITERS = 16, 18, 60    # tile size, zvals side, droplets per tile (tile job and tile set)
N, HITERS, EITERS = 128, 300, 500   # heightmap image side, droplets of the heightmap job and of the erosion job
KINDS = ["grid", "tiles", "voxel", "hmap", "erode", "relight"]


class World:
    """Inputs shared by every run, made once on a context of their own."""

    def __init__(self, tw, scene):
        self.hcfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
        self.tcfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1),
                                      scene_size=(0.5, 0.5, 4.0))
        self.sine = self.tcfg.sine_params()
        self.hp, self.ep = self.hcfg.height_params(), self.hcfg.erosion_params()
        self.thp, self.tep = self.tcfg.height_params(), self.tcfg.erosion_params()
        self.grid = self.hcfg.heightmap_grid(G, G)
        self.origins = [(tx * S * 40 - 3000, ty * S * 40 + 500) for ty in range(3) for tx in range(3)]   # ocean and mountain tiles
        self.tile_xy = np.array([(tx, ty) for ty in range(3) for tx in range(3)], np.int32)
        g = np.load(os.path.join(GOLD, "voxel_post.npz"))
        self.tables = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
        dims, seed, kw = RANDOM_FIELDS[0]
        self.vals, self.zix = random_field(dims, seed, kw.get("centre_seed", 1))
        self.vpp = post_params(tw.VoxelPostParams, dims, **kw)
        c = tw.Context(0)
        try:
            c.set_sine_params(self.sine)
            dx, dy = float(self.tcfg.dx_val), float(self.tcfg.dy_val)
            self.set_z = c.create_zvals_batch(self.origins, self.tcfg.mesh_size, dx, dy, ZV, self.thp, ITERS, self.tep, self.tep.zmin)
            self.wp = weight_cases(tw.WeightParams, np.random.default_rng(9), float(self.set_z.min()), float(self.set_z.max()), S, dx, dy)[3]
            self.tile_params = np.random.default_rng(9).uniform(-0.2, 1.3, (len(self.origins), 8)).astype(f32)
            self.img, self.info, _ = c.proc_gen_heightmap(N, N, float(self.hcfg.dx_val), float(self.hcfg.dy_val), self.hp, 0, self.ep)
            job = c.voxel_build_launch(self.vpp, vals=self.vals.copy(), zix_xy=self.zix, tables=self.tables)
            assert c.create_tiles_poll(True)
            self.cap = job.ntris + 4   # room for sentinel rows after the triangles
        finally:
            c.close()
        self.sp = tw.ShadowParams()
        sp = self.sp
        sp.x_scene_size = sp.y_scene_size = 0.5
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, float(self.tep.zmin), float(self.tep.zmax), 0
        sp.lpos[0], sp.lpos[1], sp.lpos[2] = 3.0, 2.0, 0.15
        self.hs = tw.HmapSampler(N, N, 2, 1.0, float(f32(0.0008) * f32(self.hp.mesh_height_scale)), self.info.mesh_file_scale, self.info.mesh_file_tz,
                                 self.hp.mesh_scale_z_inv)


@pytest.fixture(scope="module")
def world(tw, scene):
    return World(tw, scene)


def _ready(t):
    torch.cuda.synchronize()   # the library's streams do not wait for torch's
    return t


# Each launcher launches one job with fresh outputs (NaN / 0xAB sentinels) and returns a function that reads them once the job is complete.
def _grid(tw, c, ts, w):
    out, mm = _ready(torch.full((G, G), NAN, device="cuda")), tw.MinMax(NAN, NAN)
    c.heightgen_2d_launch(w.grid, w.hp, 1, 0, out, mm)
    return lambda: {"z": out, "mm": mm}


def _tiles(tw, c, ts, w):
    nt = len(w.origins)
    o = dict(zvals=np.full((nt, ZV, ZV), NAN, f32), mm=np.full((nt, 2), NAN, f32), bounds=(tw.TileBounds * nt)(),
             normals=np.full((nt, ZV - 1, ZV - 1, 4), 0xAB, u8), min_normal_z=np.full(nt, NAN, f32), weights=np.full((nt, ZV - 1, ZV - 1, 4), 0xAB, u8),
             has_any_grass=np.full(nt, 0xAB, u8))
    c.create_tiles_launch(w.origins, w.tcfg.mesh_size, float(w.tcfg.dx_val), float(w.tcfg.dy_val), ZV, w.thp, ITERS, w.tep, w.tep.zmin, wpz_max=float(w.tep.water_plane_z),
                          size=S, wp=w.wp, tile_params=w.tile_params, **o)
    return lambda: o


def _voxel(tw, c, ts, w):
    v, o = w.vals.copy(), np.full(w.vals.shape, 0xAB, u8)
    t = _ready(torch.full((w.cap, 3, 3), NAN, device="cuda"))
    job = c.voxel_build_launch(w.vpp, vals=v, outside=o, tris=t, zix_xy=w.zix, tables=w.tables, capacity=w.cap)
    return lambda: {"vals": v, "outside": o, "tris": t, "ntris": job.ntris, "changed": job.changed}


def _hmap(tw, c, ts, w):
    d16, vals = np.full(2 * N * N, 0xAB, u8), np.full(N * N, NAN, f32)
    job = c.proc_gen_heightmap_launch(N, N, float(w.hcfg.dx_val), float(w.hcfg.dy_val), w.hp, HITERS, w.ep, data16=d16, vals=vals, set_image=True)
    return lambda: {"data16": d16, "vals": vals, "info": job.info}


def _erode(tw, c, ts, w):
    vals = np.full(N * N, NAN, f32)
    c.erode_image_launch(w.info.val_mult, w.info.val_add, EITERS, w.ep, vals=vals)
    return lambda: {"vals": vals}


def _relight(tw, c, ts, w):
    n = len(w.tile_xy)
    L = tw.Light(w.sp, np.full((n, ZV, ZV), 0xAB, u8), np.full((n, ZV), NAN, f32), np.full((n, ZV), NAN, f32))
    rec = ts.shadows_launch(w.tile_xy, [L])
    return lambda: {"smask": L.smask, "sh_out_x": L.sh_out_x, "sh_out_y": L.sh_out_y, "recomputed": rec}


LAUNCH = dict(grid=_grid, tiles=_tiles, voxel=_voxel, hmap=_hmap, erode=_erode, relight=_relight)


# A refused launch of each kind (TW_ERR_ARG): a grid without columns, min_normal_z without the normal map, a capacity without tris, a 0-wide heightmap,
# an empty float map, a relight of a tile that is not resident.
def _refuse_grid(tw, c, ts, w):
    c.heightgen_2d_launch(tw.Grid2D(0.0, 0.0, 1.0, 1.0, 0, G), w.hp, 1, 0, _ready(torch.empty(G, device="cuda")), tw.MinMax())


def _refuse_tiles(tw, c, ts, w):
    nt = len(w.origins)
    c.create_tiles_launch(w.origins, w.tcfg.mesh_size, float(w.tcfg.dx_val), float(w.tcfg.dy_val), ZV, w.thp, ITERS, w.tep, w.tep.zmin,
                          np.empty((nt, ZV, ZV), f32), min_normal_z=np.empty(nt, f32))


def _refuse_voxel(tw, c, ts, w):
    c.voxel_build_launch(w.vpp, vals=w.vals.copy(), tables=w.tables, capacity=5)


def _refuse_hmap(tw, c, ts, w):
    c.proc_gen_heightmap_launch(0, N, float(w.hcfg.dx_val), float(w.hcfg.dy_val), w.hp, HITERS, w.ep, data16=np.empty(2 * N * N, u8))


def _refuse_erode(tw, c, ts, w):
    c.erode_launch(np.empty((0, 4), f32), 0.0, EITERS, w.ep)


def _refuse_relight(tw, c, ts, w):
    ts.shadows_launch(np.array([(7, 7)], np.int32), [tw.Light(w.sp, np.empty((1, ZV, ZV), u8))])


REFUSE = dict(grid=_refuse_grid, tiles=_refuse_tiles, voxel=_refuse_voxel, hmap=_refuse_hmap, erode=_refuse_erode, relight=_refuse_relight)


def _bits(v):
    if isinstance(v, torch.Tensor):
        return v.cpu().numpy().tobytes()
    if isinstance(v, np.ndarray):
        return v.tobytes()
    return v if isinstance(v, int) else bytes(v)   # ctypes structures and arrays


def _image(c, w):
    """The context's heightmap image, through heightmap tiles that cover it."""
    origins = [(x, y) for y in range(-N // 2, N // 2, 64) for x in range(-N // 2, N // 2, 64)]
    z = np.full((len(origins), 65, 65), NAN, f32)
    c.create_tiles_launch(origins, (64, 64), float(w.hcfg.dx_val), float(w.hcfg.dy_val), 65, None, 0, None, 0.0, z, hmap=w.hs)
    assert c.create_tiles_poll(True)
    return z.tobytes()


def _run(tw, w, steps):
    """Runs `steps` on a fresh context that has the sine params, the image and a tile set of the 3x3 tiles: a kind name launches that job, "poll" waits
    for the pending job, "poll0" polls without waiting and must find the context idle, ("refuse", kind) checks that the refused launch returns TW_ERR_ARG.
    Returns every launched job's outputs, tw_last_erosion_steps after the last step and the image."""
    c = tw.Context(0)
    try:
        c.set_sine_params(w.sine)
        c.set_heightmap(w.img.reshape(N, N, 2))
        ts = c.tile_set(ZV, 1)
        ts.put(w.tile_xy, w.set_z)
        reads = []
        for s in steps:
            if s in ("poll", "poll0"):
                assert c.create_tiles_poll(s == "poll")
            elif isinstance(s, tuple):
                with pytest.raises(tw.TwError) as e:
                    REFUSE[s[1]](tw, c, ts, w)
                assert e.value.status == tw.TW_ERR_ARG
            else:
                reads.append(LAUNCH[s](tw, c, ts, w))
        outs = [{k: _bits(v) for k, v in r().items()} for r in reads]
        return outs, c.last_erosion_steps, _image(c, w)
    finally:
        c.close()


def _same(got, exp, names):
    for name, g, e in zip(names, got, exp):
        assert g.keys() == e.keys()
        for k in e:
            assert g[k] == e[k], "%s: %s differs" % (name, k)


@pytest.mark.parametrize("b", KINDS)
@pytest.mark.parametrize("a", KINDS)
def test_launch_completes_a_job_of_any_kind(tw, world, a, b):
    exp, exp_steps, exp_img = _run(tw, world, [a, "poll", b, "poll"])
    got, steps, img = _run(tw, world, [a, b, "poll"])
    _same(got, exp, ["A (%s)" % a, "B (%s)" % b])
    assert steps == exp_steps and img == exp_img


_ALONE = {}


@pytest.mark.parametrize("b", KINDS)
@pytest.mark.parametrize("a", KINDS)
def test_refused_launch_leaves_the_job_to_complete(tw, world, a, b):
    """The refusal of a relight's request comes before the launch completes the pending job, every other one after; either way the poll that follows
    returns TW_OK with A's outputs complete, and a second poll finds nothing pending. (A refused tile launch still zeroes tw_last_erosion_steps.)"""
    if a not in _ALONE:
        _ALONE[a] = _run(tw, world, [a, "poll"])
    exp, _, exp_img = _ALONE[a]
    got, _, img = _run(tw, world, [a, ("refuse", b), "poll", "poll0"])
    _same(got, exp, ["A (%s)" % a])
    assert img == exp_img
