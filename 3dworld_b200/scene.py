"""Host-side mirror of the reference's scene/global setup for the terrain path: turns the reference's config keys
(mesh_size, scene_size, mesh_scale, mesh_height, mesh_gen_mode, mesh_gen_shape, mesh_freq_filter, mesh_seed, glaciate, hmap_* ...;
src/3DWorld.cpp:1870-2020) into the explicit POD parameter blocks of include/tw3d.h, following set_scene_constants()
(src/matrix_ops.cpp:57-86), compute_scale() (src/mesh_gen.cpp:544-548), gen_rx_ry() (:581-586) and init_terrain_mesh() /
gen_tex_height_tables() (src/mesh_gen.cpp:407-431, src/Textures.cpp:1757-1761). fp32 arithmetic is done with numpy.float32 so the
derived constants are the ones the reference computes."""
import math
from dataclasses import dataclass, field

import numpy as np

from . import (ErosionParams, Grid2D, HeightParams, Rng, VoxelParams, compute_scale, gen_rx_ry, gen_sine_params, hmap_params,
               water_z_height, MGEN_SINE)

f32 = np.float32


@dataclass
class SceneConfig:
    mesh_size: tuple = (128, 128, 1)           # mesh_size
    scene_size: tuple = (4.0, 4.0, 4.0)        # scene_size
    mesh_scale: float = 1.0
    mesh_height: float = 1.0                   # mesh_height_scale ("mesh_height" config key)
    mesh_gen_mode: int = 0
    mesh_gen_shape: int = 0
    mesh_freq_filter: int = 2                  # FREQ_FILTER
    mesh_seed: int = 0
    mesh_rgen_index: int = 0
    glaciate: int = 1
    custom_glaciate_exp: float = 0.0
    mesh_scale_z: float = 1.0                  # pow(mesh_scale, 0.7) after a zoom; 1 at start-up
    zmax_est: float = 1.0
    hmap: dict = field(default_factory=dict)   # hmap_* keys
    erode_amount: float = 1.0
    water_h_off: float = 0.0
    water_h_off_rel: float = 0.0
    relh_adj_tex: float = 0.0
    temperature: float = 20.0

    # ---- set_scene_constants (src/matrix_ops.cpp:57-86) ----
    @property
    def dx_val(self):
        return f32(f32(2.0) * f32(self.scene_size[0])) / f32(self.mesh_size[0])

    @property
    def dy_val(self):
        return f32(f32(2.0) * f32(self.scene_size[1])) / f32(self.mesh_size[1])

    @property
    def half_dxy(self):
        return f32(0.5) * f32(self.dx_val + self.dy_val)

    @property
    def MESH_HEIGHT(self):
        return f32(0.10) * f32(self.scene_size[2])

    def start_eval_sin(self):
        return compute_scale(self.mesh_scale, self.mesh_freq_filter)

    def height_params(self):
        hp = HeightParams()
        hp.gen_mode, hp.gen_shape = self.mesh_gen_mode, self.mesh_gen_shape
        hp.start_eval_sin = self.start_eval_sin()
        hp.glaciate = self.glaciate
        hp.mesh_scale = self.mesh_scale
        hp.mesh_scale_z_inv = float(f32(1.0 / float(f32(self.mesh_scale_z))))
        hp.dx_val_inv = float(f32(1.0) / self.dx_val)
        hp.dy_val_inv = float(f32(1.0) / self.dy_val)
        hp.mesh_height = float(self.MESH_HEIGHT)
        hp.mesh_height_scale = self.mesh_height
        hp.zmax_est = self.zmax_est
        hp.custom_glaciate_exp = self.custom_glaciate_exp
        hp.rx, hp.ry = gen_rx_ry(self.mesh_seed, self.mesh_rgen_index, self.mesh_gen_mode)
        hp.hmap = hmap_params(**self.hmap)
        return hp

    def sine_params(self, rng=None):
        """gen_rand_sine_table_entries(MESH_HEIGHT*mesh_height_scale) (src/mesh_gen.cpp:219,267)."""
        scaled_height = float(self.MESH_HEIGHT * f32(self.mesh_height))
        return gen_sine_params(scaled_height, mesh=self.mesh_size[:2], scene=self.scene_size[:2], seed=self.mesh_seed,
                               rgen_index=self.mesh_rgen_index, mode=self.mesh_gen_mode, rng=rng)

    def heightmap_grid(self, width, height):
        """heightmap_t::proc_gen: build_arrays(-0.5*width, -0.5*height, DX_VAL, DY_VAL, width, height) (src/heightmap.cpp:135)."""
        return Grid2D(-0.5 * width, -0.5 * height, float(self.dx_val), float(self.dy_val), width, height)

    def water_plane_z(self):
        return water_z_height(self.zmax_est, self.glaciate, self.custom_glaciate_exp, self.water_h_off, self.water_h_off_rel)

    def clip_hd1(self):
        """init_terrain_mesh + gen_tex_height_tables: clip_hd1 = 0.9*h_dirt[1] + 0.1*h_dirt[0], h_dirt[i] = pow(lttex_dirt[i].zval, glaciate_exp)
        (src/mesh_gen.cpp:407-431, src/Textures.cpp:1757-1761); only the sand/dirt entries (both below W_PLANE_Z) are needed."""
        W_PLANE_Z = f32(0.42)
        rel_wpz = f32(min(1.0, max(0.0, float(W_PLANE_Z + f32(self.water_h_off_rel)))))
        glaciate_exp = f32(1.0)
        if self.glaciate:
            glaciate_exp = f32(3.0) if self.custom_glaciate_exp == 0.0 else f32(self.custom_glaciate_exp)
        h = []
        for def_h in (f32(0.40), f32(0.44)):  # mesh_rh_dirt[0..1], src/mesh_gen.cpp:43
            if def_h < W_PLANE_Z:
                hv = f32(def_h * rel_wpz / W_PLANE_Z)
            else:
                rel_h = f32((def_h - W_PLANE_Z) / (f32(1.0) - W_PLANE_Z))
                hv = f32(float(rel_wpz) + float(rel_h) * (1.0 - float(rel_wpz)))
            h.append(f32(math.pow(float(hv), float(glaciate_exp))))  # pow(float,float) -> float
        return float(f32(0.90 * float(h[1]) + 0.10 * float(h[0])))

    def erosion_params(self, zmin=None, zmax=None):
        """The globals apply_erosion reads. zmin/zmax default to -/+zmax_est as set_zvals() leaves them (src/mesh_gen.cpp:494-504)."""
        zmin = -self.zmax_est if zmin is None else zmin
        zmax = self.zmax_est if zmax is None else zmax
        return ErosionParams(self.erode_amount, self.water_plane_z(), float(self.half_dxy), zmin, zmax, self.relh_adj_tex, self.clip_hd1())


def voxel_landscape_params(cfg, nx, ny, nz, zbottom=None, czmin=None, mag=1.0, freq=1.0, geom_rseed=123, rand_gen_index=0,
                           normalize_to_1=1, z_gradient=0.0, invert=0, xoff2=0, yoff2=0, gen_mode=None):
    """setup_voxel_landscape + gen_voxel_landscape (src/voxels.cpp:1851-1878): grid geometry from the scene, seeds (geom_rseed, 456+rand_gen_index)."""
    MX, MY = cfg.mesh_size[0], cfg.mesh_size[1]
    XSS, YSS, ZSS = (f32(v) for v in cfg.scene_size)
    dx, dy = cfg.dx_val, cfg.dy_val
    zbottom = f32(-cfg.zmax_est if zbottom is None else zbottom)
    czmin = zbottom if czmin is None else f32(czmin)
    zlo, zhi = zbottom, f32(min(czmin, zbottom) + ZSS)
    xsz = f32((2.0 * (1.0 - 0.05 / MX) * float(XSS) - float(dx)) / (nx - 1))
    ysz = f32((2.0 * (1.0 - 0.05 / MY) * float(YSS) - float(dy)) / (ny - 1))
    vsz = (xsz, ysz, f32(f32(zhi - zlo) / f32(nz)))
    center = (f32(-0.5) * dx, f32(-0.5) * dy, f32(0.5) * f32(zlo + zhi))
    # lo_pos = center - 0.5*vector3d((nx-1)*vsz.x, ...) (src/voxels.cpp:98)
    lo = tuple(f32(center[d] - f32(0.5) * f32(f32(n - 1) * vsz[d])) for d, n in enumerate((nx, ny, nz)))
    vp = VoxelParams()
    vp.nx, vp.ny, vp.nz = nx, ny, nz
    off = (f32(dx * f32(xoff2)), f32(dy * f32(yoff2)), f32(0.0))
    for d in range(3):
        vp.lo_pos[d], vp.vsz[d], vp.offset[d] = float(lo[d]), float(vsz[d]), float(off[d])
    vp.mag, vp.freq = mag, freq
    vp.gen_mode = cfg.mesh_gen_mode if gen_mode is None else gen_mode
    vp.normalize_to_1 = normalize_to_1
    vp.rseed1, vp.rseed2 = geom_rseed, 456 + rand_gen_index
    vp.octaves = max(1, 5 - cfg.mesh_freq_filter)
    vp.rx, vp.ry = gen_rx_ry(cfg.mesh_seed, cfg.mesh_rgen_index, vp.gen_mode) if vp.gen_mode != MGEN_SINE else (0.0, 0.0)
    vp.zscale = float(f32((-1.0 if invert else 1.0) * z_gradient / (nz - 1)))
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = 0, 0.0, 0.0
    return vp


def gen_mesh(ctx, cfg, erosion_iters=0, xoff2=0, yoff2=0, sine_rng=None):
    """gen_mesh(surface_type=0, keep_sin_table=0, update_zvals=1) in ground mode (src/mesh_gen.cpp:257-355): sine-table entries ->
    gen_mesh_sine_table (:201-210) -> calc_zminmax -> estimate_zminmax (:447-485, a 128x128 probe of the equation) -> set_zvals (:494-504) ->
    glaciate() (:388-404) -> apply_erosion(mesh, X, Y, zbottom, erosion_iters) (:443). All grids are evaluated on the GPU through `ctx`.
    Returns (mesh[MY, MX], dict(zmin, zmax, zmax_est, zbottom, ztop, water_plane_z), sine_params). cfg.zmax_est is updated."""
    MX, MY = cfg.mesh_size[0], cfg.mesh_size[1]
    sp = cfg.sine_params(rng=sine_rng)
    ctx.set_sine_params(sp)
    hp = cfg.height_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    mesh, (zmin, zmax) = ctx.heightgen_2d(Grid2D(float(xoff2 - MX // 2), float(yoff2 - MY // 2), dx, dy, MX, MY), hp, enable_glaciate=0, want_minmax=True)
    zmin, zmax = f32(zmin), f32(zmax)
    zmax_est = max(zmax, -zmin)
    if zmax == zmin:
        zmax_est = f32(float(zmax_est) + 1.0E-6)
    else:
        xy_scene = f32(0.5) * (f32(cfg.scene_size[0]) + f32(cfg.scene_size[1]))
        rm_scale = float(f32(1000.0 * float(xy_scene) / float(f32(cfg.mesh_scale))))
        probe = ctx.heightgen_2d(Grid2D(0.0, 0.0, rm_scale, rm_scale, 128, 128), hp, enable_glaciate=0)
        zmax_est = max(zmax_est, f32(np.abs(probe).max()))
        if cfg.mesh_gen_mode != MGEN_SINE:
            zmax_est = f32(float(zmax_est) * 1.2)
        zmax_est = f32(1.1 * float(zmax_est))
    zbottom, ztop = zmin, zmax                      # set_zvals
    zmin, zmax = -zmax_est, zmax_est
    cfg.zmax_est = float(zmax_est)
    hp = cfg.height_params()
    wpz = cfg.water_plane_z()
    if cfg.glaciate:
        zbottom, ztop = ctx.glaciate_mesh(mesh, xoff2, yoff2, (MX, MY), hp)
    ep = cfg.erosion_params(zmin=float(zmin), zmax=float(zmax))
    if erosion_iters > 0:
        ctx.erode(mesh, float(zbottom), erosion_iters, ep)
    return mesh, dict(zmin=float(zmin), zmax=float(zmax), zmax_est=float(zmax_est), zbottom=float(zbottom), ztop=float(ztop), water_plane_z=float(wpz)), sp


def gen_mesh_async(ctx, cfg, erosion_iters=0, xoff2=0, yoff2=0, sine_rng=None, prev=(0.0, 0.0, 0.0), mesh=None):
    """gen_mesh as one asynchronous job (Context.gen_mesh_launch): the sine table is made and set here, as gen_mesh does, and everything after it runs on
    the device. prev = (zbottom, ztop, water_plane_z) before the call, which a flat mesh keeps. Returns (job, sine_params); job.poll(wait) gives (mesh[MY, MX],
    info) once the job is complete, with gen_mesh's info for a mesh that is not flat. cfg.zmax_est is not updated: set it from info['zmax_est']."""
    sp = cfg.sine_params(rng=sine_rng)
    ctx.set_sine_params(sp)
    job = ctx.gen_mesh_launch(cfg.mesh_size[:2], cfg.height_params(), cfg.erosion_params(), erosion_iters, xoff2, yoff2, float(cfg.dx_val), float(cfg.dy_val),
                              cfg.scene_size[:2], cfg.water_h_off, cfg.water_h_off_rel, prev, mesh)
    return job, sp
