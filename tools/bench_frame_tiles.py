"""A frame's worth of new tiles the way an engine creates them (tile_draw_t::update): the asynchronous path (tw_create_tiles_launch, then
tw_create_tiles_poll(wait=0) until ready) against the three synchronous calls it replaces (tw_create_zvals_batch, tw_tile_bounds_batch,
tw_tile_normals_batch), alternated in one process. Default: 16 tiles of 130^2, BASELINE terrain (mode 4, 8 octaves), 1000 droplets per tile, z range +
sub-block bounds + normal map into pinned host memory; medians over --reps rounds after 3 warm-up rounds. --ao adds the AO map (the synchronous side
then calls tw_create_zvals_ao_batch instead of tw_create_zvals_batch), --weights the terrain weights texture and has_any_grass (tw_tile_weights_batch):
the asynchronous job is then tw_create_tiles_launch_ex. --shadows adds the mesh shadows of two lights (sun and moon, masks and outgoing edges into pinned
memory) through tw_create_tiles_launch_shadows; the synchronous side then also calls tw_tile_shadows_batch once per light on the zvals it made. --hmap takes
the heights from a 7168^2 terrain image built with tw_proc_gen_heightmap and kept in host memory, as an engine keeps a loaded heightmap: the job is
tw_create_tiles_launch_hmap on the image tw_set_heightmap uploaded once (its time is reported), the synchronous side the chain an engine uses without it,
tw_heightmap_sample_tiles on the host image (which uploads the whole image every call) and tw_erode_tiles, then the same tail. Prints one JSON line with the
GPU's name and power limit; writes nothing."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
ap = argparse.ArgumentParser()
ap.add_argument("--tiles", type=int, default=16)
ap.add_argument("--zvsize", type=int, default=130)
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--ao", action="store_true")
ap.add_argument("--weights", action="store_true")
ap.add_argument("--shadows", action="store_true")
ap.add_argument("--hmap", action="store_true")
a = ap.parse_args()
if a.hmap and a.ao:
    ap.error("--hmap: the tile job makes no AO map for heightmap tiles")

nt, zv, iters, size = a.tiles, a.zvsize, a.droplets, a.zvsize - 2
ctx = tw.Context(0)
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                        mesh_size=(size, size, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy, wpz_max = float(cfg.dx_val), float(cfg.dy_val), float(cfg.erosion_params().water_plane_z)
z = torch.empty((nt, zv, zv), dtype=torch.float32).pin_memory()
nrm = torch.empty((nt, zv - 1, zv - 1, 4), dtype=torch.uint8).pin_memory()
mm, mnz, bounds = np.empty((nt, 2), np.float32), np.empty(nt, np.float32), (tw.TileBounds * nt)()
hd = 0.5 * (dx + dy)
ao = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8).pin_memory() if a.ao else None
wts = torch.empty((nt, zv - 1, zv - 1, 4), dtype=torch.uint8).pin_memory() if a.weights else None
grass = np.empty(nt, np.uint8) if a.weights else None
wp, corners = None, None
if a.weights:
    ctx.set_sine_params(cfg.sine_params())
    wp = tw.WeightParams()
    for i, h in enumerate((0.40, 0.44, 0.60, 0.75, 1.0)):
        wp.h_dirt[i], wp.tex_class[i] = h, i
    wp.sthresh[0][0], wp.sthresh[0][1], wp.sthresh[1][0], wp.sthresh[1][1] = 0.68, 0.86, 0.48, 0.72
    wp.zmin, wp.zmax, wp.water_level = -2.3, 2.3, float(ep.water_plane_z)
    wp.noise_scale, wp.vnz_scale, wp.vegetation = 0.003, float(np.float32(np.sqrt(2.0))), 1.0
    wp.dx_val, wp.dy_val, wp.dxdy, wp.xy_mult = dx, dy, dx * dy, 1.0 / size
    corners = np.random.default_rng(1).uniform(-0.2, 1.3, (nt, 8)).astype(np.float32)
shading = dict(ao=ao, weights=wts, has_any_grass=grass, half_dxy=hd, wp=wp, tile_params=corners) if (a.ao or a.weights) else {}
lights = []
if a.shadows:
    for lp in ((3.0, 2.0, 0.15), (-2.0, -4.0, 0.2)):      # sun and moon
        sp = tw.ShadowParams()
        sp.x_scene_size = sp.y_scene_size = float(cfg.scene_size[0])
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
        sp.xy_sum_size, sp.zmin, sp.zmax = 2 * size, float(ep.zmin), float(ep.zmax)
        sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp
        lights.append(tw.Light(sp, torch.empty((nt, zv, zv), dtype=torch.uint8).pin_memory(), torch.empty((nt, zv)).pin_memory(), torch.empty((nt, zv)).pin_memory()))
    shading.update(lights=lights)
hmap, img, upload_ms = None, None, None
if a.hmap:
    N = 7168
    img, info, _ = ctx.proc_gen_heightmap(N, N, dx, dy, hp, 0, ep)
    img = img.reshape(N, N, 2)
    hmap = tw.HmapSampler(N, N, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), info.mesh_file_scale, info.mesh_file_tz, hp.mesh_scale_z_inv)
    t0 = time.perf_counter()
    ctx.set_heightmap(img)
    upload_ms = 1e3 * (time.perf_counter() - t0)
    shading.update(hmap=hmap)
launch_ms, ready_ms, sync_ms = [], [], []
for r in range(a.reps + 3):
    origins = [((r * 5 + t % 4) * size, (t // 4 + r) * size) for t in range(nt)]   # new tiles every frame
    t0 = time.perf_counter()
    ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, z, mm=mm, bounds=bounds, normals=nrm, min_normal_z=mnz,
                            wpz_max=wpz_max, size=size, tile_xy=np.asarray(origins, np.int32) // size if a.shadows else None, **shading)
    t1 = time.perf_counter()
    while not ctx.create_tiles_poll(wait=False):
        pass
    t2 = time.perf_counter()
    if a.hmap:
        ctx.heightmap_sample_tiles(img, hmap, origins, zv, out=z)
        ctx.erode_tiles(z, iters, ep, min_zval_all=ep.zmin)
        zn = z.numpy().reshape(nt, -1)
        mm[:, 0], mm[:, 1] = zn.min(1), zn.max(1)
    elif a.ao:
        ctx.create_zvals_ao_batch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, hd, out=z, ao=ao, want_minmax=True)
    else:
        ctx.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, out=z, want_minmax=True)
    ctx.tile_bounds(z, wpz_max, dx, dy, size)
    ctx.tile_normals(z, dx, dy, out=nrm)
    if a.weights:
        ctx.tile_weights(z, origins, cfg.mesh_size, dx, dy, hp, wp, corners, out=wts)
    for L in lights:
        ctx.tile_shadows(z, np.asarray(origins, np.int32) // size, L.sp, out=L.smask)
    t3 = time.perf_counter()
    if r >= 3:
        launch_ms.append(1e3 * (t1 - t0))
        ready_ms.append(1e3 * (t2 - t0))
        sync_ms.append(1e3 * (t3 - t2))
try:
    name, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                    capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    name, plim = None, None
extra = "".join(s for s, on in ((" + AO map", a.ao), (" + weights texture", a.weights), (" + mesh shadows of 2 lights", a.shadows)) if on)
src = "heights from a 7168^2 host heightmap image (mode 4 8-octave terrain)" if a.hmap else "mode 4 8-octave"
res = {"workload": "%d tiles of %d^2, %s + %d droplets per tile, z range + bounds + normal map%s, pinned host outputs" % (nt, zv, src, iters, extra),
       "launch_host_ms": float(np.median(launch_ms)), "launch_host_ms_max": max(launch_ms), "launch_to_ready_ms": float(np.median(ready_ms)),
       ("sync_calls_ms" if extra or a.hmap else "sync_three_calls_ms"): float(np.median(sync_ms)), "rounds": a.reps, "gpu": name, "power_limit_w": plim}
if a.hmap:
    res["set_heightmap_once_ms"] = upload_ms
print(json.dumps(res))
