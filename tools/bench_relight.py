"""Relighting resident tiles with a tile set (tw_tile_set_*) against the per-call mesh shadows, on squares of BASELINE tiles (mode 4, 8-octave domain warp,
1000 droplets per tile, made with tw_create_zvals_batch): 32 x 32 tiles of 130^2 and 16 x 16 tiles of 258^2, sun and moon, outputs in pinned host memory.
The ways are alternated in one session:
  (a) the sun moves every frame (the moon stays):
      host   - tw_tile_shadows_batch per light on the zvals in (pageable) host memory, as the engine does today;
      device - the same call on device zvals (what residency alone saves);
      set    - tw_tile_set_shadows_launch of every tile with both lights: the host time in the launch, and launch to ready (the moon comes from the cache).
  (b) a row of 16 new tiles appears on the light side: put, stale, relight of the stale tiles - tiles recomputed and put-to-ready time - against a full
      relight (every slot's params changed). The row is removed and the set relit (untimed) before the next round.
Every set relight is checked against tw_tile_shadows_batch on the same tiles once per configuration. Prints one JSON line with the GPU's name and power
limit; writes nothing."""
import argparse
import ctypes as C
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
ap.add_argument("--configs", nargs="+", default=["32x130", "16x258"], help="side x zvsize")
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--frames", type=int, default=20, help="frames per way per round in (a)")
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()
L = tw.lib


def stats(v):
    v = np.asarray(v, np.float64)
    return {"median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}


def run_config(ctx, side, zv):
    size = zv - 2
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                            mesh_size=(size, size, 1))
    hp, ep = cfg.height_params(), cfg.erosion_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    keys = [(x, y) for y in range(side) for x in range(side)]
    row = [(x, side) for x in range(16)]                         # the new row, next to the square on the sun's side (+y)
    z_all = ctx.create_zvals_batch([((x - side // 2) * size, (y + 20) * size) for x, y in keys + row], cfg.mesh_size, dx, dy, zv, hp, a.droplets, ep, ep.zmin)
    z, z_row = np.ascontiguousarray(z_all[:len(keys)]), np.ascontiguousarray(z_all[len(keys):])
    dz = torch.from_numpy(z).cuda()
    txy, rxy = np.array(keys, np.int32), np.array(row, np.int32)
    nt = len(keys)

    def light(lp):
        sp = tw.ShadowParams()
        sp.x_scene_size, sp.y_scene_size = float(cfg.scene_size[0]), float(cfg.scene_size[1])
        sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * size, float(ep.zmin), float(ep.zmax), 0
        for d in range(3):
            sp.lpos[d] = lp[d]
        return sp

    def sun(f):
        return light((3.0 + 0.01 * f, 2.0, 0.15))
    moon = light((-2.0, -4.0, 0.2))

    def pinned(shape, dtype):
        return torch.empty(shape, dtype=dtype).pin_memory()
    outs = [(pinned((nt + 16, zv, zv), torch.uint8), pinned((nt + 16, zv), torch.float32), pinned((nt + 16, zv), torch.float32)) for _ in range(2)]

    def batch(zsrc, sp, o):
        ctx._check(L.tw_tile_shadows_batch(ctx._h, tw._ptr(zsrc), tw._ptr(txy), nt, zv, C.byref(sp), o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr()))

    ts = ctx.tile_set(zv, 2)
    ts.put(keys, dz)

    def relight(req, sps):
        n = len(req)
        lights = [tw.Light(sp, o[0][:n], o[1][:n], o[2][:n]) for sp, o in zip(sps, outs)]
        t0 = time.perf_counter()
        rec = ts.shadows_launch(req, lights)
        t1 = time.perf_counter()
        while not ctx.create_tiles_poll(wait=False):
            pass
        return 1e3 * (t1 - t0), 1e3 * (time.perf_counter() - t0), rec

    # check once: the set's outputs equal tw_tile_shadows_batch on the same tiles
    identical = True
    relight(txy, [sun(0), moon])
    got = [tuple(x[:nt].numpy().copy() for x in o) for o in outs]
    for sp, g in zip((sun(0), moon), got):
        e = (np.empty((nt, zv, zv), np.uint8), np.empty((nt, zv), np.float32), np.empty((nt, zv), np.float32))
        ctx._check(L.tw_tile_shadows_batch(ctx._h, tw._ptr(z), tw._ptr(txy), nt, zv, C.byref(sp), tw._ptr(e[0]), tw._ptr(e[1]), tw._ptr(e[2])))
        identical = identical and all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(g, e))
    # warm-up of every way
    batch(z, sun(0), outs[0]); batch(dz, sun(0), outs[0]); torch.cuda.synchronize()
    # (a) the sun moves every frame
    host, dev, set_launch, set_ready = [], [], [], []
    f = 1
    for _ in range(a.rounds):
        for way in ("host", "device", "set"):
            for _ in range(a.frames):
                f += 1
                if way == "set":
                    tl, tr, rec = relight(txy, [sun(f), moon])
                    set_launch.append(tl)
                    set_ready.append(tr)
                    continue
                t0 = time.perf_counter()
                for sp, o in ((sun(f), outs[0]), (moon, outs[1])):
                    batch(z if way == "host" else dz, sp, o)
                (host if way == "host" else dev).append(1e3 * (time.perf_counter() - t0))
    # (b) a row of 16 new tiles on the sun's side
    new_ready, new_rec, full_ready = [], [], []
    all_xy = np.concatenate([txy, rxy])
    for r in range(a.rounds):
        for way in ("new_row", "full"):
            if way == "new_row":
                t0 = time.perf_counter()
                ts.put(rxy, z_row)
                stale = ts.stale([sun(f), moon])
                _, _, rec = relight(stale, [sun(f), moon])
                new_ready.append(1e3 * (time.perf_counter() - t0))
                new_rec.append(int(rec.sum()))
                ts.remove(rxy)
                relight(txy, [sun(f), moon])                   # untimed: the square is valid again
            else:
                ts.put(rxy, z_row)
                f += 1
                tl, tr, rec = relight(all_xy, [sun(f), light((-2.0, -4.0, 0.2 + 0.001 * (r + 1)))])
                full_ready.append(tr)
                ts.remove(rxy)
                relight(txy, [sun(f), moon])
    ts.close()
    return {"config": "%d x %d tiles of %d^2 (+ a row of 16)" % (side, side, zv), "tiles": nt, "outputs_identical_to_batch": identical,
            "sun_moves": {"host_zvals_batch_per_light_ms": stats(host), "device_zvals_batch_per_light_ms": stats(dev),
                          "set_relight_launch_ms": stats(set_launch), "set_relight_ready_ms": stats(set_ready)},
            "new_row_on_light_side": {"put_stale_relight_ready_ms": stats(new_ready), "tiles_recomputed": stats(new_rec),
                                      "full_relight_ready_ms": stats(full_ready), "full_relight_tiles": nt + 16}}


ctx = tw.Context(0)
res = {"workload": "BASELINE tiles (mode 4, 8 octaves, %d droplets), sun and moon, outputs in pinned host memory; %d frames x %d rounds per way" %
                   (a.droplets, a.frames, a.rounds), "results": []}
for c in a.configs:
    side, zv = (int(v) for v in c.split("x"))
    res["results"].append(run_config(ctx, side, zv))
ctx.close()
try:
    name, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                    capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    name, plim = None, None
res["gpu"], res["power_limit_w"] = name, plim
print(json.dumps(res))
sys.exit(0 if all(r["outputs_identical_to_batch"] for r in res["results"]) else 1)
