"""Brush edits of the 7168^2 BASELINE image (mode 4, made by tw_proc_gen_heightmap_launch(set_image=1)) while a 32 x 32 tile set of 130^2 heightmap tiles is
kept live on a pool of 8 shared contexts, at 60 Hz. Every frame applies one brush stroke (a square rect of 64, 256 or 512 texels, in turn, whose texels'
high byte goes up by 1 on the host image) and re-creates the tiles it touches (tw_hmap_tiles_touched) in one tile-set frame with 1000 droplets per tile,
relighting for sun and moon what tw_tile_set_stale_after names. Two ways, run one after the other from the same map and set:
  edit    tw_update_heightmap(the stroke's rect), then the frame on the next pool context
  reload  tw_set_heightmap(the whole image), then the same frame
Each way first runs one warm-up frame of the largest brush per pool context (untimed). For each: host time blocked per frame in the library calls, the wait
for the slot's previous frame included (median, p99, max; that wait also on its own), launch-to-ready per frame (polls after every frame's calls and between
frames), the wall time of the timed frames and the frames per second it gives, and whether every frame's zvals and shadow outputs are identical byte for
byte between the two ways. Then the edit kernel alone: its device time from torch.profiler over
--kernel-reps edits of each brush size on an idle context. Prints one JSON line with the GPU's name and power limit (--out also writes it there)."""
import argparse
import hashlib
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

ap = argparse.ArgumentParser()
ap.add_argument("--size", type=int, default=7168)
ap.add_argument("--frames", type=int, default=60)
ap.add_argument("--pool", type=int, default=8)
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--brushes", type=int, nargs="*", default=[64, 256, 512])
ap.add_argument("--kernel-reps", type=int, default=200)
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
S, ZV, NT = 128, 130, 32
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy = float(cfg.dx_val), float(cfg.dy_val)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
n = a.size
ctx = tw.Context(0)
pool = [ctx.shared() for _ in range(a.pool)]
map0 = torch.empty((n, n, 2), dtype=torch.uint8).pin_memory().numpy()
job = ctx.proc_gen_heightmap_launch(n, n, dx, dy, hp, 0, ep, data16=map0, set_image=True)
ctx.create_tiles_poll(True)
hs = tw.HmapSampler(n, n, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), job.info.mesh_file_scale, job.info.mesh_file_tz,
                    hp.mesh_scale_z_inv)
keys = np.array([(x, y) for y in range(-NT // 2, NT // 2) for x in range(-NT // 2, NT // 2)], np.int32)
origins = keys * S


def light(lp):
    sp = tw.ShadowParams()
    sp.x_scene_size, sp.y_scene_size = float(cfg.scene_size[0]), float(cfg.scene_size[1])
    sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * S, float(ep.zmin), float(ep.zmax), 0
    sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp
    return sp


sps = [light((3.0, 2.0, 0.15)), light((-2.0, -3.0, 0.2))]     # sun and moon
nk = len(keys)
bufs = [dict(z=torch.empty((nk, ZV, ZV), dtype=torch.float32).pin_memory(),
             m=[torch.empty((nk, ZV, ZV), dtype=torch.uint8).pin_memory() for _ in sps],
             x=[torch.empty((nk, ZV), dtype=torch.float32).pin_memory() for _ in sps],
             y=[torch.empty((nk, ZV), dtype=torch.float32).pin_memory() for _ in sps]) for _ in range(a.pool)]


def launch(ts, c, b, txy, org, rxy):
    k, r = len(txy), len(rxy)
    lights = [tw.Light(sp, b["m"][i][:r], b["x"][i][:r], b["y"][i][:r]) for i, sp in enumerate(sps)]
    ts.create_tiles_launch(org, cfg.mesh_size, dx, dy, hp, a.droplets, ep, ep.zmin, txy, zvals=b["z"][:k], relight_xy=rxy, lights=lights, hmap=hs, ctx=c)


def digest(b, k, r):
    h = hashlib.sha256(b["z"][:k].numpy().tobytes())
    for i in range(len(sps)):
        for t in (b["m"][i][:r], b["x"][i][:r], b["y"][i][:r]):
            h.update(t.numpy().tobytes())
    return h.hexdigest()[:16]


def strokes():
    """--pool warm-up strokes of the largest brush (every pool context's first frame grows its scratch and staging), then --frames timed ones."""
    rng = np.random.default_rng(1)
    lo, hi = n // 2 - NT // 2 * S, n // 2 + NT // 2 * S                  # texels the live tiles cover (mesh_scale 1)
    for f in range(a.pool + a.frames):
        w = max(a.brushes) if f < a.pool else a.brushes[f % len(a.brushes)]
        yield f >= a.pool, (int(rng.integers(lo, hi - w)), int(rng.integers(lo, hi - w)), w, w)


def run(way):
    """One way: the stats of the timed frames and every frame's output digest. A frame's host time counts everything the frame's library calls block for,
    including the wait for the slot's previous frame; a frame is ready when a poll first finds it complete, and polls run after every frame's calls (the
    reload's tw_set_heightmap completes every frame in flight) and between frames until the next 60 Hz tick."""
    img = map0.copy()
    ctx.set_heightmap(img)
    ts = ctx.tile_set(ZV, len(sps))
    launch(ts, ctx, bufs[0], keys, origins, keys)                          # the live set, fully relit
    ctx.create_tiles_poll(True)
    blocked, slot_wait, ready, digests, pending = [], [], [], {}, {}
    t_start = t_next = None

    def done(kk, t):
        f0, t_launch, k2, r2, timed = pending.pop(kk)
        if timed:
            ready.append(t - t_launch)
        digests[f0] = digest(bufs[kk], k2, r2)

    def sweep():
        for kk in list(pending):
            if pool[kk].create_tiles_poll(False):
                done(kk, time.perf_counter())

    for f, (timed, rect) in enumerate(strokes()):
        x, y, w, h = rect
        img[y:y + h, x:x + w, 1] = np.minimum(img[y:y + h, x:x + w, 1], 253) + 1      # the brush (the engine's own code)
        if timed and t_start is None:
            t_start = t_next = time.perf_counter()
        k = f % a.pool
        c, b = pool[k], bufs[k]
        t0 = time.perf_counter()
        if k in pending:                                                   # the slot's previous frame
            c.create_tiles_poll(True)
            done(k, time.perf_counter())
        t1 = time.perf_counter()
        if way == "edit":
            ctx.update_heightmap(img, [rect])
        else:
            ctx.set_heightmap(img)
        touched = tw.hmap_tiles_touched(hs, origins, ZV, [rect]) == 1
        txy = keys[touched]
        rxy = ts.stale_after(sps, put_xy=txy)
        launch(ts, c, b, txy, origins[touched], rxy)
        t2 = time.perf_counter()
        if timed:
            blocked.append(t2 - t0)
            slot_wait.append(t1 - t0)
        pending[k] = (f, t2, len(txy), len(rxy), timed)
        sweep()
        if timed:
            t_next += 1.0 / 60.0
            while time.perf_counter() < t_next:                            # busy-poll the frames in flight until the next tick
                sweep()
    for kk in list(pending):
        pool[kk].create_tiles_poll(True)
        done(kk, time.perf_counter())
    wall = time.perf_counter() - t_start
    ts.close()
    ms = lambda v: round(1e3 * float(v), 3)  # noqa: E731
    bl = np.array(blocked)
    return dict(blocked_ms_median=ms(np.median(bl)), blocked_ms_p99=ms(np.percentile(bl, 99)), blocked_ms_max=ms(bl.max()),
                slot_wait_ms_median=ms(np.median(slot_wait)), slot_wait_ms_max=ms(max(slot_wait)),
                ready_ms_median=ms(np.median(ready)), ready_ms_p99=ms(np.percentile(ready, 99)), ready_ms_max=ms(max(ready)),
                wall_s=round(wall, 3), frames_per_s=round(a.frames / wall, 2)), [digests[f] for f in range(a.pool + a.frames)]


res = {}
res["edit"], dig_edit = run("edit")
res["reload"], dig_reload = run("reload")
res["frames_identical"] = dig_edit == dig_reload

# the edit kernel alone, on an idle context: device time of hmap_scatter_kernel per edit
ctx.set_heightmap(map0)
kernel = {}
for w in a.brushes:
    rect = [((n - w) // 2, (n - w) // 2, w, w)]
    for _ in range(10):
        ctx.update_heightmap(map0, rect)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.kernel_reps):
            ctx.update_heightmap(map0, rect)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "hmap_scatter_kernel" in e.name]
    dt = [getattr(e, "device_time", None) or e.cuda_time for e in ev]
    kernel[str(w)] = dict(kernels=len(ev), us_median=round(float(np.median(dt)), 2) if dt else None,
                          gb_per_s=round(2 * 2 * w * w / (np.median(dt) * 1e-6) / 1e9, 1) if dt else None)   # read + write of 2-byte texels
res["edit_kernel"] = kernel
res.update(gpu=gpu, power_limit_w=plim, size=n, tiles=nk, zvsize=ZV, pool=a.pool, droplets=a.droplets, frames=a.frames, brushes=a.brushes)
line = json.dumps(res)
print(line)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")
