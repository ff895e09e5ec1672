"""tw_erode_launch_ex's sweeps job on the 7168^2 BASELINE image (mode 4, made by tw_proc_gen_heightmap_launch(set_image=1)) with 1e7 droplets, three ways
alternated in one session:
  sweeps  tw_erode_launch_ex(TW_EROSION_SWEEPS) on the context's image, completed by tw_create_tiles_poll(wait = 1)
  sync    the chain it replaces on a host image: tw_heightmap_to_floats_u16 -> tw_minmax_f32 -> tw_erode_sweeps -> tw_heightmap_from_floats_u16 -> tw_set_heightmap
  openmp  tw_erode_launch's OpenMP mode (num_threads = 0) on the image
For each: host time blocked in the call (for the jobs: in the launch), launch-to-ready time, droplets/s and moves/s (medians over --reps after one warm-up);
whether the sweeps job and the chain give identical image bytes and steps, and whether two sweeps runs do. Then the sweeps job alone at every --sizes
sweep (one run each after the main comparison's warm-up), and one tw_cancel right after the launch: cancel-to-poll time against the uncancelled
launch-to-ready time. Prints one JSON line with the GPU's name and power limit (--out also writes it there)."""
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
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--size", type=int, default=7168)
ap.add_argument("--droplets", type=int, default=10000000)
ap.add_argument("--sweep", type=int, default=9472)
ap.add_argument("--halo", type=int, default=64)
ap.add_argument("--sizes", type=int, nargs="*", default=[2048, 9472, 65536])
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
hp, ep = cfg.height_params(), cfg.erosion_params()
ctx = tw.Context(0)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
n, iters = a.size, a.droplets
host_img = torch.empty(2 * n * n, dtype=torch.uint8).pin_memory().numpy()   # the loaded map every way starts from
job = ctx.proc_gen_heightmap_launch(n, n, float(cfg.dx_val), float(cfg.dy_val), hp, 0, ep, data16=host_img, set_image=True)
ctx.create_tiles_poll(True)
mult, add = job.info.val_mult, job.info.val_add


def digest(x):
    return hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()[:16]


def run(way, sweep):
    """One run from the same loaded map; returns (host blocked ms, ready ms, steps, eroded floats)."""
    ctx.set_heightmap(host_img.reshape(n, n, 2))
    torch.cuda.synchronize()
    vals = torch.empty((n, n), dtype=torch.float32, device="cuda")
    t0 = time.perf_counter()
    if way == "sync":
        v = ctx.to_floats_u16(host_img, mult, add).reshape(n, n)
        zmin, _ = ctx.minmax(v)
        steps = ctx.erode_sweeps(v, zmin, iters, ep, sweep, a.halo)
        ctx.set_heightmap(ctx.from_floats_u16(v, mult, add).reshape(n, n, 2))
        t2 = time.perf_counter()
        return 1e3 * (t2 - t0), 1e3 * (t2 - t0), steps, v
    if way == "sweeps":
        ctx.erode_image_launch(mult, add, iters, ep, vals=vals, sweep=sweep, halo=a.halo)
    else:
        ctx.erode_image_launch(mult, add, iters, ep, num_threads=0, vals=vals)
    t1 = time.perf_counter()
    ctx.create_tiles_poll(True)
    t2 = time.perf_counter()
    return 1e3 * (t1 - t0), 1e3 * (t2 - t0), ctx.last_erosion_steps, vals.cpu().numpy()


ways = {"sweeps": [], "sync": [], "openmp": []}
outs = {}
for r in range(a.reps + 1):
    for way in ways:
        blocked, ready, steps, v = run(way, a.sweep)
        outs.setdefault(way, []).append((steps, v))
        if r:
            ways[way].append((blocked, ready, steps))
moves_sync, v_sync = outs["sync"][-1]
(s1, v1), (s2, v2) = outs["sweeps"][-2], outs["sweeps"][-1]
b_sync, b_job = (ctx.from_floats_u16(v, mult, add) for v in (v_sync, v1))   # the image bytes each way leaves
summary = {}
for way, rs in ways.items():
    ready_ms = float(np.median([x[1] for x in rs]))
    steps = rs[-1][2]
    summary[way] = {"host_blocked_ms": float(np.median([x[0] for x in rs])), "ready_ms": ready_ms, "steps": int(steps),
                    "droplets_per_s": iters / (ready_ms * 1e-3), "moves_per_s": steps / (ready_ms * 1e-3)}
result = {"workload": "image %d^2 (mode 4), %d droplets, sweep %d, halo %d" % (n, iters, a.sweep, a.halo), "ways": summary, "reps": a.reps,
          "sweeps_two_runs_identical": bool(s1 == s2 and np.array_equal(v1.view(np.uint32), v2.view(np.uint32))),
          "sweeps_equals_sync_chain": bool(s1 == moves_sync and np.array_equal(v1.view(np.uint32), v_sync.view(np.uint32)) and np.array_equal(b_job, b_sync)),
          "digests": {"sweeps": digest(v1), "sync": digest(v_sync)}}
by_size = {}
for sweep in a.sizes:
    _, ready, steps, _ = run("sweeps", sweep)
    by_size[str(sweep)] = {"ready_ms": ready, "steps": int(steps), "droplets_per_s": iters / (ready * 1e-3), "moves_per_s": steps / (ready * 1e-3)}
result["sweep_sizes"] = by_size
# one cancel right after the launch
ctx.set_heightmap(host_img.reshape(n, n, 2))
torch.cuda.synchronize()
ctx.erode_image_launch(mult, add, iters, ep, sweep=a.sweep, halo=a.halo)
t0 = time.perf_counter()
ctx.cancel()
try:
    ctx.create_tiles_poll(True)
    cancelled = False
except tw.TwCanceled:
    cancelled = True
result["cancel"] = {"cancel_to_poll_ms": 1e3 * (time.perf_counter() - t0), "uncancelled_ready_ms": summary["sweeps"]["ready_ms"], "cancelled": cancelled}
result.update({"gpu": gpu, "power_limit_w": plim})
line = json.dumps(result)
print(line, flush=True)
if a.out:
    with open(a.out, "w") as f:
        f.write(line + "\n")
ctx.close()
