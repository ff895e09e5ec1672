"""How long tw_cancel takes to stop each kind of long job: the time from tw_cancel (called right after the launch) to the completing poll that returns
TW_ERR_CANCELED, median over --reps, next to the job's uncancelled launch-to-ready time (one run). That time is the "what still runs" bound: the work
already enqueued behind the cancellation points (pads, tails, end-of-job copies) plus the wait for the next point. Workloads:
  serial     tw_erode_launch, serial order (speculative rounds), 1e6 droplets on an 8192^2 device float map
  image      the same on the context's 8192^2 tw_set_heightmap image (unpack, erode, pack)
  openmp1    tw_erode_launch, OpenMP mode with one thread, 1e6 droplets on the 8192^2 map (one droplet at a time)
  tiles      tw_create_tiles_launch, 64 tiles of 130^2 with 1e6 droplets each
  voxel      tw_voxel_build_launch of a 3 x 3 x 2000004 column: a flood fill of 1e6 generations
Prints one JSON line per workload with the GPU's name and power limit; --out also writes them to a file."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--droplets", type=int, default=1000000)
ap.add_argument("--no-uncancelled", action="store_true", help="skip the uncancelled runs (each takes seconds)")
ap.add_argument("--workloads", nargs="+", default=["serial", "image", "openmp1", "tiles", "voxel"])
ap.add_argument("--out", default=None)
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
from test_voxel_flood_reference import column_case, post_params  # noqa: E402

HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
tcfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(128, 128, 1))
hp, ep, thp, tep = cfg.height_params(), cfg.erosion_params(), tcfg.height_params(), tcfg.erosion_params()
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
ctx = tw.Context(0)
ctx.set_sine_params(tcfg.sine_params())
N = 8192
z0 = torch.empty((N, N), dtype=torch.float32, device="cuda")
ctx.heightgen_2d(cfg.heightmap_grid(N, N), hp, out=z0)
zmin = ctx.minmax(z0)[0]
img, info, _ = ctx.proc_gen_heightmap(N, N, float(cfg.dx_val), float(cfg.dy_val), hp, 0, ep)
origins = [(tx * 128 - 512, ty * 128 - 512) for ty in range(8) for tx in range(8)]
zt = torch.empty((len(origins), 130, 130), dtype=torch.float32, device="cuda")
nz = 2000004
vals, kw = column_case(nz)
vpp = post_params(tw.VoxelPostParams, (3, 3, nz), **kw)
vdev = torch.from_numpy(vals).cuda()


def launch(name):
    """Launches the workload's job on ctx (its inputs restored first, outside the timed window)."""
    if name in ("serial", "openmp1"):
        m = z0.clone()
        torch.cuda.synchronize()
        return lambda: ctx.erode_launch(m, zmin, a.droplets, ep, num_threads=None if name == "serial" else 1)
    if name == "image":
        ctx.set_heightmap(img.reshape(N, N, 2))
        return lambda: ctx.erode_image_launch(info.val_mult, info.val_add, a.droplets, ep)
    if name == "tiles":
        return lambda: ctx.create_tiles_launch(origins, tcfg.mesh_size, float(tcfg.dx_val), float(tcfg.dy_val), 130, thp, a.droplets, tep, tep.zmin, zt)
    if name == "voxel":
        v = vdev.clone()
        torch.cuda.synchronize()
        return lambda: ctx.voxel_build_launch(vpp, vals=v)
    raise SystemExit("unknown workload " + name)


def uncancelled(name):
    go = launch(name)
    t0 = time.perf_counter()
    go()
    assert ctx.create_tiles_poll(True)
    return time.perf_counter() - t0


def cancelled(name):
    go = launch(name)
    go()
    t0 = time.perf_counter()
    ctx.cancel()
    try:
        ctx.create_tiles_poll(True)
        stopped = False
    except tw.TwCanceled:
        stopped = True
    return time.perf_counter() - t0, stopped


lines = []
for name in a.workloads:
    cancelled(name)   # warm-up: modules, scratch, the speculative graph
    runs = [cancelled(name) for _ in range(a.reps)]
    row = {"workload": name, "droplets_or_generations": a.droplets if name != "voxel" else (nz - 2) // 2,
           "cancel_to_poll_ms_median": 1e3 * float(np.median([t for t, _ in runs])), "cancel_to_poll_ms_max": 1e3 * max(t for t, _ in runs),
           "all_cancelled": all(s for _, s in runs), "reps": a.reps,
           "uncancelled_s": None if a.no_uncancelled else uncancelled(name), "gpu": gpu, "power_limit_w": plim}
    print(json.dumps(row), flush=True)
    lines.append(row)
if a.out:
    with open(a.out, "w") as f:
        for row in lines:
            f.write(json.dumps(row) + "\n")
ctx.close()
