"""The ground-mode mesh (gen_mesh) as one asynchronous job (tw_gen_mesh_launch, scene.gen_mesh_async) against the synchronous chain it replaces
(scene.gen_mesh: tw_heightgen_2d of the mesh and of the 128^2 probe, the host's z arithmetic, tw_glaciate_mesh, tw_erode), alternated in one run on one device.
Workloads: BASELINE config 1 (128^2, sine mode, seed 6, glaciation) with 0 and 1500 droplets, and a 1024^2 mode-4 mesh with 1e5 droplets (the speculative
erosion). The mesh is a page-locked host buffer for the job and a numpy array for the chain. Medians over --reps after --warmup:
  sync_ms     host time of scene.gen_mesh (every step blocks)
  blocked_ms  host time blocked in scene.gen_mesh_async (the sine table and the launch)
  ready_ms    time from the start of that call to the poll that reports the job complete (polled with wait = 0 in a loop)
Outputs (mesh, the six z values, the step count) are checked bit for bit between the two every rep. Prints one JSON line with the GPU's name and power limit
(--out also writes it there)."""
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

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
WORKLOADS = [
    ("cfg1_128_sine_0", dict(mesh_gen_mode=0, mesh_freq_filter=2, mesh_seed=6, glaciate=1), 0),
    ("cfg1_128_sine_1500", dict(mesh_gen_mode=0, mesh_freq_filter=2, mesh_seed=6, glaciate=1), 1500),
    ("dwarp_1024_1e5", dict(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, mesh_size=(1024, 1024, 1), scene_size=(32.0, 32.0, 4.0)), 100000),
]
ZKEYS = ("zmin", "zmax", "zmax_est", "zbottom", "ztop", "water_plane_z")
ctx = tw.Context(0)
res = dict(gpu=gpu, power_limit_w=plim, reps=a.reps, workloads={})
for name, kw, iters in WORKLOADS:
    cfg = scene.SceneConfig(**kw)
    MX, MY = cfg.mesh_size[:2]
    pinned = torch.empty((MY, MX), dtype=torch.float32).pin_memory()
    sync_ms, blocked_ms, ready_ms, identical = [], [], [], True
    for rep in range(a.warmup + a.reps):
        cfg.zmax_est = 1.0
        t0 = time.perf_counter()
        want, zw, _ = scene.gen_mesh(ctx, cfg, erosion_iters=iters)
        t1 = time.perf_counter()
        steps_w = ctx.last_erosion_steps if iters else 0
        cfg.zmax_est = 1.0
        t2 = time.perf_counter()
        job, _ = scene.gen_mesh_async(ctx, cfg, iters, mesh=pinned)
        t3 = time.perf_counter()
        while True:
            r = job.poll(False)
            if r is not None:
                break
        t4 = time.perf_counter()
        got, z = r
        same = (np.array_equal(got.numpy().view(np.uint32), want.view(np.uint32)) and all(np.float32(z[k]) == np.float32(zw[k]) for k in ZKEYS)
                and z["erosion_moves"] == steps_w)
        identical = identical and same
        if rep >= a.warmup:
            sync_ms.append(1e3 * (t1 - t0)); blocked_ms.append(1e3 * (t3 - t2)); ready_ms.append(1e3 * (t4 - t2))
    res["workloads"][name] = dict(mesh=[MX, MY], droplets=iters, sync_ms=float(np.median(sync_ms)), blocked_ms=float(np.median(blocked_ms)),
                                  ready_ms=float(np.median(ready_ms)), identical=bool(identical))
ctx.close()
line = json.dumps(res)
print(line)
if a.out:
    with open(a.out, "w") as f:
        f.write(line + "\n")
