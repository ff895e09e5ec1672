"""heightmap_t::proc_gen on the 8192^2 BASELINE terrain (mesh_gen_mode 1 and 4, 8 octaves) with 1000 and 1e5 erosion droplets, two ways alternated in one session:
  sync  tw_proc_gen_heightmap (the host waits for the whole call)
  job   tw_proc_gen_heightmap_launch, completed by tw_create_tiles_poll(wait = 1)
both into device buffers. For each: host time blocked in the call (for the job: in the launch) and launch-to-ready time, medians over --reps after one warm-up,
and whether both ways give identical outputs (image, heights, info). --erode-only times tw_erode (the M_SPEC path) on the mode-4 map instead, which an older
checkout has too: with --root DIR it times that checkout's package, so two versions can be alternated in one session. Prints one JSON line per workload
with the GPU's name and power limit; writes nothing."""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--size", type=int, default=8192)
ap.add_argument("--droplets", type=int, nargs="+", default=[1000, 100000])
ap.add_argument("--modes", type=int, nargs="+", default=[1, 4])
ap.add_argument("--erode-only", action="store_true")
a = ap.parse_args()
sys.path.insert(0, os.path.abspath(a.root))
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
ctx = tw.Context(0)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
n = a.size


def cfg(mode):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)


def digest(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.cpu().numpy().tobytes() if hasattr(t, "cpu") else bytes(t))
    return h.hexdigest()[:16]


if a.erode_only:
    c = cfg(4)
    base = torch.empty((n, n), dtype=torch.float32, device="cuda")
    ctx.heightgen_2d(tw.Grid2D(-0.5 * n, -0.5 * n, float(c.dx_val), float(c.dy_val), n, n), c.height_params(), out=base)
    zmin, _ = ctx.minmax(base)
    ep = c.erosion_params()
    for iters in a.droplets:
        ms, w = [], None
        for r in range(a.reps + 1):
            w = base.clone()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.erode(w, zmin, iters, ep)
            t1 = time.perf_counter()
            if r:
                ms.append(1e3 * (t1 - t0))
        print(json.dumps({"root": os.path.abspath(a.root), "workload": "tw_erode %d^2 mode 4, %d droplets" % (n, iters), "erode_ms": float(np.median(ms)),
                          "min_ms": min(ms), "max_ms": max(ms), "reps": a.reps, "moves": ctx.last_erosion_steps, "digest": digest(w), "gpu": gpu,
                          "power_limit_w": plim}), flush=True)
    sys.exit(0)

for mode in a.modes:
    c = cfg(mode)
    hp, ep = c.height_params(), c.erosion_params()
    for iters in a.droplets:
        bufs = {w: (torch.empty(2 * n * n, dtype=torch.uint8, device="cuda"), torch.empty((n, n), dtype=torch.float32, device="cuda")) for w in ("sync", "job")}
        blocked, ready, infos = {"sync": [], "job": []}, {"sync": [], "job": []}, {}
        for r in range(a.reps + 1):
            for way in ("sync", "job"):
                img, vals = bufs[way]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if way == "sync":
                    _, info, _ = ctx.proc_gen_heightmap(n, n, float(c.dx_val), float(c.dy_val), hp, iters, ep, data16=img, vals=vals)
                    t1 = t2 = time.perf_counter()
                else:
                    job = ctx.proc_gen_heightmap_launch(n, n, float(c.dx_val), float(c.dy_val), hp, iters, ep, data16=img, vals=vals)
                    t1 = time.perf_counter()
                    ctx.create_tiles_poll(True)
                    t2 = time.perf_counter()
                    info = job.info
                infos[way] = bytes(info)
                if r:
                    blocked[way].append(1e3 * (t1 - t0))
                    ready[way].append(1e3 * (t2 - t0))
        dg = {w: digest(*bufs[w]) + ":" + hashlib.sha256(infos[w]).hexdigest()[:8] for w in bufs}
        summary = {w: {"host_blocked_ms": float(np.median(blocked[w])), "ready_ms": float(np.median(ready[w]))} for w in bufs}
        print(json.dumps({"workload": "proc_gen %d^2 mode %d, %d droplets" % (n, mode, iters), "ways": summary, "reps": a.reps,
                          "identical": len(set(dg.values())) == 1, "digests": dg, "gpu": gpu, "power_limit_w": plim}), flush=True)
