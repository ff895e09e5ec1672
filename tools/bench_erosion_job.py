"""tw_erode_launch against the synchronous chains it replaces, two ways alternated in one session, on three workloads:
  image 7168^2, 1e7 droplets, OpenMP mode (num_threads = 0)   the BASELINE terrain (mode 4, 8 octaves) made by tw_proc_gen_heightmap_launch(set_image=1);
  image 7168^2, 1e5 droplets, serial order                     heightmap_t::run_erosion on the loaded map (src/heightmap.cpp:153-187)
  float map 8192^2 on the device, 1e5 droplets, serial order
  sync  the image in host memory: tw_heightmap_to_floats_u16 -> tw_minmax_f32 -> tw_erode / tw_erode_parallel -> tw_heightmap_from_floats_u16 ->
        tw_set_heightmap (for the float map: tw_erode on the map in host memory)
  job   tw_erode_launch on the context's image (the float map: on the device tensor), completed by tw_create_tiles_poll(wait = 1)
For each: host time blocked in the call (for the job: in the launch) and launch-to-ready time, medians over --reps after one warm-up. The serial ways must give
identical eroded floats and step counts; for the OpenMP mode, whose result depends on timing, it records the properties tests/test_gpu_erosion.py holds
tw_erode_parallel to (step counts, share of identical cells, total height moved). Prints one JSON line per workload with the GPU's name and power limit;
writes nothing."""
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
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--image-size", type=int, default=7168)
ap.add_argument("--map-size", type=int, default=8192)
ap.add_argument("--omp-droplets", type=int, default=10000000)
ap.add_argument("--serial-droplets", type=int, default=100000)
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
hp, ep = cfg.height_params(), cfg.erosion_params()
ctx = tw.Context(0)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]


def digest(x):
    return hashlib.sha256(np.ascontiguousarray(x.cpu().numpy() if hasattr(x, "cpu") else x).tobytes()).hexdigest()[:16]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t1 = fn()
    t2 = time.perf_counter()
    return 1e3 * ((t1 or t2) - t0), 1e3 * (t2 - t0)


def report(workload, ways, extra):
    summary = {w: {"host_blocked_ms": float(np.median([b for b, _ in ways[w]])), "ready_ms": float(np.median([r for _, r in ways[w]]))} for w in ways}
    print(json.dumps(dict({"workload": workload, "ways": summary, "reps": a.reps, "gpu": gpu, "power_limit_w": plim}, **extra)), flush=True)


# ---- the image
n = a.image_size
host_img = torch.empty(2 * n * n, dtype=torch.uint8).pin_memory().numpy()   # the loaded map the synchronous chain starts from
job = ctx.proc_gen_heightmap_launch(n, n, float(cfg.dx_val), float(cfg.dy_val), hp, 0, ep, data16=host_img, set_image=True)
ctx.create_tiles_poll(True)
mult, add = job.info.val_mult, job.info.val_add
base = ctx.to_floats_u16(host_img, mult, add).reshape(n, n)
for iters, threads in ((a.omp_droplets, 0), (a.serial_droplets, None)):
    ways, out = {"sync": [], "job": []}, {}
    vals_job = torch.empty((n, n), dtype=torch.float32, device="cuda")
    for r in range(a.reps + 1):
        for way in ("sync", "job"):
            ctx.set_heightmap(host_img.reshape(n, n, 2))                               # the same map before every run
            if way == "sync":
                def chain():
                    v = ctx.to_floats_u16(host_img, mult, add).reshape(n, n)
                    zmin, _ = ctx.minmax(v)
                    if threads is None:
                        ctx.erode(v, zmin, iters, ep)
                    else:
                        ctx.erode_parallel(v, zmin, iters, ep, num_threads=threads)
                    out["sync"] = (v, ctx.last_erosion_steps)
                    ctx.set_heightmap(ctx.from_floats_u16(v, mult, add).reshape(n, n, 2))
                t = timed(chain)
            else:
                def launch():
                    ctx.erode_image_launch(mult, add, iters, ep, num_threads=threads, vals=vals_job)
                    t1 = time.perf_counter()
                    ctx.create_tiles_poll(True)
                    return t1
                t = timed(launch)
                out["job"] = (vals_job.cpu().numpy(), ctx.last_erosion_steps)
            if r:
                ways[way].append(t)
    (vs, ss), (vj, sj) = out["sync"], out["job"]
    extra = {"steps": {"sync": ss, "job": sj}}
    if threads is None:
        extra["identical"] = bool(ss == sj and np.array_equal(vs.view(np.uint32), vj.view(np.uint32)))
        extra["digests"] = {"sync": digest(vs), "job": digest(vj)}
    else:   # timing-dependent: the properties of test_erode_parallel_many_threads_close_to_serial, sync against job
        moved = {w: float(np.abs(v.astype(np.float64) - base).sum()) for w, v in (("sync", vs), ("job", vj))}
        extra.update({"same_cells": float((vs == vj).mean()), "height_moved": moved, "finite": bool(np.isfinite(vj).all())})
    report("image %d^2 (mode 4), %d droplets, %s" % (n, iters, "serial order" if threads is None else "OpenMP mode, num_threads %d" % threads), ways, extra)

# ---- the float map on the device
n, iters = a.map_size, a.serial_droplets
dev = torch.empty((n, n), dtype=torch.float32, device="cuda")
ctx.heightgen_2d(cfg.heightmap_grid(n, n), hp, out=dev)
zmin, _ = ctx.minmax(dev)
host = dev.cpu().numpy()
ways, out = {"sync": [], "job": []}, {}
for r in range(a.reps + 1):
    for way in ("sync", "job"):
        if way == "sync":
            m = host.copy()

            def erode():
                ctx.erode(m, zmin, iters, ep)
                out["sync"] = (m, ctx.last_erosion_steps)
            t = timed(erode)
        else:
            m = dev.clone()

            def launch():
                ctx.erode_launch(m, zmin, iters, ep)
                t1 = time.perf_counter()
                ctx.create_tiles_poll(True)
                out["job"] = (m, ctx.last_erosion_steps)
                return t1
            t = timed(launch)
        if r:
            ways[way].append(t)
(vs, ss), (vj, sj) = out["sync"], out["job"]
vj = vj.cpu().numpy()
report("float map %d^2 (mode 4) on the device, %d droplets, serial order" % (n, iters), ways,
       {"steps": {"sync": ss, "job": sj}, "identical": bool(ss == sj and np.array_equal(vs.view(np.uint32), vj.view(np.uint32))),
        "digests": {"sync": digest(vs), "job": digest(vj)}})
ctx.close()
