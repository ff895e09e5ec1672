"""Object placement as the points job (tw_points_launch) on one device: 1e5 and 1e6 TW_PQ_EXACT_ZVAL points on the BASELINE terrain in domain-warp mode
(mesh_gen_mode 4), and the same counts of TW_PQ_HMAP points on the 7168^2 image of that terrain (tw_proc_gen_heightmap_launch(set_image=1), not eroded).
xy and out are host arrays, pageable or page-locked. For each workload and memory kind, medians over --reps after --warmup:
  sync_ms        host time of tw_eval_points with the same arguments (the call the job replaces; TW_PQ_HMAP has no synchronous counterpart)
  sync_ms_frame  the same call made on the context whose frame job (below) is in flight, which completes that frame first
  blocked_ms     host time blocked in tw_points_launch
  ready_ms       time from the launch to the poll that reports the job complete (polled with wait = 0 in a loop)
  *_frame        the same two with a frame job in flight on another shared context, launched right before: 16 new 130^2 tiles with 1000 droplets each
Outputs are checked bit for bit against tw_eval_points (procedural) and against the job without a frame beside it. Prints one JSON line with the GPU's name
and power limit (--out also writes it there)."""
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
ap.add_argument("--size", type=int, default=7168)
ap.add_argument("--counts", type=int, nargs="+", default=[100000, 1000000])
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HM_CFG = dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0)   # the BASELINE terrain (scene_config/config.txt:76)
S, ZV = 128, 130
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy = float(cfg.dx_val), float(cfg.dy_val)
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
root = tw.Context(0)
frame_ctx, pts_ctx = root.shared(), root.shared()
n = a.size
job = root.proc_gen_heightmap_launch(n, n, dx, dy, hp, 0, ep, set_image=True)
root.create_tiles_poll(True)
hs = tw.HmapSampler(n, n, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), job.info.mesh_file_scale, job.info.mesh_file_tz,
                    hp.mesh_scale_z_inv)
pq_z = tw.PointQuery(tw.PQ_EXACT_ZVAL, 1.0, S, S, float(cfg.scene_size[0]), float(cfg.scene_size[1]), 0, 0, 0)
pq_h = tw.PointQuery(tw.PQ_HMAP, 1.0, 0, 0, 0.0, 0.0, 0, 0, 0)
origins = np.array([(x * S, y * S) for y in range(-2, 2) for x in range(-2, 2)], np.int32)
frame_z = torch.empty((len(origins), ZV, ZV), dtype=torch.float32).pin_memory()


def frame():
    frame_ctx.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 1000, ep, ep.zmin, frame_z)


def buf(shape, pinned, fill=None):
    t = torch.empty(shape, dtype=torch.float32)
    if fill is not None:
        t.copy_(torch.from_numpy(fill))
    return t.pin_memory().numpy() if pinned else t.numpy().copy()


def measure(xy, out, pq, with_frame):
    """(blocked, ready) in ms of one job on pts_ctx, optionally with the frame launched on frame_ctx right before."""
    if with_frame:
        frame()
    t0 = time.perf_counter()
    j = pts_ctx.points_launch(xy, hp, pq, hs, out)
    t1 = time.perf_counter()
    while j.poll(False) is None:
        pass
    t2 = time.perf_counter()
    if with_frame:
        frame_ctx.create_tiles_poll(True)
    return 1e3 * (t1 - t0), 1e3 * (t2 - t0)


rng = np.random.default_rng(1)
res = {}
for kind, pq in (("exact_zval_dwarp", pq_z), ("hmap_7168", pq_h)):
    for count in a.counts:
        if kind == "hmap_7168":
            src = rng.uniform(-n / 2 - 500, n / 2 + 500, (count, 2)).astype(np.float32)
        else:
            src = rng.uniform(-float(cfg.scene_size[0]), float(cfg.scene_size[0]), (count, 2)).astype(np.float32)
        for pinned in (False, True):
            xy, out = buf((count, 2), pinned, src), buf((count,), pinned)
            sync_out = buf((count,), pinned)
            key = "%s_n%d_%s" % (kind, count, "pinned" if pinned else "pageable")
            r = {k: [] for k in ("sync_ms", "sync_ms_frame", "blocked_ms", "ready_ms", "blocked_ms_frame", "ready_ms_frame")}
            alone = None
            for rep in range(a.warmup + a.reps):
                if kind != "hmap_7168":
                    t0 = time.perf_counter()
                    pts_ctx.eval_points(xy, hp, pq, out=sync_out)
                    ts = 1e3 * (time.perf_counter() - t0)
                    frame()
                    t0 = time.perf_counter()
                    frame_ctx.eval_points(xy, hp, pq, out=sync_out)
                    tsf = 1e3 * (time.perf_counter() - t0)
                b, d = measure(xy, out, pq, False)
                if alone is None:
                    alone = out.copy()
                    if kind != "hmap_7168":
                        assert np.array_equal(alone.view(np.uint32), sync_out.view(np.uint32)), key
                bf, df = measure(xy, out, pq, True)
                assert np.array_equal(out.view(np.uint32), alone.view(np.uint32)), key
                if rep >= a.warmup:
                    if kind != "hmap_7168":
                        r["sync_ms"].append(ts), r["sync_ms_frame"].append(tsf)
                    r["blocked_ms"].append(b), r["ready_ms"].append(d), r["blocked_ms_frame"].append(bf), r["ready_ms_frame"].append(df)
            res[key] = {k: (round(float(np.median(v)), 3) if v else None) for k, v in r.items()}
            print(key, res[key], flush=True)
t0 = time.perf_counter()
frame()
frame_ctx.create_tiles_poll(True)
res["frame_alone_ready_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
res.update(gpu=gpu, power_limit_w=plim, size=n, counts=a.counts, reps=a.reps, frame_tiles=len(origins), frame_zvsize=ZV, frame_droplets=1000, outputs_identical=True)
root.close()
line = json.dumps(res)
print(line)
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")
