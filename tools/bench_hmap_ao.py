"""tw_hmap_tile_ao_launch on a 7168^2 image (the size of BASELINE's island map; smooth synthetic hills plus texel noise, mirror edges, mesh_scale 1).
Workloads: 16 tiles of 130^2 (a frame's new tiles; host zvals and host AO, as the engine holds them) and 4096 tiles of 258^2 (device zvals and AO). For
each, over --reps launches after --warmup: host time the launch call blocks and launch-to-ready (launch plus waiting poll), medians. Against that, alternated
in the same run, the CPU path the engine has today: the window sampled on the host (oracle.hmap_sample_tiles) and oracle.tile_ao, on one thread; for 4096
tiles it runs on the first --cpu-tiles tiles only and is reported per tile. Then the frame pair on a pool of two shared contexts: a heightmap tile-set frame
of the 16 tiles (no zvals output) and the AO of its tiles from the set on the other context, launched back to back, against the frame alone (launch to
ready, alternated). Every AO is checked byte for byte against the oracle. Prints one JSON line with the GPU's name and power limit (--out also writes it)."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import oracle  # noqa: E402
from cases import convert  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--size", type=int, default=7168)
ap.add_argument("--reps", type=int, default=15)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--cpu-tiles", type=int, default=16)
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
oracle.lib()
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
n, HALF_DXY = a.size, 0.03125
rng = np.random.default_rng(1)
y, x = np.mgrid[0:n, 0:n].astype(np.float32)
v = np.clip(128.0 + 90.0 * np.sin(0.011 * x) * np.cos(0.009 * y) + 30.0 * np.sin(0.07 * x + 0.05 * y) + rng.uniform(-4, 4, (n, n)), 0, 255.99)
img = np.empty((n, n, 2), np.uint8)
img[..., 1] = np.floor(v).astype(np.uint8)
img[..., 0] = ((v - np.floor(v)) * 256).astype(np.uint8)
del x, y, v
hs = tw.HmapSampler(n, n, 2, 1.0, 0.0012, 1.7, -0.3, 0.8)
ohs = convert(hs, oracle.HmapSampler)
ctx = tw.Context(0)
ctx.set_heightmap(img)


def median_ms(ts):
    return round(float(np.median(ts)) * 1e3, 4)


def grid(side, size):
    txy = np.array([(tx, ty) for ty in range(side) for tx in range(side)], np.int32)
    return txy, txy * size - side * size // 2


def cpu_ao(origins, z):
    czv = oracle.hmap_sample_tiles(img, ohs, origins - 36, z.shape[1] - 1 + 72)
    return oracle.tile_ao(z, czv, HALF_DXY)


def workload(side, size, on_device):
    zv = size + 2
    txy, origins = grid(side, size)
    nt = len(origins)
    z = ctx.heightmap_sample_tiles(img, hs, origins, zv)
    z += np.random.default_rng(side).uniform(-0.01, 0.01, z.shape).astype(np.float32)
    zin = torch.from_numpy(z).cuda() if on_device else z
    out = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8, device="cuda") if on_device else np.empty((nt, zv - 1, zv - 1), np.uint8)
    nc = min(nt, a.cpu_tiles)
    blocked, ready, cpu = [], [], []
    for i in range(a.warmup + a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        job = ctx.hmap_tile_ao_launch(hs, origins, zin, HALF_DXY, out=out)
        t1 = time.perf_counter()
        job.poll(wait=True)
        t2 = time.perf_counter()
        exp = cpu_ao(origins[:nc], z[:nc])
        t3 = time.perf_counter()
        if i >= a.warmup:
            blocked.append(t1 - t0)
            ready.append(t2 - t0)
            cpu.append(t3 - t2)
    got = out.cpu().numpy() if on_device else out
    assert np.array_equal(got[:nc], exp), "AO differs from the oracle"
    return {"tiles": nt, "zvsize": zv, "memory": "device" if on_device else "pageable host", "launch_blocked_ms": median_ms(blocked),
            "ready_ms": median_ms(ready), "cpu_tiles": nc, "cpu_1_thread_ms": median_ms(cpu), "cpu_1_thread_ms_per_tile": round(median_ms(cpu) / nc, 4),
            "identical_to_oracle": True}


res = {"gpu": gpu, "power_limit_w": plim, "image": [n, n], "reps": a.reps, "workloads": {}}
res["workloads"]["16x130"] = workload(4, 128, False)
res["workloads"]["4096x258"] = workload(64, 256, True)

# the frame pair on a pool of shared contexts
fa, fb = ctx.shared(), ctx.shared()
ts = ctx.tile_set(130, 1)
txy, origins = grid(4, 128)
ep = tw.ErosionParams()
alone, pair, blocked = [], [], []
ao = np.empty((16, 129, 129), np.uint8)
for i in range(a.warmup + a.reps):
    for with_ao in (False, True):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ts.create_tiles_launch(origins, (128, 128), 0.0625, 0.0625, None, 0, ep, -10.0, txy, hmap=hs, ctx=fa)
        if with_ao:
            t1 = time.perf_counter()
            job = ts.hmap_ao_launch(txy, origins, hs, HALF_DXY, out=ao, ctx=fb)
            t2 = time.perf_counter()
            job.poll(wait=True)
        fa.create_tiles_poll(wait=True)
        t3 = time.perf_counter()
        if i >= a.warmup:
            (pair if with_ao else alone).append(t3 - t0)
            if with_ao:
                blocked.append(t2 - t1)
z = ctx.heightmap_sample_tiles(img, hs, origins, 130)
assert np.array_equal(ao, cpu_ao(origins, z)), "frame pair AO differs from the oracle"
res["frame_pair"] = {"tiles": 16, "zvsize": 130, "contexts": 2, "erosion": 0, "frame_alone_ready_ms": median_ms(alone), "frame_and_ao_ready_ms": median_ms(pair),
                     "ao_launch_blocked_ms": median_ms(blocked), "identical_to_oracle": True}
ts.close()
fa.close()
fb.close()
ctx.close()
line = json.dumps(res)
print(line)
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")
