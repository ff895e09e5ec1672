"""A camera flying over BASELINE terrain (mode 4, 8 octaves, 1000 droplets per tile): on every k-th frame of a 16.7 ms frame clock it launches the next row of
16 tiles of 130^2 (heights, erosion, z range, sub-block bounds, normal map, min_normal_z, all into pinned host memory) and at the start of every frame polls
the outstanding jobs without waiting, as tile_draw_t::update does. Two ways of running the jobs, alternated in one process:
  one   - one context (tw_create_tiles_launch on it completes the previous job first);
  pool  - a pool of --pool shared contexts of one parent (tw_create_shared): a launch takes a context with no job in flight, else the one launched on
          longest ago (whose job it completes first).
Reports per way and k: the host time blocked per frame in launches and polls (median, p99, max), the launch-to-ready latency per batch (readiness is also
polled between frames, those polls are not counted as blocked time), the latency of each batch alone on an idle device and each batch's latency over
that (the cost of running beside other jobs), and whether both ways produced identical outputs batch for batch. Prints one JSON line with the GPU's name and power limit; writes nothing."""
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

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
ap = argparse.ArgumentParser()
ap.add_argument("--tiles", type=int, default=16)
ap.add_argument("--zvsize", type=int, default=130)
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--frames", type=int, default=120)
ap.add_argument("--pool", type=int, default=8)
ap.add_argument("--every", type=int, nargs="+", default=[1, 2], help="k: a batch every k-th frame")
ap.add_argument("--rounds", type=int, default=2, help="alternations of the two ways per k")
a = ap.parse_args()

FRAME = 1.0 / 60.0
nt, zv, iters, size = a.tiles, a.zvsize, a.droplets, a.zvsize - 2
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                        mesh_size=(size, size, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy, wpz_max = float(cfg.dx_val), float(cfg.dy_val), float(ep.water_plane_z)
parent = tw.Context(0)


class Buffers:
    def __init__(self):
        self.z = torch.empty((nt, zv, zv), dtype=torch.float32).pin_memory()
        self.n = torch.empty((nt, zv - 1, zv - 1, 4), dtype=torch.uint8).pin_memory()
        self.mm, self.mnz, self.b = np.empty((nt, 2), np.float32), np.empty(nt, np.float32), (tw.TileBounds * nt)()

    def digest(self):
        h = hashlib.blake2b()
        for x in (self.z.numpy(), self.n.numpy(), self.mm, self.mnz):
            h.update(np.ascontiguousarray(x).tobytes())
        h.update(bytes(self.b))
        return h.hexdigest()


def row(r):
    return [((t - nt // 2) * size, (r + 20) * size) for t in range(nt)]


def launch(c, buf, r):
    c.create_tiles_launch(row(r), cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, buf.z, mm=buf.mm, bounds=buf.b, normals=buf.n, min_normal_z=buf.mnz,
                          wpz_max=wpz_max, size=size)


def run(k, slots):
    """slots: [(context, buffers)]; one slot = one context. Returns blocked ms per frame, latency ms per batch, output digest per batch."""
    busy = {}                       # slot index -> (batch, launch time)
    last = {}                       # slot index -> when it was last launched on
    blocked, latency, digests = [], {}, {}
    nbatch = 0

    def done(i, t_ready):
        b, t0 = busy.pop(i)
        latency[b] = 1e3 * (t_ready - t0)
        digests[b] = slots[i][1].digest()

    def poll_all(count):
        spent = 0.0
        for i in list(busy):
            t0 = time.perf_counter()
            ready = slots[i][0].create_tiles_poll(wait=False)
            t1 = time.perf_counter()
            spent += t1 - t0 if count else 0.0
            if ready:
                done(i, t1)
        return spent
    t_start = time.perf_counter()
    for f in range(a.frames):
        tick = t_start + f * FRAME
        while time.perf_counter() < tick:            # between frames: readiness only (not counted)
            poll_all(False)
            time.sleep(0.0002)
        spent = poll_all(True)
        if f % k == 0:
            free = [i for i in range(len(slots)) if i not in busy]
            i = free[0] if free else min(busy, key=lambda j: last[j])
            t0 = time.perf_counter()
            if i in busy:                              # what the launch would do first: complete the slot's job (its outputs are read before reuse)
                slots[i][0].create_tiles_poll(wait=True)
                done(i, time.perf_counter())
            t1 = time.perf_counter()
            launch(slots[i][0], slots[i][1], nbatch)
            t2 = time.perf_counter()
            busy[i], last[i] = (nbatch, t1), t2
            nbatch += 1
            spent += t2 - t0
        blocked.append(1e3 * spent)
    for i in list(busy):
        slots[i][0].create_tiles_poll(wait=True)
        done(i, time.perf_counter())
    return blocked, [latency[b] for b in range(nbatch)], [digests[b] for b in range(nbatch)]


one = [(parent, Buffers())]
pool = [(parent.shared(), Buffers()) for _ in range(a.pool)]
# warm-up: every context's scratch and staging, and the kernels
for c, buf in one + pool:
    launch(c, buf, 0)
    c.create_tiles_poll(wait=True)
iso = []
for r in range(a.frames // min(a.every)):             # every batch of the runs alone on an idle device: what running beside other jobs costs a batch
    t0 = time.perf_counter()
    launch(parent, one[0][1], r)
    while not parent.create_tiles_poll(wait=False):
        pass
    iso.append(1e3 * (time.perf_counter() - t0))


def stats(v):
    v = np.asarray(v, np.float64)
    return {"median": round(float(np.median(v)), 3), "p99": round(float(np.percentile(v, 99)), 3), "max": round(float(v.max()), 3)}


res = {"workload": "every k-th frame of a 60 Hz clock, a row of %d tiles of %d^2, mode 4 8-octave + %d droplets per tile, z range + bounds + normal map "
                   "+ min_normal_z into pinned host memory; %d frames per run" % (nt, zv, iters, a.frames),
       "isolated_batch_latency_ms": stats(iso), "results": []}
identical = True
for k in a.every:
    acc = {"one": ([], [], []), "pool": ([], [], [])}
    ref = None
    for _ in range(a.rounds):
        for way, slots in (("one", one), ("pool", pool)):
            blocked, lat, dig = run(k, slots)
            acc[way][0].extend(blocked)
            acc[way][1].extend(lat)
            acc[way][2].extend(x / y for x, y in zip(lat, iso))
            ref = ref or dig
            identical = identical and dig == ref
    for way in ("one", "pool"):
        res["results"].append({"way": way if way == "one" else "pool of %d shared contexts" % a.pool, "k": k, "blocked_ms_per_frame": stats(acc[way][0]),
                               "launch_to_ready_ms": stats(acc[way][1]),
                               "latency_over_isolated": stats(acc[way][2]), "batches": len(acc[way][1])})
res["identical_outputs"] = identical
try:
    name, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                    capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    name, plim = None, None
res["gpu"], res["power_limit_w"] = name, plim
parent.close()
print(json.dumps(res))
sys.exit(0 if identical else 1)
