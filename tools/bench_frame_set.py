"""A camera flying over BASELINE terrain (mode 4, 8 octaves, 1000 droplets per tile) whose live tiles are a tile set: 32 x 32 tiles of 130^2, lit by a sun
and a moon. On every frame of a 16.7 ms frame clock half a row of 16 new tiles appears on the sun's side (heights, erosion, z range, sub-block bounds,
normal map, min_normal_z, all into pinned host memory), the 16 oldest tiles are evicted (not on a run's first frame, which grows the set's slabs), and the
tiles whose shadows change - the new tiles and their downstream closure - are relit for both lights into pinned memory. At the start of every frame the
outstanding jobs are polled without waiting. Three ways, alternated in one process:
  seq   - today's steps on one context: tw_tile_set_remove, tw_create_tiles_launch_ex, a waiting poll, tw_tile_set_put, tw_tile_set_stale and
          tw_tile_set_shadows_launch (its poll comes on a later frame, or the next frame's first call completes it);
  set   - tw_tile_set_create_tiles_launch on the set's context (one frame in flight at a time);
  pool  - tw_tile_set_create_tiles_launch on a pool of --pool shared contexts: a launch takes a context with no job in flight, else the one launched on
          longest ago (whose job it completes first).
Reports per way: the host time blocked per frame in launches and polls (median, p99, max), the launch-to-ready latency of each frame, the growth frames
separately, and whether the three ways produced identical outputs frame for frame (checked in one more, untimed run of each way). Prints one JSON line with the GPU's name and power limit; writes nothing."""
import argparse
import collections
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
ap.add_argument("--side", type=int, default=32, help="the set is side x side tiles")
ap.add_argument("--tiles", type=int, default=16, help="new tiles per frame")
ap.add_argument("--zvsize", type=int, default=130)
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--frames", type=int, default=60)
ap.add_argument("--pool", type=int, default=8)
ap.add_argument("--rounds", type=int, default=2, help="alternations of the three ways")
a = ap.parse_args()

FRAME = 1.0 / 60.0
side, nt, zv, iters, size = a.side, a.tiles, a.zvsize, a.droplets, a.zvsize - 2
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                        mesh_size=(size, size, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy, wpz_max = float(cfg.dx_val), float(cfg.dy_val), float(ep.water_plane_z)
parent = tw.Context(0)


def light(lp):
    sp = tw.ShadowParams()
    sp.x_scene_size, sp.y_scene_size = float(cfg.scene_size[0]), float(cfg.scene_size[1])
    sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = 2 * size, float(ep.zmin), float(ep.zmax), 0
    sp.lpos[0], sp.lpos[1], sp.lpos[2] = lp
    return sp


SPS = [light((3.0, 2.0, 0.15)), light((-2.0, -3.0, 0.2))]      # the sun lights from +x / +y: the new tiles (larger y) are on its side
CAP = side * side + nt                                           # most tiles a relight can name


def origins(keys):
    return [((x - side // 2) * size, (y + 20) * size) for x, y in keys]


def frame_keys(f):
    """The new tiles of frame f: half a row beyond the window, alternating halves."""
    x0 = (f % 2) * (side // 2)
    return [(x0 + (t % (side // 2)), side + f // 2 + t // (side // 2)) for t in range(nt)]


class Slot:
    """A context and pinned outputs for one frame's job."""

    def __init__(self, c):
        self.c = c
        pin = lambda shape, dt: torch.empty(shape, dtype=dt).pin_memory()   # noqa: E731
        self.z, self.n = pin((nt, zv, zv), torch.float32), pin((nt, zv - 1, zv - 1, 4), torch.uint8)
        self.mm, self.mnz, self.b = np.empty((nt, 2), np.float32), np.empty(nt, np.float32), (tw.TileBounds * nt)()
        self.m = [pin((CAP, zv, zv), torch.uint8) for _ in SPS]
        self.ox, self.oy = [pin((CAP, zv), torch.float32) for _ in SPS], [pin((CAP, zv), torch.float32) for _ in SPS]
        self.req, self.rec = None, None

    def lights(self, n):
        return [tw.Light(sp, self.m[l][:n], self.ox[l][:n], self.oy[l][:n]) for l, sp in enumerate(SPS)]

    def outs(self):
        return dict(zvals=self.z, mm=self.mm, bounds=self.b, normals=self.n, min_normal_z=self.mnz, wpz_max=wpz_max, size=size)

    def digest(self):
        h = hashlib.blake2b()
        n = len(self.req)
        for x in [self.z.numpy(), self.n.numpy(), self.mm, self.mnz, np.asarray(self.req, np.int32), self.rec] + \
                 [t[:n].numpy() for t in self.m + self.ox + self.oy]:
            h.update(np.ascontiguousarray(x).tobytes())
        h.update(bytes(self.b))
        return h.hexdigest()


# the initial window: side x side tiles, generated once
init_keys = [(x, y) for y in range(side) for x in range(side)]
init_z = parent.create_zvals_batch(origins(init_keys), cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin)


def new_set():
    ts = parent.tile_set(zv, len(SPS))
    ts.put(init_keys, init_z)
    lights = [tw.Light(sp, np.empty((len(init_keys), zv, zv), np.uint8), None, None) for sp in SPS]
    ts.shadows_launch(np.array(init_keys, np.int32), lights)
    parent.create_tiles_poll(wait=True)
    return ts


def launch_seq(slot, ts, new, evict):
    if evict:
        ts.remove(evict)
    slot.c.create_tiles_launch(origins(new), cfg.mesh_size, dx, dy, zv, hp, iters, ep, ep.zmin, **slot.outs())
    slot.c.create_tiles_poll(wait=True)
    ts.put(new, slot.z)
    slot.req = [tuple(k) for k in ts.stale(SPS)]
    slot.rec = ts.shadows_launch(np.array(slot.req, np.int32), slot.lights(len(slot.req)))


def launch_frame(slot, ts, new, evict):
    slot.req = [tuple(k) for k in ts.stale_after(SPS, evict or None, new)]
    slot.rec = ts.create_tiles_launch(origins(new), cfg.mesh_size, dx, dy, hp, iters, ep, ep.zmin, new, remove_xy=evict or None, relight_xy=slot.req,
                                      lights=slot.lights(len(slot.req)), ctx=slot.c, **slot.outs())


def run(way, slots, frames, check=False):
    """Returns blocked ms per frame, launch-to-ready ms per frame, and with check the output digest per frame (hashing ~20 MB per frame takes host time that
    would hold the frame loop back, so the timed runs do not hash)."""
    ts = new_set()
    window = collections.deque(init_keys)
    busy, last = {}, {}             # slot index -> (frame, launch time); slot index -> when it was last launched on
    blocked, latency, digests = [], {}, {}

    def done(i, t_ready):
        f, t0 = busy.pop(i)
        latency[f] = 1e3 * (t_ready - t0)
        digests[f] = slots[i].digest() if check else None

    def poll_all(count):
        spent = 0.0
        for i in list(busy):
            t0 = time.perf_counter()
            ready = slots[i].c.create_tiles_poll(wait=False)
            t1 = time.perf_counter()
            spent += t1 - t0 if count else 0.0
            if ready:
                done(i, t1)
        return spent
    t_start = time.perf_counter()
    for f in range(frames):
        tick = t_start + f * FRAME
        while time.perf_counter() < tick:            # between frames: readiness only (not counted)
            poll_all(False)
            time.sleep(0.0002)
        spent = poll_all(True)
        new = frame_keys(f)
        evict = [window.popleft() for _ in range(nt)] if f else []
        window.extend(new)
        free = [i for i in range(len(slots)) if i not in busy]
        i = free[0] if free else min(busy, key=lambda j: last[j])
        t0 = time.perf_counter()
        if i in busy:                                  # what the launch would do first: complete the slot's job (its outputs are read before reuse)
            slots[i].c.create_tiles_poll(wait=True)
            done(i, time.perf_counter())
        t1 = time.perf_counter()
        (launch_seq if way == "seq" else launch_frame)(slots[i], ts, new, evict)
        t2 = time.perf_counter()
        busy[i], last[i] = (f, t1), t2
        spent += t2 - t0
        blocked.append(1e3 * spent)
    for i in list(busy):
        slots[i].c.create_tiles_poll(wait=True)
        done(i, time.perf_counter())
    ts.close()
    return blocked, [latency[f] for f in range(frames)], [digests[f] for f in range(frames)]


one = [Slot(parent)]
pool = [Slot(parent.shared()) for _ in range(a.pool)]
ways = (("seq", one), ("set", one), ("pool", pool))
for way, slots in ways:                              # warm-up: every context's scratch and staging, the kernels, the slab sizes
    run(way, slots, min(a.frames, len(slots) + 2))


def stats(v):
    v = np.asarray(v, np.float64)
    return {"median": round(float(np.median(v)), 3), "p99": round(float(np.percentile(v, 99)), 3), "max": round(float(v.max()), 3)}


acc = {way: ([], [], [], []) for way, _ in ways}     # steady blocked, steady latency, growth-frame blocked, growth-frame latency
ref, identical = None, True
for _ in range(a.rounds):
    for way, slots in ways:
        blocked, lat, _ = run(way, slots, a.frames)
        acc[way][0].extend(blocked[1:])
        acc[way][1].extend(lat[1:])
        acc[way][2].append(blocked[0])
        acc[way][3].append(lat[0])
for way, slots in ways:                              # the outputs, frame for frame, in an untimed run of each way
    dig = run(way, slots, a.frames, check=True)[2]
    ref = ref or dig
    identical = identical and dig == ref
res = {"workload": "a %d x %d tile set of %d^2 tiles, sun + moon; every frame of a 60 Hz clock %d new tiles on the sun's side (mode 4 8-octave + %d droplets per "
                   "tile, z range + bounds + normal map + min_normal_z into pinned memory), the %d oldest evicted, the new tiles' downstream closure relit for "
                   "both lights into pinned memory; %d frames per run, the first of each run grows the slabs" % (side, side, zv, nt, iters, nt, a.frames),
       "results": []}
names = {"seq": "remove + launch + waiting poll + put + relight on one context", "set": "tw_tile_set_create_tiles_launch on the set's context",
         "pool": "tw_tile_set_create_tiles_launch on a pool of %d shared contexts" % a.pool}
for way, _ in ways:
    res["results"].append({"way": names[way], "blocked_ms_per_frame": stats(acc[way][0]), "launch_to_ready_ms": stats(acc[way][1]),
                           "growth_frame_blocked_ms": [round(v, 3) for v in acc[way][2]], "growth_frame_launch_to_ready_ms": [round(v, 3) for v in acc[way][3]],
                           "frames": len(acc[way][0])})
res["identical_outputs"] = identical
try:
    name, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                    capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    name, plim = None, None
res["gpu"], res["power_limit_w"] = name, plim
for s in pool:
    s.c.close()
parent.close()
print(json.dumps(res))
sys.exit(0 if identical else 1)
