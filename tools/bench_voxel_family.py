"""Brush strokes of a resident voxel model on the thread's context (every stroke first completes the previous one) against strokes on the slots of a pool
of shared contexts (tw_voxel_model_edit_launch_on: a stroke waits for the previous one on the device only), beside a tile frame per display frame.
Workload: the 512^3 GLM simplex terrain of tools/bench_voxel_edit.py in 32 x 32-column blocks; one brush of radius 6 voxels every --settings frames
(alternately adding and digging at a surface point of a random column), and per 60 Hz frame 16 new 130^2 tiles (tw_create_tiles_launch, mode 4, 1000
droplets each) on a pool of --pool shared contexts; --frames frames per setting (remove_unconnected:stroke interval). A frame: launch the tiles, launch the
stroke, then poll without waiting until the frame's 16.7 ms are over.
Per stroke, readiness is tracked per job, not per context: device done = a CUDA event recorded on the stroke's stream right after its launch has
completed (seen by the frame's poll loop); results on the host = the job was completed, either by a poll that found it still the pending job of its
context, or by the return of a later launch on that context (which completes it first). Host time blocked per frame is the time spent inside launches.
Both ways run the same strokes on two models; the final fields and flags and every stroke's block table must be equal. Prints one JSON line per setting
with the GPU's name and power limit, and writes them all to --out."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=120)
ap.add_argument("--n", type=int, default=512)
ap.add_argument("--block", type=int, default=32)
ap.add_argument("--pool", type=int, default=8)
ap.add_argument("--settings", nargs="+", default=["0:1", "3:1", "3:3"], help="remove_unconnected:frames between strokes")
ap.add_argument("--out", default=os.path.join(HERE, "results", "h100", "voxel_family.json"))
a = ap.parse_args()
sys.path.insert(0, HERE)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(HERE, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
R, FRAME, NT, ZV, ITERS = 6, 1.0 / 60.0, 16, 130, 1000
parent = tw.Context(0)
slots = [parent.shared() for _ in range(a.pool)]
tcfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                         mesh_size=(ZV - 2, ZV - 2, 1))
hp, ep = tcfg.height_params(), tcfg.erosion_params()
dx, dy = float(tcfg.dx_val), float(tcfg.dy_val)


def params(rm):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)
    vp = scene.voxel_landscape_params(cfg, a.n, a.n, a.n, z_gradient=-2.0)
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = vp.nx, vp.ny, vp.nz
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    p.isolevel, p.invert, p.make_closed_surface, p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = -1.0, 0, 1, rm, 0, 1, 0
    return vp, p


def brush(rng, raw, flags, frame):
    """A ball of radius R around the first outside voxel of a random column: +1 (inside) on even frames, -2 (outside) on odd ones."""
    n = raw.shape[0]
    x, y = (int(v) for v in rng.integers(R, n - R, 2))
    col = flags[y, x]
    z = min(max(int(np.argmax(col == 1)) if (col == 1).any() else n // 2, R), n - R - 1)
    box = raw[y - R:y + R + 1, x - R:x + R + 1, z - R:z + R + 1].copy()
    yy, xx, zz = np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="ij")
    box[xx ** 2 + yy ** 2 + zz ** 2 <= R * R] = 1.0 if frame % 2 == 0 else -2.0
    return (x - R, y - R, z - R, 2 * R + 1, 2 * R + 1, 2 * R + 1), box


class Pool:
    """tw3d::tile_job_pool's slot choice: a slot with nothing in flight, else the one launched on longest ago (whose launch completes its job).
    freed(c) is called for every slot whose poll completed its job (or found none)."""

    def __init__(self, ctxs):
        self.ctxs, self.launched, self.clock = ctxs, [0] * len(ctxs), 0

    def next(self, freed):
        pick = None
        for i, c in enumerate(self.ctxs):
            if c.create_tiles_poll(wait=False):
                freed(c, time.perf_counter())
                pick = i
                break
        if pick is None:
            pick = int(np.argmin(self.launched))
        self.clock += 1
        self.launched[pick] = self.clock
        return self.ctxs[pick]


def tiles_outputs():
    return torch.empty((NT, ZV, ZV), device="cuda"), np.empty((NT, 2), np.float32)


def run(way, m, strokes, every):
    pool = Pool(slots)
    outs = [tiles_outputs() for _ in range(a.pool)]
    mv = torch.empty((4 << 20, 3), device="cuda")
    mi = torch.empty((8 << 20, 3), dtype=torch.int32, device="cuda")
    blocked, dev_ready, host_ready, tables = [], [], [], []
    pending = {}       # id(context) -> the stroke whose job is that context's pending job
    launch = {}        # stroke -> (job, launch time, its event, whether the device is done)

    def completed(c, t):                        # c's pending job was completed at t (a poll, or a later launch on c, returned)
        k = pending.pop(id(c), None)
        if k is not None:
            j, t0, _, _ = launch[k]
            host_ready.append(1e3 * (t - t0))
            tables.append((k, j.blocks.tobytes(), j.nverts, j.ntris, j.changed))

    def launched(c, t):
        completed(c, t)

    t_next = time.perf_counter()
    nstroke = 0
    for f in range(len(strokes) * every):
        t_next += FRAME
        t0 = time.perf_counter()
        c = pool.next(completed)
        z, mm = outs[slots.index(c)]
        org = [((f * 4 + t % 4) * (ZV - 2), (t // 4 + 20) * (ZV - 2)) for t in range(NT)]
        c.create_tiles_launch(org, tcfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, mm=mm)
        launched(c, time.perf_counter())
        if f % every == 0:
            box, vals = strokes[nstroke]
            sc = parent if way == "thread" else pool.next(completed)
            ts = time.perf_counter()
            job = m.edit_launch([box], vals, verts=mv, indices=mi, ctx=sc)
            tl = time.perf_counter()
            launched(sc, tl)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.ExternalStream(sc.stream))
            launch[nstroke] = [job, ts, ev, False]
            pending[id(sc)] = nstroke
            nstroke += 1
        blocked.append(1e3 * (time.perf_counter() - t0))
        ctx_of = {id(x): x for x in [parent] + slots}
        while True:                              # the rest of the frame: polls and event queries that never wait
            now = time.perf_counter()
            for k, rec in launch.items():
                if not rec[3] and rec[2].query():
                    rec[3] = True
                    dev_ready.append(1e3 * (now - rec[1]))
            for cid in list(pending):
                if ctx_of[cid].create_tiles_poll(wait=False):
                    completed(ctx_of[cid], time.perf_counter())
            if time.perf_counter() >= t_next:
                break
    for rec in launch.values():
        if not rec[3]:
            rec[2].synchronize()
            dev_ready.append(1e3 * (time.perf_counter() - rec[1]))
    for c in [parent] + slots:
        assert c.create_tiles_poll(wait=True)
        completed(c, time.perf_counter())
    assert len(tables) == len(strokes) and len(dev_ready) == len(strokes)
    return blocked, dev_ready, host_ready, sorted(tables, key=lambda t: t[0])


def stats(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "p99": float(np.percentile(v, 99)), "max": float(v.max())}


try:
    gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                   capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    gpu, plim = None, None

rows = []
for setting in a.settings:
    rm, every = (int(v) for v in setting.split(":"))
    vp, p = params(rm)
    res, finals = {}, {}
    for way in ("thread", "pool", "thread_again"):           # the thread's way twice, before and after the pool's, for the session's spread
        m = parent.voxel_model(p, TABLES, bx=a.block, by=a.block)
        m.build_launch(fill=vp)
        assert parent.create_tiles_poll(wait=True)
        raw, _, flags = m.read()
        rng = np.random.default_rng(rm + 1)
        strokes = [brush(rng, raw, flags, f) for f in range(a.frames // every + 1)]
        w = "pool" if way == "pool" else "thread"
        run(w, m, strokes[:1], 1)                                                  # warm-up stroke
        blocked, dev_ready, host_ready, tables = run(w, m, strokes[1:], every)
        finals[way] = (m.read(), tables)
        res[way] = {"host_blocked_ms_per_frame": stats(blocked), "stroke_device_done_ms": stats(dev_ready), "stroke_results_on_host_ms": stats(host_ready)}
        m.close()
        torch.cuda.empty_cache()
    (ft, tt), (fp, tp) = finals["thread"], finals["pool"]
    equal = all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(ft, fp)) and tt == tp
    row = {"workload": "glm%d_brush_r%d_beside_%d_tiles_%d2_per_frame" % (a.n, R, NT, ZV), "remove_unconnected": rm, "frames_per_stroke": every,
           "blocks": "%dx%d" % (a.block, a.block), "frames": a.frames, "pool": a.pool, "final_model_and_block_tables_equal": bool(equal), "gpu": gpu,
           "power_limit_w": plim, "strokes_on_thread_context": res["thread"], "strokes_on_pool_slots": res["pool"],
           "strokes_on_thread_context_repeat": res["thread_again"]}
    print(json.dumps(row), flush=True)
    rows.append(row)
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(rows, f)
    f.write("\n")
parent.close()
