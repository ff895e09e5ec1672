"""The voxel build job with the unwelded triangle soup against the same job with the welded indexed mesh (tw_voxel_build_launch_ex, no soup), on the 512^3
sine grid (BASELINE config 4, remove_unconnected 3) and a 512^3 GLM simplex terrain, with device and with page-locked host outputs, the four ways alternated
in one session. For each: host time blocked in the launch, launch-to-ready time (median over --reps after one warm-up round) and output bytes. Also times
the sequential welding of tests/voxel_mesh_ref.c (a per-edge cache filled cube by cube, what a caller without this library does on the host) on the job's field and
flags, and checks that its mesh equals the device's. Prints one JSON line per workload with the GPU's name and power limit, and writes them all to --out."""
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
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--workloads", nargs="+", default=["sine512", "glm512"])
ap.add_argument("--out", default=os.path.join(HERE, "results", "h100", "voxel_mesh.json"))
a = ap.parse_args()
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "tests"))
import torch  # noqa: E402

from voxel_mesh_ref import voxel_mesh as welded  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(HERE, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
ctx = tw.Context(0)


def workload(name):
    """(fill VoxelParams, post params, description), as tools/bench_voxel_build.py builds them."""
    cfg = lambda mode: scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)  # noqa: E731
    if name == "sine512":
        vp = scene.voxel_landscape_params(cfg(0), 512, 512, 512)
        vp.offset[0], vp.offset[1] = 0.5, -0.25
        iso, desc = 0.0, "512^3 sine fill (BASELINE config 4), isolevel 0, remove_unconnected 3"
    elif name == "glm512":
        vp = scene.voxel_landscape_params(cfg(1), 512, 512, 512, z_gradient=-2.0)
        iso, desc = -1.0, "512^3 GLM simplex terrain (z_gradient -2), isolevel -1, remove_unconnected 3"
    else:
        raise SystemExit("unknown workload " + name)
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = vp.nx, vp.ny, vp.nz
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    p.isolevel, p.invert, p.make_closed_surface, p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = iso, 0, 1, 3, 0, 1, 0
    return vp, p, desc


def run(vp, p, way, counts):
    """One job; way = (output 'soup' or 'mesh', buffers 'device' or 'pinned'). Returns (outputs, s blocked in the launch, s launch-to-ready, bytes)."""
    out, kind = way
    ntris, nverts, mtris = counts
    alloc = (lambda *s, dt=torch.float32: torch.empty(s, dtype=dt, device="cuda")) if kind == "device" else \
        (lambda *s, dt=torch.float32: torch.empty(s, dtype=dt).pin_memory())
    if out == "soup":
        bufs = (alloc(ntris, 3, 3),)
        nbytes = ntris * 36
    else:
        bufs = (alloc(nverts, 3), alloc(mtris, 3, dt=torch.int32))
        nbytes = nverts * 12 + mtris * 12
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if out == "soup":
        j = ctx.voxel_build_launch(p, fill=vp, tables=TABLES, tris=bufs[0])
    else:
        j = ctx.voxel_build_launch(p, fill=vp, tables=TABLES, mesh=bufs, soup=False)
    t1 = time.perf_counter()
    while not ctx.create_tiles_poll(wait=False):
        pass
    t2 = time.perf_counter()
    assert (j.ntris if out == "soup" else (j.nverts, j.mesh_ntris)) == (ntris if out == "soup" else (nverts, mtris))
    return bufs, t1 - t0, t2 - t0, nbytes


def digest(bufs):
    return int(sum(int(np.frombuffer(b.cpu().numpy().tobytes(), np.uint32).sum(dtype=np.uint64)) for b in bufs))


try:
    gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                   capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    gpu, plim = None, None

rows = []
WAYS = [("soup", "device"), ("mesh", "device"), ("soup", "pinned"), ("mesh", "pinned")]
for name in a.workloads:
    vp, p, desc = workload(name)
    shape = (p.ny, p.nx, p.nz)
    v, o = torch.empty(shape, device="cuda"), torch.empty(shape, dtype=torch.uint8, device="cuda")
    j = ctx.voxel_build_launch(p, vals=v, outside=o, fill=vp, tables=TABLES, mesh=(None, None))     # the counts, the field and the flags
    assert ctx.create_tiles_poll(wait=True)
    counts = (j.ntris, j.nverts, j.mesh_ntris)
    vals, flags = v.cpu().numpy(), o.cpu().numpy()
    del v, o
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    hv, hi = welded(vals, flags, p, TABLES)
    host_s = time.perf_counter() - t0
    del vals, flags
    res, dig = {w: ([], []) for w in WAYS}, {}
    mesh_equal = None
    for r in range(a.reps + 1):     # round 0 warms every shape up
        for w in WAYS:
            bufs, blocked, ready, nbytes = run(vp, p, w, counts)
            d = digest(bufs)
            assert dig.setdefault(w, d) == d, "%s: outputs differ between rounds" % (w,)
            if w[0] == "mesh" and mesh_equal is None:
                gv, gi = bufs[0].cpu().numpy(), bufs[1].cpu().numpy().view(np.uint32)
                mesh_equal = bool(np.array_equal(gv.view(np.uint32), hv.view(np.uint32)) and np.array_equal(gi, hi))
            if r:
                res[w][0].append(1e3 * blocked)
                res[w][1].append(1e3 * ready)
            del bufs
            torch.cuda.empty_cache()
    row = {"workload": name, "desc": desc, "ntris_soup": counts[0], "nverts_mesh": counts[1], "ntris_mesh": counts[2],
           "host_welding_s": host_s, "device_mesh_equals_host": mesh_equal, "reps": a.reps, "gpu": gpu, "power_limit_w": plim}
    for (out, kind), (blk, rdy) in res.items():
        key = "%s_%s" % (out, kind)
        row[key] = {"launch_blocked_ms_median": float(np.median(blk)), "ready_ms_median": float(np.median(rdy)), "ready_ms_min": min(rdy),
                    "ready_ms_max": max(rdy), "output_bytes": counts[0] * 36 if out == "soup" else counts[1] * 12 + counts[2] * 12}
    print(json.dumps(row), flush=True)
    rows.append(row)
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(rows, f)
    f.write("\n")
