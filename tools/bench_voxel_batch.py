"""Many small voxel grids: n rock / asteroid models (64^3, atten_to_sphere mode 3, centre_seed, remove_unconnected 3, the welded mesh into page-locked
buffers) built three ways, alternated in one session:
  batch     one tw_voxel_build_batch_launch on one context, polled once
  one_ctx   n tw_voxel_build_launch_ex on one context, each polled before the next
  pool8     n tw_voxel_build_launch_ex spread over 8 shared contexts (a launch completes its context's previous job first), all polled at the end
For each (GLM simplex and sine fills, n = 16 / 64 / 256): the host time blocked in the library's launch calls, the launch-to-ready time (median and p99
over --reps after one warm-up), the kernel launches per build (tw_launch_count), and whether the three ways give identical meshes and counts. Prints one
JSON line per (fill, n) with the GPU's name and power limit; writes nothing."""
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
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
ap.add_argument("--modes", type=int, nargs="+", default=[1, 0], help="gen modes: 1 GLM simplex, 0 sine")
a = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
TABLES = tuple(np.ascontiguousarray(t, dt) for t, dt in zip((g["edge_table"], g["tri_table"], g["edge_to_vals"]), (np.uint32, np.int32, np.uint32)))
N = 64


def rock(mode, k):
    """Grid k of a workload: a 64^3 sphere-attenuated fill whose offset moves with k, so every rock differs."""
    cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)
    vp = scene.voxel_landscape_params(cfg, N, N, N)
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = 3, 0.9, 0.3
    vp.offset[0], vp.offset[1], vp.offset[2] = 0.37 * k, -0.21 * k, 0.13 * k
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = N, N, N
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    p.isolevel, p.remove_unconnected, p.centre_seed = 0.0, 3, 1
    return vp, p


def pinned(shape, dtype):
    return torch.zeros(shape, dtype=dtype).pin_memory()


def digest(meshes, counts):
    h = hashlib.sha256()
    for (v, i), c in zip(meshes, counts):
        h.update(v.numpy().tobytes()); h.update(i.numpy().tobytes()); h.update(np.asarray(c, np.uint64).tobytes())
    return h.hexdigest()[:16]


def pct(x, q):
    return float(np.percentile(np.asarray(x), q))


gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                capture_output=True, text=True, check=True).stdout.strip().split(",")]
parent = tw.Context(0)
pool = [parent.shared() for _ in range(8)]
for mode in a.modes:
    for n in a.sizes:
        rocks = [rock(mode, k) for k in range(n)]
        caps = []
        for vp, p in rocks:   # the counts, for exact page-locked buffers
            job = parent.voxel_build_launch(p, fill=vp, tables=TABLES, mesh=(None, None), soup=False)
            parent.create_tiles_poll(wait=True)
            caps.append((job.nverts, job.mesh_ntris))
        meshes = {w: [(pinned((nv, 3), torch.float32), pinned((nt, 3), torch.int32)) for nv, nt in caps] for w in ("batch", "one_ctx", "pool8")}

        def run(way):
            """(host ms blocked in launches, launch-to-ready ms, kernel launches, per-grid counts)"""
            ms, blocked = meshes[way], 0.0
            ctxs = [parent] if way != "pool8" else pool
            l0 = sum(tw.lib.tw_launch_count(c._h) for c in ctxs)
            t0 = time.perf_counter()
            if way == "batch":
                job = parent.voxel_build_batch_launch([{"vpp": p, "fill": vp, "mesh": m} for (vp, p), m in zip(rocks, ms)], TABLES)
                blocked = time.perf_counter() - t0
                parent.create_tiles_poll(wait=True)
                counts = list(zip(job.nverts, job.ntris, job.changed))
            else:
                jobs = []
                for k, ((vp, p), m) in enumerate(zip(rocks, ms)):
                    c = ctxs[k % len(ctxs)]
                    s = time.perf_counter()
                    jobs.append(c.voxel_build_launch(p, fill=vp, tables=TABLES, mesh=m, soup=False))
                    blocked += time.perf_counter() - s
                    if way == "one_ctx":
                        c.create_tiles_poll(wait=True)
                for c in ctxs:
                    c.create_tiles_poll(wait=True)
                counts = [(j.nverts, j.mesh_ntris, j.changed) for j in jobs]
            ready = time.perf_counter() - t0
            return blocked * 1e3, ready * 1e3, sum(tw.lib.tw_launch_count(c._h) for c in ctxs) - l0, counts

        res = {w: {"blocked": [], "ready": []} for w in meshes}
        dig = {}
        for rep in range(a.reps + 1):
            for w in meshes:
                b, r, launches, counts = run(w)
                if rep == 0:   # warm-up; its outputs are the ones compared
                    dig[w] = digest(meshes[w], counts)
                    res[w]["launches"] = launches
                    continue
                res[w]["blocked"].append(b); res[w]["ready"].append(r)
        out = {"workload": "%d x 64^3 %s rocks (atten 3, centre_seed, remove_unconnected 3, welded mesh to page-locked buffers)" % (n, ("sine", "GLM simplex")[mode]),
               "n": n, "reps": a.reps, "identical": len(set(dig.values())) == 1, "digest": dig["batch"], "gpu": gpu, "power_limit_w": plim}
        for w, r in res.items():
            out[w] = {"host_blocked_ms_median": round(pct(r["blocked"], 50), 3), "ready_ms_median": round(pct(r["ready"], 50), 3),
                      "ready_ms_p99": round(pct(r["ready"], 99), 3), "launches": r["launches"]}
        print(json.dumps(out), flush=True)
for c in pool:
    c.close()
parent.close()
