"""Many small resident voxel models: n rock / asteroid models (64^3 GLM simplex, atten_to_sphere mode 3, centre_seed, remove_unconnected 3, blocks of 16 x 16
cube columns, welded block meshes into page-locked buffers) built and then edited three ways, alternated in one session:
  batch     one tw_voxel_model_build_batch_launch / tw_voxel_model_edit_batch_launch on one context, polled once
  one_ctx   n tw_voxel_model_build_launch_on / tw_voxel_model_edit_launch_on on one context, each polled before the next
  pool8     the n single-model jobs spread over 8 shared contexts (a launch completes its context's previous job first), all polled at the end
Workloads: the build; a frame where every model takes one radius-4 sphere brush (with a change list); a frame where a quarter of the models take one.
For each (workload, n = 16 / 64 / 256): host time blocked in the launch calls, launch-to-ready time (median and p99 over --reps after one warm-up),
kernel launches (tw_launch_count), and whether the three ways give identical models (tw_voxel_model_read), block tables, meshes and change lists. Prints
one JSON line per (workload, n) with the GPU's name and power limit; with --out also writes them there as a JSON list."""
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
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
ap.add_argument("--out", default=None)
a = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(ROOT, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
N, BLOCK, R = 64, 16, 4
WAYS = ("batch", "one_ctx", "pool8")


def rock(k):
    """Model k: a 64^3 sphere-attenuated GLM fill whose offset moves with k, so every rock differs."""
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)
    vp = scene.voxel_landscape_params(cfg, N, N, N)
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = 3, 0.9, 0.3
    vp.offset[0], vp.offset[1], vp.offset[2] = 0.37 * k, -0.21 * k, 0.13 * k
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = N, N, N
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    p.isolevel, p.remove_unconnected, p.centre_seed = 0.0, 3, 1
    return vp, p


def brush(rng):
    """A radius-R sphere of +1 (inside) or -1 (outside) at a random centre, as one box of raw values (the box's other voxels keep a rock-like -1)."""
    c = [int(v) for v in rng.integers(R + 8, N - R - 8, 3)]
    yy, xx, zz = np.meshgrid(*[np.arange(-R, R + 1)] * 3, indexing="ij")
    vals = np.where(xx ** 2 + yy ** 2 + zz ** 2 <= R * R, 1.0 if rng.random() < 0.5 else -1.0, -1.0).astype(np.float32)
    return [(c[0] - R, c[1] - R, c[2] - R, 2 * R + 1, 2 * R + 1, 2 * R + 1)], vals.ravel()


def pinned(shape, dtype):
    return torch.zeros(shape, dtype=dtype).pin_memory()


def pct(x, q):
    return float(np.percentile(np.asarray(x), q))


gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                capture_output=True, text=True, check=True).stdout.strip().split(",")]
parent = tw.Context(0)
pool = [parent.shared() for _ in range(8)]
results = []
for n in a.sizes:
    rocks = [rock(k) for k in range(n)]
    models = {w: [parent.voxel_model(p, TABLES, bx=BLOCK, by=BLOCK) for _, p in rocks] for w in WAYS}
    caps = []
    for m, (vp, _) in zip(models["batch"], rocks):   # the build's counts: buffers of twice that for every job
        job = m.build_launch(fill=vp)
        parent.create_tiles_poll(wait=True)
        caps.append((2 * job.nverts + 64, 2 * job.ntris + 64))
    bufs = {w: [(pinned((nv, 3), torch.float32), pinned((nt, 3), torch.int32), pinned((N ** 3,), torch.int32)) for nv, nt in caps] for w in WAYS}

    def run(way, work, edits):
        """(host ms blocked in launches, launch-to-ready ms, kernel launches, jobs); edits[k] = (boxes, values) or None for a build"""
        ms, blocked = models[way], 0.0
        ctxs = [parent] if way != "pool8" else pool
        l0 = sum(c.launch_count for c in ctxs)
        t0 = time.perf_counter()
        if way == "batch":
            if work == "build":
                entries = [{"model": m, "fill": vp, "verts": b[0], "indices": b[1]} for m, (vp, _), b in zip(ms, rocks, bufs[way])]
                jobs = parent.voxel_model_build_batch_launch(entries)
            else:
                entries = [{"model": m, "boxes": e[0], "values": e[1], "verts": b[0], "indices": b[1], "changes": (b[2], None, None)}
                           for m, e, b in zip(ms, edits, bufs[way]) if e is not None]
                jobs = parent.voxel_model_edit_batch_launch(entries)
            blocked = time.perf_counter() - t0
            parent.create_tiles_poll(wait=True)
        else:
            jobs, k = [], 0
            for m, (vp, _), e, b in zip(ms, rocks, edits, bufs[way]):
                if work != "build" and e is None:
                    continue
                c = ctxs[k % len(ctxs)]
                k += 1
                s = time.perf_counter()
                if work == "build":
                    jobs.append(m.build_launch(fill=vp, verts=b[0], indices=b[1], ctx=c))
                else:
                    jobs.append(m.edit_launch(e[0], e[1], verts=b[0], indices=b[1], changes=(b[2], None, None), ctx=c))
                blocked += time.perf_counter() - s
                if way == "one_ctx":
                    c.create_tiles_poll(wait=True)
            for c in ctxs:
                c.create_tiles_poll(wait=True)
        ready = time.perf_counter() - t0
        return blocked * 1e3, ready * 1e3, sum(c.launch_count for c in ctxs) - l0, jobs

    def digest(way, jobs, edits):
        """the job's tables, counts, meshes and change lists, and every model's read"""
        h = hashlib.sha256()
        hit = [k for k, e in enumerate(edits) if e is not None]
        for k, j in zip(hit, jobs):
            v, i, ch = bufs[way][k]
            h.update(j.blocks.tobytes()); h.update(np.asarray([j.nverts, j.ntris, j.changed, j.nchanged], np.uint64).tobytes())
            h.update(v.numpy()[:min(j.nverts, len(v))].tobytes()); h.update(i.numpy()[:min(j.ntris, len(i))].tobytes())
            h.update(ch.numpy()[:min(j.nchanged, len(ch))].tobytes())
        for m in models[way]:
            for arr in m.read():
                h.update(arr.tobytes())
        return h.hexdigest()[:16]

    rng = np.random.default_rng(n)
    for work in ("build", "every model hit", "a quarter hit"):
        res = {w: {"blocked": [], "ready": []} for w in WAYS}
        dig = {}
        for rep in range(a.reps + 1):
            edits = [()] * n if work == "build" else [brush(rng) if (work == "every model hit" or k % 4 == 0) else None for k in range(n)]
            for w in WAYS:
                b, r, launches, jobs = run(w, work, edits)
                if rep == 0:   # warm-up; its outputs are the ones compared
                    dig[w] = digest(w, jobs, edits)
                    res[w]["launches"] = launches
                    continue
                res[w]["blocked"].append(b); res[w]["ready"].append(r)
        out = {"workload": "%s: %d x 64^3 GLM rocks (atten 3, centre_seed, remove_unconnected 3, %dx%d blocks, welded block meshes to page-locked buffers%s)"
                           % (work, n, BLOCK, BLOCK, "" if work == "build" else ", radius-%d sphere brushes with change lists" % R),
               "n": n, "reps": a.reps, "identical": len(set(dig.values())) == 1, "digest": dig["batch"], "gpu": gpu, "power_limit_w": plim}
        for w, r in res.items():
            out[w] = {"host_blocked_ms_median": round(pct(r["blocked"], 50), 3), "ready_ms_median": round(pct(r["ready"], 50), 3),
                      "ready_ms_p99": round(pct(r["ready"], 99), 3), "launches": r["launches"]}
        print(json.dumps(out), flush=True)
        results.append(out)
    for w in WAYS:
        for m in models[w]:
            m.close()
if a.out:
    with open(a.out, "w") as f:
        json.dump(results, f, indent=1)
for c in pool:
    c.close()
parent.close()
