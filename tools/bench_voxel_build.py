"""The voxel path of create_procedural + voxel_model::build (fill, outside flags, remove_unconnected with interior holes, marching cubes) on the 512^3 sine grid
(BASELINE config 4), a 512^3 GLM simplex terrain and the one-voxel column that needs 20000 flood generations, four ways alternated in one session:
  sync_host    the synchronous calls on host arrays (what tw3d::voxel_build does: count, then emit)
  sync_device  the same calls on CUDA tensors
  job_device   tw_voxel_build_launch with device outputs
  job_pinned   tw_voxel_build_launch with page-locked host outputs
For each: host time blocked in the calls (for the job: in the launch) and launch-to-ready time (median over --reps after one warm-up), and whether all ways
give identical outputs (field, flags, triangles, counts). --remove-only times only the synchronous tw_voxel_remove_unconnected on device tensors of the same
inputs, which an older checkout has too: with --root DIR it times that checkout's package, so two versions can be alternated in one session. Prints one
JSON line per workload with the GPU's name and power limit; writes nothing."""
import argparse
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
ap.add_argument("--workloads", nargs="+", default=["sine512", "glm512", "column20000"])
ap.add_argument("--remove-only", action="store_true")
a = ap.parse_args()
sys.path.insert(0, os.path.abspath(a.root))
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
g = np.load(os.path.join(HERE, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
ctx = tw.Context(0)


def post(dims, geom=None, **kw):
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = dims
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = (geom.lo_pos[d], geom.vsz[d]) if geom is not None else ((-1.0, 0.5, 0.25)[d], (0.05, 0.07, 0.04)[d])
    p.isolevel, p.invert, p.make_closed_surface = kw.get("isolevel", 0.0), 0, 1
    p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = kw.get("rm", 3), 0, 1, 0
    return p


def workload(name):
    """(fill VoxelParams or None, input field or None, post params, description)"""
    cfg = lambda mode: scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)  # noqa: E731
    if name == "sine512":
        vp = scene.voxel_landscape_params(cfg(0), 512, 512, 512)
        vp.offset[0], vp.offset[1] = 0.5, -0.25
        return vp, None, post((512, 512, 512), vp), "512^3 sine fill (BASELINE config 4), isolevel 0, remove_unconnected 3"
    if name == "glm512":
        vp = scene.voxel_landscape_params(cfg(1), 512, 512, 512, z_gradient=-2.0)
        return vp, None, post((512, 512, 512), vp, isolevel=-1.0), "512^3 GLM simplex terrain (z_gradient -2), isolevel -1, remove_unconnected 3"
    if name == "column20000":
        return None, np.ones((3, 3, 40002), np.float32), post((3, 3, 40002), rm=1), "3x3x40002 column: a flood of 20000 generations"
    raise SystemExit("unknown workload " + name)


def sync_chain(vp, field, p, dev):
    """tw_voxel_fill (or the given field) -> outside -> remove_unconnected -> triangles (count, then emit), on host arrays or CUDA tensors."""
    shape = (p.ny, p.nx, p.nz)
    if vp is not None:
        v = torch.empty(shape, device="cuda") if dev else np.empty(shape, np.float32)
        ctx.voxel_fill(vp, out=v)
    else:
        v = torch.from_numpy(field).cuda() if dev else field.copy()
    o = torch.empty(shape, dtype=torch.uint8, device="cuda") if dev else None
    o = ctx.voxel_outside(v, p, out=o)
    ch = ctx.voxel_remove_unconnected(v, o, p)
    if dev:
        n = C_count(v, o, p)
        t = torch.empty((n, 3, 3), device="cuda")
        if n:
            ctx.voxel_triangles(v, o, p, TABLES, out=t)
    else:
        t = ctx.voxel_triangles(v, o, p, TABLES)
    return v, o, t, len(t), ch


def C_count(v, o, p):
    import ctypes as C
    e, t, x = (np.ascontiguousarray(TABLES[0], np.uint32), np.ascontiguousarray(TABLES[1], np.int32), np.ascontiguousarray(TABLES[2], np.uint32))
    n = C.c_uint64()
    ctx._check(tw.lib.tw_voxel_triangles(ctx._h, tw._ptr(v), tw._ptr(o), C.byref(p), tw._ptr(e), tw._ptr(t), tw._ptr(x), None, 0, C.byref(n)))
    return n.value


def job(vp, field, p, kind, cap):
    """Returns (outputs, seconds blocked in the launch, seconds from launch to ready)."""
    shape = (p.ny, p.nx, p.nz)
    if kind == "device":
        v = torch.from_numpy(field).cuda() if field is not None else torch.empty(shape, device="cuda")
        o, t = torch.empty(shape, dtype=torch.uint8, device="cuda"), torch.empty((cap, 3, 3), device="cuda")
    else:
        v = torch.from_numpy(field).pin_memory() if field is not None else torch.empty(shape).pin_memory()
        o, t = torch.empty(shape, dtype=torch.uint8).pin_memory(), torch.empty((cap, 3, 3)).pin_memory()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    j = ctx.voxel_build_launch(p, vals=v, outside=o, tris=t, fill=vp, tables=TABLES, capacity=cap)
    t1 = time.perf_counter()
    while not ctx.create_tiles_poll(wait=False):
        pass
    t2 = time.perf_counter()
    return (v, o, t, j.ntris, j.changed), t1 - t0, t2 - t0


def digest(out):
    v, o, t, n, ch = out
    v, o, t = (x.cpu().numpy() if hasattr(x, "cpu") else x for x in (v, o, t))
    return (int(np.frombuffer(v.tobytes(), np.uint32).sum(dtype=np.uint64)), int(o.sum(dtype=np.uint64)),
            int(np.frombuffer(t[:n].tobytes(), np.uint32).sum(dtype=np.uint64)), int(n), int(ch))


try:
    gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                   capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    gpu, plim = None, None

for name in a.workloads:
    vp, field, p, desc = workload(name)
    if a.remove_only:   # the synchronous remove_unconnected alone, on device tensors prepared outside the timed window
        shape = (p.ny, p.nx, p.nz)
        v0 = torch.empty(shape, device="cuda") if vp is not None else torch.from_numpy(field).cuda()
        if vp is not None:
            ctx.voxel_fill(vp, out=v0)
        o0 = torch.empty(shape, dtype=torch.uint8, device="cuda")
        ctx.voxel_outside(v0, p, out=o0)
        ms, out = [], None
        for r in range(a.reps + 1):
            v, o = v0.clone(), o0.clone()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ch = ctx.voxel_remove_unconnected(v, o, p)
            dt = time.perf_counter() - t0
            if r:
                ms.append(1e3 * dt)
            out = (v, o, torch.zeros((0, 3, 3)), 0, ch)
        print(json.dumps({"root": os.path.abspath(a.root), "workload": name, "desc": desc, "remove_unconnected_ms": float(np.median(ms)), "min_ms": min(ms),
                          "max_ms": max(ms), "reps": a.reps, "digest": digest(out), "gpu": gpu, "power_limit_w": plim}), flush=True)
        del v0, o0, v, o
        torch.cuda.empty_cache()
        continue
    res, digests = {}, {}
    for r in range(a.reps + 1):     # round 0 warms every shape up
        for way in ("sync_host", "sync_device", "job_device", "job_pinned"):
            if way.startswith("sync"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = sync_chain(vp, field, p, way == "sync_device")
                blocked = ready = time.perf_counter() - t0
            else:
                out, blocked, ready = job(vp, field, p, way[4:], max(1, digests.get("sync_host", (0, 0, 0, 1))[3]))
            digests[way] = digest(out)
            if r:
                res.setdefault(way, []).append((1e3 * blocked, 1e3 * ready))
            del out
    same = len(set(digests.values())) == 1
    summary = {w: {"blocked_ms": float(np.median([b for b, _ in v])), "ready_ms": float(np.median([q for _, q in v]))} for w, v in res.items()}
    print(json.dumps({"root": os.path.abspath(a.root), "workload": name, "desc": desc, "ways": summary, "reps": a.reps, "ntris": digests["sync_host"][3],
                      "changed": digests["sync_host"][4], "identical": same, "digests": digests if not same else None, "gpu": gpu, "power_limit_w": plim}), flush=True)
    torch.cuda.empty_cache()
