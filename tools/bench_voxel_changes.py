"""The change list of a voxel model edit (tw_voxel_model_edit_launch_ex) against the two ways an engine has without it, alternated frame by frame in one
session: the edit alone (the engine's copy of the field goes stale), the edit with the list, and the edit followed by a whole-grid tw_voxel_model_read
of the field and flags. Workload: the 512^3 GLM simplex terrain of tools/bench_voxel_edit.py in 32 x 32-column blocks, brushes of radius 6 voxels
(alternately adding and digging at a surface point of a random column), remove_unconnected 0 and 3; mesh, list and read outputs in page-locked memory.
Each frame runs the three ways on three brushes, in an order that rotates every frame. Per way: host time blocked (the launch, and for the read way the
read) and launch-to-ready (median, p99), the bytes of field and flags brought to the host per edit, and for the list the changes per edit (median, max).
Every frame a CPU mirror of the field and flags, patched from the list after the list's edit, is compared with a whole-grid read. Prints one JSON line
per setting with the GPU's name and power limit, and writes them all to --out."""
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
ap.add_argument("--frames", type=int, default=30)
ap.add_argument("--n", type=int, default=512)
ap.add_argument("--block", type=int, default=32)
ap.add_argument("--capacity", type=int, default=1 << 22)
ap.add_argument("--remove", type=int, nargs="+", default=[0, 3])
ap.add_argument("--out", default=os.path.join(HERE, "results", "h100", "voxel_changes.json"))
a = ap.parse_args()
sys.path.insert(0, HERE)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(HERE, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
ctx = tw.Context(0)
R = 6
WAYS = ("edit", "edit_list", "edit_read")


def params(rm):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)
    vp = scene.voxel_landscape_params(cfg, a.n, a.n, a.n, z_gradient=-2.0)
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = vp.nx, vp.ny, vp.nz
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = vp.lo_pos[d], vp.vsz[d]
    p.isolevel, p.invert, p.make_closed_surface, p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = -1.0, 0, 1, rm, 0, 1, 0
    return vp, p


def brush(rng, raw, flags, k):
    """A ball of radius R around the first outside voxel of a random column: +1 (inside) for even k, -2 (outside) for odd k."""
    n = raw.shape[0]
    x, y = (int(v) for v in rng.integers(R, n - R, 2))
    col = flags[y, x]
    z = int(np.argmax(col == 1)) if (col == 1).any() else n // 2
    z = min(max(z, R), n - R - 1)
    x0, y0, z0 = x - R, y - R, z - R
    box = raw[y0:y0 + 2 * R + 1, x0:x0 + 2 * R + 1, z0:z0 + 2 * R + 1].copy()
    yy, xx, zz = np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="ij")
    box[xx ** 2 + yy ** 2 + zz ** 2 <= R * R] = 1.0 if k % 2 == 0 else -2.0
    return (x0, y0, z0, 2 * R + 1, 2 * R + 1, 2 * R + 1), box


def read_grid(m, rv, ro):
    """tw_voxel_model_read of the field and flags only (VoxelModel.read also copies the raw field)."""
    ctx._check(tw.lib.tw_voxel_model_read(m._h, None, tw._ptr(rv), tw._ptr(ro)))


def ready(t0):
    while not ctx.create_tiles_poll(wait=False):
        pass
    return time.perf_counter() - t0


try:
    gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                   capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    gpu, plim = None, None

rows = []
for rm in a.remove:
    vp, p = params(rm)
    n = a.n
    shape = (n, n, n)
    m = ctx.voxel_model(p, TABLES, bx=a.block, by=a.block)
    first = m.build_launch(fill=vp)
    assert ctx.create_tiles_poll(wait=True)
    cap_v, cap_t = int(first.nverts * 1.2) + 100000, int(first.ntris * 1.2) + 100000
    mv, mi = torch.empty((cap_v, 3)).pin_memory(), torch.empty((cap_t, 3), dtype=torch.int32).pin_memory()
    li = torch.empty(a.capacity, dtype=torch.int32).pin_memory()
    lv = torch.empty(a.capacity, dtype=torch.float32).pin_memory()
    lo = torch.empty(a.capacity, dtype=torch.uint8).pin_memory()
    rv, ro = torch.empty(shape).pin_memory(), torch.empty(shape, dtype=torch.uint8).pin_memory()
    raw, _, _ = m.read()
    read_grid(m, rv, ro)
    mirror_v, mirror_o = rv.numpy().ravel().copy(), ro.numpy().ravel().copy()     # the engine's copy of the field and flags
    flags = ro.numpy().copy()
    rng = np.random.default_rng(rm + 1)
    res = {w: {"blocked": [], "ready": [], "bytes": [], "changes": []} for w in WAYS}
    mirror_equal, overflows, k = True, 0, 0
    for frame in range(a.frames + 1):          # frame 0 warms every way up
        for w in WAYS[frame % 3:] + WAYS[:frame % 3]:
            box, vals = brush(rng, raw, flags, k)
            k += 1
            x0, y0, z0, bw, bh, bd = box
            raw[y0:y0 + bh, x0:x0 + bw, z0:z0 + bd] = vals
            t0 = time.perf_counter()
            job = m.edit_launch([box], vals, verts=mv, indices=mi, changes=(li, lv, lo) if w == "edit_list" else None)
            t1 = time.perf_counter()
            if w == "edit_read":
                read_grid(m, rv, ro)        # completes the edit, then copies the grid
                t2 = time.perf_counter()
                blocked, t_ready, nbytes = t2 - t0, t2 - t0, 5 * n ** 3
            else:
                t_ready = ready(t0)
                blocked, nbytes = t1 - t0, (9 * min(job.nchanged, a.capacity) if w == "edit_list" else 0)
            assert job.nverts <= cap_v and job.ntris <= cap_t
            if w == "edit_list":
                c = job.nchanged
                if c <= a.capacity:
                    idx = li.numpy()[:c].view(np.uint32)
                    mirror_v[idx], mirror_o[idx] = lv.numpy()[:c], lo.numpy()[:c]
                else:
                    overflows += 1
                read_grid(m, rv, ro)        # the check, untimed
                if c > a.capacity:
                    mirror_v[:], mirror_o[:] = rv.numpy().ravel(), ro.numpy().ravel()
                mirror_equal = mirror_equal and bool(np.array_equal(mirror_v.view(np.uint32), rv.numpy().ravel().view(np.uint32)) and
                                                     np.array_equal(mirror_o, ro.numpy().ravel()))
            else:
                if w == "edit":
                    read_grid(m, rv, ro)    # the mirror follows, untimed
                mirror_v[:], mirror_o[:] = rv.numpy().ravel(), ro.numpy().ravel()
            if frame:
                r = res[w]
                r["blocked"].append(1e3 * blocked)
                r["ready"].append(1e3 * t_ready)
                r["bytes"].append(nbytes)
                r["changes"].append(job.nchanged)
        if frame % 4 == 0:
            flags = ro.numpy().copy()
    row = {"workload": "glm%d_brush_r%d" % (n, R), "remove_unconnected": rm, "blocks": "%dx%d" % (a.block, a.block), "frames": a.frames,
           "list_capacity": a.capacity, "list_overflows": overflows, "mirror_patched_from_list_equals_read_every_frame": mirror_equal, "gpu": gpu,
           "power_limit_w": plim}
    for w, r in res.items():
        row[w] = {"host_blocked_ms_median": float(np.median(r["blocked"])), "host_blocked_ms_p99": float(np.percentile(r["blocked"], 99)),
                  "ready_ms_median": float(np.median(r["ready"])), "ready_ms_p99": float(np.percentile(r["ready"], 99)),
                  "field_bytes_to_host_per_edit_median": int(np.median(r["bytes"]))}
        if w == "edit_list":
            row[w]["changes_per_edit_median"] = float(np.median(r["changes"]))
            row[w]["changes_per_edit_max"] = int(max(r["changes"]))
    row["list_cost_ready_ms_median"] = row["edit_list"]["ready_ms_median"] - row["edit"]["ready_ms_median"]
    print(json.dumps(row), flush=True)
    rows.append(row)
    m.close()
    del mv, mi, li, lv, lo, rv, ro
    torch.cuda.empty_cache()
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(rows, f)
    f.write("\n")
