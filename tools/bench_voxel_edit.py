"""Brush edits of a resident voxel model (tw_voxel_model_edit_launch) against rebuilding the whole welded mesh (tw_voxel_build_launch_ex, mesh only, no fill)
on the same edited field, alternated frame by frame in one session. Workload: the 512^3 GLM simplex terrain of tools/bench_voxel_mesh.py in 32 x 32-column
blocks; every frame one brush of radius 6 voxels (alternately adding and digging, at a surface point of a random column) written by the bench into a 13^3
box; --frames frames, with remove_unconnected 0 and 3. Outputs go to page-locked memory for both ways. Per way: host time blocked in the launch and
launch-to-ready (median, p99), the bytes written to the page-locked outputs per frame, and the blocks re-meshed per edit; every frame the model's field and
flags are compared with the rebuild's. Prints one JSON line per setting with the GPU's name and power limit, and writes them all to --out."""
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
ap.add_argument("--frames", type=int, default=60)
ap.add_argument("--n", type=int, default=512)
ap.add_argument("--block", type=int, default=32)
ap.add_argument("--remove", type=int, nargs="+", default=[0, 3])
ap.add_argument("--out", default=os.path.join(HERE, "results", "h100", "voxel_edit.json"))
a = ap.parse_args()
sys.path.insert(0, HERE)
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
g = np.load(os.path.join(HERE, "tests", "golden", "voxel_post.npz"))
TABLES = (g["edge_table"], g["tri_table"], g["edge_to_vals"])
ctx = tw.Context(0)
R = 6


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
    z = int(np.argmax(col == 1)) if (col == 1).any() else n // 2
    z = min(max(z, R), n - R - 1)
    x0, y0, z0 = x - R, y - R, z - R
    box = raw[y0:y0 + 2 * R + 1, x0:x0 + 2 * R + 1, z0:z0 + 2 * R + 1].copy()
    yy, xx, zz = np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="ij")
    box[xx ** 2 + yy ** 2 + zz ** 2 <= R * R] = 1.0 if frame % 2 == 0 else -2.0
    return (x0, y0, z0, 2 * R + 1, 2 * R + 1, 2 * R + 1), box


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
    full = ctx.voxel_build_launch(p, fill=vp, tables=TABLES, mesh=(None, None), soup=False)
    assert ctx.create_tiles_poll(wait=True)
    fv, fi = torch.empty((int(full.nverts * 1.2) + 100000, 3)).pin_memory(), torch.empty((int(full.mesh_ntris * 1.2) + 100000, 3), dtype=torch.int32).pin_memory()
    raw, _, flags = m.read()
    d_raw = torch.from_numpy(raw).cuda()
    d_o = torch.empty(shape, dtype=torch.uint8, device="cuda")
    r_v, r_o = torch.empty(shape, device="cuda"), torch.empty(shape, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(rm + 1)
    res = {"edit": ([], [], [], []), "rebuild": ([], [], [], [])}
    equal = True
    for frame in range(a.frames + 1):          # frame 0 warms both ways up
        box, vals = brush(rng, raw, flags, frame)
        x0, y0, z0, w, h, d = box
        raw[y0:y0 + h, x0:x0 + w, z0:z0 + d] = vals
        d_raw[y0:y0 + h, x0:x0 + w, z0:z0 + d] = torch.from_numpy(vals).cuda()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        job = m.edit_launch([box], vals, verts=mv, indices=mi)
        t1 = time.perf_counter()
        t_ready = ready(t0)
        assert job.nverts <= cap_v and job.ntris <= cap_t
        if frame:
            res["edit"][0].append(1e3 * (t1 - t0))
            res["edit"][1].append(1e3 * t_ready)
            res["edit"][2].append(12 * (job.nverts + job.ntris))
            res["edit"][3].append(len(job.blocks))
        t0 = time.perf_counter()
        fj = ctx.voxel_build_launch(p, vals=d_raw, outside=d_o, tables=TABLES, mesh=(fv, fi), soup=False)
        t1 = time.perf_counter()
        t_ready = ready(t0)
        if frame:
            res["rebuild"][0].append(1e3 * (t1 - t0))
            res["rebuild"][1].append(1e3 * t_ready)
            res["rebuild"][2].append(12 * (fj.nverts + fj.mesh_ntris))
            res["rebuild"][3].append(-1)
        # the build job leaves d_raw holding the field after remove_unconnected: compare with the model's, then restore the raw field
        m.read(vals=r_v, outside=r_o)
        equal = equal and bool(torch.equal(r_v.view(torch.int32), d_raw.view(torch.int32)) and torch.equal(r_o, d_o))
        d_raw.copy_(torch.from_numpy(raw).cuda())
        flags = r_o.cpu().numpy() if frame % 8 == 0 else flags
    row = {"workload": "glm%d_brush_r%d" % (n, R), "remove_unconnected": rm, "blocks": "%dx%d" % (a.block, a.block), "frames": a.frames,
           "field_and_flags_equal_every_frame": equal, "gpu": gpu, "power_limit_w": plim}
    for k, (blk, rdy, nb, nbl) in res.items():
        row[k] = {"launch_blocked_ms_median": float(np.median(blk)), "launch_blocked_ms_p99": float(np.percentile(blk, 99)),
                  "ready_ms_median": float(np.median(rdy)), "ready_ms_p99": float(np.percentile(rdy, 99)),
                  "pinned_bytes_per_frame_median": int(np.median(nb))}
        if k == "edit":
            row[k]["blocks_per_edit_median"] = float(np.median(nbl))
            row[k]["blocks_per_edit_max"] = int(max(nbl))
    print(json.dumps(row), flush=True)
    rows.append(row)
    m.close()
    del mv, mi, fv, fi, d_raw, d_o, r_v, r_o
    torch.cuda.empty_cache()
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(rows, f)
    f.write("\n")
