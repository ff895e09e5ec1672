"""tw_create_zvals_ao_batch on the workloads of tools/bench_frame_tiles.py (BASELINE terrain, mode 4 8-octave, 1000 droplets per tile, zvals, AO map and
z range into pinned host memory): median over --reps rounds after 3 warm-up rounds, new tiles every round. --root DIR times the package of another
checkout (for example the parent commit's, built there) so two versions can be compared in one session: run it once per checkout, alternating. Prints one
JSON line with the GPU's name and power limit, the step count and a checksum of the outputs (equal outputs give equal checksums); writes nothing."""
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
ap.add_argument("--tiles", type=int, default=16)
ap.add_argument("--zvsize", type=int, default=130)
ap.add_argument("--droplets", type=int, default=1000)
ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()
sys.path.insert(0, os.path.abspath(a.root))
import torch  # noqa: E402

tw = importlib.import_module("3dworld_b200")
scene = importlib.import_module("3dworld_b200.scene")
nt, zv, size = a.tiles, a.zvsize, a.zvsize - 2
ctx = tw.Context(0)
cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=dict(sine_mag=5.0, sine_freq=0.001, sine_bias=-4.0), zmax_est=2.3,
                        mesh_size=(size, size, 1))
hp, ep = cfg.height_params(), cfg.erosion_params()
dx, dy = float(cfg.dx_val), float(cfg.dy_val)
z = torch.empty((nt, zv, zv), dtype=torch.float32).pin_memory()
ao = torch.empty((nt, zv - 1, zv - 1), dtype=torch.uint8).pin_memory()
ms = []
for r in range(a.reps + 3):
    if nt <= 64:
        origins = [((r * 5 + t % 4) * size, (t // 4 + r) * size) for t in range(nt)]        # bench_frame_tiles.py's frames
    else:
        origins = [((r * 64 + t % 64) * size, (t // 64) * size) for t in range(nt)]
    t0 = time.perf_counter()
    ctx.create_zvals_ao_batch(origins, cfg.mesh_size, dx, dy, zv, hp, a.droplets, ep, ep.zmin, 0.5 * (dx + dy), out=z, ao=ao, want_minmax=True)
    if r >= 3:
        ms.append(1e3 * (time.perf_counter() - t0))
try:
    name, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                                    capture_output=True, text=True, timeout=30).stdout.split(",")[:2]]
except Exception:   # noqa: BLE001 - descriptive only
    name, plim = None, None
print(json.dumps({"root": os.path.abspath(a.root), "workload": "%d tiles of %d^2, mode 4 8-octave + %d droplets per tile, zvals + AO + z range, pinned host outputs" % (nt, zv, a.droplets),
                  "create_zvals_ao_batch_ms": float(np.median(ms)), "min_ms": min(ms), "max_ms": max(ms), "rounds": a.reps, "steps": ctx.last_erosion_steps,
                  "checksum": int(np.frombuffer(z.numpy().tobytes(), np.uint32).sum(dtype=np.uint64) + ao.numpy().sum(dtype=np.uint64)), "gpu": name, "power_limit_w": plim}))
