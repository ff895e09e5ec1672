"""tw_read_heightmap_launch on the 7168^2 BASELINE-sized image (random texels; the read does not look at them): the whole image into device memory laid out
like the image, into device memory one texel off the image's phase (the staged path: shift copy and second kernel), into page-locked and into pageable
host memory; and square rects of 64, 256 and 512 texels at an odd x, into the engine's pageable whole-image copy (pitch 2*7168) and into device memory. For each workload,
over --reps launches after --warmup: the host time the launch call blocks (median), launch-to-ready (the launch and a waiting poll, which for host memory
includes moving the rows; median), the bytes read over that time, and in the same run the median time of one plain copy of the same bytes between the same
kinds of memory (torch copy_, synchronised) and its bytes/s. Every read is checked byte for byte. Prints one JSON line with the GPU's name and power limit
(--out also writes it there)."""
import argparse
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

ap = argparse.ArgumentParser()
ap.add_argument("--size", type=int, default=7168)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--out")
a = ap.parse_args()

tw = importlib.import_module("3dworld_b200")
gpu, plim = [v.strip() for v in subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                               capture_output=True, text=True).stdout.strip().split(",")]
n = a.size
ctx = tw.Context(0)
img = torch.randint(0, 256, (n, n, 2), dtype=torch.uint8)
img_np = img.numpy()
ctx.set_heightmap(img_np)
img_dev = img.cuda()
torch.cuda.synchronize()


def median_ms(ts):
    return round(float(np.median(ts)) * 1e3, 4)


def time_read(rects, out, check):
    blocked, ready = [], []
    for i in range(a.warmup + a.reps):
        t0 = time.perf_counter()
        job = ctx.read_heightmap_launch(rects, out)
        t1 = time.perf_counter()
        job.poll(wait=True)
        t2 = time.perf_counter()
        if i >= a.warmup:
            blocked.append(t1 - t0)
            ready.append(t2 - t0)
    assert check(), "read differs"
    return blocked, ready


def time_copy(dst, src):
    ts = []
    for i in range(a.warmup + a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst.copy_(src, non_blocking=dst.is_cuda or dst.is_pinned())
        torch.cuda.synchronize()
        if i >= a.warmup:
            ts.append(time.perf_counter() - t0)
    return ts


def entry(nbytes, blocked, ready, copy):
    r, c = float(np.median(ready)), float(np.median(copy))
    return {"bytes": nbytes, "launch_blocked_ms": median_ms(blocked), "ready_ms": median_ms(ready), "read_GB_per_s": round(nbytes / r / 1e9, 2),
            "memcpy_ms": median_ms(copy), "memcpy_GB_per_s": round(nbytes / c / 1e9, 2)}


res = {"gpu": gpu, "power_limit_w": plim, "image": [n, n], "reps": a.reps, "whole": {}, "rects": {}}
whole = [(0, 0, n, n)]
nb = 2 * n * n
dev_out = torch.empty((n, n, 2), dtype=torch.uint8, device="cuda")
copy_dst = torch.empty_like(dev_out)
b, r = time_read(whole, dev_out, lambda: torch.equal(dev_out, img_dev))
res["whole"]["device"] = entry(nb, b, r, time_copy(copy_dst, img_dev))
raw = torch.empty(nb + 64, dtype=torch.uint8, device="cuda")
off_out = torch.as_strided(raw, (n, n, 2), (2 * n, 2, 1), 2)                                     # one texel past a 16-byte boundary
b, r = time_read(whole, off_out, lambda: torch.equal(off_out, img_dev))
res["whole"]["device_one_texel_off"] = entry(nb, b, r, time_copy(torch.as_strided(raw, (nb,), (1,), 2), img_dev.view(-1)))
del raw, off_out, copy_dst
pin_out = torch.empty((n, n, 2), dtype=torch.uint8).pin_memory()
b, r = time_read(whole, pin_out, lambda: torch.equal(pin_out, img))
res["whole"]["pinned"] = entry(nb, b, r, time_copy(torch.empty_like(pin_out).pin_memory(), img_dev))
page_out = np.empty((n, n, 2), np.uint8)
b, r = time_read(whole, page_out, lambda: np.array_equal(page_out, img_np))
res["whole"]["pageable"] = entry(nb, b, r, time_copy(torch.empty((n, n, 2), dtype=torch.uint8), img_dev))
for s in (64, 256, 512):
    rect = [(1001, 2002, s, s)]
    nbr = 2 * s * s
    src = img_dev[2002:2002 + s, 1001:1001 + s].contiguous()
    torch.cuda.synchronize()
    e = {}
    b, r = time_read(rect, page_out, lambda: np.array_equal(page_out[2002:2002 + s, 1001:1001 + s], img_np[2002:2002 + s, 1001:1001 + s]))
    e["pageable_image"] = entry(nbr, b, r, time_copy(torch.empty((s, s, 2), dtype=torch.uint8), src))
    b, r = time_read(rect, dev_out, lambda: torch.equal(dev_out[2002:2002 + s, 1001:1001 + s], src))
    e["device"] = entry(nbr, b, r, time_copy(torch.empty_like(src), src))
    res["rects"][str(s)] = e
ctx.close()
line = json.dumps(res)
print(line)
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")
