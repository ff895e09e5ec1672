"""No GPU: tw_hmap_tiles_touched (the live tiles an image edit changes) against a brute-force enumeration of every cell's texels written here, and against the
oracle's sampler (a tile whose samples change is always flagged); the new exports, the tw_hmap_rect layout and the unchanged ABI version."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clamp(x, y, W, H, mode):
    """clamp_no_scale (src/heightmap.cpp:315-341) on arrays of cells: (x, y, on the texture)."""
    x, y = x + W // 2, y + H // 2
    inside = (x >= 0) & (y >= 0) & (x < W) & (y < H)
    if mode == 0:
        return np.clip(x, 0, W - 1), np.clip(y, 0, H - 1), np.ones_like(inside)
    if mode == 1:
        return x, y, inside

    def mirror(v, n):
        mod, div = np.abs(v) % n, np.sign(v) * (np.abs(v) // n)     # C's % of abs() and truncating division
        return np.where(div & 1, n - mod - 1, mod)
    return np.where(inside, x, mirror(x, W)), np.where(inside, y, mirror(y, H)), np.ones_like(inside)


def _round_fp(v):
    return np.where(v > 0, (v + np.float32(0.5)).astype(np.float32).astype(np.int64), (v - np.float32(0.5)).astype(np.float32).astype(np.int64))


def read_mask(hs, x1, y1, zv):
    """Every texel the zv^2 cells of the tile at (x1, y1) read, cell by cell: bool [H, W]."""
    W, H, ms = hs.width, hs.height, np.float32(hs.mesh_scale)
    j, i = np.meshgrid(np.arange(zv), np.arange(zv), indexing="ij")
    x, y = (x1 + i).ravel(), (y1 + j).ravel()
    m = np.zeros((H, W), bool)
    if ms < 1:
        sx, sy = ms * x.astype(np.float32), ms * y.astype(np.float32)
        xlo, ylo = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        xhi, yhi = np.ceil(sx).astype(np.int64), np.ceil(sy).astype(np.int64)
        xlo, ylo, ok_lo = _clamp(xlo, ylo, W, H, hs.edge_mode)
        xhi, yhi, ok_hi = _clamp(xhi, yhi, W, H, hs.edge_mode)
        ok = ok_lo & ok_hi
        for a, b in ((xlo, ylo), (xhi, ylo), (xlo, yhi), (xhi, yhi)):
            m[b[ok], a[ok]] = True
    else:
        xs, ys = _round_fp(ms * (x.astype(np.float32) + np.float32(0))), _round_fp(ms * (y.astype(np.float32) + np.float32(0)))
        xs, ys, ok = _clamp(xs, ys, W, H, hs.edge_mode)
        m[ys[ok], xs[ok]] = True
    return m


def brute(hs, origins, zv, rects):
    out = np.zeros(len(origins), np.uint8)
    for t, (x1, y1) in enumerate(origins):
        m = read_mask(hs, x1, y1, zv)
        out[t] = any(m[y:y + h, x:x + w].any() for x, y, w, h in rects)
    return out


def _rects(rng, W, H, n):
    rs = [(0, 0, 1, 1), (W - 1, H - 1, 1, 1), (W - 3, 0, 3, 2), (0, H - 2, 2, 2), (0, H // 2, W, 1), (W // 2, 0, 1, H)]   # corners, a row, a column
    for _ in range(n):
        w, h = int(rng.integers(1, max(2, W // 4))), int(rng.integers(1, max(2, H // 4)))
        rs.append((int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h))
    return rs


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ms", [0.37, 0.5, 1.0, 1.5, 2.0, 3.3])
def test_tiles_touched_equals_brute_force(tw, mode, ms):
    rng = np.random.default_rng(int(ms * 100) + mode)
    for W, H, zv in ((37, 53, 9), (61, 29, 17)):
        hs = tw.HmapSampler(W, H, mode, ms, 1.0, 1.0, 0.0, 1.0)
        grid = [(tx * (zv - 1) - 5 * (zv - 1), ty * (zv - 1) - 4 * (zv - 1)) for ty in range(9) for tx in range(10)]
        far = [(-3 * W - 11, 2 * H + 7), (5 * W + 3, -4 * H - 1), (-7 * W, -9 * H), (40 * W + 1, 33 * H)]   # mirror repeats; clamp edges; cliff: nothing
        origins = np.array(grid + far, np.int32)
        for k in range(8):
            rects = _rects(rng, W, H, 2) if k else [(0, 0, W, H)]
            one = [rects[int(rng.integers(0, len(rects)))]]
            for rs in (rects, one):
                got = tw.hmap_tiles_touched(hs, origins, zv, rs)
                assert np.array_equal(got, brute(hs, origins, zv, rs)), (W, H, rs)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ms", [0.5, 1.0, 2.0])
def test_tiles_touched_sound_against_oracle(tw, oracle, mode, ms):
    rng = np.random.default_rng(31 + mode)
    W, H, zv = 47, 35, 11
    hs = tw.HmapSampler(W, H, mode, ms, 0.0012, 1.7, -0.3, 0.8)
    ohs = oracle.HmapSampler(W, H, mode, ms, 0.0012, 1.7, -0.3, 0.8)
    origins = np.array([(tx * 10 - 60, ty * 10 - 50) for ty in range(11) for tx in range(12)], np.int32)
    img = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
    before = oracle.hmap_sample_tiles(img, ohs, origins, zv)
    for _ in range(6):
        rects = _rects(rng, W, H, 1)[-2:]
        new = img.copy()
        for x, y, w, h in rects:
            new[y:y + h, x:x + w] = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        after = oracle.hmap_sample_tiles(new, ohs, origins, zv)
        changed = np.any(before.view(np.uint32) != after.view(np.uint32), axis=(1, 2))
        touched = tw.hmap_tiles_touched(hs, origins, zv, rects)
        assert not np.any(changed & (touched == 0)), rects
        assert np.any(touched)


def test_tiles_touched_refusals(tw):
    hs = tw.HmapSampler(16, 16, 0, 1.0, 1.0, 1.0, 0.0, 1.0)
    org, out, rect = np.zeros(2, np.int32), np.zeros(1, np.uint8), (tw.HmapRect * 1)(tw.HmapRect(0, 0, 1, 1))
    L = tw.lib
    assert L.tw_hmap_tiles_touched(None, tw._ptr(org), 1, 4, rect, 1, tw._ptr(out)) == tw.TW_ERR_ARG
    for mode in (-1, 3):
        assert L.tw_hmap_tiles_touched(C.byref(tw.HmapSampler(16, 16, mode, 1.0, 1.0, 1.0, 0.0, 1.0)), tw._ptr(org), 1, 4, rect, 1, tw._ptr(out)) == tw.TW_ERR_ARG
    assert L.tw_hmap_tiles_touched(C.byref(hs), None, 1, 4, rect, 1, tw._ptr(out)) == tw.TW_ERR_ARG
    assert L.tw_hmap_tiles_touched(C.byref(hs), tw._ptr(org), 1, 4, rect, 1, None) == tw.TW_ERR_ARG
    assert L.tw_hmap_tiles_touched(C.byref(hs), tw._ptr(org), 1, 4, None, 1, tw._ptr(out)) == tw.TW_ERR_ARG
    assert L.tw_hmap_tiles_touched(C.byref(hs), tw._ptr(org), 1, 1, rect, 1, tw._ptr(out)) == tw.TW_ERR_ARG
    assert L.tw_hmap_tiles_touched(C.byref(hs), None, 0, 4, None, 0, None) == tw.TW_OK
    out[0] = 7
    assert L.tw_hmap_tiles_touched(C.byref(hs), tw._ptr(org), 1, 4, None, 0, tw._ptr(out)) == tw.TW_OK and out[0] == 0


def test_exports_layout_and_abi(tw, tmp_path):
    assert tw.lib.tw_abi_version() == 1
    for name in ("tw_update_heightmap", "tw_hmap_tiles_touched"):
        assert name in tw.ABI_SYMBOLS and hasattr(tw.lib, name)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tw3d.h"\nint main(void) {printf("%zu %zu %zu %zu %zu", sizeof(tw_hmap_rect), '
                   'offsetof(tw_hmap_rect, x), offsetof(tw_hmap_rect, y), offsetof(tw_hmap_rect, w), offsetof(tw_hmap_rect, h)); return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    R = tw.HmapRect
    assert got == [C.sizeof(R), R.x.offset, R.y.offset, R.w.offset, R.h.offset]


def test_update_refuses_without_context(tw):
    img = np.zeros((4, 4, 2), np.uint8)
    rect = (tw.HmapRect * 1)(tw.HmapRect(0, 0, 1, 1))
    assert tw.lib.tw_update_heightmap(None, tw._ptr(img), 8, rect, 1) == tw.TW_ERR_ARG
