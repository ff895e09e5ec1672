"""CPU: the windowed domain-warp kernel (csrc/tw_heightgen.cu dwarp_windows, csrc/tw_noise2.cuh DWARP_WIN_OCTAVES) indexes its tables by lattice
coordinates shifted into per-stage, per-octave windows instead of reducing them mod 289. This restates in numpy fp32 the host's windows (the box of
each fBm stage's inputs, the lattice indices at its two corners) and checks that
  * every cell inside a box has lattice indices inside the corner windows (brute force at random, edge and corner positions, several grids, bands
    and origins), and the shifted indices stay inside the repeating tables;
  * the repeating tables' entries equal the 580 / 291-entry tables' entries at the reduced index, bit for bit, and the three gradient addresses the
    windowed octave forms (denormal adds, as the kernel) are the parent's addresses of the same gradient entries."""
import numpy as np
import pytest

f32 = np.float32
SPAN = 600                                     # DWARP_WIN_SPAN at 7 windowed octaves
WLUT_N, WHASH_N = 578 + SPAN, 290 + SPAN
ENTRY = 128
CY = f32(0.366025403784439)
OFF = [(0.0, 0.0), (5.2, 1.3), (1.7, 9.2), (8.3, 2.8), (0.0, 0.0)]
RX, RY = f32(1.1808359622955322), f32(1.3357980251312256)   # mesh_seed 1, mode 4 (the headline's rx, ry)


def permute(x):
    v = (x * f32(34.0) + f32(1.0)) * x
    return v - np.floor(v * (f32(1.0) / f32(289.0))) * f32(289.0)


def bits(v):
    """The float whose bit pattern is the non-negative integer v"""
    return np.asarray(v, np.int64).astype(np.uint32).view(f32)


def octaves():
    out, freq, rx, ry = [], f32(1.0), RX, RY
    for _ in range(8):
        out.append((freq, rx, ry))
        freq, rx, ry = f32(freq * f32(1.92)), f32(rx * f32(1.5)), f32(ry * f32(1.5))
    return out


def lattice(x, y, o):
    f, rx, ry = o
    px, py = f32(f * x) + rx, f32(f * y) + ry
    s = f32(px * CY) + f32(py * CY)
    return np.floor(px + s), np.floor(py + s)


def coord(i, d, o, inv):
    return f32(f32(f32(f32(i) * d) + o) * inv) * f32(0.0007)


def boxes(x0, y0, nx, r0, r1, d=f32(0.0625), margin=f32(0.45)):
    """The boxes of dwarp_windows for the cells [0, nx) x [r0, r1) of a grid with origin (x0, y0) in cells (mesh_scale 1)"""
    inv = f32(1.0) / d
    xs = [coord(0, d, f32(d * f32(x0)), inv), coord(nx - 1, d, f32(d * f32(x0)), inv)]
    ys = [coord(r0, d, f32(d * f32(y0)), inv), coord(r1 - 1, d, f32(d * f32(y0)), inv)]
    out = []
    for s in range(5):
        m = margin if s >= 2 else f32(0.0)
        out.append((f32(float(f32(min(xs) - m)) + OFF[s][0]), f32(float(f32(min(ys) - m)) + OFF[s][1]),
                    f32(float(f32(max(xs) + m)) + OFF[s][0]), f32(float(f32(max(ys) + m)) + OFF[s][1])))
    return out


GRIDS = [(-4096, -4096, 8192, 0, 8192), (-4096, -4096, 8192, 512, 1024), (-37, 5000, 1001, 0, 777), (600000, -600000, 256, 0, 256), (3, 9, 1, 0, 1)]


@pytest.mark.parametrize("grid", GRIDS)
def test_corner_windows_hold_every_cell_in_the_box(grid):
    rng = np.random.default_rng(7)
    for s, (bx0, by0, bx1, by1) in enumerate(boxes(*grid)):
        t = rng.random((2, 20000))
        x = np.concatenate([f32(bx0) + (f32(bx1) - f32(bx0)) * t[0].astype(f32), [bx0, bx1, bx0, bx1], np.full(64, bx0), np.full(64, bx1)]).astype(f32)
        y = np.concatenate([f32(by0) + (f32(by1) - f32(by0)) * t[1].astype(f32), [by0, by1, by1, by0],
                            np.linspace(by0, by1, 64, dtype=f32), np.linspace(by0, by1, 64, dtype=f32)]).astype(f32)
        inside = (x >= bx0) & (x <= bx1) & (y >= by0) & (y <= by1)
        x, y = x[inside], y[inside]
        for k, o in enumerate(octaves()[:7]):
            lo, hi = lattice(f32(bx0), f32(by0), o), lattice(f32(bx1), f32(by1), o)
            ix, iy = lattice(x, y, o)
            assert ix.min() >= lo[0] and ix.max() <= hi[0] and iy.min() >= lo[1] and iy.max() <= hi[1], (grid, s, k)
            if max(hi[0] - lo[0], hi[1] - lo[1]) > SPAN:
                continue                                  # the host keeps the reducing kernel for this launch
            cx, cy = 289 * np.floor(lo[0] / 289), 289 * np.floor(lo[1] / 289)
            assert (ix - cx).max() + 288 + 1 < WLUT_N and (iy - cy).max() + 1 < WHASH_N   # gradient P + ix' + 1, hash entry iy' + 1


def test_headline_windows_fit_the_tables():
    worst = 0
    for s in boxes(-4096, -4096, 8192, 0, 8192):
        for o in octaves()[:7]:
            lo, hi = lattice(f32(s[0]), f32(s[1]), o), lattice(f32(s[2]), f32(s[3]), o)
            worst = max(worst, hi[0] - lo[0], hi[1] - lo[1])
    assert 500 < worst <= SPAN, worst


def lut_entry(k):
    """simplex_lut_entry: {a0, h, n, permute(k)} of the hashed index"""
    pk = permute(k)
    t = pk * f32(0.024390243902439)
    X = f32(2.0) * (t - np.floor(t)) - f32(1.0)
    h = np.abs(X) - f32(0.5)
    a0 = X - np.floor(X + f32(0.5))
    n = f32(1.79284291400159) - f32(0.85373472095314) * (a0 * a0 + h * h)
    return np.stack([a0, h, n, pk], axis=1)


def hash_entry(k):
    p0, p1 = permute(k).astype(np.int64), permute(k + f32(1.0)).astype(np.int64)
    return np.stack([bits(ENTRY * p0), bits(ENTRY * (p0 + 1)), bits(ENTRY * (p1 + 1)), bits(0 * p0)], axis=1)


def test_repeating_tables_match_the_reduced_tables():
    k = np.arange(WLUT_N)
    grad, grad580 = lut_entry((k % 289).astype(f32)), lut_entry(np.arange(580, dtype=f32))
    assert np.array_equal(grad[:580].view(np.uint32), grad580.view(np.uint32))            # the parent's entries, bit for bit
    assert np.array_equal(grad.view(np.uint32), grad580[k % 289].view(np.uint32))
    r = np.arange(WHASH_N)
    hsh, hsh291 = hash_entry((r % 289).astype(f32)), hash_entry(np.arange(291, dtype=f32))
    assert np.array_equal(hsh[:291].view(np.uint32), hsh291.view(np.uint32))
    assert np.array_equal(hsh.view(np.uint32), hsh291[r % 289].view(np.uint32))


@pytest.mark.parametrize("lo", [(-700, 3), (0, -289), (1000, 1733), (-32000, 31000)])
def test_windowed_addresses_reach_the_parents_gradients(lo):
    """For every (ix, iy) of a full-width window: the windowed octave's addresses (shifted bases, no reduction) read gradient entries equal to the ones
    the parent reads (mod_int289_lazy indices into the 580-entry table)."""
    grad, grad580 = lut_entry((np.arange(WLUT_N) % 289).astype(f32)), lut_entry(np.arange(580, dtype=f32))
    hsh = hash_entry((np.arange(WHASH_N) % 289).astype(f32))
    ix, iy = np.meshgrid(np.arange(lo[0], lo[0] + SPAN + 1, dtype=f32), np.arange(lo[1], lo[1] + SPAN + 1, 7, dtype=f32), indexing="ij")
    ix, iy = ix.ravel(), iy.ravel()
    cx, cy = 289 * (lo[0] // 289), 289 * (lo[1] // 289)
    shift_x = -np.float32(np.ldexp(np.float64(ENTRY * cx), -149))      # the host's denormal shifts -128*c_x, -16*c_y
    shift_y = -np.float32(np.ldexp(np.float64(16 * cy), -149))
    Lb, lane = (1 << 10) + 5 * 16, 5 * 16
    gb, hb = f32(bits(Lb) + shift_x), f32(bits(Lb - lane) + shift_y)    # one exact add each
    assert gb.view(np.uint32) == (np.uint32(Lb - ENTRY * cx) if Lb - ENTRY * cx >= 0 else np.uint32(0x80000000 | (ENTRY * cx - Lb)))
    bx = ix * bits(ENTRY) + gb
    j = (iy * bits(16) + hb).view(np.uint32).astype(np.int64) - (Lb - lane)   # byte offset of the hash entry
    assert j.min() >= 0 and j.max() // 16 + 1 < WHASH_N
    ixm = ix - np.floor(ix * (f32(1.0) / f32(289.0))) * f32(289.0)            # mod_int289_lazy
    iym = iy - np.floor(iy * (f32(1.0) / f32(289.0))) * f32(289.0)
    for i1y in (0, 1):
        i1x = 1 - i1y
        words = [hsh[j // 16, 0], hsh[j // 16 + 1, 0] if i1y else hsh[j // 16, 1], hsh[j // 16, 2]]
        for w, qy, dx in ((words[0], iym, 0), (words[1], iym + f32(i1y), i1x), (words[2], iym + f32(1.0), 1)):
            e = ((w + bx).view(np.uint32).astype(np.int64) - Lb)
            assert e.min() >= 0 and np.all(e % ENTRY == 0) and e.max() // ENTRY < WLUT_N
            want = (permute(qy) + ixm + f32(dx)).astype(np.int64)               # the parent's second-permute argument
            assert np.array_equal(grad[e // ENTRY].view(np.uint32), grad580[want].view(np.uint32))
