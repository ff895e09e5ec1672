"""GPU: every path of the windowed domain-warp kernel (noise_grid2_kernel<simplex, warp, shape 0, windowed>; dwarp_windows() in csrc/tw_heightgen.cu
computes its per-launch lattice windows), each case asserting which kernel ran (from the context's count of windowed launches) and matching its
reference bit for bit (NaN == NaN):
  * windows exactly as wide as the tables hold (SPAN) and one wider, along x and along y, at mesh_scale 0.5, 1, 1.3 and 4, on non-square cells and at
    a fractional origin: the first runs windowed, the second the reducing kernel;
  * such windows whose lowest index is 0 or 288 mod 289, positive and negative: the shifted indices then reach the first and the last table entries;
  * the largest |lattice index| at 32767 (windowed) and 32768 (reducing), on either side and along either axis;
  * grids whose whole-grid windows do not fit but whose 1024-row bands do: device output runs the reducing kernel, banded host output the windowed
    one band by band, and both are identical;
  * origins whose coordinates overflow to +-inf (reducing); a grid with more chunk groups than one wave of resident blocks (windowed, striding);
  * variant builds of csrc/tw_heightgen.cu: TW_DWARP_WARP_MARGIN 0 (every pair of fBm stages 2-4 leaves its box and takes the reducing loop inside
    the windowed kernel), 0.05 (pairs inside and outside their box in one warp) and TW_DWARP_WIN_OCTAVES=5 (170-wide tables, 512-thread blocks). Each
    is linked with the shipped build's other objects into a temporary copy of the package, and a child process runs this file's cases against it.
Grids are chosen with a numpy restatement of dwarp_windows (test_dwarp_windows.py's, for any cell size and mesh_scale), so the host's windows sit
exactly where a case claims. The reference is a batch of one tile (which always runs the reducing kernel) for square grids at integer origins, the
CPU oracle otherwise."""
import json
import os
import re
import shutil
import subprocess
import sys
from collections import namedtuple

import numpy as np
import pytest

from cases import convert, HM_CFG
from test_dwarp_windows import OFF, lattice, octaves

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32

# The build these cases run against: the shipped library, or (set by test_variant_build for its child process) a variant's lib, margin and octaves
BUILD = json.loads(os.environ.get("TW_DWARP_TEST_BUILD", "{}"))
MARGIN = f32(BUILD.get("margin", 0.45))                   # TW_DWARP_WARP_MARGIN
WIN_OCTAVES = BUILD.get("octaves", 7)                     # TW_DWARP_WIN_OCTAVES
SPAN = 600 if WIN_OCTAVES > 5 else 170                    # twn2::DWARP_WIN_SPAN
GUARD = 32768                                             # dwarp_windows: |lattice index| < 2^15
THIN = 9                                                  # cells across a width-limit grid (odd: pairs straddle its rows)

Setting = namedtuple("Setting", "hp dx dy xy")
SETTINGS = {"unit": (1.0, 4.0), "scale0.5": (0.5, 4.0), "scale1.3": (1.3, 4.0), "scale4": (4.0, 4.0), "nonsquare": (1.0, 5.76)}  # mesh_scale, scene_size y


@pytest.fixture(scope="module", autouse=True)
def variant_library(tw):
    """In a variant's child process, the package must be the variant's copy"""
    if BUILD:
        assert os.path.realpath(tw.LIB_PATH) == os.path.realpath(BUILD["lib"]), tw.LIB_PATH


@pytest.fixture(scope="module")
def settings(scene):
    out = {}
    for name, (ms, sy) in SETTINGS.items():
        cfg = scene.SceneConfig(scene_size=(4.0, sy, 4.0), mesh_scale=ms, mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
        hp = cfg.height_params()
        hp.start_eval_sin = 10                            # 8 octaves at every mesh_scale (the windowed kernel's)
        out[name] = Setting(hp, f32(cfg.dx_val), f32(cfg.dy_val), f32(f32(0.0007) * f32(ms)))   # xy: N.xy_scale
    return out


# ---- the host's windows, restated (as test_dwarp_windows.py does at mesh_scale 1 and square cells) ----
def boxes(st, x0, y0, nx, r0, r1):
    """[stage] -> (x_lo, y_lo, x_hi, y_hi): dwarp_windows' boxes for the cells [0, nx) x [r0, r1) of the grid at origin (x0, y0) with cells st.dx x st.dy"""
    def coord(i, d, x0, inv):                             # xv, yv as the kernel computes them: ((i*d + d*x0)*inv)*xy_scale
        return f32(f32(f32(f32(i) * d) + f32(d * f32(x0))) * inv) * st.xy
    xs = [coord(i, st.dx, x0, f32(st.hp.dx_val_inv)) for i in (0, nx - 1)]
    ys = [coord(i, st.dy, y0, f32(st.hp.dy_val_inv)) for i in (r0, r1 - 1)]
    out = []
    for s in range(5):
        m = MARGIN if s >= 2 else f32(0.0)
        out.append((f32(float(f32(min(xs) - m)) + OFF[s][0]), f32(float(f32(min(ys) - m)) + OFF[s][1]),
                    f32(float(f32(max(xs) + m)) + OFF[s][0]), f32(float(f32(max(ys) + m)) + OFF[s][1])))
    return out


def windows(st, x0, y0, nx, r0, r1):
    """lo, hi [stage, octave, axis]: dwarp_windows' lattice windows for the cells [0, nx) x [r0, r1) of the grid at origin (x0, y0)"""
    with np.errstate(over="ignore", invalid="ignore"):
        b = np.array(boxes(st, x0, y0, nx, r0, r1), f32)
        lo = np.array([lattice(b[:, 0], b[:, 1], o) for o in octaves()[:WIN_OCTAVES]])     # [octave, axis, stage]
        hi = np.array([lattice(b[:, 2], b[:, 3], o) for o in octaves()[:WIN_OCTAVES]])
    return lo.transpose(2, 0, 1), hi.transpose(2, 0, 1)


def fits(lo, hi):
    """dwarp_windows' verdict: true = the windowed kernel runs (NaN and inf fail)"""
    with np.errstate(invalid="ignore"):
        return bool(np.all(np.abs(lo) < GUARD) and np.all(np.abs(hi) < GUARD) and np.all(hi - lo <= SPAN))


def first(pred, a, b):
    """The least n in [a, b] with pred(n), for pred monotone (false, then true)"""
    assert pred(b)
    while a < b:
        m = (a + b) // 2
        a, b = (a, m) if pred(m) else (m + 1, b)
    return a


def limit_grid(st, axis, width, x0, y0):
    """(nx, ny): THIN cells across and the fewest cells along `axis` whose widest window along that axis is `width` (windows grow with the grid)"""
    def size(n):
        return (n, THIN) if axis == 0 else (THIN, n)

    def widest(n):
        nx, ny = size(n)
        lo, hi = windows(st, x0, y0, nx, 0, ny)
        return (hi - lo)[..., axis].max()
    n = first(lambda n: widest(n) >= width, 2, 1 << 17)
    assert widest(n) == width, (axis, width, x0, y0, n)
    return size(n)


def boundary_grid(st, axis, r, sign):
    """(x0, y0, nx, ny): a limit grid (limit_grid, width SPAN) one of whose SPAN-wide windows along `axis` starts at lo = r (mod 289), lo of `sign`.
    lo depends on the origin only (the box's low corner): move the origin along `axis` until the widest window's lo reaches the residue, then try the
    next few origins, whose widths differ by rounding, until a SPAN-wide window has it."""
    def org(t):
        return (t, 37) if axis == 0 else (37, t)

    def at(t):
        x0, y0 = org(t)
        nx, ny = limit_grid(st, axis, SPAN, x0, y0)
        lo, hi = windows(st, x0, y0, nx, 0, ny)
        return (x0, y0, nx, ny), lo[..., axis], (hi - lo)[..., axis]
    t0 = sign * 20000                                           # far enough out that every stage's octave-6 window has lo of that sign
    _, lo, w = at(t0)
    s, k = np.unravel_index(np.argmax(w), w.shape)
    target = lo[s, k] + (r - lo[s, k]) % 289                    # the next lo >= the current one with the residue
    t = first(lambda t: windows(st, *org(t), THIN, 0, THIN)[0][s, k, axis] >= target, t0, t0 + 20000)
    for t in range(t, t + 64):
        g, lo, w = at(t)
        hit = (w == SPAN) & (lo % 289 == r) & (np.sign(lo) == sign)
        if hit.any():
            return g
    pytest.fail("no origin near %d puts a %d-wide window at %d mod 289" % (t0, SPAN, r))


# ---- runs and references ----
@pytest.fixture(scope="module")
def wctx(tw, ctx, settings):
    """ctx with its noise tables staged: the first height call on a context launches one more kernel, which builds them"""
    ctx.heightgen_2d(tw.Grid2D(0.0, 0.0, 0.0625, 0.0625, 2, 1), settings["unit"].hp)
    return ctx


def launches(ctx, fn):
    """fn()'s result and the kernels it launched on ctx: (result, windowed domain-warp launches, reducing ones - the only other kernel of the call)"""
    n0, w0 = ctx.launch_count, ctx.dwarp_window_launches
    out = fn()
    n, w = ctx.launch_count - n0, ctx.dwarp_window_launches - w0
    return out, w, n - w


def device(tw, ctx, st, x0, y0, nx, ny):
    """The grid to device memory: (heights, windowed launches, reducing launches)"""
    import torch
    g = tw.Grid2D(float(x0), float(y0), float(st.dx), float(st.dy), nx, ny)
    z = torch.full((ny, nx), float("nan"), dtype=torch.float32, device="cuda")

    def run():
        ctx.heightgen_2d(g, st.hp, out=z)
        ctx.sync()
        return z.cpu().numpy()
    return launches(ctx, run)


def host(tw, ctx, st, x0, y0, nx, ny):
    """The grid to host memory (row bands from 32 MiB on): (heights, windowed launches, reducing launches)"""
    g = tw.Grid2D(float(x0), float(y0), float(st.dx), float(st.dy), nx, ny)
    z = np.full((ny, nx), np.nan, np.float32)
    return launches(ctx, lambda: ctx.heightgen_2d(g, st.hp, out=z))


def oracle_grid(oracle, st, x0, y0, nx, ny, dx=None, dy=None):
    g = oracle.Grid2D(float(x0), float(y0), float(st.dx if dx is None else dx), float(st.dy if dy is None else dy), nx, ny)
    return oracle.heightgen_2d(g, convert(st.hp, oracle.HeightParams), None, 1, 0)


def assert_oracle_rows(oracle, beq, st, z, x0, y0, rows):
    """Rows of a grid at an integer origin with power-of-two cells (so row r is the one-row grid at y0 + r) against the oracle"""
    assert float(x0).is_integer() and float(y0).is_integer() and float(st.dy) == 0.0625
    for r in sorted(rows):
        assert beq(z[r:r + 1], oracle_grid(oracle, st, x0, y0 + r, z.shape[1], 1)) == 0, (x0, y0, r)


def one_tile(ctx, st, x0, y0, n):
    """The n x n grid at integer origin (x0, y0) as a batch of one tile (mesh size 2: the tile's grid starts one cell before its origin)"""
    return ctx.heightgen_tiles([(x0 + 1, y0 + 1)], (2, 2), float(st.dx), float(st.dy), n, st.hp)[0]


def band_rows(nx, ny):
    """band_rows_for: rows per band of a host-bound grid"""
    return ny if nx * ny * 4 < (32 << 20) else max(64, ((ny + 15) // 16 + 63) & ~63)


# ---- cases ----
def test_headline(tw, wctx, beq, settings):
    st = settings["unit"]
    assert fits(*windows(st, -4096, -4096, 8192, 0, 8192))
    ref = one_tile(wctx, st, -4096, -4096, 8192)
    assert np.isfinite(ref).all()
    z, win, red = device(tw, wctx, st, -4096, -4096, 8192, 8192)
    assert (win, red) == (1, 0)
    assert beq(z, ref) == 0
    z, win, red = host(tw, wctx, st, -4096, -4096, 8192, 8192)
    assert (win, red) == (8192 // band_rows(8192, 8192), 0)       # one launch per band, each band with its own windows
    assert beq(z, ref) == 0


WIDTH_CASES = [(name, -4096, 1234) for name in SETTINGS] + [("unit", -4096.37, 1234.71)]   # the last: fractional origin


@pytest.mark.parametrize("over", [0, 1], ids=["span", "span+1"])
@pytest.mark.parametrize("axis", [0, 1], ids=["x", "y"])
@pytest.mark.parametrize("name,x0,y0", WIDTH_CASES, ids=[c[0] + ("_frac" if not float(c[1]).is_integer() else "") for c in WIDTH_CASES])
def test_width_limit(tw, wctx, oracle, beq, settings, name, x0, y0, axis, over):
    st = settings[name]
    nx, ny = limit_grid(st, axis, SPAN + over, x0, y0)
    lo, hi = windows(st, x0, y0, nx, 0, ny)
    assert (hi - lo)[..., 1 - axis].max() < SPAN                  # the other axis stays inside the tables
    assert fits(lo, hi) == (over == 0)
    z, win, red = device(tw, wctx, st, x0, y0, nx, ny)
    assert (win, red) == ((1, 0) if over == 0 else (0, 1))
    assert beq(z, oracle_grid(oracle, st, x0, y0, nx, ny)) == 0


@pytest.mark.parametrize("sign", [1, -1], ids=["pos", "neg"])
@pytest.mark.parametrize("r", [0, 288])
@pytest.mark.parametrize("axis", [0, 1], ids=["x", "y"])
def test_window_shift_on_289_boundary(tw, wctx, oracle, beq, settings, axis, r, sign):
    st = settings["unit"]
    x0, y0, nx, ny = boundary_grid(st, axis, r, sign)
    assert fits(*windows(st, x0, y0, nx, 0, ny))
    z, win, red = device(tw, wctx, st, x0, y0, nx, ny)
    assert (win, red) == (1, 0)
    assert beq(z, oracle_grid(oracle, st, x0, y0, nx, ny)) == 0


@pytest.mark.parametrize("bound", [GUARD - 1, GUARD])
@pytest.mark.parametrize("sign", [1, -1], ids=["pos", "neg"])
@pytest.mark.parametrize("axis", [0, 1], ids=["x", "y"])
def test_index_guard(tw, wctx, beq, settings, axis, sign, bound):
    """The largest |lattice index| of any window (hi on the positive side, lo on the negative one) at the guard and one below it"""
    st, n = settings["unit"], 96

    def extreme(t):
        lo, hi = windows(st, *((sign * t, 5) if axis == 0 else (5, sign * t)), n, 0, n)
        return (hi if sign > 0 else -lo).max()
    t = first(lambda t: extreme(t) >= bound, 0, 1 << 22)
    assert extreme(t) == bound
    x0, y0 = (sign * t, 5) if axis == 0 else (5, sign * t)
    assert fits(*windows(st, x0, y0, n, 0, n)) == (bound < GUARD)
    z, win, red = device(tw, wctx, st, x0, y0, n, n)
    assert (win, red) == ((1, 0) if bound < GUARD else (0, 1))
    assert beq(z, one_tile(wctx, st, x0, y0, n)) == 0


@pytest.mark.parametrize("nx,ny", [(1024, 16384), (1023, 16385)])
def test_band_windows(tw, wctx, oracle, beq, settings, nx, ny):
    """Whole-grid windows too tall for the tables, each band's windows inside them; 1023 x 16385: 1088-row bands, a 65-row last band whose last pair
    straddles the grid's end"""
    st, x0, y0 = settings["unit"], -512, -8192
    assert not fits(*windows(st, x0, y0, nx, 0, ny))
    br = band_rows(nx, ny)
    bands = [(r0, min(ny, r0 + br)) for r0 in range(0, ny, br)]
    assert len(bands) > 1 and all(fits(*windows(st, x0, y0, nx, r0, r1)) for r0, r1 in bands)
    zd, win, red = device(tw, wctx, st, x0, y0, nx, ny)
    assert (win, red) == (0, 1)
    zh, win, red = host(tw, wctx, st, x0, y0, nx, ny)
    assert (win, red) == (len(bands), 0)
    assert beq(zh, zd) == 0
    assert_oracle_rows(oracle, beq, st, zh, x0, y0, {ny // 2} | {r for b in bands for r in (b[0], b[1] - 1)})


@pytest.mark.parametrize("x0,y0,dx,dy", [(1.0e38, 3.0, 4.0, 4.0),             # x overflows to +inf
                                         (-5.0, -1.0e38, 4.0, 4.0)])          # y overflows to -inf
def test_non_finite_coordinates(tw, wctx, oracle, beq, settings, x0, y0, dx, dy):
    """Cells 4 wide on a scene whose coordinates count 1/16 ones: the origin's product overflows, the windows are not finite"""
    st = settings["unit"]._replace(dx=f32(dx), dy=f32(dy))
    with np.errstate(over="ignore"):
        assert not np.isfinite(f32(dx) * f32(x0)) or not np.isfinite(f32(dy) * f32(y0))
    assert not fits(*windows(st, x0, y0, 65, 0, 33))
    z, win, red = device(tw, wctx, st, x0, y0, 65, 33)
    assert (win, red) == (0, 1)
    assert beq(z, oracle_grid(oracle, st, x0, y0, 65, 33)) == 0


def test_persistent_striding(tw, wctx, oracle, beq, settings):
    """More chunk groups than one wave of resident blocks: each block strides over many of them with its staged tables"""
    import torch
    st, x0, y0, nx, ny = settings["unit"], -3000, -1500, 6000, 3001
    assert fits(*windows(st, x0, y0, nx, 0, ny))
    assert (nx * ny + 2047) // 2048 > 4 * torch.cuda.get_device_properties(0).multi_processor_count
    z, win, red = device(tw, wctx, st, x0, y0, nx, ny)
    assert (win, red) == (1, 0)
    assert_oracle_rows(oracle, beq, st, z, x0, y0, {0, 1, 2, ny // 2, ny - 2, ny - 1})


# ---- variant builds ----
VARIANTS = {"margin0": (dict(margin=0.0), "-DTW_DWARP_WARP_MARGIN=0.0f", "headline or width_limit or shift_on_289 or band_windows"),
            "margin0.05": (dict(margin=0.05), "-DTW_DWARP_WARP_MARGIN=0.05f", "headline or width_limit"),
            "octaves5": (dict(octaves=5), "-DTW_DWARP_WIN_OCTAVES=5", "headline or width_limit or band_windows")}


@pytest.fixture(scope="module")
def variant_builds(tw, tmp_path_factory):
    """Compiles csrc/tw_heightgen.cu once per variant, all at once, and links each with the shipped build's other objects into its own copy of the
    package (the shipped library is never touched). Returns {name: (package root, nvcc process, link command)}."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("tw_build", os.path.join(ROOT, "3dworld_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    shipped = os.path.join(ROOT, "3dworld_b200", "build")
    others = [os.path.join(shipped, s.rsplit(".", 1)[0] + ".o") for s in b.SOURCES if s != "tw_heightgen.cu"]
    missing = [o for o in others if not os.path.exists(o)]
    assert not missing, "the shipped build's objects are missing (build() leaves them in 3dworld_b200/build): %s" % missing
    flags = [f for f in b.NVCC_FLAGS if f != "--use_fast_math=false"]
    out = {}
    for name, (_, define, _) in VARIANTS.items():
        d = tmp_path_factory.mktemp("variant")
        pkg = d / "3dworld_b200"
        pkg.mkdir()
        for f in os.listdir(os.path.dirname(tw.LIB_PATH)):
            if f.endswith(".py"):
                shutil.copy(os.path.join(os.path.dirname(tw.LIB_PATH), f), pkg / f)
        obj = str(d / "tw_heightgen.o")
        nvcc = subprocess.Popen([b.nvcc()] + flags + [define, "-x", "cu", "-c", os.path.join(b.CSRC, "tw_heightgen.cu"), "-o", obj],
                                stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        link = ([b.nvcc(), "-shared", "-Wno-deprecated-gpu-targets", "-o", str(pkg / "lib3dworld_b200.so"), obj] + others +
                ["-Xlinker", "--no-undefined", "-lcudart_static", "-lpthread", "-ldl", "-lrt"])         # as build.build links
        out[name] = (str(d), nvcc, link)
    yield out
    for _, nvcc, _ in out.values():
        if nvcc.poll() is None:
            nvcc.kill()
            nvcc.wait()


@pytest.mark.skipif(bool(BUILD), reason="runs in the shipped build's process only")
@pytest.mark.parametrize("name", list(VARIANTS))
def test_variant_build(ctx, variant_builds, name):            # ctx: skips without a CUDA device
    consts, _, select = VARIANTS[name]
    root, nvcc, link = variant_builds[name]
    log, _ = nvcc.communicate()
    assert nvcc.returncode == 0, log
    subprocess.check_call(link)
    lib = os.path.join(root, "3dworld_b200", "lib3dworld_b200.so")
    script = ("import importlib, sys; sys.path.insert(0, %r); importlib.import_module('3dworld_b200'); import pytest; "
              "sys.exit(pytest.main([%r, '-q', '-m', 'gpu', '-p', 'no:cacheprovider', '-k', %r]))" % (root, os.path.abspath(__file__), select))
    env = dict(os.environ, TW_DWARP_TEST_BUILD=json.dumps(dict(consts, lib=lib)), PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", script], cwd=root, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    tail = r.stdout[-8000:]
    assert r.returncode == 0, tail
    assert re.search(r"\d+ passed", tail) and " skipped" not in tail and "deselected" in tail, tail
