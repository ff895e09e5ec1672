"""CPU: the asynchronous points job on the host side - tw_points_launch is exported and listed in ABI_SYMBOLS, PQ_HMAP and the ctypes mirror of tw_points_job
match the header, a NULL context is refused; a numpy restatement of the heightmap point sampler (hmap_points_kernel: get_clamped_height at float cells)
held to the oracle's tile sampler at integer cells, which the GPU tests then hold the kernel to at fractional ones; and the SASS of the point and tile
kernels the job reuses, against the digests of the build before the job existed."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _clamp(x, y, W, H, mode):
    """clamp_no_scale (src/heightmap.cpp:315-341) on int64 arrays of texel coordinates: (x, y, on the texture)."""
    x, y = x + W // 2, y + H // 2
    inside = (x >= 0) & (y >= 0) & (x < W) & (y < H)
    if mode == 0:
        return np.clip(x, 0, W - 1), np.clip(y, 0, H - 1), np.ones_like(inside)
    if mode == 1:
        return x, y, inside

    def mirror(v, n):
        mod, div = np.abs(v) % n, np.sign(v) * (np.abs(v) // n)     # C's abs() % n and truncating division
        return np.where(div & 1, n - mod - 1, mod)
    return np.where(inside, x, mirror(x, W)), np.where(inside, y, mirror(y, H)), np.ones_like(inside)


def _scaled(ms, v):
    """twh::clamp_scaled(mesh_scale*v) in fp32: NaN goes to -2^30."""
    s = (F(ms) * v.astype(F)).astype(F)
    return np.clip(np.where(np.isnan(s), F(-2.0 ** 30), s), F(-2.0 ** 30), F(2.0 ** 30)).astype(F)


def hmap_points_np(img, hs, xy):
    """hmap_points_kernel, expression for expression in fp32: img = uint8 [H, W, 2] (low byte, high byte), hs = HmapSampler, xy = float32 [n, 2]."""
    W, H, ms = hs.width, hs.height, F(hs.mesh_scale)
    xy = np.asarray(xy, F).reshape(-1, 2)
    hsc, mfs, tz, zinv = F(hs.h_scale), F(hs.mesh_file_scale), F(hs.mesh_file_tz), F(hs.mesh_scale_z_inv)
    scale = lambda v: ((hsc * mfs * v + tz) * zinv).astype(F)  # noqa: E731  scale_mh_texture_val
    tex = scale((img[..., 0].astype(np.float64) / 256.0 + img[..., 1].astype(np.float64)).astype(F))   # get_heightmap_value, exact in fp32
    zero = scale(F(0.0))
    if ms < 1:
        sx, sy = _scaled(ms, xy[:, 0]), _scaled(ms, xy[:, 1])
        xlo, ylo = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        xhi, yhi = np.ceil(sx).astype(np.int64), np.ceil(sy).astype(np.int64)
        xv, yv = (sx - xlo.astype(F)).astype(F), (sy - ylo.astype(F)).astype(F)
        xlo, ylo, ok_lo = _clamp(xlo, ylo, W, H, hs.edge_mode)
        xhi, yhi, ok_hi = _clamp(xhi, yhi, W, H, hs.edge_mode)
        ok = ok_lo & ok_hi
        g = lambda a, b: tex[np.where(ok, b, 0), np.where(ok, a, 0)]  # noqa: E731
        one = F(1.0)
        z = (yv * (xv * g(xhi, yhi) + (one - xv) * g(xlo, yhi)) + (one - yv) * (xv * g(xhi, ylo) + (one - xv) * g(xlo, ylo))).astype(F)
        return np.where(ok, z, zero).astype(F)

    def near(v):                                             # round_fp(mesh_scale*(x + 0.0f))
        s = _scaled(ms, (v.astype(F) + F(0.0)).astype(F))
        return np.where(s > 0, (s + F(0.5)).astype(F), (s - F(0.5)).astype(F)).astype(np.int64)
    x, y, ok = _clamp(near(xy[:, 0]), near(xy[:, 1]), W, H, hs.edge_mode)
    return np.where(ok, tex[np.where(ok, y, 0), np.where(ok, x, 0)], zero).astype(F)


def tile_cells(origins, zv):
    """The cells (x1 + i, y1 + j) of tiles at origins, in tw_heightmap_sample_tiles' output order, as float32 [nt*zv*zv, 2]."""
    j, i = np.meshgrid(np.arange(zv), np.arange(zv), indexing="ij")
    o = np.asarray(origins, np.int64).reshape(-1, 1, 1, 2)
    return np.stack([o[..., 0] + i, o[..., 1] + j], -1).reshape(-1, 2).astype(F)


def sampler_cases(W, H, zv):
    """Tile origins inside the image, across its edges and far outside it (mirror periods, clamp edges, cliff)."""
    inner = [(tx * (zv - 1) - W // 2 - 3, ty * (zv - 1) - H // 2 - 2) for ty in range(4) for tx in range(5)]
    far = [(-3 * W - 11, 2 * H + 7), (5 * W + 3, -4 * H - 1), (-7 * W, -9 * H), (40 * W + 1, 33 * H), (-(1 << 20), 1 << 21)]
    return np.array(inner + far, np.int32)


def test_entry_point_is_exported(tw):
    assert "tw_points_launch" in tw.ABI_SYMBOLS and hasattr(tw.lib, "tw_points_launch")
    hdr = open(os.path.join(ROOT, "include", "tw3d.h")).read()
    assert int(re.search(r"#define TW_PQ_HMAP\s+(\d+)", hdr).group(1)) == tw.PQ_HMAP == 3
    assert tw.lib.tw_abi_version() == 1


def test_points_job_layout(tw, tmp_path):
    fields = [f for f, _ in tw.PointsJobArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tw3d.h"\nint main(void) {printf("%zu", sizeof(tw_points_job)); '
                   + "".join('printf(" %%zu", offsetof(tw_points_job, %s)); ' % f for f in fields) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(tw.PointsJobArgs)] + [getattr(tw.PointsJobArgs, f).offset for f in fields]


def test_launch_refuses_null_context(tw):
    xy, out = np.zeros((1, 2), np.float32), np.zeros(1, np.float32)
    a = tw.PointsJobArgs(tw._ptr(xy), 1, None, None, None, tw._ptr(out))
    assert tw.lib.tw_points_launch(None, C.byref(a)) == tw.TW_ERR_ARG


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ms", [0.5, 1.0, 2.0, 1.3, 0.37])
def test_numpy_sampler_equals_oracle_tiles(tw, oracle, mode, ms):
    rng = np.random.default_rng(int(ms * 100) + mode)
    for W, H, zv in ((37, 53, 9), (61, 29, 17), (64, 48, 5)):
        img = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
        hs = tw.HmapSampler(W, H, mode, ms, 0.0012, 1.7, -0.3, 0.8)
        origins = sampler_cases(W, H, zv)
        want = oracle.hmap_sample_tiles(img, oracle.HmapSampler(W, H, mode, ms, 0.0012, 1.7, -0.3, 0.8), origins, zv).ravel()
        got = hmap_points_np(img, hs, tile_cells(origins, zv))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (W, H)


def test_numpy_sampler_holds_absurd_coordinates_on_the_image(tw):
    """NaN, infinities and huge floats read texels of the image (the clamp of the scaled coordinate keeps every index in int range)."""
    img = np.arange(2 * 7 * 5, dtype=np.uint8).reshape(5, 7, 2)
    xy = np.array([[np.nan, 0], [np.inf, -np.inf], [3e9, -3e9], [1e30, 2.5], [-0.0, 1e-30]], np.float32)
    for mode in (0, 1, 2):
        for ms in (0.5, 1.0, 4.0):
            z = hmap_points_np(img, tw.HmapSampler(7, 5, mode, ms, 1.0, 1.0, 0.0, 1.0), xy)
            assert np.all(np.isfinite(z))


# SHA-256 of each kernel's SASS instruction words (the encodings cuobjdump -sass prints) in the build before tw_points_launch existed, CUDA 12.9: the job reuses
# these kernels, and their code must not change with it
SASS_CUDA = "12.9"
SASS_PARENT = {
    "points_kernel<0,0,0>": "a838e4e42bae64d3fd88cd489544345b7c79e0a19fecb4dfad4dd35de99a7513",
    "points_kernel<0,0,1>": "bf5546986d6e9eadceb3a8e76fc73742f83e5bab206dd5e0e416061a85307861",
    "points_kernel<0,0,2>": "3ec4caef18575a74582c8f564ab66199286aa8891a85fb5852c04f80d2c6b5b6",
    "points_kernel<1,0,0>": "91065a32e74592b2f349974e79835f8a44d1f943ada21b2aa37cdbb574772d06",
    "points_kernel<1,0,1>": "fbf1f766145af3037fc3c5f3bf4faeef15516ca7628476066061a76a185ab94e",
    "points_kernel<1,0,2>": "ab24216f0f1e68ccac68ea91da8012eb6bdd60c7d7f4626d3328b085871966eb",
    "points_kernel<1,1,0>": "ac1ed6a9348ebbf768e8553ec9ef9b94475eeb7d3711b90d71e5a365e6558802",
    "points_kernel<1,1,1>": "91123382340e0fe354e5a484dcbddd88483cfba6de6a668d9512f165b76a6f64",
    "points_kernel<1,1,2>": "56ac6e2eb428a31645a7e7fa179ad77380b47a31d230fbd12f262d504f649b63",
    "hmap_sample_tiles_kernel": "ac354798e03a45249bb60979713cfc3a1053deda5663976404e019006bd39e9f",
}


def kernel_sass(lib):
    """{short kernel name: SHA-256 of its SASS instruction words} for the kernels of SASS_PARENT."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, name, buf = {}, None, []

    def flush():
        if name:
            res[name] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            flush()
            f, buf = m.group(1), []
            t = re.match(r"_Z13points_kernelILb(\d)ELb(\d)ELi(\d)E", f)
            name = ("points_kernel<%s,%s,%s>" % t.groups()) if t else ("hmap_sample_tiles_kernel" if "24hmap_sample_tiles_kernel" in f else None)
        elif name:
            buf.extend(re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line))   # the instruction words only: cuobjdump also prints section headers that name source paths
    flush()
    return res


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_reused_kernels_keep_their_sass(tw):
    release = re.search(r"release (\d+\.\d+)", subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != SASS_CUDA:
        pytest.skip("the digests are those of CUDA %s" % SASS_CUDA)
    assert kernel_sass(tw.LIB_PATH) == SASS_PARENT
