"""GPU: the voxel path (tw_voxel_fill, tw_voxel_outside, tw_voxel_remove_unconnected, tw_voxel_triangles) at the launch shapes and sizes where its kernels
change behaviour, bit for bit against the plain-C oracle and, for remove_unconnected, against the scipy reference of tests/test_voxel_flood_reference.py:
  fill         the sine kernel's 8-column passes, 64-column blocks and 128-voxel z blocks; the GLM kernel's 128- and 256-thread z blocks (nz 128 / 129) and
               several z blocks; every attenuation mode; the 65535 limits; the full 512^3 sine grid (BASELINE config 4) and a y slab of the 512^3 GLM grids
  post chain   outside -> remove_unconnected -> triangles on GLM grids of 256^3 and 512^3 (131072 marching-cubes blocks: 128 passes of the block scan)
  triangles    grids of exactly 1024 and 1025 blocks, capacity cut at a block boundary and inside the second scan pass
  flood fills  known answers: fills that end one generation before, at and after a multiple of 8 (the frontier is checked every 8 launches) and after
               20000 generations; a cut serpentine corridor (pass 0) and a cut outside corridor winding down from the top plane (pass 1)."""
import os

import numpy as np
import pytest

from cases import convert
from test_voxel_flood_reference import column_case, column_generations, corridor_case, post_params, remove_unconnected_ref, serpentine_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAN = float("nan")


@pytest.fixture(scope="module")
def tables():
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _cfg(scene, mode):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)


def _vp(scene, mode, nx, ny, nz, atten=0):
    """The voxel grid of tests/test_gpu_voxel.py: geometry (lo_pos, vsz) of a 40x24x36 grid, any dimensions (so grids 1 voxel wide are allowed)."""
    vp = scene.voxel_landscape_params(_cfg(scene, mode), 40, 24, 36)
    vp.nx, vp.ny, vp.nz = nx, ny, nz
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = atten, 0.7, 0.4
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    return vp


def _nan_cuda(shape, dtype=None):
    """A CUDA tensor filled with NaN (or 0xAB bytes), so elements a kernel never writes show; waits for it, as the context's stream does not wait for torch's."""
    import torch
    t = torch.full(shape, NAN, device="cuda") if dtype is None else torch.full(shape, 0xAB, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    return t


def _check_fill(ctx, oracle, beq, vp):
    exp = oracle.voxel_fill(convert(vp, oracle.VoxelParams))
    got = ctx.voxel_fill(vp)
    assert beq(got, exp) == 0, "host %dx%dx%d mode %d: %d values differ" % (vp.nx, vp.ny, vp.nz, vp.gen_mode, beq(got, exp))
    d = _nan_cuda((vp.ny, vp.nx, vp.nz))
    ctx.voxel_fill(vp, out=d)
    assert beq(d.cpu().numpy(), exp) == 0, "device %dx%dx%d mode %d" % (vp.nx, vp.ny, vp.nz, vp.gen_mode)


# ---- fill shapes ----
@pytest.mark.parametrize("nx", [7, 8, 9, 63, 64, 65, 72])
def test_sine_fill_shapes(scene, oracle, ctx, beq, nx):
    """voxel_sine_kernel: x passes of 8 columns, blocks of 64 columns and of 128 z values, each just below, at and above its size."""
    for nz in (127, 128, 129, 257):
        _check_fill(ctx, oracle, beq, _vp(scene, 0, nx, 3, nz))


def test_sine_fill_wider_than_65535(scene, oracle, ctx, beq):
    _check_fill(ctx, oracle, beq, _vp(scene, 0, 65537, 1, 2))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("nx", [31, 32, 33, 65])
def test_glm_fill_shapes(scene, oracle, ctx, beq, mode, nx):
    """voxel_glm_kernel: 128-thread z blocks up to nz = 128, 256-thread blocks above, several z blocks; x runs of 32 columns per block."""
    for nz in (128, 129, 256, 257, 513):
        _check_fill(ctx, oracle, beq, _vp(scene, mode, nx, 2, nz))


@pytest.mark.parametrize("mode", [1, 2])
def test_glm_fill_65535_rows(scene, oracle, ctx, beq, mode):
    _check_fill(ctx, oracle, beq, _vp(scene, mode, 1, 65535, 1))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("atten", [1, 2, 3, 4, 5])
def test_glm_fill_atten_modes(scene, oracle, ctx, beq, mode, atten):
    _check_fill(ctx, oracle, beq, _vp(scene, mode, 31, 17, 45, atten=atten))


@pytest.mark.parametrize("mode,dims", [(0, (1, 65536, 1)), (1, (1, 65536, 1)), (2, (1, 65536, 1)), (1, (65536, 1, 1)), (2, (65536, 1, 1))])
def test_fill_size_refusals(tw, scene, ctx, mode, dims):
    with pytest.raises(tw.TwError) as e:
        ctx.voxel_fill(_vp(scene, mode, *dims))
    assert e.value.status == tw.TW_ERR_ARG


def test_sine_fill_512_cube(scene, oracle, ctx, beq):
    """BASELINE config 4: the whole 512^3 sine grid."""
    vp = scene.voxel_landscape_params(_cfg(scene, 0), 512, 512, 512)
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    d = _nan_cuda((512, 512, 512))
    ctx.voxel_fill(vp, out=d)
    exp = oracle.voxel_fill(convert(vp, oracle.VoxelParams), nthreads=os.cpu_count() or 1)
    assert beq(d.cpu().numpy(), exp) == 0


@pytest.mark.parametrize("mode", [1, 2])
def test_glm_fill_512_cube_slab(scene, oracle, ctx, beq, mode):
    """The 512^3 GLM grid: its first 16 rows are the 512x16x512 grid of the same geometry (true without attenuation only, which depends on ny)."""
    vp = scene.voxel_landscape_params(_cfg(scene, mode), 512, 512, 512)
    d = _nan_cuda((512, 512, 512))
    ctx.voxel_fill(vp, out=d)
    assert not d.isnan().any().item()
    slab = convert(vp, type(vp))
    slab.ny = 16
    assert beq(d[:16].cpu().numpy(), oracle.voxel_fill(convert(slab, oracle.VoxelParams))) == 0


# ---- post-processing chain ----
def _glm_field(tw, scene, ctx, dims, z_gradient=0.0):
    """A GLM simplex grid filled on the device; returns (VoxelParams, CUDA tensor)."""
    vp = scene.voxel_landscape_params(_cfg(scene, 1), *dims, z_gradient=z_gradient)
    d = _nan_cuda((dims[1], dims[0], dims[2]))
    ctx.voxel_fill(vp, out=d)
    return vp, d


def _post(tw, vp, **kw):
    p = post_params(tw.VoxelPostParams, (vp.nx, vp.ny, vp.nz), **kw)
    for k in range(3):
        p.lo_pos[k], p.vsz[k] = vp.lo_pos[k], vp.vsz[k]
    return p


CHAIN = [(256, rm, kae, mesh) for rm in (1, 3) for kae in (0, 1) for mesh in (0, 1)] + [(512, 1, 0, 0), (512, 3, 1, 1), (512, 3, 0, 0), (512, 1, 1, 1)]


@pytest.mark.parametrize("n,rm,kae,mesh", CHAIN)
def test_post_chain(tw, scene, oracle, ctx, beq, tables, n, rm, kae, mesh):
    """A terrain-like GLM grid (inside below a noisy surface, caves and floating pieces) through the device-resident chain; every stage against the
    oracle stage on the same input, remove_unconnected also against the scipy reference."""
    import torch
    vp, dv = _glm_field(tw, scene, ctx, (n, n, n), z_gradient=-2.0)
    vals = dv.cpu().numpy()
    p = _post(tw, vp, isolevel=-1.0, remove_unconnected=rm, keep_at_edge=kae, centre_seed=int(not mesh), skip_under_mesh=mesh)
    po = convert(p, oracle.VoxelPostParams)
    zix = np.random.default_rng(n + 8 * rm + 2 * kae + mesh).integers(n // 16, n // 4, (n, n)).astype(np.uint32) if mesh else None
    dz = None if zix is None else torch.from_numpy(zix.astype(np.int32)).cuda()
    do = _nan_cuda((n, n, n), torch.uint8)
    ctx.voxel_outside(dv, p, dz, out=do)
    out_o = oracle.voxel_outside(vals, po, zix)
    assert np.array_equal(do.cpu().numpy(), out_o)
    ch = ctx.voxel_remove_unconnected(dv, do, p)
    v_o, o_o, ch_o = oracle.voxel_remove_unconnected(vals, out_o, po)
    assert np.array_equal(do.cpu().numpy(), o_o) and beq(dv.cpu().numpy(), v_o) == 0 and ch == ch_o
    v_r, o_r, ch_r = remove_unconnected_ref(vals, out_o, po)
    assert np.array_equal(o_r, o_o) and beq(v_r, v_o) == 0 and ch_r == ch_o
    assert 0 < ch_o < n ** 3 // 8
    t_o = oracle.voxel_triangles(v_o, o_o, po, tables)
    assert len(t_o) > 100000
    t = ctx.voxel_triangles(dv, do, p, tables)
    assert t.shape == t_o.shape and beq(t, t_o) == 0
    dt = _nan_cuda((len(t_o), 3, 3))
    _, cnt = ctx.voxel_triangles(dv, do, p, tables, out=dt)
    assert cnt == len(t_o) and beq(dt.cpu().numpy(), t_o) == 0


@pytest.mark.parametrize("dims", [(128, 64, 128), (1025, 32, 32), (32, 1024, 32), (32, 1025, 32)])
def test_triangles_block_counts(tw, scene, oracle, ctx, beq, tables, dims):
    """Grids of exactly 1024 and 1025 marching-cubes blocks (1024 cubes each): the block scan runs one full pass, or a second pass of one block. With
    nx*nz = 1024 every block is one y plane, so the last valid plane is the last block of the first pass."""
    vp, dv = _glm_field(tw, scene, ctx, dims)
    vals = dv.cpu().numpy()
    p = _post(tw, vp)
    po = convert(p, oracle.VoxelPostParams)
    o = oracle.voxel_outside(vals, po)
    t_o = oracle.voxel_triangles(vals, o, po, tables)
    assert len(t_o) > 10000
    t = ctx.voxel_triangles(vals, o, p, tables)
    assert t.shape == t_o.shape and beq(t, t_o) == 0
    import torch
    do = torch.from_numpy(o).cuda()
    dt = _nan_cuda((len(t_o), 3, 3))
    _, cnt = ctx.voxel_triangles(dv, do, p, tables, out=dt)
    assert cnt == len(t_o) and beq(dt.cpu().numpy(), t_o) == 0


def test_triangles_capacity_in_second_scan_pass(tw, scene, oracle, ctx, beq, tables):
    """32x1100x32: block b is plane y = b, so the triangles of blocks < b are those of the grid's first b+1 planes (make_closed_surface off: the flags are
    per voxel). Capacities at the boundary of the two scan passes, at a block boundary inside the second pass and one past it; host and device outputs;
    nothing is written past the capacity."""
    import torch
    vp, dv = _glm_field(tw, scene, ctx, (32, 1100, 32))
    vals = dv.cpu().numpy()
    p = _post(tw, vp, make_closed_surface=0)
    po = convert(p, oracle.VoxelPostParams)
    o = oracle.voxel_outside(vals, po)
    t_o = oracle.voxel_triangles(vals, o, po, tables)
    do = torch.from_numpy(o).cuda()

    def before(b):
        pb = convert(po, oracle.VoxelPostParams)
        pb.ny = b + 1
        return len(oracle.voxel_triangles(vals[:b + 1], o[:b + 1], pb, tables))

    caps = [before(1024), before(1050), before(1050) + 1]
    assert 0 < caps[0] < caps[1] < caps[2] < len(t_o)
    for cap in caps:
        host = np.full((cap, 3, 3), NAN, np.float32)
        assert ctx.voxel_triangles(vals, o, p, tables, out=host) is host and beq(host, t_o[:cap]) == 0
        dt = _nan_cuda((cap + 4, 3, 3))
        _, cnt = ctx.voxel_triangles(dv, do, p, tables, out=dt[:cap])
        got = dt.cpu().numpy()
        assert cnt == len(t_o) and beq(got[:cap], t_o[:cap]) == 0 and np.isnan(got[cap:]).all()


# ---- flood fills with known answers ----
def _remove_both(tw, ctx, vals, outside, p):
    """remove_unconnected on host arrays and on CUDA tensors; returns the two results (vals, outside, changed)."""
    import torch
    v, o = vals.copy(), outside.copy()
    ch = ctx.voxel_remove_unconnected(v, o, p)
    dv, do = torch.from_numpy(vals).cuda(), torch.from_numpy(outside).cuda()
    torch.cuda.synchronize()
    dch = ctx.voxel_remove_unconnected(dv, do, p)
    return (v, o, ch), (dv.cpu().numpy(), do.cpu().numpy(), dch)


@pytest.mark.parametrize("nz", [16, 18, 20, 32, 34, 36, 40002])
def test_deep_fill_column(tw, ctx, beq, nz):
    """The fill along a 1-voxel line ends after 7, 8, 9, 15, 16, 17 and 20000 generations and must reach all of it."""
    vals, kw = column_case(nz)
    p = post_params(tw.VoxelPostParams, (3, 3, nz), **kw)
    outside = ctx.voxel_outside(vals, p)
    assert (outside == 0).sum() == nz - 2 and column_generations(nz) in (7, 8, 9, 15, 16, 17, 20000)
    for v, o, ch in _remove_both(tw, ctx, vals, outside, p):
        assert ch == 0 and np.array_equal(o, outside) and beq(v, vals) == 0


@pytest.mark.parametrize("case", [serpentine_case, corridor_case])
def test_deep_fill_corridors(tw, ctx, beq, case):
    vals, kw, exp_o, exp_v = case()
    ny, nx, nz = vals.shape
    p = post_params(tw.VoxelPostParams, (nx, ny, nz), **kw)
    outside = ctx.voxel_outside(vals, p)
    assert np.array_equal(outside, (vals < 0).astype(np.uint8))
    for v, o, ch in _remove_both(tw, ctx, vals, outside, p):
        assert np.array_equal(o, exp_o) and beq(v, exp_v) == 0 and ch == int((exp_o != outside).sum())


# ---- argument checks ----
@pytest.mark.parametrize("dims", [(65536, 65536, 1), (65537, 65535, 1), (1, 65537, 65535)])
def test_post_refuses_2_32_voxels(tw, ctx, tables, dims):
    p = post_params(tw.VoxelPostParams, dims)
    vals, flags = np.zeros(8, np.float32), np.zeros(8, np.uint8)
    for call in (lambda: ctx.voxel_outside(vals, p, out=flags), lambda: ctx.voxel_remove_unconnected(vals, flags, p),
                 lambda: ctx.voxel_triangles(vals, flags, p, tables)):
        with pytest.raises(tw.TwError) as e:
            call()
        assert e.value.status == tw.TW_ERR_ARG


def test_remove_unconnected_refuses_unaligned_device_flags(tw, ctx):
    import torch
    p = post_params(tw.VoxelPostParams, (4, 4, 4))
    buf = torch.zeros(65, dtype=torch.uint8, device="cuda")
    with pytest.raises(tw.TwError) as e:
        ctx.voxel_remove_unconnected(np.ones(64, np.float32), buf[1:], p)
    assert e.value.status == tw.TW_ERR_ARG


@pytest.mark.parametrize("dims", [(9, 7, 15), (9, 7, 14), (9, 7, 13)])
def test_remove_unconnected_device_flags_not_multiple_of_4(tw, oracle, ctx, beq, dims):
    """n % 4 = 1, 2, 3: a device flag buffer gives the host result, and the bytes after it are left alone."""
    import torch
    from test_voxel_flood_reference import random_field
    nx, ny, nz = dims
    n = nx * ny * nz
    vals, _ = random_field(dims, n, True)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=3)
    outside = ctx.voxel_outside(vals, p)
    exp = oracle.voxel_remove_unconnected(vals, outside, convert(p, oracle.VoxelPostParams))
    assert exp[2] > 0
    v, o = vals.copy(), outside.copy()
    assert ctx.voxel_remove_unconnected(v, o, p) == exp[2] and np.array_equal(o, exp[1]) and beq(v, exp[0]) == 0
    buf = _nan_cuda((n + 8,), torch.uint8)
    buf[:n].copy_(torch.from_numpy(outside.ravel()))
    dv = torch.from_numpy(vals).cuda()
    torch.cuda.synchronize()
    assert ctx.voxel_remove_unconnected(dv, buf[:n], p) == exp[2]
    got = buf.cpu().numpy()
    assert np.array_equal(got[:n], exp[1].ravel()) and (got[n:] == 0xAB).all() and beq(dv.cpu().numpy(), exp[0]) == 0
