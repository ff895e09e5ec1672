"""GPU: the welded marching-cubes mesh - tw_voxel_mesh_welded (Context.voxel_mesh) and the voxel build job with mesh outputs (tw_voxel_build_launch_ex).

The device derives every vertex from its owner cube's neighbourhood; the sequential reference of tests/voxel_mesh_ref.c fills a per-edge cache cube by
cube. The two are held equal bit for bit (vertices, indices, both counts) on the golden cases, smoothed random fields with every option, odd and tiny grids, the constructed orientation and
degenerate fields of tests/test_voxel_mesh_host.py, a 512^3 sine fill and 256^3 GLM terrain through the job, with host, page-locked and device buffers.
The job's soup must stay what tw_voxel_build_launch gives, capacities must be honoured with counts still reported, and the job must follow the job rules:
a shared context beside tile jobs, and tw_cancel with the counts left unwritten."""
import ctypes as C
import os

import numpy as np
import pytest

from cases import convert
from test_gpu_voxel_build import _buf, _input, _post_for, _scfg
from test_voxel_flood_reference import RANDOM_FIELDS, column_case, post_params, random_field
from test_voxel_mesh_host import CASES, check_mesh, degenerate_case, make_case, orientation_case
from voxel_mesh_ref import voxel_mesh as welded

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAN = float("nan")
SENT = 0xDEADBEEF


@pytest.fixture(scope="module")
def tables():
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def _same_mesh(got, exp):
    gv, gi = np.asarray(_np(got[0]), np.float32), np.asarray(_np(got[1]), np.uint32)
    ev, ei = exp
    assert gv.shape == ev.shape and gi.shape == ei.shape
    assert np.array_equal(gv.view(np.uint32), ev.view(np.uint32))
    assert np.array_equal(gi, ei)


def _mesh_bufs(kind, nv, nt, extra=3):
    """verts / indices buffers of nv + extra, nt + extra rows filled with sentinels: 'host' numpy, 'pinned' page-locked torch, 'device' CUDA tensors."""
    import torch
    if kind == "host":
        return np.full((nv + extra, 3), NAN, np.float32), np.full((nt + extra, 3), SENT, np.uint32)
    dev = "cuda" if kind == "device" else "cpu"
    v = torch.full((nv + extra, 3), NAN, dtype=torch.float32, device=dev)
    i = torch.full((nt + extra, 3), SENT - (1 << 32), dtype=torch.int32, device=dev)   # the sentinel's bits as int32
    if kind == "pinned":
        v, i = v.pin_memory(), i.pin_memory()
    torch.cuda.synchronize()
    return v, i


def _untouched(v, i, nv, nt):
    v, i = _np(v), np.asarray(_np(i)).view(np.uint32)
    return bool(np.isnan(v[nv:]).all() and (i[nt:] == SENT).all())


# ---- the synchronous call against the sequential reference ----
@pytest.mark.parametrize("case", CASES)
def test_sync_vs_reference(tw, oracle, ctx, tables, case):
    vals, outside, p = make_case(oracle, tw.VoxelPostParams, case)
    exp = welded(vals, outside, p, tables)
    _same_mesh(ctx.voxel_mesh(vals, outside, p, tables), exp)
    soup = ctx.voxel_triangles(vals, outside, p, tables)
    check_mesh(exp[0], exp[1], soup, outside, p)     # the device soup against the device mesh's vertices (equal to the reference's)


@pytest.mark.parametrize("dims,seed,kw", [((2, 2, 2), 1, dict(remove_unconnected=0, make_closed_surface=0)), ((5, 7, 9), 2, dict(remove_unconnected=1)),
                                          ((33, 17, 65), 3, dict(remove_unconnected=3, invert=1, isolevel=0.1)),
                                          ((64, 40, 48), 4, dict(remove_unconnected=3, centre_seed=0, skip_under_mesh=1)),
                                          ((1, 9, 9), 5, dict(remove_unconnected=0)), ((70, 3, 200), 6, dict(remove_unconnected=1, make_closed_surface=0))])
def test_shapes_and_options(tw, oracle, ctx, tables, dims, seed, kw):
    """Odd sizes, a single cube, a flat grid without cubes, grids of many 1024-cube blocks; invert, make_closed_surface, skip_under_mesh with zix_xy."""
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    po = post_params(oracle.VoxelPostParams, dims, **kw)
    v2, o2, _ = oracle.voxel_remove_unconnected(vals, oracle.voxel_outside(vals, po, zix), po)
    p = post_params(tw.VoxelPostParams, dims, **kw)
    exp = welded(v2, o2, po, tables)
    _same_mesh(ctx.voxel_mesh(v2, o2, p, tables), exp)


def test_orientation_case(tw, oracle, ctx, tables):
    vals, outside, p, own, last = orientation_case(tw.VoxelPostParams, tables)
    verts, indices = ctx.voxel_mesh(vals, outside, p, tables)
    _same_mesh((verts, indices), welded(vals, outside, p, tables))
    vb = verts.view(np.uint32)
    assert (vb == own.view(np.uint32)).all(1).any() and not (vb == last.view(np.uint32)).all(1).any()
    soup = ctx.voxel_triangles(vals, outside, p, tables)
    assert (soup[-1].view(np.uint32) == last.view(np.uint32)).all(1).any()


def test_degenerate_case(tw, oracle, ctx, tables):
    vals, outside, p, _ = degenerate_case(tw.VoxelPostParams, oracle, tables)
    verts, indices = ctx.voxel_mesh(vals, outside, p, tables)
    _same_mesh((verts, indices), welded(vals, outside, p, tables))
    assert len(indices) != len(ctx.voxel_triangles(vals, outside, p, tables))


@pytest.mark.parametrize("kind", ["host", "pinned", "device"])
def test_buffer_kinds_and_capacities(tw, oracle, ctx, tables, kind):
    """Inputs and outputs of one kind; capacities 0, partial and exact, with the counts always reported and nothing written past a capacity."""
    import torch
    vals, outside, p = make_case(oracle, tw.VoxelPostParams, ("random", 0))
    ev, ei = welded(vals, outside, p, tables)
    nv, nt = len(ev), len(ei)
    if kind == "host":
        v_in, o_in = vals, outside
    else:
        v_in, o_in = torch.from_numpy(vals.copy()), torch.from_numpy(outside.copy())
        v_in, o_in = (v_in.cuda(), o_in.cuda()) if kind == "device" else (v_in.pin_memory(), o_in.pin_memory())
    for cv, ct in ((nv, nt), (0, 0), (nv // 3, 0), (0, nt // 2), (17, 5)):
        big_v, big_i = _mesh_bufs(kind, cv, ct, extra=3)
        _, _, gnv, gnt = ctx.voxel_mesh(v_in, o_in, p, tables, verts=big_v[:cv], indices=big_i[:ct])
        assert (gnv, gnt) == (nv, nt)
        assert _untouched(big_v, big_i, cv, ct)
        gv, gi = _np(big_v)[:cv], np.asarray(_np(big_i)).view(np.uint32)[:ct]
        assert np.array_equal(gv.view(np.uint32), ev[:cv].view(np.uint32)) and np.array_equal(gi, ei[:ct])


def test_refusals(tw, ctx, tables):
    p = post_params(tw.VoxelPostParams, (1130, 1130, 1130))     # 3*n >= 2^32 (n itself is below 2^32)
    e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
    dummy = np.zeros(16, np.float32)
    nv, nt = C.c_uint64(7), C.c_uint64(7)
    m = tw.VoxelMesh(None, 0, None, 0, C.cast(C.pointer(nv), C.c_void_p), C.cast(C.pointer(nt), C.c_void_p))
    call = lambda p, m: tw.lib.tw_voxel_mesh_welded(ctx._h, tw._ptr(dummy), tw._ptr(dummy), C.byref(p), tw._ptr(e), tw._ptr(t), tw._ptr(v), C.byref(m))  # noqa: E731
    assert call(p, m) == tw.TW_ERR_ARG and nv.value == 7
    p2 = post_params(tw.VoxelPostParams, (2, 2, 4))
    bad = tw.VoxelMesh(None, 4, None, 0, C.cast(C.pointer(nv), C.c_void_p), C.cast(C.pointer(nt), C.c_void_p))
    assert call(p2, bad) == tw.TW_ERR_ARG
    nocount = tw.VoxelMesh(None, 0, None, 0, None, None)
    assert call(p2, nocount) == tw.TW_ERR_ARG
    # the job: pageable outputs, a mesh without tables, soup buffers without ntris, the index limit
    vals = _input("device", np.ones((4, 2, 2), np.float32))
    with pytest.raises(tw.TwError):
        ctx.voxel_build_launch(p2, vals=vals, tables=tables, mesh=(np.zeros((8, 3), np.float32), None))
    with pytest.raises(tw.TwError):
        ctx.voxel_build_launch(p2, vals=vals, mesh=(None, None))
    with pytest.raises(tw.TwError):
        ctx.voxel_build_launch(p2, vals=vals, tables=tables, tris=_buf("device", (4, 3, 3), np.float32, NAN), mesh=(None, None), soup=False)
    big = post_params(tw.VoxelPostParams, (1130, 1130, 1130))
    with pytest.raises(tw.TwError):
        ctx.voxel_build_launch(big, vals=vals, tables=tables, mesh=(None, None))
    assert ctx.create_tiles_poll(wait=True)      # nothing was enqueued


# ---- the job ----
def _job(ctx, p, tables, exp_mesh, vals=None, fill=None, zix=None, kind="device", soup_cap=None, soup=True):
    """One job with mesh outputs of exactly the mesh's size plus sentinel rows (and the soup when soup_cap is given); returns (job, verts, indices, tris)."""
    nv, nt = len(exp_mesh[0]), len(exp_mesh[1])
    v, i = _mesh_bufs(kind, nv, nt)
    tris = None if soup_cap is None else _buf("device" if kind == "device" else "pinned", (soup_cap + 2, 3, 3), np.float32, NAN)
    vin = None if vals is None else _input("device", vals)
    job = ctx.voxel_build_launch(p, vals=vin, tris=tris, fill=fill, zix_xy=zix, tables=tables, capacity=soup_cap, mesh=(v, i), soup=soup)
    assert ctx.create_tiles_poll(wait=True)
    assert (job.nverts, job.mesh_ntris) == (nv, nt) and _untouched(v, i, nv, nt)
    return job, _np(v)[:nv], np.asarray(_np(i)).view(np.uint32)[:nt], (None if tris is None else _np(tris))


@pytest.mark.parametrize("case", [("golden", "mesh"), ("random", 3), ("random", 2)])
@pytest.mark.parametrize("kind", ["device", "pinned"])
def test_job_vs_sync(tw, oracle, ctx, beq, tables, case, kind):
    """The job from the raw field (outside flags and remove_unconnected inside it) equals the synchronous chain + tw_voxel_mesh_welded, and its soup
    equals tw_voxel_build_launch's."""
    if case[0] == "golden":
        g = np.load(os.path.join(GOLD, "voxel_post.npz"))
        vals0, zix = g["mesh_vals"], g["mesh_zix"]
        _, _, p = make_case(oracle, tw.VoxelPostParams, case)
    else:
        dims, seed, kw = RANDOM_FIELDS[case[1]]
        vals0, zix = random_field(dims, seed, kw.get("centre_seed", 1))
        p = post_params(tw.VoxelPostParams, dims, **kw)
    o = ctx.voxel_outside(vals0, p, zix)
    v2 = vals0.copy()
    ctx.voxel_remove_unconnected(v2, o, p)
    sync = ctx.voxel_mesh(v2, o, p, tables)
    soup = ctx.voxel_triangles(v2, o, p, tables)
    job, gv, gi, tris = _job(ctx, p, tables, sync, vals=vals0, zix=zix, kind=kind, soup_cap=len(soup))
    _same_mesh((gv, gi), sync)
    assert job.ntris == len(soup) and beq(tris[:len(soup)], soup) == 0 and np.isnan(tris[len(soup):]).all()
    pt = _buf("device", (len(soup), 3, 3), np.float32, NAN)
    plain = ctx.voxel_build_launch(p, vals=_input("device", vals0), zix_xy=zix, tables=tables, tris=pt)
    assert ctx.create_tiles_poll(wait=True) and plain.ntris == len(soup) and beq(_np(pt), tris[:len(soup)]) == 0
    # mesh only: no soup passes, the same mesh
    job2, gv2, gi2, _ = _job(ctx, p, tables, sync, vals=vals0, zix=zix, kind=kind, soup=False)
    _same_mesh((gv2, gi2), sync)
    assert job2.ntris == 0


def test_job_capacities(tw, oracle, ctx, tables):
    vals, _, p = make_case(oracle, tw.VoxelPostParams, ("random", 0))
    p.remove_unconnected = 0
    ev, ei = welded(vals, ctx.voxel_outside(vals, p), p, tables)
    for cv, ct in ((0, 0), (len(ev) // 2, len(ei) // 3), (len(ev), len(ei))):
        v, i = _mesh_bufs("pinned", cv, ct)
        job = ctx.voxel_build_launch(p, vals=_input("device", vals), tables=tables, mesh=(v[:cv] if cv else None, i[:ct] if ct else None), soup=False)
        assert ctx.create_tiles_poll(wait=True)
        assert (job.nverts, job.mesh_ntris) == (len(ev), len(ei)) and _untouched(v, i, cv, ct)
        assert np.array_equal(v.numpy()[:cv].view(np.uint32), ev[:cv].view(np.uint32)) and np.array_equal(i.numpy()[:ct].view(np.uint32), ei[:ct])


def test_fill_sine_512(tw, scene, oracle, ctx, tables):
    """BASELINE config 4 through the job: the welded mesh of the job's own field and flags equals the sequential reference's."""
    import torch
    vp = scene.voxel_landscape_params(_scfg(scene, 0), 512, 512, 512)
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    p = _post_for(tw, vp, remove_unconnected=3)
    shape = (512, 512, 512)
    v, o = torch.empty(shape, device="cuda"), torch.empty(shape, dtype=torch.uint8, device="cuda")
    cnt = ctx.voxel_build_launch(p, vals=v, outside=o, fill=vp, tables=tables, mesh=(None, None), soup=False)
    assert ctx.create_tiles_poll(wait=True)
    vals, outside = v.cpu().numpy(), o.cpu().numpy()
    exp = welded(vals, outside, p, tables)
    assert (cnt.nverts, cnt.mesh_ntris) == (len(exp[0]), len(exp[1])) and len(exp[1]) > 100000
    gv, gi = torch.empty((len(exp[0]), 3), device="cuda"), torch.empty((len(exp[1]), 3), dtype=torch.int32, device="cuda")
    job = ctx.voxel_build_launch(p, fill=vp, tables=tables, mesh=(gv, gi), soup=False)
    assert ctx.create_tiles_poll(wait=True)
    assert (job.nverts, job.mesh_ntris) == (len(exp[0]), len(exp[1]))
    _same_mesh((gv, gi.cpu().numpy().view(np.uint32)), exp)


def test_fill_glm_256_terrain(tw, scene, oracle, ctx, tables):
    import torch
    n = 256
    vp = scene.voxel_landscape_params(_scfg(scene, 1), n, n, n, z_gradient=-2.0)
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=3, centre_seed=0, skip_under_mesh=1)
    zix = np.random.default_rng(7).integers(n // 16, n // 4, (n, n)).astype(np.uint32)
    v, o = torch.empty((n, n, n), device="cuda"), torch.empty((n, n, n), dtype=torch.uint8, device="cuda")
    cnt = ctx.voxel_build_launch(p, vals=v, outside=o, fill=vp, zix_xy=zix, tables=tables, mesh=(None, None), soup=False)
    assert ctx.create_tiles_poll(wait=True)
    exp = welded(v.cpu().numpy(), o.cpu().numpy(), p, tables)
    assert (cnt.nverts, cnt.mesh_ntris) == (len(exp[0]), len(exp[1])) and len(exp[1]) > 10000
    _, gv, gi, _ = _job(ctx, p, tables, exp, fill=vp, zix=zix, kind="pinned")
    _same_mesh((gv, gi), exp)


def test_shared_context_beside_tile_jobs(tw, scene, oracle, tables):
    import torch
    from test_gpu_shared_ctx import _cfg as tile_cfg
    from test_gpu_tiles_shading import ITERS, ZV, _origins
    P = tw.Context(0)
    try:
        cfg = tile_cfg(scene, 0)
        P.set_sine_params(cfg.sine_params())
        hp, ep = cfg.height_params(), cfg.erosion_params()
        A = P.shared()
        origins = _origins(4)
        dims, seed, kw = RANDOM_FIELDS[2]
        vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
        p = post_params(tw.VoxelPostParams, dims, **kw)
        po = convert(p, oracle.VoxelPostParams)
        v2, o2, _ = oracle.voxel_remove_unconnected(vals, oracle.voxel_outside(vals, po, zix), po)
        exp = welded(v2, o2, po, tables)
        z = torch.full((len(origins), ZV, ZV), NAN).pin_memory()
        P.create_tiles_launch(origins, cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), ZV, hp, ITERS, ep, ep.zmin, z)
        v, i = _mesh_bufs("device", len(exp[0]), len(exp[1]))
        job = A.voxel_build_launch(p, vals=_input("device", vals), zix_xy=zix, tables=tables, mesh=(v, i), soup=False)
        for c in (A, P):
            assert c.create_tiles_poll(wait=True)
        assert (job.nverts, job.mesh_ntris) == (len(exp[0]), len(exp[1]))
        _same_mesh((v[:len(exp[0])], i[:len(exp[1])].cpu().numpy().view(np.uint32)), exp)
        assert not np.isnan(z.numpy()).any()
    finally:
        P.close()


def test_cancel_before_the_flood(tw, ctx, tables):
    """A 3 x 3 column whose flood runs 1e6 generations: cancelled right after the launch, the poll raises TwCanceled and leaves the mesh counts alone."""
    import torch
    c = tw.Context(0)
    try:
        nz = 2_000_004
        vals, kw = column_case(nz)
        p = post_params(tw.VoxelPostParams, (3, 3, nz), **kw)
        v = torch.from_numpy(vals).cuda()
        torch.cuda.synchronize()
        job = c.voxel_build_launch(p, vals=v, tables=tables, mesh=(None, None))
        job._nverts.value, job._mesh_ntris.value = 12345, 54321
        c.cancel()
        with pytest.raises(tw.TwCanceled):
            c.create_tiles_poll(True)
        assert (job.nverts, job.mesh_ntris) == (12345, 54321)
    finally:
        c.close()
