"""GPU: tw_voxel_build_launch (Context.voxel_build_launch) - the fill, the outside flags, remove_unconnected and the marching cubes of a voxel grid as one
asynchronous job. Every case is held to the plain-C oracle, the golden outputs of the reference's voxel_manager functions or the scipy reference of
tests/test_voxel_flood_reference.py (the synchronous tw_voxel_remove_unconnected runs the same flood as the job, so equality with it alone would prove
little): field, flags, triangles, the triangle count and the number of flipped voxels, with host, page-locked and device buffers."""
import ctypes as C
import os

import numpy as np
import pytest

from cases import convert
from test_voxel_flood_reference import RANDOM_FIELDS, column_case, corridor_case, post_params, random_field, remove_unconnected_ref, serpentine_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAN = float("nan")


@pytest.fixture(scope="module")
def tables():
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _buf(kind, shape, dtype, fill):
    """A buffer of the given kind ('host' numpy, 'pinned' page-locked torch, 'device' CUDA tensor) filled with `fill`, ready before the job starts."""
    import torch
    tdt = {np.float32: torch.float32, np.uint8: torch.uint8}[dtype]
    if kind == "host":
        return np.full(shape, fill, dtype)
    t = torch.full(shape, fill, dtype=tdt, device="cuda" if kind == "device" else "cpu")
    if kind == "pinned":
        t = t.pin_memory()
    torch.cuda.synchronize()
    return t


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def _input(kind, vals):
    import torch
    if kind == "host":
        return vals.copy()
    t = torch.from_numpy(vals.copy())
    t = t.cuda() if kind == "device" else t.pin_memory()
    torch.cuda.synchronize()
    return t


def _expected(oracle, vals, p, zix, tables):
    """The oracle's chain: (vals, outside, triangles, changed)."""
    po = convert(p, oracle.VoxelPostParams)
    o = oracle.voxel_outside(vals, po, zix)
    v2, o2, ch = oracle.voxel_remove_unconnected(vals, o, po)
    return v2, o2, oracle.voxel_triangles(v2, o2, po, tables), ch


def _run(ctx, p, tables, vals=None, kind="device", tri_kind=None, fill=None, zix=None, extra=4, want_vals=True):
    """One job with outputs of the given kind (tris in page-locked memory for host outputs), NaN / 0xAB sentinels everywhere; returns
    (vals, outside, tris, ntris, changed) as numpy, tris with its `extra` sentinel rows."""
    shape = (p.ny, p.nx, p.nz)
    if vals is not None:
        v = _input(kind, vals)
    else:
        v = _buf(kind, shape, np.float32, NAN) if want_vals else None
    o = _buf(kind, shape, np.uint8, 0xAB)
    cap = _count(ctx, p, tables, vals, fill, zix) if tables is not None else 0
    t = _buf(tri_kind or ("device" if kind == "device" else "pinned"), (cap + extra, 3, 3), np.float32, NAN)
    job = ctx.voxel_build_launch(p, vals=v, outside=o, tris=t, fill=fill, zix_xy=zix, tables=tables, capacity=cap)
    assert ctx.create_tiles_poll(wait=True)
    return (None if v is None else _np(v)), _np(o), _np(t), job.ntris, job.changed


def _count(ctx, p, tables, vals, fill, zix):
    """The triangle count from a counting job (no tris)."""
    job = ctx.voxel_build_launch(p, vals=None if vals is None else vals.copy(), fill=fill, zix_xy=zix, tables=tables)
    assert ctx.create_tiles_poll(wait=True)
    return job.ntris


def _check(beq, got, exp, extra=4):
    v, o, t, ntris, ch = got
    ev, eo, et, ech = exp
    if v is not None:
        assert beq(v, ev) == 0
    assert np.array_equal(o, eo)
    assert ntris == len(et) and ch == ech
    assert beq(t[:len(et)], et) == 0 and np.isnan(t[len(et):]).all() and len(t) == len(et) + extra


# ---- the golden cases and the random fields ----
def _golden_params(tw, a):
    p = tw.VoxelPostParams()
    p.nx, p.ny, p.nz = int(a[0]), int(a[1]), int(a[2])
    for d in range(3):
        p.lo_pos[d], p.vsz[d] = float(a[3 + d]), float(a[6 + d])
    p.isolevel, p.invert, p.make_closed_surface, p.remove_unconnected, p.keep_at_edge, p.centre_seed, p.skip_under_mesh = (
        float(a[9]), int(a[10]), int(a[11]), int(a[12]), int(a[13]), int(a[14]), int(a[15]))
    return p


@pytest.mark.parametrize("kind", ["host", "pinned", "device"])
@pytest.mark.parametrize("name", ["sine", "inv", "mesh"])
def test_golden(tw, ctx, beq, tables, name, kind):
    g = np.load(os.path.join(GOLD, "voxel_post.npz"))
    p = _golden_params(tw, g[name + "_params"])
    zix = g[name + "_zix"] if (name + "_zix") in g.files else None
    exp = (g[name + "_vals2"], g[name + "_outside2"], g[name + "_tris"], int((g[name + "_outside2"] != g[name + "_outside"]).sum()))
    _check(beq, _run(ctx, p, tables, vals=g[name + "_vals"], kind=kind, zix=zix), exp)


@pytest.mark.parametrize("dims,seed,kw", RANDOM_FIELDS)
def test_random_fields(tw, oracle, ctx, beq, tables, dims, seed, kw):
    """The four fields of test_voxel_post_vs_oracle_random_fields (17x19x23: n % 4 = 1), with their under-mesh heights."""
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    p = post_params(tw.VoxelPostParams, dims, **kw)
    exp = _expected(oracle, vals, p, zix, tables)
    assert exp[3] > 0
    for kind in ("host", "device"):
        _check(beq, _run(ctx, p, tables, vals=vals, kind=kind, zix=zix), exp)


# ---- the fill inside the job ----
def _scfg(scene, mode):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=2, mesh_seed=3, scene_size=(16.0, 16.0, 4.0), mesh_size=(128, 128, 64), zmax_est=1.0)


def _post_for(tw, vp, **kw):
    p = post_params(tw.VoxelPostParams, (vp.nx, vp.ny, vp.nz), **kw)
    for k in range(3):
        p.lo_pos[k], p.vsz[k] = vp.lo_pos[k], vp.vsz[k]
    return p


def test_fill_sine_512(tw, scene, oracle, ctx, beq, tables):
    """BASELINE config 4: the 512^3 sine grid filled, cleaned and meshed in one job; the fill against the oracle, remove_unconnected against the scipy
    reference, the triangles against the oracle."""
    vp = scene.voxel_landscape_params(_scfg(scene, 0), 512, 512, 512)
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    p = _post_for(tw, vp, remove_unconnected=3)
    field = oracle.voxel_fill(convert(vp, oracle.VoxelParams), nthreads=os.cpu_count() or 1)
    po = convert(p, oracle.VoxelPostParams)
    o = oracle.voxel_outside(field, po)
    v2, o2, ch = remove_unconnected_ref(field, o, po)
    del o
    t = oracle.voxel_triangles(v2, o2, po, tables)
    assert len(t) > 100000
    _check(beq, _run(ctx, p, tables, fill=vp), (v2, o2, t, ch))


@pytest.mark.parametrize("mesh", [0, 1])
@pytest.mark.parametrize("mode", [1, 2])
def test_fill_glm_256_terrain(tw, scene, oracle, ctx, beq, tables, mode, mesh):
    """GLM simplex / Perlin 256^3 terrain (z_gradient -2, isolevel -1, as test_post_chain), with and without under-mesh heights: the job's field equals the
    synchronous fill (its first 16 rows also the oracle's), every later stage equals the oracle's on that field."""
    import torch
    n = 256
    vp = scene.voxel_landscape_params(_scfg(scene, mode), n, n, n, z_gradient=-2.0)
    d = _buf("device", (n, n, n), np.float32, NAN)
    ctx.voxel_fill(vp, out=d)
    field = d.cpu().numpy()
    del d
    slab = convert(vp, type(vp))
    slab.ny = 16
    assert beq(field[:16], oracle.voxel_fill(convert(slab, oracle.VoxelParams))) == 0
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=3, centre_seed=int(not mesh), skip_under_mesh=mesh)
    zix = np.random.default_rng(mode * 2 + mesh).integers(n // 16, n // 4, (n, n)).astype(np.uint32) if mesh else None
    exp = _expected(oracle, field, p, zix, tables)
    assert exp[3] > 0
    _check(beq, _run(ctx, p, tables, fill=vp, zix=zix), exp)
    if mesh:   # device zix
        _check(beq, _run(ctx, p, tables, fill=vp, zix=torch.from_numpy(zix.astype(np.int32)).cuda(), kind="pinned"), exp)


@pytest.mark.parametrize("atten", [0, 1, 2, 3, 4, 5])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fill_small_every_attenuation(tw, scene, oracle, ctx, beq, tables, mode, atten):
    vp = scene.voxel_landscape_params(_scfg(scene, mode), 40, 24, 36)
    vp.nx, vp.ny, vp.nz = 31, 17, 45
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = atten, 0.7, 0.4
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    field = oracle.voxel_fill(convert(vp, oracle.VoxelParams))
    p = _post_for(tw, vp, remove_unconnected=3)
    exp = _expected(oracle, field, p, None, tables)
    _check(beq, _run(ctx, p, tables, fill=vp, kind="host"), exp)
    rdata = np.empty(420, np.float32)
    tw.lib.tw_noise3d_gen_sines(vp.rseed1, vp.rseed2, vp.mag, vp.freq, tw._ptr(rdata))
    if mode == 0:   # the coefficients given instead of generated
        job = ctx.voxel_build_launch(p, fill=vp, rdata=rdata, tables=tables)
        assert ctx.create_tiles_poll(wait=True) and job.ntris == len(exp[2]) and job.changed == exp[3]


def test_fill_triangles_only(tw, scene, oracle, ctx, beq, tables):
    """vals == NULL with a fill: only the triangles (and the flags) come out."""
    vp = scene.voxel_landscape_params(_scfg(scene, 1), 64, 48, 40, z_gradient=-2.0)
    field = oracle.voxel_fill(convert(vp, oracle.VoxelParams))
    p = _post_for(tw, vp, isolevel=-1.0, remove_unconnected=3)
    exp = _expected(oracle, field, p, None, tables)
    for kind in ("pinned", "device"):
        v, o, t, ntris, ch = _run(ctx, p, tables, fill=vp, kind=kind, want_vals=False)
        assert v is None
        _check(beq, (None, o, t, ntris, ch), exp)


# ---- options, the interior-holes bail-out, deep fills ----
@pytest.mark.parametrize("rm", [0, 1, 3])
@pytest.mark.parametrize("kae", [0, 1])
@pytest.mark.parametrize("mesh", [0, 1])
def test_options(tw, oracle, ctx, beq, tables, rm, kae, mesh):
    dims = (31, 27, 23)
    vals, zix = random_field(dims, 11, centre_seed=not mesh)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=rm, keep_at_edge=kae, centre_seed=int(not mesh), skip_under_mesh=mesh, isolevel=0.1,
                    make_closed_surface=int(not kae))
    exp = _expected(oracle, vals, p, zix, tables)
    assert (exp[3] > 0) == (rm > 0)
    _check(beq, _run(ctx, p, tables, vals=vals, kind="device", zix=zix), exp)


def test_interior_holes_without_a_top_seed(tw, oracle, ctx, beq, tables):
    """remove_unconnected 3 on a grid whose top plane is all inside: remove_interior_holes bails out, so the outside pockets stay."""
    dims = (30, 26, 22)
    vals, _ = random_field(dims, 5, True)
    vals[:, :, -1] = 5.0                                   # an inside top plane, joined to the centre seed by an inside column
    vals[dims[1] // 2, dims[0] // 2, dims[2] // 2:] = 5.0
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=3, make_closed_surface=0)
    exp = _expected(oracle, vals, p, None, tables)
    p1 = post_params(tw.VoxelPostParams, dims, remove_unconnected=1, make_closed_surface=0)
    exp1 = _expected(oracle, vals, p1, None, tables)
    assert np.array_equal(exp[1], exp1[1]) and exp[3] == exp1[3] and (exp[1] == 1).sum() > 0
    _check(beq, _run(ctx, p, tables, vals=vals, kind="host"), exp)
    v_r, o_r, ch_r = remove_unconnected_ref(vals, oracle.voxel_outside(vals, convert(p, oracle.VoxelPostParams)), p)
    assert np.array_equal(o_r, exp[1]) and beq(v_r, exp[0]) == 0 and ch_r == exp[3]


@pytest.mark.parametrize("nz", [16, 18, 20, 32, 34, 36, 40002])
def test_deep_fill_column(tw, ctx, beq, nz):
    """The one-voxel line that needs 7 ... 20000 generations: the fill reaches all of it, nothing changes."""
    vals, kw = column_case(nz)
    p = post_params(tw.VoxelPostParams, (3, 3, nz), **kw)
    outside = ctx.voxel_outside(vals, p)
    for kind in ("host", "device"):
        v, o, _, _, ch = _run(ctx, p, None, vals=vals, kind=kind, extra=0)
        assert ch == 0 and np.array_equal(o, outside) and beq(v, vals) == 0


@pytest.mark.parametrize("case", [serpentine_case, corridor_case])
def test_deep_fill_corridors(tw, ctx, beq, case):
    vals, kw, exp_o, exp_v = case()
    ny, nx, nz = vals.shape
    p = post_params(tw.VoxelPostParams, (nx, ny, nz), **kw)
    for kind in ("host", "device"):
        v, o, _, _, ch = _run(ctx, p, None, vals=vals, kind=kind, extra=0)
        assert np.array_equal(o, exp_o) and beq(v, exp_v) == 0 and ch == int((exp_o != (vals < 0)).sum())


# ---- triangle capacity ----
def _registered(shape):
    """A numpy buffer page-locked with cudaHostRegister (flags 0: mapped and portable on a UVA system); returns (array, unregister)."""
    import torch
    a = np.full(shape, NAN, np.float32)
    rt = torch.cuda.cudart()
    assert int(rt.cudaHostRegister(a.ctypes.data, a.nbytes, 0)) == 0
    return a, lambda: rt.cudaHostUnregister(a.ctypes.data)


def test_capacity(tw, oracle, ctx, beq, tables):
    """Capacity 0, 7, exactly ntris and larger, into device memory, torch's page-locked memory (cudaHostAlloc) and cudaHostRegister'ed memory: the first
    min(ntris, capacity) triangles are written, the NaN sentinels after them survive."""
    import torch
    dims, seed, kw = RANDOM_FIELDS[1]
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    p = post_params(tw.VoxelPostParams, dims, **kw)
    exp = _expected(oracle, vals, p, zix, tables)
    nt = len(exp[2])
    for cap in (0, 7, nt, nt + 5):
        for kind in ("device", "pinned", "registered"):
            undo = None
            if kind == "registered":
                t, undo = _registered((cap + 3, 3, 3))
            else:
                t = _buf(kind, (cap + 3, 3, 3), np.float32, NAN)
            try:
                job = ctx.voxel_build_launch(p, vals=vals.copy(), tris=t, zix_xy=zix, tables=tables, capacity=cap)
                assert ctx.create_tiles_poll(wait=True)
                got = _np(t)
                k = min(cap, nt)
                assert job.ntris == nt and job.changed == exp[3]
                assert beq(got[:k], exp[2][:k]) == 0 and np.isnan(got[k:]).all(), (cap, kind)
            finally:
                if undo:
                    undo()
    del torch


# ---- refusals ----
def test_refusals_change_nothing(tw, scene, ctx, beq, tables):
    """Each TW_ERR_ARG case of the header, and pageable tris: nothing is enqueued, no output and no host count changes."""
    import torch
    L = tw.lib
    dims = (12, 10, 9)
    vals, _ = random_field(dims, 3, True)
    p = post_params(tw.VoxelPostParams, dims, remove_unconnected=3)
    vp = scene.voxel_landscape_params(_scfg(scene, 1), *dims)
    e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
    dt = _buf("device", (16, 3, 3), np.float32, NAN)
    o = np.full((dims[1], dims[0], dims[2]), 0xAB, np.uint8)
    vin = vals.copy()
    ntris, changed = C.c_uint64(77), C.c_uint64(88)
    P = C.cast(C.pointer(p), C.c_void_p)

    def build(**kw):
        f = dict(fill=None, rdata420=None, post=P, zix_xy=None, edge_table256=tw._ptr(e), tri_table256x16=tw._ptr(t), edge_to_vals12x2=tw._ptr(v), vals=tw._ptr(vin),
                 outside=tw._ptr(o), tris=tw._ptr(dt), capacity=16, ntris=C.cast(C.pointer(ntris), C.c_void_p), changed=C.cast(C.pointer(changed), C.c_void_p))
        f.update(kw)
        return tw.VoxelBuild(**f)

    bad_vp = convert(vp, type(vp))
    bad_vp.nz = 8
    big_vp = convert(vp, type(vp))
    big_p = post_params(tw.VoxelPostParams, (70000, 3, 2))
    big_vp.nx, big_vp.ny, big_vp.nz = 70000, 3, 2                      # GLM fill wider than 65535
    mode_vp = convert(vp, type(vp))
    mode_vp.gen_mode = 9
    empty = post_params(tw.VoxelPostParams, (0, 3, 3))
    huge = post_params(tw.VoxelPostParams, (65536, 65536, 1))
    pageable = np.full((16, 3, 3), NAN, np.float32)
    cases = [build(post=None), build(post=C.cast(C.pointer(empty), C.c_void_p)), build(post=C.cast(C.pointer(huge), C.c_void_p)),
             build(fill=C.cast(C.pointer(bad_vp), C.c_void_p)), build(fill=C.cast(C.pointer(mode_vp), C.c_void_p)),
             build(fill=C.cast(C.pointer(big_vp), C.c_void_p), post=C.cast(C.pointer(big_p), C.c_void_p)), build(vals=None),
             build(tri_table256x16=None), build(edge_table256=None, edge_to_vals12x2=None), build(ntris=None), build(tris=None),
             build(tris=tw._ptr(pageable))]
    for b in cases:
        assert L.tw_voxel_build_launch(ctx._h, C.byref(b)) == tw.TW_ERR_ARG, L.tw_last_error(ctx._h)
        assert ctx.create_tiles_poll(wait=False)                       # nothing pending
    assert beq(vin, vals) == 0 and (o == 0xAB).all() and np.isnan(dt.cpu().numpy()).all() and np.isnan(pageable).all()
    assert ntris.value == 77 and changed.value == 88
    # TW_ERR_STATE where tw_voxel_fill returns it: a context without the sin table
    h = C.c_void_p()
    assert L.tw_create(0, C.byref(h)) == tw.TW_OK
    try:
        assert L.tw_voxel_build_launch(h, C.byref(build(fill=C.cast(C.pointer(vp), C.c_void_p)))) == tw.TW_ERR_STATE
        assert L.tw_voxel_fill(h, C.byref(vp), None, tw._ptr(np.empty((dims[1], dims[0], dims[2]), np.float32))) == tw.TW_ERR_STATE
    finally:
        L.tw_destroy(h)
    assert (o == 0xAB).all() and ntris.value == 77
    del torch


# ---- the job's place among the context's work ----
def _sine_512(tw, scene):
    vp = scene.voxel_landscape_params(_scfg(scene, 0), 512, 512, 512)
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    return vp, _post_for(tw, vp, remove_unconnected=3)


def test_poll_reports_not_ready_then_completes(tw, scene, ctx, beq, tables):
    """A warmed 512^3 build with device outputs: the launch returns before the device is done, poll(0) says so, poll(1) completes it with the same
    outputs as the first (warming) run."""
    import torch
    vp, p = _sine_512(tw, scene)
    v, o = _buf("device", (512, 512, 512), np.float32, NAN), _buf("device", (512, 512, 512), np.uint8, 0)
    first = ctx.voxel_build_launch(p, vals=v, outside=o, fill=vp, tables=tables)
    assert ctx.create_tiles_poll(wait=True)
    v0, o0 = v.clone(), o.clone()
    torch.cuda.synchronize()
    job = ctx.voxel_build_launch(p, vals=v, outside=o, fill=vp, tables=tables)
    assert not ctx.create_tiles_poll(wait=False)
    assert ctx.heightgen_2d_poll(wait=True)
    assert job.ntris == first.ntris > 0 and job.changed == first.changed
    assert torch.equal(o, o0) and beq(v.cpu().numpy(), v0.cpu().numpy()) == 0


def test_other_entry_point_completes_the_job(tw, oracle, ctx, beq, tables):
    dims, seed, kw = RANDOM_FIELDS[2]
    vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
    p = post_params(tw.VoxelPostParams, dims, **kw)
    exp = _expected(oracle, vals, p, zix, tables)
    v, o, t = _input("device", vals), _buf("pinned", (dims[1], dims[0], dims[2]), np.uint8, 0xAB), _buf("device", (len(exp[2]), 3, 3), np.float32, NAN)
    job = ctx.voxel_build_launch(p, vals=v, outside=o, tris=t, zix_xy=zix, tables=tables)
    small = post_params(tw.VoxelPostParams, (4, 4, 4))
    ctx.voxel_outside(np.ones((4, 4, 4), np.float32), small)          # completes the build first
    assert job.ntris == len(exp[2]) and job.changed == exp[3]
    assert beq(v.cpu().numpy(), exp[0]) == 0 and np.array_equal(o.numpy(), exp[1]) and beq(t.cpu().numpy(), exp[2]) == 0


def test_shared_context_beside_tile_jobs(tw, scene, oracle, beq, tables):
    """A build on a shared context while tile jobs run on the parent and on another shared context: every output equals the same job run alone, and the
    build also equals the oracle."""
    import torch
    from test_gpu_shared_ctx import _cfg as tile_cfg
    from test_gpu_tiles_shading import ITERS, ZV, _origins
    P = tw.Context(0)
    try:
        cfg = tile_cfg(scene, 0)
        P.set_sine_params(cfg.sine_params())
        hp, ep = cfg.height_params(), cfg.erosion_params()
        dx, dy = float(cfg.dx_val), float(cfg.dy_val)
        A, B = P.shared(), P.shared()
        origins = _origins(4)
        dims, seed, kw = RANDOM_FIELDS[2]
        vals, zix = random_field(dims, seed, kw.get("centre_seed", 1))
        p = post_params(tw.VoxelPostParams, dims, **kw)
        exp = _expected(oracle, vals, p, zix, tables)

        def tiles(c):
            z = torch.full((len(origins), ZV, ZV), NAN).pin_memory()
            mm = np.empty((len(origins), 2), np.float32)
            c.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, mm=mm)
            return z, mm

        def build(c):
            o, t = _buf("pinned", (dims[1], dims[0], dims[2]), np.uint8, 0xAB), _buf("device", (len(exp[2]), 3, 3), np.float32, NAN)
            v = _input("device", vals)
            return v, o, t, c.voxel_build_launch(p, vals=v, outside=o, tris=t, zix_xy=zix, tables=tables)

        zp, mp = tiles(P)
        zb, mb = tiles(B)
        v, o, t, job = build(A)
        for c in (A, P, B):
            assert c.create_tiles_poll(wait=True)
        alone = [tiles(P)]
        assert P.create_tiles_poll(wait=True)
        alone.append(tiles(B))
        assert B.create_tiles_poll(wait=True)
        v1, o1, t1, job1 = build(A)
        assert A.create_tiles_poll(wait=True)
        for (z, mm), (z1, mm1) in zip(((zp, mp), (zb, mb)), alone):
            assert beq(z.numpy(), z1.numpy()) == 0 and beq(mm, mm1) == 0
        assert job.ntris == job1.ntris == len(exp[2]) and job.changed == job1.changed == exp[3]
        assert torch.equal(o, o1) and np.array_equal(o.numpy(), exp[1])
        assert beq(v.cpu().numpy(), exp[0]) == 0 and beq(v1.cpu().numpy(), exp[0]) == 0
        assert beq(t.cpu().numpy(), exp[2]) == 0 and beq(t1.cpu().numpy(), exp[2]) == 0
    finally:
        P.close()
