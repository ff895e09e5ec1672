"""GPU: tw_voxel_build_batch_launch (Context.voxel_build_batch_launch) - many small voxel grids built in one job. Every grid of a batch is held bit for bit
to tw_voxel_build_launch_ex run alone on the same context with the same buffers (field, flags, welded vertices and indices up to the capacities, both
counts and the flipped voxels), which the other voxel suites hold to the oracle and the reference goldens. Covered: mixed shapes up to the 2^18-voxel
limit, every gen mode and attenuation, the remove_unconnected options, host and device input fields, a flood of thousands of generations, interior
holes without a top seed, capacities, batches of 1 / 7 / 300 grids, two batches on two shared contexts, the launch count and the refusals."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_voxel_build import _post_for, _scfg
from test_voxel_flood_reference import corridor_case, post_params, random_field, serpentine_case

pytestmark = pytest.mark.gpu
NAN = float("nan")
SENT = 0xDEADBEEF


@pytest.fixture(scope="module")
def tables():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_post.npz"))
    return g["edge_table"], g["tri_table"], g["edge_to_vals"]


def _mesh(nv, nt):
    import torch
    v = torch.full((nv, 3), NAN, dtype=torch.float32, device="cuda")
    i = torch.full((nt, 3), SENT - (1 << 32), dtype=torch.int32, device="cuda")
    return v, i


def _inputs(spec):
    """Fresh buffers for one run of a grid: its input field (host numpy or CUDA tensor, as the spec says) and its outputs."""
    import torch
    p = spec["vpp"]
    shape = (p.ny, p.nx, p.nz)
    g = {"vpp": p, "fill": spec.get("fill"), "zix_xy": spec.get("zix"), "rdata": spec.get("rdata")}
    if spec.get("vals") is not None:
        v = spec["vals"].copy()
        g["vals"] = torch.from_numpy(v).cuda() if spec.get("kind") == "device" else v
    else:
        g["vals"] = np.full(shape, NAN, np.float32)
    g["outside"] = np.full(shape, 0xEE, np.uint8)
    return g


def _counts(ctx, spec, tables):
    g = _inputs(spec)
    job = ctx.voxel_build_launch(g["vpp"], vals=g["vals"], outside=g["outside"], fill=g["fill"], rdata=g["rdata"], zix_xy=g["zix_xy"], tables=tables,
                                 mesh=(None, None), soup=False)
    assert ctx.create_tiles_poll(wait=True)
    return job.nverts, job.mesh_ntris


def _caps(ctx, spec, tables):
    """(vcap, tcap): the spec's, else the counts plus 3 spare rows."""
    if "cap" in spec:
        return spec["cap"]
    nv, nt = _counts(ctx, spec, tables)
    return nv + 3, nt + 3


def _result(g, mesh, nv, nt, ch):
    v = g["vals"]
    return (v if isinstance(v, np.ndarray) else v.cpu().numpy(), g["outside"], mesh[0].cpu().numpy(), mesh[1].cpu().numpy().view(np.uint32), nv, nt, ch)


def _single(ctx, spec, tables, caps):
    g = _inputs(spec)
    mesh = _mesh(*caps)
    job = ctx.voxel_build_launch(g["vpp"], vals=g["vals"], outside=g["outside"], fill=g["fill"], rdata=g["rdata"], zix_xy=g["zix_xy"], tables=tables,
                                 mesh=mesh, soup=False)
    assert ctx.create_tiles_poll(wait=True)
    return _result(g, mesh, job.nverts, job.mesh_ntris, job.changed)


def _batch(ctx, specs, tables, caps, poll=True):
    gs = [_inputs(s) for s in specs]
    meshes = [_mesh(*c) for c in caps]
    for g, m in zip(gs, meshes):
        g["mesh"] = m
    job = ctx.voxel_build_batch_launch(gs, tables)
    if not poll:
        return gs, meshes, job
    assert ctx.create_tiles_poll(wait=True)
    return [_result(g, m, job.nverts[i], job.ntris[i], job.changed[i]) for i, (g, m) in enumerate(zip(gs, meshes))]


def _same(got, exp):
    for k, (a, b) in enumerate(zip(got, exp)):
        if isinstance(a, np.ndarray):
            assert a.shape == b.shape, k
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k   # bit for bit, NaN sentinels included
        else:
            assert a == b, k


def _check_batch(ctx, specs, tables):
    caps = [_caps(ctx, s, tables) for s in specs]
    exp = [_single(ctx, s, tables, c) for s, c in zip(specs, caps)]
    got = _batch(ctx, specs, tables, caps)
    for i, (g, e) in enumerate(zip(got, exp)):
        try:
            _same(g, e)
        except AssertionError as err:
            raise AssertionError("grid %d (%s): output %s differs" % (i, tuple(specs[i]["vpp"].__getattribute__(a) for a in ("nx", "ny", "nz")), err))
    return got


def _fill_spec(tw, scene, mode, dims, atten=3, **kw):
    nx, ny, nz = dims
    vp = scene.voxel_landscape_params(_scfg(scene, mode), max(nx, 2), max(ny, 2), max(nz, 2))
    vp.nx, vp.ny, vp.nz = nx, ny, nz
    vp.atten_mode, vp.atten_val, vp.atten_inner_radius = atten, 0.7, 0.4
    vp.offset[0], vp.offset[1] = 0.5, -0.25
    kw.setdefault("remove_unconnected", 3)
    kw.setdefault("centre_seed", 1)
    return {"vpp": _post_for(tw, vp, **kw), "fill": vp}


def _field_spec(tw, dims, seed, kind="host", zix=False, **kw):
    cs = kw.get("centre_seed", 0)
    vals, z = random_field(dims, seed, cs)
    p = post_params(tw.VoxelPostParams, dims, **kw)
    return {"vpp": p, "vals": vals, "kind": kind, "zix": z if zix else None}


def test_mixed_shapes(tw, scene, ctx, tables):
    """2x2x2, odd sizes, nz not a multiple of 32, the 2^18-voxel shapes 8x8x4096, 512x512x1 and 64^3, in one batch with every gen mode."""
    shapes = [(2, 2, 2), (5, 7, 9), (3, 4, 37), (17, 9, 70), (8, 8, 4096), (512, 512, 1), (64, 64, 64), (33, 31, 65)]
    specs = [_fill_spec(tw, scene, k % 3, s) for k, s in enumerate(shapes)]
    got = _check_batch(ctx, specs, tables)
    assert sum(g[5] for g in got) > 1000


def test_every_gen_mode_and_attenuation(tw, scene, ctx, tables):
    specs = [_fill_spec(tw, scene, mode, (31, 17, 45), atten=atten, centre_seed=int(atten >= 3)) for mode in (0, 1, 2) for atten in range(6)]
    rdata = np.empty(420, np.float32)
    vp = specs[0]["fill"]
    tw.lib.tw_noise3d_gen_sines(vp.rseed1, vp.rseed2, vp.mag, vp.freq, tw._ptr(rdata))
    specs.append(dict(specs[0], rdata=rdata))   # the coefficients given instead of generated
    got = _check_batch(ctx, specs, tables)
    assert any(g[6] > 0 for g in got)


def test_options_and_input_fields(tw, ctx, tables):
    """remove_unconnected 0 / 1 / 3, centre_seed, keep_at_edge, skip_under_mesh with zix_xy, invert, make_closed_surface; host and device input fields."""
    specs, seed = [], 0
    for rm in (0, 1, 3):
        for cs, kae, mesh in ((1, 0, 0), (0, 1, 1), (0, 0, 1), (1, 1, 0)):
            for inv, mcs in ((0, 0), (1, 1)):
                seed += 1
                specs.append(_field_spec(tw, (13 + seed % 5, 11, 19 + seed % 7), seed, kind=("device" if seed % 2 else "host"), zix=bool(mesh),
                                         remove_unconnected=rm, centre_seed=cs, keep_at_edge=kae, skip_under_mesh=mesh, invert=inv, make_closed_surface=mcs))
    got = _check_batch(ctx, specs, tables)
    assert sum(g[6] for g in got) > 0


def test_deep_floods(tw, ctx, tables):
    """A serpentine corridor (pass 0) and an outside corridor from the top plane (pass 1) whose floods take thousands of generations, beside a small grid."""
    specs = []
    for case in (serpentine_case, corridor_case):
        vals, kw, exp_o, exp_v = case()
        ny, nx, nz = vals.shape
        specs.append({"vpp": post_params(tw.VoxelPostParams, (nx, ny, nz), **kw), "vals": vals, "kind": "device", "exp": (exp_o, exp_v)})
    specs.append(_field_spec(tw, (6, 5, 7), 99, remove_unconnected=3, centre_seed=1))
    got = _check_batch(ctx, specs, tables)
    for s, g in zip(specs[:2], got[:2]):
        assert np.array_equal(g[1], s["exp"][0]) and np.array_equal(g[0].view(np.uint32), s["exp"][1].view(np.uint32))


def test_interior_holes_without_a_top_seed(tw, ctx, tables):
    """remove_unconnected 3 where the top plane holds no outside voxel: pass 1 seeds nothing, so the enclosed outside pocket stays."""
    vals = np.full((12, 12, 12), 1.0, np.float32)    # inside everywhere (val > isolevel 0)...
    vals[2:5, 2:5, 2:5] = -1.0                        # ...around an outside pocket away from the centre seed
    p = post_params(tw.VoxelPostParams, (12, 12, 12), isolevel=0.0, make_closed_surface=0, remove_unconnected=3, centre_seed=1)
    spec = {"vpp": p, "vals": vals, "kind": "host"}
    got = _check_batch(ctx, [spec, dict(spec, kind="device")], tables)
    assert (got[0][1][2:5, 2:5, 2:5] == 1).all() and got[0][6] == 0


def test_capacities(tw, scene, ctx, tables):
    """Capacities below the counts, zero and exact: counts complete, nothing written past a capacity."""
    base = _fill_spec(tw, scene, 1, (24, 20, 28))
    nv, nt = _counts(ctx, base, tables)
    assert nv > 10 and nt > 10
    specs = [dict(base, cap=c) for c in ((nv // 2, nt // 3), (0, 0), (nv, nt), (0, nt), (nv, 0))]
    got = _check_batch(ctx, specs, tables)
    for g in got:
        assert g[4] == nv and g[5] == nt


@pytest.mark.parametrize("n", [1, 7, 300])
def test_batch_sizes(tw, scene, ctx, tables, n):
    specs = []
    for k in range(n):
        if k % 3 == 2:
            specs.append(_fill_spec(tw, scene, k % 3, (9 + k % 4, 10, 11 + k % 9), atten=k % 6))
        else:
            specs.append(_field_spec(tw, (8 + k % 5, 7 + k % 3, 9 + k % 11), k, kind="device" if k % 2 else "host", remove_unconnected=(0, 1, 3)[k % 3],
                                     centre_seed=1))
    _check_batch(ctx, specs, tables)


def test_two_batches_on_two_shared_contexts(tw, scene, ctx, tables):
    import torch
    P = tw.Context(0)
    try:
        A, B = P.shared(), P.shared()
        sa = [_fill_spec(tw, scene, k % 3, (20 + k, 18, 22)) for k in range(5)]
        sb = [_field_spec(tw, (15, 16 + k, 17), 40 + k, remove_unconnected=3, centre_seed=1) for k in range(6)]
        ca, cb = [_caps(A, s, tables) for s in sa], [_caps(B, s, tables) for s in sb]
        ea, eb = [_single(A, s, tables, c) for s, c in zip(sa, ca)], [_single(B, s, tables, c) for s, c in zip(sb, cb)]
        ra, rb = _batch(A, sa, tables, ca, poll=False), _batch(B, sb, tables, cb, poll=False)   # both in flight
        for ctx_, (gs, ms, job), exp in ((A, ra, ea), (B, rb, eb)):
            assert ctx_.create_tiles_poll(wait=True)
            for i, (g, m) in enumerate(zip(gs, ms)):
                _same(_result(g, m, job.nverts[i], job.ntris[i], job.changed[i]), exp[i])
        torch.cuda.synchronize()
    finally:
        P.close()


def test_launch_count_does_not_grow_with_the_batch(tw, scene, ctx, tables):
    """One option mix - a sine grid, a GLM grid and an input field, every third grid each - launches the same kernels for 3 grids as for 300."""
    def mix(n):
        return [_fill_spec(tw, scene, k % 3, (10, 9, 12)) if k % 3 < 2 else _field_spec(tw, (10, 9, 12), k, remove_unconnected=3, centre_seed=1)
                for k in range(n)]
    counts = []
    for n in (3, 300, 3, 300):   # the first two warm up the context's tables
        before = tw.lib.tw_launch_count(ctx._h)
        _batch(ctx, mix(n), tables, [(50, 50)] * n)
        counts.append(tw.lib.tw_launch_count(ctx._h) - before)
    assert counts[2] == counts[3] == 6


def test_cancel_changes_nothing(tw, scene, ctx, tables):
    specs = [_fill_spec(tw, scene, k % 3, (30, 28, 26)) for k in range(4)]
    caps = [_caps(ctx, s, tables) for s in specs]
    exp = [_single(ctx, s, tables, c) for s, c in zip(specs, caps)]
    gs, ms, job = _batch(ctx, specs, tables, caps, poll=False)
    ctx.cancel()
    assert ctx.create_tiles_poll(wait=True)
    for i, (g, m) in enumerate(zip(gs, ms)):
        _same(_result(g, m, job.nverts[i], job.ntris[i], job.changed[i]), exp[i])


def test_refusals_enqueue_nothing(tw, ctx, tables):
    """An oversized grid, tables that differ, soup fields set and pageable mesh buffers: TW_ERR_ARG naming the grid, nothing launched, no job pending."""
    import torch
    ok = _field_spec(tw, (8, 8, 8), 1, remove_unconnected=1, centre_seed=1)
    big = _field_spec(tw, (65, 64, 64), 2)
    tabs = tuple(np.ascontiguousarray(t, dt) for t, dt in zip(tables, (np.uint32, np.int32, np.uint32)))
    other = tuple(t.copy() for t in tabs)
    cnt = C.c_uint64(0)
    vbuf, ibuf = torch.zeros((10, 3), device="cuda"), torch.zeros((10, 3), dtype=torch.int32, device="cuda")
    pageable = np.zeros((10, 3), np.float32)
    keep = []

    def build(specs, tabsets, soup=(), verts=None):
        bs, ms = (tw.VoxelBuild * len(specs))(), (tw.VoxelMesh * len(specs))()
        for i, (s, t) in enumerate(zip(specs, tabsets)):
            v = s["vals"].copy()
            keep.append(v)
            bs[i] = tw.VoxelBuild(None, None, C.cast(C.pointer(s["vpp"]), C.c_void_p), None, tw._ptr(t[0]), tw._ptr(t[1]), tw._ptr(t[2]), tw._ptr(v), None,
                                  None, 0, C.cast(C.pointer(cnt), C.c_void_p) if i in soup else None, None)
            vv = verts if (verts is not None and i == 1) else vbuf
            ms[i] = tw.VoxelMesh(tw._ptr(vv), 10, tw._ptr(ibuf), 10, C.cast(C.pointer(cnt), C.c_void_p), C.cast(C.pointer(cnt), C.c_void_p))
        return bs, ms

    cases = [build([ok, big], [tabs, tabs]), build([ok, ok], [tabs, other]), build([ok, ok], [tabs, tabs], soup=(1,)),
             build([ok, ok], [tabs, tabs], verts=pageable)]
    ctx.create_tiles_poll(wait=True)
    before = tw.lib.tw_launch_count(ctx._h)
    for bs, ms in cases:
        assert tw.lib.tw_voxel_build_batch_launch(ctx._h, bs, ms, 2) == tw.TW_ERR_ARG
        assert b"grid 1" in tw.lib.tw_last_error(ctx._h)
    bs, ms = cases[0]
    assert tw.lib.tw_voxel_build_batch_launch(ctx._h, bs, ms, 0) == tw.TW_ERR_ARG
    assert tw.lib.tw_voxel_build_batch_launch(ctx._h, None, ms, 1) == tw.TW_ERR_ARG
    assert tw.lib.tw_launch_count(ctx._h) == before and cnt.value == 0
