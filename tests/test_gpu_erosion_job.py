"""GPU: tw_erode_launch - tw_erode / tw_erode_parallel of one map, or of the context's set_heightmap image between its unpack and its pack, as one
asynchronous job. Float maps are held bit for bit to tw_erode (on both sides of the M_SPEC threshold, and at 8192^2) and to the oracle, the OpenMP mode to
tw_erode (one thread) or to the properties of tw_erode_parallel's test (many), the image to the chain of synchronous calls and to the oracle's chain; then
poll(0), completion by other calls, shared contexts, the image rules and every refusal."""
import ctypes as C

import numpy as np
import pytest
import torch

from cases import convert, HM_CFG

pytestmark = pytest.mark.gpu
f32 = np.float32


def _cfg(scene, mode=4, zmax_est=2.3):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=zmax_est)


@pytest.fixture(scope="module")
def jctx(tw):
    c = tw.Context(0)
    yield c
    c.close()


_TERRAIN = {}


def _terrain(c, scene, n, mode=4):
    key = (n, mode)
    if key not in _TERRAIN:
        cfg = _cfg(scene, mode, 2.3 if mode == 4 else 2.0)
        _TERRAIN[key] = (cfg, c.heightgen_2d(cfg.heightmap_grid(n, n), cfg.height_params()))
    return _TERRAIN[key]


def _ready(*ts):
    """The library's context streams do not wait for torch's stream: inputs made by torch are complete before a launch reads them."""
    torch.cuda.synchronize()
    return ts[0] if len(ts) == 1 else ts


def _place(kind, a):
    if kind == "device":
        return _ready(torch.from_numpy(a.copy()).cuda())
    if kind == "pinned":
        return torch.from_numpy(a.copy()).pin_memory()
    return a.copy()


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


def _bits(a):
    return np.ascontiguousarray(_host(a), np.float32).view(np.uint32)


def _spec(n, iters):
    """twi_erode_spec_eligible for one map: M_SPEC takes maps of >= 2^20 padded cells (PAD = 4) with >= 64 droplets."""
    return (n + 8) ** 2 >= 1 << 20 and iters >= 64


# 1000^2 (1008^2 padded cells) takes the tile-style path, 1024^2 M_SPEC, 1024^2 with 63 droplets the tile-style path again
@pytest.mark.parametrize("kind", ["device", "pinned", "pageable"])
@pytest.mark.parametrize("n,iters,spec", [(1000, 2000, False), (1024, 2000, True), (1024, 63, False)])
def test_serial_matches_tw_erode_and_the_oracle(tw, scene, oracle, jctx, n, iters, spec, kind):
    assert _spec(n, iters) == spec
    cfg, z = _terrain(jctx, scene, n)
    zmin, ep = float(z.min()), cfg.erosion_params()
    ref = jctx.erode(z.copy(), zmin, iters, ep)
    steps = jctx.last_erosion_steps
    zo, so = oracle.apply_erosion(z, zmin, iters, convert(ep, oracle.ErosionParams))
    assert np.array_equal(_bits(ref), _bits(zo)) and steps == so > 0
    m = _place(kind, z)
    job = jctx.erode_launch(m, zmin, iters, ep)
    assert job.heightmap is m
    assert jctx.create_tiles_poll(True)
    assert np.array_equal(_bits(m), _bits(ref)) and jctx.last_erosion_steps == steps


@pytest.mark.parametrize("iters", [1000, 100000])
def test_8192_matches_tw_erode(tw, scene, jctx, iters):
    cfg, n = _cfg(scene), 8192
    ep = cfg.erosion_params()
    z = torch.empty((n, n), dtype=torch.float32, device="cuda")
    jctx.heightgen_2d(cfg.heightmap_grid(n, n), cfg.height_params(), out=z)
    zmin, _ = jctx.minmax(z)
    ref, m = _ready(z.clone(), z.clone())
    jctx.erode(ref, zmin, iters, ep)
    steps = jctx.last_erosion_steps
    jctx.erode_launch(m, zmin, iters, ep)
    assert jctx.create_tiles_poll(True)
    assert steps > 0 and jctx.last_erosion_steps == steps
    assert torch.equal(m.view(torch.int32), ref.view(torch.int32))


@pytest.mark.parametrize("n", [1000, 1024])
def test_openmp_one_thread_is_tw_erode(tw, scene, jctx, n):
    cfg, z = _terrain(jctx, scene, n)
    zmin, ep, iters = float(z.min()), cfg.erosion_params(), 2000
    ref = jctx.erode(z.copy(), zmin, iters, ep)
    steps = jctx.last_erosion_steps
    par = jctx.erode_parallel(z.copy(), zmin, iters, ep, num_threads=1)
    assert np.array_equal(_bits(par), _bits(ref)) and jctx.last_erosion_steps == steps
    for kind in ("device", "pageable"):
        m = _place(kind, z)
        jctx.erode_launch(m, zmin, iters, ep, num_threads=1)
        assert jctx.create_tiles_poll(True)
        assert np.array_equal(_bits(m), _bits(ref)) and jctx.last_erosion_steps == steps


@pytest.mark.parametrize("threads", [0, 7, 4096])
def test_openmp_many_threads_close_to_serial(tw, scene, oracle, jctx, threads):
    """The properties tests/test_gpu_erosion.py::test_erode_parallel_many_threads_close_to_serial holds tw_erode_parallel to, on the same terrain."""
    cfg, z = _terrain(jctx, scene, 2048, mode=1)
    zmin, zmax = float(z.min()), float(z.max())
    ep, iters = cfg.erosion_params(), 5000
    zc, steps = oracle.apply_erosion(z, zmin, iters, convert(ep, oracle.ErosionParams))
    m = _place("device", z)
    jctx.erode_launch(m, zmin, iters, ep, num_threads=threads)
    assert jctx.create_tiles_poll(True)
    zg = _host(m)
    assert np.isfinite(zg).all()
    assert abs(jctx.last_erosion_steps - steps) <= 0.1 * steps
    assert (zg != z).sum() > 0.9 * (zc != z).sum()
    same = (zg == zc).mean()
    moved_serial = np.abs(zc.astype(np.float64) - z).sum()
    moved_par = np.abs(zg.astype(np.float64) - z).sum()
    print("threads %d: identical cells %.4f, moved %.6g vs %.6g, steps %d vs %d (z range %.3g)" % (threads, same, moved_par, moved_serial, jctx.last_erosion_steps,
                                                                                                  steps, zmax - zmin))
    assert same > 0.5, same
    assert np.abs(zg - z).max() < 3.0 * np.abs(zc - z).max()
    assert abs(moved_par - moved_serial) < (0.3 if 0 < threads < 64 else 0.5) * moved_serial


# ---- the image
def _image(c, scene, n):
    """A generated 16-bit image and its heightmap_t scalars (proc_gen without erosion)."""
    cfg = _cfg(scene)
    img, info, _ = c.proc_gen_heightmap(n, n, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), 0, cfg.erosion_params())
    return cfg, img, info


def _chain(c, img, info, n, iters, ep, threads=None):
    """tw_heightmap_to_floats_u16 -> tw_minmax_f32 -> tw_erode (tw_erode_parallel) -> tw_heightmap_from_floats_u16."""
    vals = c.to_floats_u16(img, info.val_mult, info.val_add).reshape(n, n)
    zmin, _ = c.minmax(vals)
    if threads is None:
        c.erode(vals, zmin, iters, ep)
    else:
        c.erode_parallel(vals, zmin, iters, ep, num_threads=threads)
    steps = c.last_erosion_steps
    return vals, c.from_floats_u16(vals, info.val_mult, info.val_add), steps


def _sampler(tw, cfg, info, n):
    hp = cfg.height_params()
    return tw.HmapSampler(n, n, 2, 1.0, float(f32(0.0008) * f32(hp.mesh_height_scale)), info.mesh_file_scale, info.mesh_file_tz, hp.mesh_scale_z_inv)


def _origins(n, S=64):
    return [(x, y) for y in range(-n // 2, n // 2, S) for x in range(-n // 2, n // 2, S)]


def _image_tiles(c, cfg, hs, n, S=64):
    """Heightmap tiles over the whole of the context's image (tw_create_tiles_launch_hmap)."""
    origins, zv = _origins(n, S), S + 1
    z = np.full((len(origins), zv, zv), np.nan, np.float32)
    c.create_tiles_launch(origins, (S, S), float(cfg.dx_val), float(cfg.dy_val), zv, None, 0, None, 0.0, z, hmap=hs)
    assert c.create_tiles_poll(True)
    return z


def _sampled(c, img, hs, n, S=64):
    return c.heightmap_sample_tiles(img, hs, _origins(n, S), S + 1)


@pytest.mark.parametrize("threads", [None, 1])
@pytest.mark.parametrize("kind", ["device", "pinned", "pageable", None])
def test_image_matches_the_chain_and_the_oracle(tw, scene, oracle, kind, threads):
    n, iters = 1024, 3000
    c = tw.Context(0)
    try:
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        vals_ref, img_ref, steps = _chain(c, img, info, n, iters, ep, threads)
        vo = oracle.to_floats_u16(img, info.val_mult, info.val_add).reshape(n, n)
        vo, so = oracle.apply_erosion(vo, float(vo.min()), iters, convert(ep, oracle.ErosionParams))
        io, bad = oracle.from_floats_u16(vo, info.val_mult, info.val_add)
        assert bad == 0 and so == steps and np.array_equal(_bits(vo), _bits(vals_ref)) and np.array_equal(io, img_ref)
        hs = _sampler(tw, cfg, info, n)
        c.set_heightmap(img.reshape(n, n, 2))
        vals = None if kind is None else _place(kind, np.full(n * n + 64, np.nan, np.float32))
        job = c.erode_image_launch(info.val_mult, info.val_add, iters, ep, num_threads=threads, vals=None if vals is None else vals[:n * n])
        assert c.create_tiles_poll(True)
        assert c.last_erosion_steps == steps
        if vals is not None:
            hv = _host(vals)
            assert job.vals is not None and np.array_equal(hv[:n * n].view(np.uint32), _bits(vals_ref).ravel()) and np.all(np.isnan(hv[n * n:]))
        assert np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), _bits(_sampled(c, img_ref, hs, n)))
    finally:
        c.close()


def test_image_from_the_heightmap_job(tw, scene):
    """proc_gen_heightmap_launch(set_image) followed at once by this job (whose launch completes the heightmap job) equals the chain on proc_gen's image."""
    n, iters = 1024, 2000
    c = tw.Context(0)
    try:
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        vals_ref, img_ref, steps = _chain(c, img, info, n, iters, ep)
        hjob = c.proc_gen_heightmap_launch(n, n, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), 0, ep, set_image=True)
        vals = torch.empty((n, n), dtype=torch.float32, device="cuda")
        c.erode_image_launch(info.val_mult, info.val_add, iters, ep, vals=vals)
        assert c.create_tiles_poll(True)
        assert hjob.info.val_mult == info.val_mult and c.last_erosion_steps == steps
        assert torch.equal(vals.view(torch.int32).cpu(), torch.from_numpy(_bits(vals_ref).view(np.int32)))
        hs = _sampler(tw, cfg, info, n)
        assert np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), _bits(_sampled(c, img_ref, hs, n)))
    finally:
        c.close()


def test_no_work_keeps_the_image(tw, scene):
    n = 256
    c = tw.Context(0)
    try:
        cfg, img, info = _image(c, scene, n)
        hs = _sampler(tw, cfg, info, n)
        c.set_heightmap(img.reshape(n, n, 2))
        ref = _sampled(c, img, hs, n)
        vals = np.full(n * n, np.nan, np.float32)
        no_erosion = cfg.erosion_params()
        no_erosion.erode_amount = 0.0
        for iters, ep in ((0, cfg.erosion_params()), (100, no_erosion)):
            c.erode_image_launch(info.val_mult, info.val_add, iters, ep, vals=vals)
            assert c.create_tiles_poll(True) and c.last_erosion_steps == 0
            assert np.all(np.isnan(vals)) and np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), _bits(ref))
        z = _terrain(c, scene, 256)[1]
        m = z.copy()
        c.erode_launch(m, float(z.min()), 0, cfg.erosion_params())
        assert c.create_tiles_poll(True) and c.last_erosion_steps == 0 and np.array_equal(_bits(m), _bits(z))
    finally:
        c.close()


def test_pack_error_reported_by_the_poll(tw, scene):
    """An image whose scalars put the packed values above 256 (a val_add that swamps val_mult: the round trip through float loses the low bits): the
    completing poll returns TW_ERR_ARG with tw_heightmap_from_floats_u16's message, and the context is left without an image."""
    n = 256
    c = tw.Context(0)
    try:
        cfg = _cfg(scene)
        img = np.full(2 * n * n, 0xFF, np.uint8)
        mult, add = float(f32(4.6 * 2.0 ** -14 / 255.99)), 1000.0
        vals = c.to_floats_u16(img, mult, add)
        with pytest.raises(tw.TwError) as e:
            c.from_floats_u16(vals, mult, add)
        assert e.value.status == tw.TW_ERR_ARG
        c.set_heightmap(img.reshape(n, n, 2))
        c.erode_image_launch(mult, add, 100, cfg.erosion_params())
        with pytest.raises(tw.TwError) as e2:
            c.create_tiles_poll(True)
        assert e2.value.status == tw.TW_ERR_ARG and str(e2.value) == str(e.value)
        hs = tw.HmapSampler(n, n, 2, 1.0, 0.0008, 1.0, 0.0, 1.0)
        with pytest.raises(tw.TwError) as e3:
            _image_tiles(c, cfg, hs, n)
        assert e3.value.status == tw.TW_ERR_STATE
    finally:
        c.close()


def test_poll_zero_is_not_ready(tw, scene, jctx):
    cfg, n = _cfg(scene), 8192
    z = torch.empty((n, n), dtype=torch.float32, device="cuda")
    jctx.heightgen_2d(cfg.heightmap_grid(n, n), cfg.height_params(), out=z)
    zmin, _ = jctx.minmax(z)
    ep = cfg.erosion_params()
    m = _ready(z.clone())
    jctx.erode_launch(m, zmin, 100000, ep)                                               # warm-up: the graph and the scratch exist
    assert jctx.create_tiles_poll(True)
    ref, steps = m.clone(), jctx.last_erosion_steps
    _ready(m.copy_(z))
    jctx.erode_launch(m, zmin, 100000, ep)
    assert jctx.create_tiles_poll(False) is False
    assert jctx.create_tiles_poll(True)
    assert torch.equal(m, ref) and jctx.last_erosion_steps == steps


def test_completed_by_another_call_and_by_destroy(tw, scene):
    n, iters = 1024, 2000
    c = tw.Context(0)
    cfg, z = _terrain(c, scene, n)
    zmin, ep = float(z.min()), cfg.erosion_params()
    ref = c.erode(z.copy(), zmin, iters, ep)
    steps = c.last_erosion_steps
    m = _place("device", z)
    c.erode_launch(m, zmin, iters, ep)
    c.minmax(np.arange(16, dtype=np.float32))                                             # another entry point completes the job first
    assert np.array_equal(_bits(m), _bits(ref)) and c.last_erosion_steps == steps
    pinned = _place("pinned", z)
    c.erode_launch(pinned, zmin, iters, ep)
    c.close()                                                                             # tw_destroy completes it as a poll would
    assert np.array_equal(_bits(pinned), _bits(ref))


def test_shared_context_beside_a_tile_job(tw, scene):
    """A float-map job on one shared context and a tile job on another, in flight together, give what each gives alone."""
    cfg, n, iters = _cfg(scene), 2048, 20000
    hp, ep = cfg.height_params(), cfg.erosion_params()
    c = tw.Context(0)
    a, b = c.shared(), c.shared()
    try:
        S, zv = 128, 130
        origins = [(x * S, y * S) for y in range(-4, 4) for x in range(-4, 4)]

        def tiles():
            zt = np.empty((len(origins), zv, zv), np.float32)
            b.create_tiles_launch(origins, (S, S), float(cfg.dx_val), float(cfg.dy_val), zv, hp, 1000, ep, ep.zmin, zt)
            return zt
        z = c.heightgen_2d(cfg.heightmap_grid(n, n), hp)
        zmin = float(z.min())
        ref = a.erode(z.copy(), zmin, iters, ep)
        steps = a.last_erosion_steps
        z_ref = tiles()
        assert b.create_tiles_poll(True)
        m = _place("device", z)
        a.erode_launch(m, zmin, iters, ep)
        zt = tiles()
        assert b.create_tiles_poll(True) and a.create_tiles_poll(True)
        assert np.array_equal(zt.view(np.uint32), z_ref.view(np.uint32))
        assert np.array_equal(_bits(m), _bits(ref)) and a.last_erosion_steps == steps
    finally:
        c.close()


def test_image_rules_on_shared_contexts(tw, scene):
    """The image job is refused on a shared context; while the parent's runs, a shared context's heightmap tile launch gets TW_ERR_STATE and the parent's
    own completes the job first; after the poll both sample the eroded image."""
    n, iters = 1024, 3000
    c = tw.Context(0)
    s = c.shared()
    try:
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        _, img_ref, _ = _chain(c, img, info, n, iters, ep)
        hs = _sampler(tw, cfg, info, n)
        c.set_heightmap(img.reshape(n, n, 2))
        before = _image_tiles(s, cfg, hs, n)
        with pytest.raises(tw.TwError) as e:
            s.erode_image_launch(info.val_mult, info.val_add, iters, ep)
        assert e.value.status == tw.TW_ERR_ARG
        assert np.array_equal(_bits(_image_tiles(s, cfg, hs, n)), _bits(before))           # the refusal left the parent's image alone
        c.erode_image_launch(info.val_mult, info.val_add, iters, ep)
        with pytest.raises(tw.TwError) as e:
            _image_tiles(s, cfg, hs, n)
        assert e.value.status == tw.TW_ERR_STATE
        want = _bits(_sampled(c, img_ref, hs, n))
        c.set_heightmap(img.reshape(n, n, 2))                                                # completes the job; the original image again
        c.erode_image_launch(info.val_mult, info.val_add, iters, ep)
        assert np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), want)                      # completes the job first
        assert np.array_equal(_bits(_image_tiles(s, cfg, hs, n)), want)
    finally:
        c.close()


def test_refusals_change_nothing(tw, scene):
    n = 256
    L = tw.lib
    c = tw.Context(0)
    s = c.shared()
    fresh = tw.Context(0)                                                                   # sin table, no image
    raw = C.c_void_p()
    assert L.tw_create(0, C.byref(raw)) == tw.TW_OK                                         # no sin table
    try:
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        hs = _sampler(tw, cfg, info, n)
        c.set_heightmap(img.reshape(n, n, 2))
        img_tiles = _bits(_image_tiles(c, cfg, hs, n))
        z = _terrain(c, scene, n)[1]
        zmin = float(z.min())
        m = z.copy()
        vals = np.full(n * n, np.nan, np.float32)
        c.erode(z.copy(), zmin, 100, ep)
        steps = c.last_erosion_steps
        epp = C.cast(C.pointer(ep), C.c_void_p)
        mp, vp = C.c_void_p(m.ctypes.data), C.c_void_p(vals.ctypes.data)
        S, O = tw.TW_EROSION_SERIAL, tw.TW_EROSION_OPENMP
        J = tw.ErosionJobArgs
        cases = [
            (c, None, tw.TW_ERR_ARG),
            (c, J(mp, n, n, zmin, 0, 0, 100, None, S, 0, None), tw.TW_ERR_ARG),              # no ep
            (c, J(mp, 0, n, zmin, 0, 0, 100, epp, S, 0, None), tw.TW_ERR_ARG),               # empty map
            (c, J(mp, n, -1, zmin, 0, 0, 100, epp, S, 0, None), tw.TW_ERR_ARG),
            (c, J(mp, n, n, zmin, 0, 0, 100, epp, S, 0, vp), tw.TW_ERR_ARG),                 # vals with a float map
            (c, J(mp, n, n, zmin, 0, 0, 100, epp, 2, 0, None), tw.TW_ERR_ARG),               # bad mode
            (c, J(mp, n, n, zmin, 0, 0, 100, epp, -1, 0, None), tw.TW_ERR_ARG),
            (c, J(mp, n, n, zmin, 0, 0, 100, epp, S, 3, None), tw.TW_ERR_ARG),               # num_threads in the serial order
            (c, J(None, n, n, 0, info.val_mult, info.val_add, 100, epp, S, 0, vp), tw.TW_ERR_ARG),   # sizes with the image
            (c, J(None, n, 0, 0, info.val_mult, info.val_add, 100, epp, O, 0, vp), tw.TW_ERR_ARG),
            (s, J(None, 0, 0, 0, info.val_mult, info.val_add, 100, epp, S, 0, vp), tw.TW_ERR_ARG),   # the image on a shared context
            (fresh, J(None, 0, 0, 0, info.val_mult, info.val_add, 100, epp, S, 0, vp), tw.TW_ERR_STATE),  # no image
            (raw, J(mp, n, n, zmin, 0, 0, 100, epp, S, 0, None), tw.TW_ERR_STATE),           # no sin table
            (raw, J(mp, n, n, zmin, 0, 0, 100, epp, O, 0, None), tw.TW_ERR_STATE),
        ]
        for k, (cx, j, want) in enumerate(cases):
            handle = cx if isinstance(cx, C.c_void_p) else cx._h
            rc = L.tw_erode_launch(handle, C.byref(j) if j is not None else None)
            assert rc == want, (k, rc, L.tw_last_error(handle))
            assert L.tw_create_tiles_poll(handle, 0) == tw.TW_OK                           # nothing pending
            assert np.array_equal(_bits(m), _bits(z)) and np.all(np.isnan(vals)), k
        assert c.last_erosion_steps == steps
        assert np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), img_tiles)
        assert np.array_equal(_bits(_image_tiles(s, cfg, hs, n)), img_tiles)
    finally:
        L.tw_destroy(raw)
        fresh.close()
        c.close()
