"""GPU: tw_proc_gen_heightmap_launch - heightmap_t::proc_gen as one asynchronous job. Its outputs after the completing poll are held to the oracle's
restatement of proc_gen (every gen mode, no erosion, the tile-style erosion path and the speculative M_SPEC path) and, at 8192^2, to the composition of the
independent synchronous calls; then the output placements, set_image, poll(0), completion by other calls, shared contexts and every refusal."""
import ctypes as C

import numpy as np
import pytest
import torch

from cases import convert, HM_CFG

pytestmark = pytest.mark.gpu
f32 = np.float32


def _cfg(scene, mode):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)


@pytest.fixture(scope="module")
def jctx(tw, scene):
    c = tw.Context(0)
    c.set_sine_params(_cfg(scene, 0).sine_params())
    yield c
    c.close()


def _launch(c, cfg, w, h, iters, **kw):
    return c.proc_gen_heightmap_launch(w, h, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), iters, cfg.erosion_params(), **kw)


def _info(i):
    return (i.min_z, i.max_z, i.val_mult, i.val_add, i.mesh_file_scale, i.mesh_file_tz, i.erosion_moves)


def _scalars(min_z, max_z, hp):
    """set_mesh_height_scales_for_zval_range + get_mh_texture_mult/add as tw_proc_gen_heightmap's host code computes them (src/mesh_gen.cpp:124-131)."""
    min_z, max_z = f32(min_z), f32(max_z)
    dz = max(f32(1.0E-12), f32(max_z - min_z))
    dz255 = f32(float(dz) / 255.0)
    mhs, mszi, R = f32(hp.mesh_height_scale), f32(hp.mesh_scale_z_inv), f32(0.0008)
    mfs = f32(dz255 / f32(f32(R * mhs) * mszi))
    mtz = f32(min_z / mszi)
    return float(f32(f32(f32(R * mhs) * mfs) * mszi)), float(f32(mtz * mszi)), float(mfs), float(mtz)


_HEIGHTS = {}


def _oracle(oracle, cfg, w, h, iters):
    """heightmap_t::proc_gen restated from the oracle pieces, as test_gpu_callers._oracle_proc_gen does (the generated grid cached per mode and size)."""
    hp = cfg.height_params()
    key = (cfg.mesh_gen_mode, w, h)
    if key not in _HEIGHTS:
        sp = cfg.sine_params() if cfg.mesh_gen_mode == 0 else None
        _HEIGHTS[key] = oracle.heightgen_2d(oracle.Grid2D(-0.5 * w, -0.5 * h, float(cfg.dx_val), float(cfg.dy_val), w, h), convert(hp, oracle.HeightParams), sp, 1, 0)
    vals, moves = _HEIGHTS[key].copy(), 0
    if iters:
        vals, moves = oracle.apply_erosion(vals, float(vals.min()), iters, convert(cfg.erosion_params(), oracle.ErosionParams))
    mult, add, mfs, mtz = _scalars(vals.min(), vals.max(), hp)
    img, bad = oracle.from_floats_u16(vals, mult, add)
    assert bad == 0
    return img, vals, (float(vals.min()), float(vals.max()), mult, add, mfs, mtz, moves)


# no erosion; the tile-style path (< 2^20 padded cells); M_SPEC at 1024^2 with one window (64), one droplet more (65) and many rounds (2000)
@pytest.mark.parametrize("iters,w,h", [(0, 320, 200), (800, 256, 256), (64, 1024, 1024), (65, 1024, 1024), (2000, 1024, 1024)])
@pytest.mark.parametrize("mode", [0, 1, 2, 4])
def test_matches_oracle(tw, scene, oracle, jctx, beq, mode, iters, w, h):
    cfg = _cfg(scene, mode)
    img_o, vals_o, info_o = _oracle(oracle, cfg, w, h, iters)
    vals = torch.empty((h, w), dtype=torch.float32, device="cuda")
    img = torch.empty(2 * w * h, dtype=torch.uint8, device="cuda")
    job = _launch(jctx, cfg, w, h, iters, data16=img, vals=vals)
    assert jctx.create_tiles_poll(True)
    assert beq(vals.cpu().numpy(), vals_o) == 0
    assert np.array_equal(img.cpu().numpy(), img_o)
    assert _info(job.info) == info_o
    assert jctx.last_erosion_steps == info_o[-1]


@pytest.mark.parametrize("iters", [1000, 100000])
def test_8192_matches_the_synchronous_calls(tw, scene, jctx, iters):
    """tw_heightgen_2d -> tw_erode -> tw_minmax_f32 -> tw_heightmap_from_floats_u16 on device tensors, with the scalars of tw_proc_gen_heightmap's host code."""
    cfg, n = _cfg(scene, 4), 8192
    hp, ep = cfg.height_params(), cfg.erosion_params()
    ref = torch.empty((n, n), dtype=torch.float32, device="cuda")
    jctx.heightgen_2d(tw.Grid2D(-0.5 * n, -0.5 * n, float(cfg.dx_val), float(cfg.dy_val), n, n), hp, out=ref)
    zmin, _ = jctx.minmax(ref)
    jctx.erode(ref, zmin, iters, ep)
    moves = jctx.last_erosion_steps
    mn, mx = jctx.minmax(ref)
    mult, add, mfs, mtz = _scalars(mn, mx, hp)
    ref_img = torch.empty(2 * n * n, dtype=torch.uint8, device="cuda")
    jctx.from_floats_u16(ref, mult, add, out=ref_img)
    vals = torch.empty_like(ref)
    img = torch.empty_like(ref_img)
    job = _launch(jctx, cfg, n, n, iters, data16=img, vals=vals)
    assert jctx.create_tiles_poll(True)
    assert moves > 0 and _info(job.info) == (mn, mx, mult, add, mfs, mtz, moves)
    assert jctx.last_erosion_steps == moves
    assert torch.equal(vals.view(torch.int32), ref.view(torch.int32))
    assert torch.equal(img, ref_img)


def _alloc(kind, n, dtype, fill):
    if kind == "device":
        return torch.full((n,), fill, dtype=dtype, device="cuda")
    if kind == "pinned":
        return torch.full((n,), fill, dtype=dtype).pin_memory()
    return np.full(n, fill, {torch.float32: np.float32, torch.uint8: np.uint8}[dtype])


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


@pytest.mark.parametrize("kind", ["device", "pinned", "pageable"])
def test_output_placements(tw, scene, jctx, kind):
    """data16 and vals on the device, in page-locked and in pageable host memory, and vals absent: each equals the synchronous call, and the 64 elements
    after each output (NaN / 0xEE sentinels) stay untouched."""
    cfg, w, h, iters = _cfg(scene, 1), 300, 200, 700
    img_s, info_s, vals_s = jctx.proc_gen_heightmap(w, h, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), iters, cfg.erosion_params(), vals=np.empty((h, w), f32))
    for with_vals in (True, False):
        img = _alloc(kind, 2 * w * h + 64, torch.uint8, 0xEE)
        vals = _alloc(kind, w * h + 64, torch.float32, float("nan")) if with_vals else None
        job = _launch(jctx, cfg, w, h, iters, data16=img[:2 * w * h], vals=vals[:w * h] if with_vals else None)
        assert jctx.create_tiles_poll(True)
        hi = _host(img)
        assert np.array_equal(hi[:2 * w * h], img_s) and np.all(hi[2 * w * h:] == 0xEE)
        if with_vals:
            hv = _host(vals)
            assert np.array_equal(hv[:w * h].view(np.uint32), vals_s.ravel().view(np.uint32)) and np.all(np.isnan(hv[w * h:]))
        assert _info(job.info) == _info(info_s)


def _hmap_tiles(tw, c, cfg, hs, origins, zv, S):
    z = np.full((len(origins), zv, zv), np.nan, np.float32)
    c.create_tiles_launch(origins, (S, S), float(cfg.dx_val), float(cfg.dy_val), zv, None, 0, None, 0.0, z, hmap=hs)
    assert c.create_tiles_poll(True)
    return z


def test_set_image(tw, scene):
    """After the poll, heightmap tiles on the parent and on a shared context equal those of the tw_set_heightmap(data16) route; between launch and poll a
    shared context has no image and the parent's own hmap launch completes the job first; set_image on a shared context is refused."""
    cfg, w, h, iters, S, zv = _cfg(scene, 1), 257, 300, 400, 64, 65
    hp = cfg.height_params()
    c = tw.Context(0)
    s = c.shared()
    try:
        img_s, info_s, _ = c.proc_gen_heightmap(w, h, float(cfg.dx_val), float(cfg.dy_val), hp, iters, cfg.erosion_params())
        hs = tw.HmapSampler(w, h, 2, 1.0, float(f32(0.0008) * f32(hp.mesh_height_scale)), info_s.mesh_file_scale, info_s.mesh_file_tz, hp.mesh_scale_z_inv)
        origins = [(-200, -150), (0, 0), (64, -64), (130, 100)]
        c.set_heightmap(img_s.reshape(h, w, 2))
        z_ref = _hmap_tiles(tw, c, cfg, hs, origins, zv, S)
        with pytest.raises(tw.TwError) as e:
            _launch(s, cfg, w, h, iters, set_image=True)
        assert e.value.status == tw.TW_ERR_ARG
        assert np.array_equal(_hmap_tiles(tw, s, cfg, hs, origins, zv, S), z_ref)      # the refusal left the parent's image alone
        for data16 in (None, torch.empty(2 * w * h, dtype=torch.uint8, device="cuda")):
            job = _launch(c, cfg, w, h, iters, data16=data16, set_image=True)
            with pytest.raises(tw.TwError) as e:                                          # no image until the job completes
                _hmap_tiles(tw, s, cfg, hs, origins, zv, S)
            assert e.value.status == tw.TW_ERR_STATE
            assert np.array_equal(_hmap_tiles(tw, c, cfg, hs, origins, zv, S), z_ref)   # completes the job first, then samples the new image
            assert _info(job.info) == _info(info_s)
            assert np.array_equal(_hmap_tiles(tw, s, cfg, hs, origins, zv, S), z_ref)
            if data16 is not None:
                assert np.array_equal(data16.cpu().numpy(), img_s)
    finally:
        c.close()


def test_poll_zero_is_not_ready(tw, scene, jctx):
    cfg, n = _cfg(scene, 4), 8192
    img = torch.empty(2 * n * n, dtype=torch.uint8, device="cuda")
    _launch(jctx, cfg, n, n, 100000, data16=img)                                           # warm-up: the graph and the scratch exist
    assert jctx.create_tiles_poll(True)
    ref = img.clone()
    job = _launch(jctx, cfg, n, n, 100000, data16=img)
    assert jctx.create_tiles_poll(False) is False
    assert jctx.create_tiles_poll(True)
    assert torch.equal(img, ref) and job.info.erosion_moves > 0


def test_completed_by_another_call_and_by_destroy(tw, scene):
    cfg, w, h, iters = _cfg(scene, 4), 1024, 1024, 2000
    c = tw.Context(0)
    img_s, info_s, _ = c.proc_gen_heightmap(w, h, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), iters, cfg.erosion_params())
    img = torch.empty(2 * w * h, dtype=torch.uint8, device="cuda")
    job = _launch(c, cfg, w, h, iters, data16=img)
    c.minmax(np.arange(16, dtype=np.float32))                                              # another entry point completes the job first
    assert np.array_equal(img.cpu().numpy(), img_s) and _info(job.info) == _info(info_s)
    assert c.last_erosion_steps == info_s.erosion_moves
    pinned = torch.empty(2 * w * h, dtype=torch.uint8).pin_memory()
    job = _launch(c, cfg, w, h, iters, data16=pinned)
    c.close()                                                                              # tw_destroy completes it as a poll would
    assert np.array_equal(pinned.numpy(), img_s) and _info(job.info) == _info(info_s)


def test_shared_context_beside_a_tile_job(tw, scene):
    """A heightmap job on one shared context and a tile job on another, in flight together, give what each gives alone."""
    cfg, w, h, iters = _cfg(scene, 4), 2048, 2048, 20000
    hp, ep = cfg.height_params(), cfg.erosion_params()
    c = tw.Context(0)
    a, b = c.shared(), c.shared()
    try:
        S, zv = 128, 130
        origins = [(x * S, y * S) for y in range(-4, 4) for x in range(-4, 4)]

        def tiles():
            z = np.empty((len(origins), zv, zv), np.float32)
            b.create_tiles_launch(origins, (S, S), float(cfg.dx_val), float(cfg.dy_val), zv, hp, 1000, ep, ep.zmin, z)
            return z
        img_s, info_s, vals_s = a.proc_gen_heightmap(w, h, float(cfg.dx_val), float(cfg.dy_val), hp, iters, ep, vals=np.empty((h, w), f32))
        z_ref = tiles()
        assert b.create_tiles_poll(True)
        img = torch.empty(2 * w * h, dtype=torch.uint8, device="cuda")
        vals = torch.empty((h, w), dtype=torch.float32, device="cuda")
        job = _launch(a, cfg, w, h, iters, data16=img, vals=vals)
        z = tiles()
        assert b.create_tiles_poll(True) and a.create_tiles_poll(True)
        assert np.array_equal(z.view(np.uint32), z_ref.view(np.uint32))
        assert np.array_equal(img.cpu().numpy(), img_s) and np.array_equal(vals.cpu().numpy().view(np.uint32), vals_s.view(np.uint32))
        assert _info(job.info) == _info(info_s) and a.last_erosion_steps == info_s.erosion_moves
    finally:
        c.close()


def test_refusals_change_nothing(tw, scene):
    cfg, w, h = _cfg(scene, 1), 64, 48
    hp, ep = cfg.height_params(), cfg.erosion_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    L = tw.lib
    c = tw.Context(0)
    s = c.shared()
    raw = C.c_void_p()
    assert L.tw_create(0, C.byref(raw)) == tw.TW_OK                                        # no sin table
    try:
        c.proc_gen_heightmap(w, h, dx, dy, hp, 100, ep)
        steps = c.last_erosion_steps
        img = np.full(2 * w * h, 0xEE, np.uint8)
        vals = np.full((h, w), np.nan, np.float32)
        info = tw.HeightmapInfo(-1, -1, -1, -1, -1, -1, 7)

        def out(data16=True, set_image=0):
            return C.byref(tw.HeightmapOutputs(img.ctypes.data if data16 else None, vals.ctypes.data, C.cast(C.pointer(info), C.c_void_p), set_image))
        bad_mode, bad_start, sine = cfg.height_params(), cfg.height_params(), _cfg(scene, 0).height_params()
        bad_mode.gen_mode, bad_start.start_eval_sin = 7, 100000
        cases = [(c, w, h, hp, out(), tw.TW_ERR_ARG) for hp in (None,)] + [
            (c, w, h, cfg.height_params(), None, tw.TW_ERR_ARG),
            (c, 0, h, cfg.height_params(), out(), tw.TW_ERR_ARG),
            (c, w, 0, cfg.height_params(), out(), tw.TW_ERR_ARG),
            (c, w, h, cfg.height_params(), out(data16=False), tw.TW_ERR_ARG),
            (s, w, h, cfg.height_params(), out(set_image=1), tw.TW_ERR_ARG),
            (c, w, h, bad_mode, out(), tw.TW_ERR_ARG),
            (c, w, h, bad_start, out(), tw.TW_ERR_ARG),
            (c, w, h, sine, out(), tw.TW_ERR_STATE),                                          # sine mode before tw_set_sine_params
            (raw, w, h, cfg.height_params(), out(), tw.TW_ERR_STATE),
        ]
        for k, (cx, ww, hh, p, o, want) in enumerate(cases):
            handle = cx if isinstance(cx, C.c_void_p) else cx._h
            rc = L.tw_proc_gen_heightmap_launch(handle, ww, hh, dx, dy, C.byref(p) if p is not None else None, 100, C.byref(ep), o)
            assert rc == want, (k, rc, L.tw_last_error(handle))
            assert L.tw_create_tiles_poll(handle, 0) == tw.TW_OK                            # nothing pending
            assert np.all(img == 0xEE) and np.all(np.isnan(vals)) and _info(info) == (-1, -1, -1, -1, -1, -1, 7), k
        assert c.last_erosion_steps == steps
    finally:
        L.tw_destroy(raw)
        c.close()
