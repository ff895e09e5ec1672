"""GPU: tw_erode_launch_ex's TW_EROSION_SWEEPS mode - tw_erode_sweeps of one map, or of the context's set_heightmap image between its unpack and its pack,
as one asynchronous job whose sweeps end on the device. Float maps are held bit for bit to tw_erode_sweeps (device, pinned and pageable; short, exact,
ragged and 2000+ sweeps; odd shapes and 8192^2) and to the CPU oracle, the image to the chain of synchronous calls; then the refusals, the other two modes
through tw_erode_launch_ex(NULL), shared contexts side by side, tw_cancel on a long job and a cancel that comes too late."""
import ctypes as C

import numpy as np
import pytest
import torch

from cases import convert, HM_CFG
from test_gpu_cancel import _big_map, _cut_short, _fresh, _next_jobs_exact, world  # noqa: F401 (world is a fixture)
from test_gpu_erosion_job import _bits, _host, _image, _image_tiles, _place, _ready, _sampled, _sampler

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def sctx(tw):
    c = tw.Context(0)
    yield c
    c.close()


_TERRAIN = {}


def _terrain(c, scene, n, m):
    if (n, m) not in _TERRAIN:
        cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.0)
        _TERRAIN[(n, m)] = (cfg, c.heightgen_2d(cfg.heightmap_grid(n, m), cfg.height_params()))
    return _TERRAIN[(n, m)]


def _sync(c, z, zmin, iters, ep, sweep, halo):
    """tw_erode_sweeps on a host copy: the map and the moves."""
    h = np.ascontiguousarray(_host(z)).copy()
    moves = c.erode_sweeps(h, zmin, iters, ep, sweep, halo)
    return h, moves


# n x m, droplets, sweep, halo: below one sweep, exactly one, not a multiple of the sweep, 2858 sweeps of 7 droplets, 2500 sweeps of 8
CASES = [(300, 200, 100, 256, 48), (300, 200, 256, 256, 48), (512, 512, 20000, 1000, 64), (512, 512, 20000, 7, 44), (130, 97, 20000, 8, 44)]


@pytest.mark.parametrize("kind", ["device", "pinned", "pageable"])
@pytest.mark.parametrize("n,m,iters,sweep,halo", CASES)
def test_float_map_equals_tw_erode_sweeps(tw, scene, sctx, kind, n, m, iters, sweep, halo):
    cfg, z = _terrain(sctx, scene, n, m)
    zmin, ep = float(z.min()), cfg.erosion_params()
    ref, moves = _sync(sctx, z, zmin, iters, ep, sweep, halo)
    assert moves > 0 and not np.array_equal(ref, z)
    h = _place(kind, z)
    job = sctx.erode_launch(h, zmin, iters, ep, sweep=sweep, halo=halo)
    assert job.heightmap is h
    assert sctx.create_tiles_poll(True)
    assert np.array_equal(_bits(h), _bits(ref)) and sctx.last_erosion_steps == moves


@pytest.mark.parametrize("n,m,iters,sweep", [(4097, 1023, 30000, 4096), (8192, 8192, 100000, 8192)])
def test_large_maps(tw, scene, sctx, n, m, iters, sweep):
    cfg, z = _terrain(sctx, scene, n, m)
    zmin, ep = float(z.min()), cfg.erosion_params()
    ref, moves = _sync(sctx, z, zmin, iters, ep, sweep, 64)
    h = _ready(torch.from_numpy(z.copy()).cuda())
    sctx.erode_launch(h, zmin, iters, ep, sweep=sweep, halo=64)
    assert sctx.create_tiles_poll(True)
    assert np.array_equal(_bits(h), _bits(ref)) and sctx.last_erosion_steps == moves > 0


@pytest.mark.parametrize("n,m,iters,sweep,halo", [(130, 97, 777, 50, 44), (20, 30, 500, 7, 44), (200, 260, 3000, 3000, 100)])
def test_float_map_equals_the_oracle(tw, scene, oracle, sctx, n, m, iters, sweep, halo):
    """Both parameter sets of the oracle's sweeps test, the second with the rock threshold inside the map's range (walks that go NaN end as the oracle's do)."""
    cfg, z = _terrain(sctx, scene, n, m)
    zmin, zmax = float(z.min()), float(z.max())
    for ep in (tw.ErosionParams(1.0, zmin - 10, 0.0625, zmin - 0.1, zmax + 0.1, 0.0, 0.5), tw.ErosionParams(1.0, zmin + 0.2 * (zmax - zmin), 0.0625, zmin - 0.1, zmax + 0.1, 0.0, 2.0)):
        zo, mo = oracle.erode_sweeps(z, zmin, iters, convert(ep, oracle.ErosionParams), sweep, halo)
        h = z.copy()
        sctx.erode_launch(h, zmin, iters, ep, sweep=sweep, halo=halo)
        assert sctx.create_tiles_poll(True)
        assert np.array_equal(_bits(h), _bits(zo)) and sctx.last_erosion_steps == mo
        assert np.isfinite(h).all()


def test_early_out(tw, scene, sctx):
    cfg, z = _terrain(sctx, scene, 300, 200)
    ep = cfg.erosion_params()
    h = z.copy()
    sctx.erode_launch(h, float(z.min()), 0, ep, sweep=64, halo=44)
    assert sctx.create_tiles_poll(True)
    assert np.array_equal(_bits(h), _bits(z)) and sctx.last_erosion_steps == 0


@pytest.mark.parametrize("kind", ["device", "pageable", None])
def test_image_matches_the_chain(tw, scene, kind):
    n, iters, sweep, halo = 1024, 30000, 2048, 64
    c = tw.Context(0)
    try:
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        vals_ref = c.to_floats_u16(img, info.val_mult, info.val_add).reshape(n, n)
        zmin, _ = c.minmax(vals_ref)
        moves = c.erode_sweeps(vals_ref, zmin, iters, ep, sweep, halo)
        img_ref = c.from_floats_u16(vals_ref, info.val_mult, info.val_add)
        hs = _sampler(tw, cfg, info, n)
        c.set_heightmap(img.reshape(n, n, 2))
        vals = None if kind is None else _place(kind, np.full(n * n, np.nan, np.float32))
        c.erode_image_launch(info.val_mult, info.val_add, iters, ep, vals=vals, sweep=sweep, halo=halo)
        assert c.create_tiles_poll(True)
        assert c.last_erosion_steps == moves > 0
        if vals is not None:
            assert np.array_equal(_bits(vals).ravel(), _bits(vals_ref).ravel())
        assert np.array_equal(_bits(_image_tiles(c, cfg, hs, n)), _bits(_sampled(c, img_ref, hs, n)))   # the context holds the eroded image
    finally:
        c.close()


def _args(tw, h, xs, ys, ep, mode=2, num_threads=0, iters=100):
    return tw.ErosionJobArgs(C.cast(h.ctypes.data, C.c_void_p), xs, ys, float(h.min()), 0.0, 0.0, iters, C.cast(C.pointer(ep), C.c_void_p), mode, num_threads, None)


def test_refusals_enqueue_nothing(tw, scene, sctx):
    cfg, z = _terrain(sctx, scene, 300, 200)
    ep = cfg.erosion_params()
    L, h = tw.lib, z.copy()
    ok = tw.SweepParams(64, 44)
    cases = [(_args(tw, h, 300, 200, ep), tw.SweepParams(0, 44)),                      # sweep == 0
             (_args(tw, h, 300, 200, ep), tw.SweepParams(64, 43)),                     # halo < view + 12
             (_args(tw, h, 300, 200, ep, iters=0), tw.SweepParams(0, 44)),             # checked without work too
             (_args(tw, h, 300, 200, ep, num_threads=4), ok),                          # num_threads in the sweeps mode
             (_args(tw, h, 300, 200, ep), None),                                       # no tw_sweep_params
             (_args(tw, h, 300, 200, ep, mode=tw.TW_EROSION_SERIAL), ok),              # tw_sweep_params with the other modes
             (_args(tw, h, 300, 200, ep, mode=tw.TW_EROSION_OPENMP), ok),
             (_args(tw, h, 300, 200, ep, mode=3), ok),                                 # bad mode
             (_args(tw, h, 0, 200, ep), ok)]                                           # empty map
    for a, sw in cases:
        n0 = sctx.launch_count
        assert L.tw_erode_launch_ex(sctx._h, C.byref(a), None if sw is None else C.byref(sw)) == tw.TW_ERR_ARG
        assert sctx.launch_count == n0 and sctx.create_tiles_poll(False)
    assert np.array_equal(h, z)
    a = _args(tw, h, 0, 0, ep)
    a.heightmap = None
    c = tw.Context(0)
    try:   # the image without one set
        assert L.tw_erode_launch_ex(c._h, C.byref(a), C.byref(ok)) == tw.TW_ERR_STATE
    finally:
        c.close()


@pytest.mark.parametrize("mode,threads", [(0, 0), (1, 1)])
def test_other_modes_through_the_ex_entry_point(tw, scene, sctx, mode, threads):
    cfg, z = _terrain(sctx, scene, 512, 512)
    ep = cfg.erosion_params()
    out = []
    for ex in (False, True):
        h = z.copy()
        a = _args(tw, h, 512, 512, ep, mode=mode, num_threads=threads, iters=3000)
        rc = tw.lib.tw_erode_launch_ex(sctx._h, C.byref(a), None) if ex else tw.lib.tw_erode_launch(sctx._h, C.byref(a))
        assert rc == tw.TW_OK and sctx.create_tiles_poll(True)
        out.append((_bits(h).copy(), sctx.last_erosion_steps))
    assert np.array_equal(out[0][0], out[1][0]) and out[0][1] == out[1][1] > 0


def test_shared_contexts_side_by_side(tw, scene, sctx):
    cfg, z = _terrain(sctx, scene, 512, 512)
    zmin, ep = float(z.min()), cfg.erosion_params()
    params = [(20000, 1000, 64), (15000, 333, 44), (20000, 7, 44)]
    refs = [_sync(sctx, z, zmin, it, ep, sw, ha) for it, sw, ha in params]
    parent = tw.Context(0)
    try:
        shared = [parent.shared() for _ in params]
        maps = [_ready(torch.from_numpy(z.copy()).cuda()) for _ in params]
        for c, h, (it, sw, ha) in zip(shared, maps, params):
            c.erode_launch(h, zmin, it, ep, sweep=sw, halo=ha)
        for c, h, (ref, moves) in zip(shared, maps, refs):
            assert c.create_tiles_poll(True)
            assert np.array_equal(_bits(h), _bits(ref)) and c.last_erosion_steps == moves
    finally:
        parent.close()


LONG = 2_000_000   # droplets of the long jobs: 2000 sweeps of 1000 on 8192^2


def test_cancel_a_long_float_map_job(tw, world):
    c, ts = _fresh(tw, world)
    try:
        z, zmin = _big_map(c, world)
        c.erode_launch(z, zmin, LONG, world.ep, sweep=1000, halo=64)
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_cancel_a_long_image_job_leaves_no_image(tw, world):
    c, ts = _fresh(tw, world)
    try:
        big = 8192
        img, info, _ = c.proc_gen_heightmap(big, big, float(world.hcfg.dx_val), float(world.hcfg.dy_val), world.hp, 0, world.ep)
        c.set_heightmap(img.reshape(big, big, 2))
        c.erode_image_launch(info.val_mult, info.val_add, LONG, world.ep, sweep=1000, halo=64)
        _cut_short(tw, c)
        z = np.empty((1, 65, 65), f32)
        with pytest.raises(tw.TwError) as e:
            c.create_tiles_launch([(0, 0)], (64, 64), float(world.hcfg.dx_val), float(world.hcfg.dy_val), 65, None, 0, None, 0.0, z, hmap=world.hs)
        assert e.value.status == tw.TW_ERR_STATE
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_cancel_after_the_job_ended(tw, scene, sctx):
    cfg, z = _terrain(sctx, scene, 512, 512)
    zmin, ep = float(z.min()), cfg.erosion_params()
    ref, moves = _sync(sctx, z, zmin, 20000, ep, 1000, 64)
    h = z.copy()
    sctx.erode_launch(h, zmin, 20000, ep, sweep=1000, halo=64)
    torch.cuda.ExternalStream(sctx.stream).synchronize()
    sctx.cancel()
    assert sctx.create_tiles_poll(True)
    assert np.array_equal(_bits(h), _bits(ref)) and sctx.last_erosion_steps == moves
