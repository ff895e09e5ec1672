"""GPU: tw_cancel. A job cancelled right after its launch ends in well under its uncancelled time and its poll raises TwCanceled; a cancel that comes
after the job has ended changes nothing; after a cancelled job, the next job of every kind on the same context gives what it gives on a fresh context,
bit for bit (the speculative erosion's cached graph included); cancelling one shared context leaves a sibling's job exact; a tile set's job refuses the
cancel and completes unaffected; any call other than a poll completes a cancelled job without an error and does its own work. Every cancel here
acts on a real job, once."""
import time

import numpy as np
import pytest
import torch

from test_gpu_job_kinds import KINDS, LAUNCH, N, S, ZV, World, _bits, _image, _ready, _run
from test_voxel_flood_reference import column_case, post_params

pytestmark = pytest.mark.gpu
f32 = np.float32
BIG = 8192           # side of the float maps of the long erosion jobs
LONG = 1_000_000     # droplets of the long erosion jobs (about 6 s in the serial order on 8192^2)
BOUND = 2.0          # seconds from the cancel to the completing poll, with room for a shared GPU


@pytest.fixture(scope="module")
def world(tw, scene):
    return World(tw, scene)


_ALONE = {}


def _alone(tw, w, kind):
    """Outputs, erosion steps and image of one job of `kind` on a fresh context (tests/test_gpu_job_kinds.py's set-up)."""
    if kind not in _ALONE:
        _ALONE[kind] = _run(tw, w, [kind, "poll"])
    return _ALONE[kind]


def _fresh(tw, w):
    c = tw.Context(0)
    c.set_sine_params(w.sine)
    c.set_heightmap(w.img.reshape(N, N, 2))
    ts = c.tile_set(ZV, 1)
    ts.put(w.tile_xy, w.set_z)
    return c, ts


def _same(got, exp, what):
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], "%s: %s differs" % (what, k)


def _next_jobs_exact(tw, c, ts, w):
    """Every kind of job, one after the other on c, equals the same job on a fresh context: outputs, erosion steps, and the image it leaves."""
    for kind in KINDS:
        c.set_heightmap(w.img.reshape(N, N, 2))
        read = LAUNCH[kind](tw, c, ts, w)
        assert c.create_tiles_poll(True)
        exp, exp_steps, exp_img = _alone(tw, w, kind)
        _same({k: _bits(v) for k, v in read().items()}, exp[0], kind)
        if kind in ("tiles", "hmap", "erode"):        # the jobs that set tw_last_erosion_steps
            assert c.last_erosion_steps == exp_steps, kind
        if kind in ("hmap", "erode"):
            assert _image(c, w) == exp_img, kind


def _cut_short(tw, c):
    """Cancels c's pending job at once; the completing poll must raise TwCanceled within BOUND seconds. Returns that time."""
    t0 = time.perf_counter()
    c.cancel()
    with pytest.raises(tw.TwCanceled) as e:
        c.create_tiles_poll(True)
    dt = time.perf_counter() - t0
    assert e.value.status == tw.TW_ERR_CANCELED and isinstance(e.value, tw.TwError)
    assert dt < BOUND, "the cancelled job took %.2f s to complete" % dt
    assert c.last_erosion_steps == 0
    assert c.create_tiles_poll(False)   # nothing pending any more
    return dt


def _big_map(c, w):
    z = torch.empty((BIG, BIG), dtype=torch.float32, device="cuda")
    c.heightgen_2d(w.hcfg.heightmap_grid(BIG, BIG), w.hp, out=z)
    return z, c.minmax(z)[0]


def test_cancel_without_a_job(tw, world):
    c, ts = _fresh(tw, world)
    try:
        c.cancel()                              # nothing pending
        read = LAUNCH["erode"](tw, c, ts, world)
        assert c.create_tiles_poll(True)
        c.cancel()                              # the job is complete and polled
        assert c.create_tiles_poll(False)
        _same({k: _bits(v) for k, v in read().items()}, _alone(tw, world, "erode")[0][0], "erode")
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "relight"])
def test_cancel_after_the_job_ended(tw, world, kind):
    """The stream is synchronised from outside (tw_stream) before the cancel: the poll returns TW_OK with the uncancelled outputs."""
    c, ts = _fresh(tw, world)
    try:
        read = LAUNCH[kind](tw, c, ts, world)
        torch.cuda.ExternalStream(c.stream).synchronize()
        c.cancel()
        assert c.create_tiles_poll(True)
        exp, exp_steps, exp_img = _alone(tw, world, kind)
        _same({k: _bits(v) for k, v in read().items()}, exp[0], kind)
        assert c.last_erosion_steps == exp_steps and _image(c, world) == exp_img
    finally:
        c.close()


@pytest.mark.parametrize("num_threads", [None, 1])
def test_long_erosion_job(tw, world, num_threads):
    """1e6 droplets on an 8192^2 device map, in the serial order (the speculative rounds) or the OpenMP mode with one thread (one droplet at a time)."""
    c, ts = _fresh(tw, world)
    try:
        z, zmin = _big_map(c, world)
        c.erode_launch(z, zmin, LONG, world.ep, num_threads=num_threads)
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_openmp_many_threads(tw, world):
    """Many droplets in flight end too fast for a time bound: only the status (cancelled, or complete if every droplet had been drawn)."""
    c, ts = _fresh(tw, world)
    try:
        z, zmin = _big_map(c, world)
        c.erode_launch(z, zmin, LONG, world.ep, num_threads=0)
        c.cancel()
        try:
            assert c.create_tiles_poll(True)
        except tw.TwCanceled:
            assert c.last_erosion_steps == 0
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_long_image_erosion_leaves_no_image(tw, world):
    c, ts = _fresh(tw, world)
    try:
        img, info, _ = c.proc_gen_heightmap(BIG, BIG, float(world.hcfg.dx_val), float(world.hcfg.dy_val), world.hp, 0, world.ep)
        c.set_heightmap(img.reshape(BIG, BIG, 2))
        c.erode_image_launch(info.val_mult, info.val_add, LONG, world.ep)
        _cut_short(tw, c)
        z = np.empty((1, 65, 65), f32)
        with pytest.raises(tw.TwError) as e:
            c.create_tiles_launch([(0, 0)], (64, 64), float(world.hcfg.dx_val), float(world.hcfg.dy_val), 65, None, 0, None, 0.0, z, hmap=world.hs)
        assert e.value.status == tw.TW_ERR_STATE
        _next_jobs_exact(tw, c, ts, world)      # set_heightmap gives the context an image again
    finally:
        c.close()


def test_spec_graph_reused_after_cancel(tw, world):
    """A cancelled speculative erosion job keeps the cached round graph; the same job again reuses it and equals tw_erode."""
    c, ts = _fresh(tw, world)
    try:
        n, iters = 1024, 20000
        z0 = torch.empty((n, n), dtype=torch.float32, device="cuda")
        c.heightgen_2d(world.hcfg.heightmap_grid(n, n), world.hp, out=z0)
        zmin = c.minmax(z0)[0]
        ref = _ready(z0.clone())
        c.erode(ref, zmin, iters, world.ep)
        steps = c.last_erosion_steps
        c.erode_launch(_ready(z0.clone()), zmin, iters, world.ep)
        _cut_short(tw, c)
        m = _ready(z0.clone())
        c.erode_launch(m, zmin, iters, world.ep)
        assert c.create_tiles_poll(True)
        assert c.last_erosion_steps == steps and torch.equal(m.view(torch.int32), ref.view(torch.int32))
    finally:
        c.close()


def test_long_tile_job(tw, world):
    """64 tiles of 1e6 droplets each."""
    c, ts = _fresh(tw, world)
    try:
        origins = [(tx * S * 40 - 3000, ty * S * 40 + 500) for ty in range(8) for tx in range(8)]
        zv = torch.empty((len(origins), ZV, ZV), dtype=torch.float32, device="cuda")   # a pageable host output would make the launch wait for the job
        c.create_tiles_launch(origins, world.tcfg.mesh_size, float(world.tcfg.dx_val), float(world.tcfg.dy_val), ZV, world.thp, LONG, world.tep, world.tep.zmin, zv)
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_long_voxel_fill(tw, world):
    """A 3 x 3 column whose flood fill runs 1e6 generations (the field in vals, no fill)."""
    c, ts = _fresh(tw, world)
    try:
        nz = 2_000_004
        vals, kw = column_case(nz)
        p = post_params(tw.VoxelPostParams, (3, 3, nz), **kw)
        v = _ready(torch.from_numpy(vals).cuda())
        c.voxel_build_launch(p, vals=v)
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_shared_sibling_unaffected(tw, world):
    parent = tw.Context(0)
    try:
        parent.set_sine_params(world.sine)
        a, b = parent.shared(), parent.shared()
        z, zmin = _big_map(b, world)
        b.erode_launch(z, zmin, LONG, world.ep)
        read = LAUNCH["tiles"](tw, a, None, world)
        _cut_short(tw, b)
        assert a.create_tiles_poll(True)
        _same({k: _bits(v) for k, v in read().items()}, _alone(tw, world, "tiles")[0][0], "sibling's tiles")
    finally:
        parent.close()


def test_tile_set_jobs_refuse(tw, world):
    """A relight and a frame into the set: tw_cancel returns TW_ERR_STATE and the job completes as if it had not been called."""
    c, ts = _fresh(tw, world)
    try:
        read = LAUNCH["relight"](tw, c, ts, world)
        with pytest.raises(tw.TwError) as e:
            c.cancel()
        assert e.value.status == tw.TW_ERR_STATE and not isinstance(e.value, tw.TwCanceled)
        assert c.create_tiles_poll(True)
        _same({k: _bits(v) for k, v in read().items()}, _alone(tw, world, "relight")[0][0], "relight")
        frame = []
        for cancel in (False, True):
            cf, tf = _fresh(tw, world)
            try:
                tf.remove(world.tile_xy[:3])
                zv = np.full((3, ZV, ZV), np.nan, f32)
                tf.create_tiles_launch(world.origins[:3], world.tcfg.mesh_size, float(world.tcfg.dx_val), float(world.tcfg.dy_val), world.thp, 60, world.tep,
                                       world.tep.zmin, world.tile_xy[:3], zvals=zv)
                if cancel:
                    with pytest.raises(tw.TwError) as e:
                        cf.cancel()
                    assert e.value.status == tw.TW_ERR_STATE
                assert cf.create_tiles_poll(True)
                L = tw.Light(world.sp, np.zeros((len(world.tile_xy), ZV, ZV), np.uint8))
                rec = tf.shadows_launch(world.tile_xy, [L])
                assert cf.create_tiles_poll(True)
                frame.append((zv.tobytes(), L.smask.tobytes(), rec.tobytes()))
            finally:
                cf.close()
        assert frame[0] == frame[1]
    finally:
        c.close()


def test_throughput_mode_tile_job(tw, world):
    """2048 tiles of 1e6 droplets: more walks than stay resident, so the throughput mode (M_GLOBAL, with M_WINDOW for the heaviest) walks them."""
    c, ts = _fresh(tw, world)
    try:
        origins = [(tx * S * 4 - 3000, ty * S * 4 + 500) for ty in range(32) for tx in range(64)]
        zv = torch.empty((len(origins), ZV, ZV), dtype=torch.float32, device="cuda")
        c.create_tiles_launch(origins, world.tcfg.mesh_size, float(world.tcfg.dx_val), float(world.tcfg.dy_val), ZV, world.thp, LONG, world.tep, world.tep.zmin, zv)
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_shadow_waves(tw, world):
    """A tile job without erosion whose only cancellation point is the mesh shadows: a strip of 2048 tiles toward the light is 2048 dependency waves
    (one CUDA graph in the job)."""
    c, ts = _fresh(tw, world)
    try:
        n = 2048
        origins = [(tx * S, 500) for tx in range(n)]
        txy = np.array([(tx, 0) for tx in range(n)], np.int32)
        zv = torch.empty((n, ZV, ZV), dtype=torch.float32, device="cuda")
        smask = torch.empty((n, ZV, ZV), dtype=torch.uint8, device="cuda")
        c.create_tiles_launch(origins, world.tcfg.mesh_size, float(world.tcfg.dx_val), float(world.tcfg.dy_val), ZV, world.thp, 0, world.tep, world.tep.zmin, zv,
                              tile_xy=txy, lights=[tw.Light(world.sp, smask)])
        _cut_short(tw, c)
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()


def test_other_calls_complete_a_cancelled_job(tw, world):
    """No poll between the cancel and the next call: that call completes the cut-short job without an error and does its own work - tw_set_heightmap
    loads the new map, the next launch launches, a parent's table setter completes its shared context's cancelled job, tw_destroy is quick."""
    c, ts = _fresh(tw, world)
    try:
        z, zmin = _big_map(c, world)
        c.erode_launch(z, zmin, LONG, world.ep)
        c.cancel()
        c.set_heightmap(world.img.reshape(N, N, 2))                  # the map-reload recipe: no TwCanceled, the new image is in place
        assert c.create_tiles_poll(False) and c.last_erosion_steps == 0
        assert _image(c, world) == _alone(tw, world, "grid")[2]
        c.erode_image_launch(world.info.val_mult, world.info.val_add, LONG, world.ep)
        c.cancel()
        read = LAUNCH["tiles"](tw, c, ts, world)                      # the next launch completes the cancelled job first, then runs
        assert c.create_tiles_poll(True)
        exp, exp_steps, _ = _alone(tw, world, "tiles")
        _same({k: _bits(v) for k, v in read().items()}, exp[0], "tiles after a cancelled job")
        assert c.last_erosion_steps == exp_steps
        c.set_heightmap(world.img.reshape(N, N, 2))                  # the cancelled image erosion left no image
        _next_jobs_exact(tw, c, ts, world)
    finally:
        c.close()
    parent = tw.Context(0)
    try:
        parent.set_sine_params(world.sine)
        s = parent.shared()
        z, zmin = _big_map(s, world)
        s.erode_launch(z, zmin, LONG, world.ep)
        s.cancel()
        parent.set_heightmap(world.img.reshape(N, N, 2))             # completes the shared context's job first
        assert s.create_tiles_poll(False)
        s.erode_launch(z, zmin, LONG, world.ep)
        s.cancel()
        t0 = time.perf_counter()
        s.close()                                                     # tw_destroy completes the cancelled job
        assert time.perf_counter() - t0 < BOUND
    finally:
        parent.close()
