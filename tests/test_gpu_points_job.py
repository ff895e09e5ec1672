"""GPU: tw_points_launch, the asynchronous points job. Procedural kinds bit for bit against tw_eval_points for every kind x gen mode x shape, at n = 1, 255,
256, 257 and 1e7, with pageable, pinned and device xy / out, the caller's host xy overwritten right after the launch; TW_PQ_HMAP at integer cells against
tw_heightmap_sample_tiles in every edge mode and at mesh_scale 0.5, 1, 2 and 1.3 (inside the image, on its edges, far outside), at fractional cells
against the numpy restatement; the edit ordering of tw_update_heightmap; and the job rules (shared contexts, completion by other calls and tw_destroy,
tw_cancel, errors that enqueue nothing)."""
import ctypes as C
import os

import numpy as np
import pytest

from cases import HM_ALL, HM_CFG
from test_oracle_golden import point_cases
from test_points_job_host import hmap_points_np, sampler_cases, tile_cells

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MEM = ("pageable", "pinned", "device")


@pytest.fixture(scope="module")
def pctx(tw):
    c = tw.Context(0)
    yield c
    c.close()


def put(a, mem):
    import torch
    a = np.ascontiguousarray(a)
    if mem == "pageable":
        return a.copy()
    t = torch.from_numpy(a.copy())
    return t.pin_memory() if mem == "pinned" else t.cuda()


def empty(n, mem):
    import torch
    if mem == "pageable":
        return np.full(n, np.nan, np.float32)
    t = torch.full((n,), float("nan"), dtype=torch.float32)
    return t.pin_memory() if mem == "pinned" else t.cuda()


def host(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def run(c, xy, mem, hp=None, pq=None, hs=None, out_mem=None):
    """One job with xy and out in memory kind mem (out: out_mem); host xy is overwritten as soon as the launch returns."""
    xy_m, out = put(xy, mem), empty(len(xy), out_mem or mem)
    job = c.points_launch(xy_m, hp, pq, hs, out)
    if mem != "device":
        xy_m[:] = 1e30                                        # the launch copied it
    got = job.poll(True)
    assert got is out
    return host(got).copy()


def same(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def test_golden_cases_equal_eval_points(tw, pctx):
    h = np.load(os.path.join(GOLD, "points.npz"))
    n = 0
    for key, hp, pq, xy, sp, exp in point_cases(tw, h):
        if sp is not None:
            pctx.set_sine_params(sp)
        want = pctx.eval_points(xy, hp, pq)
        assert same(want, exp), key
        for k, mem in enumerate(MEM):
            assert same(run(pctx, xy, mem, hp, pq, out_mem=MEM[(k + 1) % 3]), want), (key, mem)
        n += 1
    assert n >= 50


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_every_kind_and_shape_equals_eval_points(tw, scene, pctx, mode):
    import torch
    rng = np.random.default_rng(10 + mode)
    for shape in range(3):
        cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_gen_shape=shape, mesh_freq_filter=1, mesh_seed=3, hmap=HM_ALL, zmax_est=2.3)
        hp = cfg.height_params()
        pctx.set_sine_params(cfg.sine_params())
        for qi, (kind, xy_scale) in enumerate(((tw.PQ_EXACT_ZVAL, 1.0), (tw.PQ_SIN_TERMS_SCALED, 16.0), (tw.PQ_SIN_TERMS, 1.0))):
            pq = tw.PointQuery(kind, xy_scale, 128, 128, 4.0, 4.0, -3000, 777, 0)
            for n in (1, 255, 256, 257):
                xy = rng.uniform(-60.0, 60.0, (n, 2)).astype(np.float32)
                want = pctx.eval_points(xy, hp, pq)
                for mem in MEM:
                    assert same(run(pctx, xy, mem, hp, pq), want), (shape, kind, n, mem)
            n = 10 ** 7
            d_xy = torch.empty((n, 2), dtype=torch.float32, device="cuda").uniform_(-60.0, 60.0)
            want = torch.empty(n, dtype=torch.float32, device="cuda")
            pctx.eval_points(d_xy, hp, pq, out=want)
            mem = MEM[(shape + qi) % 3]
            got = run(pctx, d_xy.cpu().numpy(), mem, hp, pq)
            assert same(got, want.cpu().numpy()), (shape, kind, mem)


def test_eval_points_still_refuses_hmap_kind(tw, pctx):
    with pytest.raises(tw.TwError) as e:
        pctx.eval_points(np.zeros((4, 2), np.float32), tw.HeightParams(), tw.PointQuery(tw.PQ_HMAP, 1.0, 128, 128, 4.0, 4.0, 0, 0, 0))
    assert e.value.status == tw.TW_ERR_ARG


def hq(tw):
    return tw.PointQuery(tw.PQ_HMAP, 1.0, 0, 0, 0.0, 0.0, 0, 0, 0)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ms", [0.5, 1.0, 2.0, 1.3])
def test_hmap_cells_equal_tile_sampler(tw, pctx, mode, ms):
    rng = np.random.default_rng(int(ms * 10) + 7 * mode)
    for W, H, zv in ((61, 45, 17), (128, 96, 33)):
        img = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
        pctx.set_heightmap(img)
        hs = tw.HmapSampler(W, H, mode, ms, 0.0012, 1.7, -0.3, 0.8)
        origins = sampler_cases(W, H, zv)
        want = pctx.heightmap_sample_tiles(img, hs, origins, zv).ravel()
        cells = tile_cells(origins, zv)
        for k, mem in enumerate(MEM):
            assert same(run(pctx, cells, mem, pq=hq(tw), hs=hs, out_mem=MEM[(k + 2) % 3]), want), (W, H, mem)
        frac = cells + rng.uniform(0.0, 1.0, cells.shape).astype(np.float32)
        odd = np.array([[np.nan, 0], [np.inf, -np.inf], [3e9, -3e9], [1e30, 2.5], [-0.0, 1e-30], [-0.5, 0.5]], np.float32)
        frac = np.concatenate([frac, odd]).astype(np.float32)
        assert same(run(pctx, frac, MEM[mode], pq=hq(tw), hs=hs), hmap_points_np(img, hs, frac)), (W, H)


def _image(rng, W, H):
    return rng.integers(0, 256, (H, W, 2), dtype=np.uint8)


def test_edit_ordering(tw, scene):
    """launch, tw_update_heightmap, launch again, no poll between: the first job reads the old image, the second the new one; then the same on a shared
    context while the root runs a heightmap tile job, whose zvals are those of the old image."""
    rng = np.random.default_rng(5)
    W, H = 301, 203
    old = _image(rng, W, H)
    new = old.copy()
    new[40:120, 10:200] = rng.integers(0, 256, (80, 190, 2), dtype=np.uint8)
    hs = tw.HmapSampler(W, H, 2, 0.5, 0.0012, 1.7, -0.3, 0.8)
    xy = (rng.uniform(-400, 400, (200000, 2))).astype(np.float32)
    want_old, want_new = hmap_points_np(old, hs, xy), hmap_points_np(new, hs, xy)
    assert not same(want_old, want_new)
    root = tw.Context(0)
    try:
        s = root.shared()
        for c in (root, s):
            root.set_heightmap(old)
            tiles = None
            if c is s:   # the root's heightmap tile job stays pending through everything below
                zv, org = 65, np.array([(x, y) for y in (-128, -64, 0, 64) for x in (-128, -64, 0, 64)], np.int32)
                tiles = np.empty((len(org), zv, zv), np.float32)
                root.create_tiles_launch(org, (zv, zv), 1.0, 1.0, zv, None, 0, None, 0.0, tiles, hmap=hs)
            a = c.points_launch(xy, pq=hq(tw), hs=hs)
            root.update_heightmap(new, [(10, 40, 190, 80)])
            b_out = np.empty(len(xy), np.float32)
            b = c.points_launch(xy, pq=hq(tw), hs=hs, out=b_out)    # completes a
            assert same(a.out, want_old) and same(b.poll(True), want_new), c is s
            if tiles is not None:
                assert root.create_tiles_poll(True)
                assert same(tiles.ravel(), hmap_points_np(old, hs, tile_cells(org, zv)))
    finally:
        root.close()


def _frame(tw, scene, c):
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(64, 64, 1))
    hp, ep = cfg.height_params(), cfg.erosion_params()
    org = np.array([(x * 64, y * 64) for y in range(-2, 2) for x in range(-2, 2)], np.int32)
    z = np.empty((16, 66, 66), np.float32)
    c.create_tiles_launch(org, cfg.mesh_size, float(cfg.dx_val), float(cfg.dy_val), 66, hp, 2000, ep, ep.zmin, z)
    return z


def test_beside_a_tile_job_on_a_shared_context(tw, scene):
    cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)
    hp = cfg.height_params()
    pq = tw.PointQuery(tw.PQ_EXACT_ZVAL, 1.0, 128, 128, 4.0, 4.0, 5, -9, 0)
    xy = np.random.default_rng(2).uniform(-3.0, 3.0, (10 ** 6, 2)).astype(np.float32)
    root = tw.Context(0)
    try:
        s1, s2 = root.shared(), root.shared()
        z_alone = _frame(tw, scene, s1)
        assert s1.create_tiles_poll(True)
        p_alone = run(s2, xy, "pinned", hp, pq)
        z = _frame(tw, scene, s1)
        job = s2.points_launch(put(xy, "pinned"), hp, pq, out=empty(len(xy), "pinned"))
        p = host(job.poll(True)).copy()
        assert s1.create_tiles_poll(True)
        assert same(z, z_alone) and same(p, p_alone)
    finally:
        root.close()


def test_other_calls_complete_it(tw, pctx, scene):
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=2, hmap=HM_CFG, zmax_est=2.3)
    hp = cfg.height_params()
    pq = tw.PointQuery(tw.PQ_EXACT_ZVAL, 1.0, 128, 128, 4.0, 4.0, 0, 0, 0)
    xy = np.random.default_rng(3).uniform(-3.0, 3.0, (100000, 2)).astype(np.float32)
    want = pctx.eval_points(xy, hp, pq)
    job = pctx.points_launch(xy, hp, pq)
    pctx.eval_points(xy[:1], hp, pq)                          # any entry point completes the pending job first
    assert same(job.out, want) and job.poll(False) is job.out
    job = pctx.points_launch(xy, hp, pq)
    assert tw.lib.tw_heightgen_2d_poll(pctx._h, 1) == tw.TW_OK and same(job.out, want)
    job = pctx.points_launch(xy, hp, pq)
    while job.poll(False) is None:
        pass
    assert same(job.out, want)
    s = pctx.shared()
    job = s.points_launch(xy, hp, pq)
    s.close()                                                 # tw_destroy completes the job
    assert same(job.out, want)


def test_cancel_is_refused(tw, pctx, scene):
    hp = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=2, hmap=HM_CFG, zmax_est=2.3).height_params()
    pq = tw.PointQuery(tw.PQ_EXACT_ZVAL, 1.0, 128, 128, 4.0, 4.0, 0, 0, 0)
    xy = np.random.default_rng(4).uniform(-3.0, 3.0, (10 ** 6, 2)).astype(np.float32)
    want = pctx.eval_points(xy, hp, pq)
    job = pctx.points_launch(xy, hp, pq)
    with pytest.raises(tw.TwError) as e:
        pctx.cancel()
    assert e.value.status == tw.TW_ERR_STATE
    assert same(job.poll(True), want)


def test_errors_enqueue_nothing(tw, scene):
    cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_freq_filter=1, mesh_seed=2, hmap=HM_CFG, zmax_est=2.3)
    hp = cfg.height_params()
    pq = tw.PointQuery(tw.PQ_EXACT_ZVAL, 1.0, 128, 128, 4.0, 4.0, 0, 0, 0)
    xy = np.random.default_rng(6).uniform(-3.0, 3.0, (1000, 2)).astype(np.float32)
    out = np.zeros(len(xy), np.float32)
    W, H = 40, 30
    img = _image(np.random.default_rng(7), W, H)
    hs = tw.HmapSampler(W, H, 0, 1.0, 1.0, 1.0, 0.0, 1.0)
    root = tw.Context(0)
    try:
        s = root.shared()

        def status(c, xy_, hp_, pq_, hs_, out_, n=None):
            ref = lambda v: C.cast(C.pointer(v), C.c_void_p) if v is not None else None  # noqa: E731
            a = tw.PointsJobArgs(tw._ptr(xy_), len(xy) if n is None else n, ref(hp_), ref(pq_), ref(hs_), tw._ptr(out_))
            before = c.launch_count
            rc = tw.lib.tw_points_launch(c._h, C.byref(a))
            assert c.launch_count == before
            return rc
        ARG, STATE = tw.TW_ERR_ARG, tw.TW_ERR_STATE
        assert status(root, xy, hp, pq, None, out) == STATE                       # sine mode without the sine params
        assert status(root, xy, None, hq(tw), hs, out) == STATE                   # no image
        root.set_sine_params(cfg.sine_params())
        root.set_heightmap(img)
        assert tw.lib.tw_points_launch(root._h, None) == ARG
        bad = lambda **kw: tw.PointQuery(kw.get("kind", tw.PQ_EXACT_ZVAL), 1.0, 128, 128, 4.0, 4.0, 0, 0, 0)  # noqa: E731
        hp_bad = cfg.height_params()
        hp_bad.start_eval_sin = 91
        for c in (root, s):
            assert status(c, None, hp, pq, None, out) == ARG
            assert status(c, xy, hp, None, None, out) == ARG
            assert status(c, xy, hp, pq, None, None) == ARG
            assert status(c, xy, None, pq, None, out) == ARG
            assert status(c, xy, hp, bad(kind=7), None, out) == ARG
            assert status(c, xy, hp, bad(kind=-1), None, out) == ARG
            assert status(c, xy, hp_bad, pq, None, out) == ARG
            assert status(c, xy, None, hq(tw), None, out) == ARG
            assert status(c, xy, None, hq(tw), tw.HmapSampler(W + 1, H, 0, 1.0, 1.0, 1.0, 0.0, 1.0), out) == ARG
            assert status(c, xy, None, hq(tw), tw.HmapSampler(W, H, 3, 1.0, 1.0, 1.0, 0.0, 1.0), out) == ARG
            assert status(c, None, None, None, None, None, n=0) == tw.TW_OK
        ep = cfg.erosion_params()
        root.erode_image_launch(1.0, 0.0, 0, ep)                                   # no image while it is pending
        assert status(s, xy, None, hq(tw), hs, out) == STATE
        assert root.create_tiles_poll(True)
        for c in (root, s):                                                        # the next job's output is the normal one
            assert same(run(c, xy, "pageable", hp, pq), root.eval_points(xy, hp, pq))
    finally:
        root.close()
