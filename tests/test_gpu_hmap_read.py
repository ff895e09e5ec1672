"""GPU: tw_read_heightmap_launch / tw_read_heightmap - the context's heightmap image read back, whole or by rects, as a job ordered with its edits. Every
comparison is byte for byte: whole images of odd and large sizes, rects at every texel phase, narrow, wide and overlapping, a pitch wider than the image,
device / page-locked / pageable destinations (device ones at every texel offset and pitch phase), the round trip with tw_update_heightmap, the image after each
writer (erosion in three modes, a set_image heightmap job, an edit), the ordering on shared contexts beside a heightmap tile frame, the brush workflow,
an image of more than 2^31 bytes, tw_cancel, the refusals and nrects == 0."""
import ctypes as C

import numpy as np
import pytest
import torch

from cases import HM_CFG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rctx(tw):
    c = tw.Context(0)
    yield c
    c.close()


def _img(rng, w, h):
    return rng.integers(0, 256, (h, w, 2), dtype=np.uint8)


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


def _rects_of(img, rects, out):
    """out with img's texels inside rects (a copy)."""
    out = out.copy()
    for x, y, w, h in rects:
        out[y:y + h, x:x + w] = img[y:y + h, x:x + w]
    return out


def _dest(kind, rows, cols, fill=0x5a, byte_offset=0):
    """A uint8 [rows, cols, 2] destination filled with `fill`: pageable numpy, page-locked or CUDA tensor; a CUDA one starts byte_offset bytes into its
    allocation (a view of it)."""
    if kind == "pageable":
        return np.full((rows, cols, 2), fill, np.uint8)
    if kind == "pinned":
        return torch.full((rows, cols, 2), fill, dtype=torch.uint8).pin_memory()
    buf = torch.full((rows * cols * 2 + byte_offset + 32,), fill, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    return torch.as_strided(buf, (rows, cols, 2), (2 * cols, 2, 1), byte_offset)


# ---- whole images
@pytest.mark.parametrize("w,h", [(1, 1), (3, 7), (7, 5), (8, 5), (9, 5), (4097, 3), (7168, 7168)])
def test_whole_image_after_set_heightmap(tw, rctx, w, h):
    img = _img(np.random.default_rng(w * 31 + h), w, h)
    rctx.set_heightmap(img)
    assert np.array_equal(rctx.read_heightmap(), img)
    for kind in ("device", "pinned"):
        out = _dest(kind, h, w)
        assert np.array_equal(_host(rctx.read_heightmap(out=out)), img), kind


# ---- rects
def _rect_cases(W, H, rng):
    cases = [[(8 * k + p, 3 + p, 37, 2) for p in range(8)] for k in (0, 5)]                       # every start phase
    cases.append([(p * 9, 10 + p, w, 3) for p, w in enumerate((1, 2, 3, 5, 7))])                  # narrower than 8 texels
    cases.append([(p, 20 + 2 * p, W - p - 1 - (p % 3), 2) for p in range(8)])                      # wider than one warp's 16-byte words (256 texels)
    cases.append([(10, 30, 100, 40), (50, 50, 120, 30), (10, 30, 100, 40), (0, 0, W, 1)])         # overlapping
    cases.append([(0, 0, W, H)])
    cases.append([(int(rng.integers(0, W - 60)), int(rng.integers(0, H - 40)), int(rng.integers(1, 60)), int(rng.integers(1, 40))) for _ in range(40)])
    return cases


@pytest.mark.parametrize("kind", ["device", "pinned", "pageable"])
def test_rects(tw, rctx, kind):
    rng = np.random.default_rng(3)
    W, H = 333, 120
    img = _img(rng, W, H)
    rctx.set_heightmap(img)
    for rects in _rect_cases(W, H, rng):
        for extra in (0, 13):                                                                     # dst_pitch = 2*W, and greater
            out = _dest(kind, H, W + extra)
            got = _host(rctx.read_heightmap(rects, out))
            want = _rects_of(np.pad(img, ((0, 0), (0, extra), (0, 0)), constant_values=0x5a), rects, np.full((H, W + extra, 2), 0x5a, np.uint8))
            assert np.array_equal(got, want), (kind, extra, rects)


@pytest.mark.parametrize("byte_offset,extra", [(2, 0), (6, 3), (4, 4), (14, 5), (16, 1), (10, 7)])
def test_device_destination_at_any_offset(tw, rctx, byte_offset, extra):
    """A device dst16 whose rows have another phase than the image's: every texel offset from a 16-byte boundary, and pitches that shift the phase from row
    to row (extra = 4: rows in and out of phase alternate; odd extra: every shift over 8 rows). Nothing outside the rects' texels is written, before dst16
    included."""
    rng = np.random.default_rng(byte_offset)
    W, H = 1029, 37
    img = _img(rng, W, H)
    rctx.set_heightmap(img)
    for rects in ([(0, 0, W, H)], [(3, 1, 700, 5), (0, 9, 9, 9), (511, 20, 518, 17), (1, 30, 5, 7)]):
        out = _dest("device", H, W + extra, byte_offset=byte_offset)
        got = _host(rctx.read_heightmap(rects, out))
        full = np.full((H, W + extra, 2), 0x5a, np.uint8)
        full[:, :W] = img
        assert np.array_equal(got, _rects_of(full, rects, np.full((H, W + extra, 2), 0x5a, np.uint8))), (byte_offset, extra, rects)
        whole = out._base.cpu().numpy()
        assert (whole[:byte_offset] == 0x5a).all() and (whole[byte_offset + out.numel():] == 0x5a).all()


def test_odd_device_destination_is_refused(tw, rctx):
    """Texels are 16-bit words: a device dst16 at an odd address or with an odd dst_pitch is TW_ERR_ARG, and nothing is written."""
    rctx.set_heightmap(_img(np.random.default_rng(8), 40, 10))
    buf = torch.full((2000,), 0x5a, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for off, pitch in ((1, 80), (0, 81), (3, 83)):
        arr, n = tw._rects([(0, 0, 40, 10)])
        a = tw.HmapReadArgs(C.cast(arr, C.c_void_p), n, C.c_void_p(buf.data_ptr() + off), pitch)
        assert tw.lib.tw_read_heightmap_launch(rctx._h, C.byref(a)) == tw.TW_ERR_ARG, (off, pitch)
    assert rctx.create_tiles_poll(True)
    assert bool((buf == 0x5a).all())


def test_read_then_update_changes_nothing(tw, rctx):
    rng = np.random.default_rng(4)
    W, H = 700, 300
    img = _img(rng, W, H)
    rctx.set_heightmap(img)
    rects = [(5, 7, 100, 30), (300, 200, 399, 100), (0, 0, 1, 1), (50, 20, 90, 60)]
    buf = np.zeros((H, W + 9, 2), np.uint8)
    rctx.read_heightmap(rects, buf)
    rctx.update_heightmap(buf, rects)
    assert np.array_equal(rctx.read_heightmap(), img)


# ---- what each writer leaves
def _cfg(scene):
    return scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3)


def _image(c, scene, n):
    cfg = _cfg(scene)
    img, info, _ = c.proc_gen_heightmap(n, n, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), 0, cfg.erosion_params())
    return cfg, img.reshape(n, n, 2), info


def _chain(c, img, info, n, iters, ep, mode):
    """to_floats -> minmax -> erode (serial, 1-thread OpenMP or sweeps) -> from_floats."""
    vals = c.to_floats_u16(img.reshape(-1), info.val_mult, info.val_add).reshape(n, n)
    zmin, _ = c.minmax(vals)
    if mode == "serial":
        c.erode(vals, zmin, iters, ep)
    elif mode == "openmp":
        c.erode_parallel(vals, zmin, iters, ep, num_threads=1)
    else:
        c.erode_sweeps(vals, zmin, iters, ep, 512, 64)
    return c.from_floats_u16(vals, info.val_mult, info.val_add).reshape(n, n, 2)


def _erode_image(c, info, iters, ep, mode):
    if mode == "serial":
        return c.erode_image_launch(info.val_mult, info.val_add, iters, ep)
    if mode == "openmp":
        return c.erode_image_launch(info.val_mult, info.val_add, iters, ep, num_threads=1)
    return c.erode_image_launch(info.val_mult, info.val_add, iters, ep, sweep=512, halo=64)


@pytest.mark.parametrize("mode", ["serial", "openmp", "sweeps"])
def test_after_erosion_of_the_image(tw, scene, rctx, mode):
    n, iters = 512, 4000
    cfg, img, info = _image(rctx, scene, n)
    ep = cfg.erosion_params()
    want = _chain(rctx, img, info, n, iters, ep, mode)
    assert not np.array_equal(want, img)
    rctx.set_heightmap(img)
    _erode_image(rctx, info, iters, ep, mode)
    assert np.array_equal(rctx.read_heightmap(), want)                                            # the read completes the erosion first


def test_after_a_set_image_heightmap_job(tw, scene, rctx):
    cfg = _cfg(scene)
    n, iters = 640, 3000
    args = (n, n, float(cfg.dx_val), float(cfg.dy_val), cfg.height_params(), iters, cfg.erosion_params())
    data16 = np.zeros(2 * n * n, np.uint8)
    rctx.proc_gen_heightmap_launch(*args, data16=data16)
    assert rctx.create_tiles_poll(True)
    rctx.proc_gen_heightmap_launch(*args, set_image=True)
    out = _dest("device", n, n)
    rctx.read_heightmap_launch(out=out)                                                           # completes the heightmap job first
    assert rctx.create_tiles_poll(True)
    assert np.array_equal(_host(out).reshape(-1), data16)


def test_after_update_heightmap(tw, rctx):
    rng = np.random.default_rng(5)
    W, H = 900, 400
    img = _img(rng, W, H)
    rctx.set_heightmap(img)
    for rects in ([(3, 3, 5, 5)], [(100, 0, 800, 400), (0, 399, 900, 1)], [(int(rng.integers(0, 800)), int(rng.integers(0, 300)), 77, 55) for _ in range(30)]):
        for x, y, w, h in rects:
            img[y:y + h, x:x + w] = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        rctx.update_heightmap(img, rects)
        assert np.array_equal(rctx.read_heightmap(), img)


# ---- ordering
def _frame(tw, c, W, H, zv=128):
    """A heightmap tile frame over the whole image (unit sampler: each cell is hi + lo/256 of one texel), launched on c; returns its zvals."""
    hs = tw.HmapSampler(W, H, 0, 1.0, 1.0, 1.0, 0.0, 1.0)
    nx, ny = -(-W // zv), -(-H // zv)
    org = np.array([(tx * zv - W // 2, ty * zv - H // 2) for ty in range(ny) for tx in range(nx)], np.int32)
    z = np.empty((len(org), zv, zv), np.float32)
    c.create_tiles_launch(org, (zv, zv), 1.0, 1.0, zv, None, 0, None, 0.0, z, hmap=hs)
    return z


def test_shared_contexts_see_the_edits_made_before_their_launch(tw):
    rng = np.random.default_rng(6)
    W, H = 4000, 3000
    old = _img(rng, W, H)
    new = old.copy()
    rects = [(100, 200, 3000, 1000), (7, 2900, 3993, 100)]
    for x, y, w, h in rects:
        new[y:y + h, x:x + w] = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
    c = tw.Context(0)
    try:
        a, b, f = c.shared(), c.shared(), c.shared()
        c.set_heightmap(old)
        z_old = _frame(tw, c, W, H)
        assert c.create_tiles_poll(True)
        for with_frame in (False, True):
            c.set_heightmap(old)
            z = _frame(tw, f, W, H) if with_frame else None                                      # a frame in flight on a third context
            before = a.read_heightmap_launch(out=_dest("pinned", H, W))
            c.update_heightmap(new, rects)
            after = b.read_heightmap_launch(out=_dest("device", H, W))
            assert np.array_equal(_host(before.poll(wait=True)), old)
            assert np.array_equal(_host(after.poll(wait=True)), new)
            if with_frame:
                assert f.create_tiles_poll(True)
                assert np.array_equal(z.view(np.uint32), z_old.view(np.uint32))
    finally:
        c.close()


def test_shared_read_while_the_root_erodes_the_image(tw, scene):
    n, iters = 512, 3000
    c = tw.Context(0)
    try:
        s = c.shared()
        cfg, img, info = _image(c, scene, n)
        ep = cfg.erosion_params()
        want = _chain(c, img, info, n, iters, ep, "serial")
        c.set_heightmap(img)
        assert np.array_equal(s.read_heightmap(), img)
        c.erode_image_launch(info.val_mult, info.val_add, iters, ep)
        with pytest.raises(tw.TwError) as e:
            s.read_heightmap(out=np.zeros((n, n, 2), np.uint8))
        assert e.value.status == tw.TW_ERR_STATE
        assert np.array_equal(c.read_heightmap(), want)                                           # the root's read completes the erosion first
        assert np.array_equal(s.read_heightmap(), want)
    finally:
        c.close()


def test_brush_after_erosion(tw, scene, rctx):
    """Erode on the device, read the image back, change a rect of the CPU copy, update_heightmap: the eroded image outside the rect, the edit inside."""
    n, iters = 512, 4000
    cfg, img, info = _image(rctx, scene, n)
    ep = cfg.erosion_params()
    eroded = _chain(rctx, img, info, n, iters, ep, "serial")
    rctx.set_heightmap(img)
    rctx.erode_image_launch(info.val_mult, info.val_add, iters, ep)
    cpu = rctx.read_heightmap()
    assert np.array_equal(cpu, eroded)
    x, y, w, h = 130, 77, 41, 29
    cpu[y:y + h, x:x + w, 1] ^= 0x11
    rctx.update_heightmap(cpu, [(x, y, w, h)])
    got = rctx.read_heightmap()
    inside = np.zeros((n, n), bool)
    inside[y:y + h, x:x + w] = True
    assert np.array_equal(got[~inside], eroded[~inside]) and np.array_equal(got[inside], cpu[inside])
    assert not np.array_equal(got[inside], eroded[inside])


# ---- an image of more than 2^31 bytes
def test_image_beyond_2_31_bytes(tw):
    W, H = 32768, 32769                                                                           # 2*W*H = 2^31 + 2^16 bytes
    nbytes = 2 * W * H
    if torch.cuda.mem_get_info()[0] < 3 * nbytes + (2 << 30):
        pytest.skip("not enough free device memory for three %d-byte images" % nbytes)
    c = tw.Context(0)
    try:
        src = torch.randint(0, 256, (H, W, 2), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        c.set_heightmap(src)
        out = torch.zeros_like(src)
        torch.cuda.synchronize()
        c.read_heightmap(out=out)
        assert torch.equal(out, src)
        rect = (W - 1000, H - 3, 1000, 3)                                                         # a rect in the last rows: offsets beyond 2^31 bytes
        out.zero_()
        torch.cuda.synchronize()
        c.read_heightmap([rect], out)
        assert torch.equal(out[H - 3:, W - 1000:], src[H - 3:, W - 1000:])
        assert int(out[:, :W - 1000].count_nonzero()) == 0 and int(out[:H - 3].count_nonzero()) == 0
        small = np.zeros((3, W, 2), np.uint8)                                                     # a host destination holding only those rows
        c.read_heightmap([rect], _dest_rows(small, H))
        assert np.array_equal(small[:, W - 1000:], src[H - 3:, W - 1000:].cpu().numpy()) and not small[:, :W - 1000].any()
    finally:
        c.close()


def _dest_rows(a, H):
    """A host view whose row y = H - len(a) + i is a[i]: a destination for a rect in the image's last rows (a strided numpy view starting before a)."""
    rows = a.shape[0]
    base = a.ctypes.data - (H - rows) * a.strides[0]
    buf = (C.c_uint8 * (H * a.strides[0])).from_address(base)
    return np.ndarray((H, a.shape[1], 2), np.uint8, buffer=buf, strides=a.strides)


# ---- cancel, refusals, nothing to do
def test_cancel_changes_nothing(tw, rctx):
    img = _img(np.random.default_rng(7), 2048, 1024)
    rctx.set_heightmap(img)
    out = np.zeros_like(img)
    job = rctx.read_heightmap_launch(out=out)
    assert tw.lib.tw_cancel(rctx._h) == tw.TW_ERR_STATE
    assert np.array_equal(job.poll(wait=True), img)


def test_refusals_and_nothing_to_do(tw):
    c = tw.Context(0)
    try:
        buf = np.zeros((40, 40, 2), np.uint8)

        def launch(rects, dst, pitch, n=None):
            arr, m = tw._rects(rects)
            a = tw.HmapReadArgs(C.cast(arr, C.c_void_p) if arr is not None else None, m if n is None else n, dst, pitch)
            return tw.lib.tw_read_heightmap_launch(c._h, C.byref(a))
        p = C.c_void_p(buf.ctypes.data)
        assert launch([(0, 0, 1, 1)], p, 80) == tw.TW_ERR_STATE                                   # no image
        c.set_heightmap(np.zeros((30, 20, 2), np.uint8))
        n0 = c.launch_count
        for rects, dst, pitch, n in (([], p, 80, 1), ([(0, 0, 1, 1)], None, 80, None), ([(0, 0, 0, 1)], p, 80, None), ([(0, 0, 1, 0)], p, 80, None),
                                     ([(19, 0, 2, 1)], p, 80, None), ([(0, 29, 1, 2)], p, 80, None), ([(-1, 0, 2, 1)], p, 80, None),
                                     ([(0, 0, 20, 30), (5, 5, 10, 1)], p, 29, None), ([(5, 5, 10, 1)], p, 29, None)):
            assert launch(rects, dst, pitch, n) == tw.TW_ERR_ARG, (rects, pitch)
        assert tw.lib.tw_read_heightmap_launch(c._h, None) == tw.TW_ERR_ARG
        assert launch([], None, 0) == tw.TW_OK and launch([(0, 0, 5, 5)], p, 80, 0) == tw.TW_OK    # nrects == 0
        assert launch([(5, 5, 10, 1)], p, 30) == tw.TW_OK                                          # dst_pitch = 2*(x + w) exactly
        assert c.create_tiles_poll(True)
        assert c.launch_count == n0 + 1
    finally:
        c.close()
