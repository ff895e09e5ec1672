"""GPU: mesh shadows of one whole mesh (tw_mesh_shadows, tw_mesh_shadows_launch, tw_gen_mesh_launch_shadows) bit for bit against the oracle's
calc_mesh_shadows: square and non-square meshes from 2x2 to 4096x1024 on non-square cells, lights in every octant, on an axis, diagonal, below zmin,
no_shadow and straight overhead, incoming rows with MESH_MIN_Z entries; host, pinned and device buffers and several lights in one launch; a mesh of more than
2^31 cells against a known answer; each golden tile traced alone with its neighbours' fixture edges; and the ground-mode job with shadows against the chain
scene.gen_mesh -> tw_mesh_shadows over every gen mode and erosion path, beside a tile job on a shared context, cancelled, and refused."""
import ctypes as C
import os

import numpy as np
import pytest

from cases import HM_CFG, convert

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = np.float32
MIN_Z = F(-1.0e6)


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def host(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def assert_same(got, want):
    (m, ox, oy), (mw, oxw, oyw) = [tuple(host(v) for v in r) for r in (got, want)]
    assert np.array_equal(m, mw), "smask differs in %d cells" % int((m != mw).sum())
    assert np.array_equal(bits(ox), bits(oxw)) and np.array_equal(bits(oy), bits(oyw)), "sh_out differs"


def shadow_params(tw, xs, ys, lpos, zmin, zmax, dx=0.0625, dy=0.046875, no_shadow=0):
    sp = tw.ShadowParams()
    for d in range(3):
        sp.lpos[d] = lpos[d]
    sp.dx_val, sp.dy_val = dx, dy
    sp.x_scene_size, sp.y_scene_size = float(F(0.5) * F(dx) * F(xs)), float(F(0.5) * F(dy) * F(ys))
    sp.dx_val_inv, sp.dy_val_inv = float(F(1.0) / F(dx)), float(F(1.0) / F(dy))
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = xs + ys, zmin, zmax, no_shadow
    return sp


def terrain(xs, ys, seed):
    rng = np.random.default_rng(seed)
    x, y = np.meshgrid(np.linspace(0, 7, xs, dtype=F), np.linspace(0, 5, ys, dtype=F))
    return (F(0.6) * np.sin(x * F(1.3)) * np.cos(y * F(0.9)) + F(0.25) * rng.standard_normal((ys, xs)).astype(F)).astype(F)


LIGHTS = [(3.0, 2.0, 1.0), (-4.0, 1.0, 0.5), (1.0, -5.0, 0.7), (-2.0, -2.0, 3.0), (0.3, 6.0, 0.2), (-6.0, -0.4, 0.15), (5.0, 0.0, 1.0), (0.0, -3.0, 2.0),
          (2.0, 2.0, 1.0), (-1.0, 1.0, 8.0), (0.0, 0.0, 5.0), (2.0, 1.0, -3.0)]          # octants, steep / grazing, axes, diagonals, overhead, below zmin


def incoming(z, rng):
    six = np.where(rng.random(z.shape[1]) < 0.3, MIN_Z, z[0] + rng.uniform(-0.2, 0.6, z.shape[1])).astype(F)
    siy = np.where(rng.random(z.shape[0]) < 0.3, MIN_Z, z[:, 0] + rng.uniform(-0.2, 0.6, z.shape[0])).astype(F)
    return six, siy


@pytest.mark.parametrize("xs,ys", [(2, 2), (3, 2), (2, 513), (64, 200), (333, 97), (1000, 37), (256, 256), (4096, 1024)])
def test_blocking_call_matches_oracle(tw, oracle, ctx, xs, ys):
    z = terrain(xs, ys, xs * 7 + ys)
    rng = np.random.default_rng(xs + ys)
    zlo, zhi = float(z.min()) - 0.5, float(z.max()) + 0.5
    lights = LIGHTS if xs * ys <= 1 << 20 else LIGHTS[::3] + [LIGHTS[-1]]
    for lp in lights:
        sp = shadow_params(tw, xs, ys, lp, zlo, zhi)
        for with_in in (0, 1):
            six, siy = incoming(z, rng) if with_in else (None, None)
            assert_same(ctx.mesh_shadows(z, sp, six, siy), oracle.calc_mesh_shadows(convert(sp, oracle.ShadowParams), z, six, siy))
    sp = shadow_params(tw, xs, ys, (1.0, 2.0, 0.5), zlo, zhi, no_shadow=1)
    assert_same(ctx.mesh_shadows(z, sp), oracle.calc_mesh_shadows(convert(sp, oracle.ShadowParams), z))


def test_buffers_and_lights_in_one_launch(tw, oracle, ctx):
    import torch
    xs, ys = 300, 170
    z = terrain(xs, ys, 3)
    six, siy = incoming(z, np.random.default_rng(4))
    zlo, zhi = float(z.min()) - 0.5, float(z.max()) + 0.5
    sps = [shadow_params(tw, xs, ys, lp, zlo, zhi) for lp in LIGHTS]
    want = [oracle.calc_mesh_shadows(convert(sp, oracle.ShadowParams), z, six, siy) for sp in sps]
    outs = {"host": lambda shape, dt: np.empty(shape, dt),
            "pinned": lambda shape, dt: torch.empty(shape, dtype=dt).pin_memory(),
            "device": lambda shape, dt: torch.empty(shape, dtype=dt, device="cuda")}
    tdt = {np.uint8: torch.uint8, np.float32: torch.float32}
    for mesh_kind in ("host", "pinned", "device"):
        mesh = z if mesh_kind == "host" else torch.from_numpy(z).pin_memory() if mesh_kind == "pinned" else torch.from_numpy(z).cuda()
        for out_kind, make in outs.items():
            mk = (lambda s, d: make(s, d)) if out_kind == "host" else (lambda s, d: make(s, tdt[d]))
            lights = [tw.Light(sp, mk((ys, xs), np.uint8), mk(xs, np.float32), mk(ys, np.float32),
                               six if mesh_kind != "device" else torch.from_numpy(six).cuda(), siy) for sp in sps]
            job = ctx.mesh_shadows_launch(mesh, lights)
            got = job.poll(True)
            for g, w in zip(got, want):
                assert_same(g, w)
    # each light of one launch equals its own blocking call, also without incoming rows and without outputs other than the mask
    got = ctx.mesh_shadows_launch(z, sps).poll(True)
    for g, sp in zip(got, sps):
        assert_same(g, ctx.mesh_shadows(z, sp))


def test_refusals_enqueue_nothing(tw, ctx):
    import torch
    xs, ys = 40, 30
    z = terrain(xs, ys, 5)
    sp = shadow_params(tw, xs, ys, (1.0, 1.0, 1.0), -2.0, 2.0)
    m, ox, oy = np.empty((ys, xs), np.uint8), np.empty(xs, F), np.empty(ys, F)
    dm = torch.empty(xs * ys + 8, dtype=torch.uint8, device="cuda")
    ARG, L = tw.TW_ERR_ARG, tw.lib
    P = tw._ptr

    def refused(call):
        before = ctx.launch_count
        assert call() == ARG
        assert ctx.launch_count == before and ctx.create_tiles_poll(False)
    refused(lambda: L.tw_mesh_shadows(ctx._h, None, xs, ys, C.byref(sp), None, None, P(m), P(ox), P(oy)))
    refused(lambda: L.tw_mesh_shadows(ctx._h, P(z), xs, ys, None, None, None, P(m), P(ox), P(oy)))
    refused(lambda: L.tw_mesh_shadows(ctx._h, P(z), xs, ys, C.byref(sp), None, None, None, P(ox), P(oy)))
    for bx, by in ((1, ys), (xs, 1), (0, 0), (-5, ys), (1 << 29, 1 << 29)):
        refused(lambda: L.tw_mesh_shadows(ctx._h, P(z), bx, by, C.byref(sp), None, None, P(m), P(ox), P(oy)))
    refused(lambda: L.tw_mesh_shadows(ctx._h, P(z), xs, ys, C.byref(sp), None, None, C.c_void_p(dm.data_ptr() + 1), None, None))  # misaligned device smask
    assert L.tw_mesh_shadows(None, P(z), xs, ys, C.byref(sp), None, None, P(m), None, None) == ARG
    light = tw.TileLight(sp, None, None, P(m), P(ox), P(oy))
    refused(lambda: L.tw_mesh_shadows_launch(ctx._h, C.byref(tw.MeshShadowsJobArgs(P(z), xs, ys, 0, C.cast(C.pointer(light), C.c_void_p)))))
    refused(lambda: L.tw_mesh_shadows_launch(ctx._h, C.byref(tw.MeshShadowsJobArgs(P(z), xs, ys, 1, None))))
    refused(lambda: L.tw_mesh_shadows_launch(ctx._h, None))
    good = ctx.mesh_shadows(z, sp)                                 # the context works normally afterwards; an aligned device mask is taken
    dm4 = dm[4:4 + xs * ys].view(ys, xs)
    ctx.mesh_shadows_launch(z, [tw.Light(sp, dm4)]).poll(True)
    assert np.array_equal(dm4.cpu().numpy(), good[0])


def known_answer(xs, ys, spikes, dx):
    """Flat zero mesh, light (1, 0, 1) (rays run along rows toward -x, dir_ratio exactly 1), spikes (row, col, k) of height (k + 0.5)*dx in the last row:
    each shades the k cells before it in its row with heights h - j*dx, and those are the sh_out_x entries (every ray ends in its own row); sh_out_y stays
    MESH_MIN_Z (no shadowed cell at x = 0)."""
    m, ox, oy = np.zeros((ys, xs), np.uint8), np.full(xs, MIN_Z), np.full(ys, MIN_Z)
    for r, c, k in spikes:
        h = F((k + 0.5) * dx)
        for j in range(1, k + 1):
            m[r, c - j] = 2
            ox[c - j] = F(float(h) - j * dx)
    return m, ox, oy


def spike_params(tw, xs, ys, dx):
    sp = tw.ShadowParams()
    sp.lpos[0], sp.lpos[1], sp.lpos[2] = 1.0, 0.0, 1.0
    sp.dx_val = sp.dy_val = dx
    sp.x_scene_size, sp.y_scene_size = float(F(dx) * F(xs) * F(0.5)), float(F(dx) * F(ys) * F(0.5))
    sp.dx_val_inv = sp.dy_val_inv = 1.0 / dx
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = xs + ys, -1.0, 1.0, 0
    return sp


def test_mesh_beyond_2_31_cells(tw, oracle, ctx):
    import torch
    dx = 2.0 ** -6
    # the known answer, first held to the oracle on a small mesh of the same kind
    xs, ys = 400, 5
    spikes = [(ys - 1, 380, 10), (ys - 1, 200, 3), (ys - 1, 40, 25)]
    z = np.zeros((ys, xs), F)
    for r, c, k in spikes:
        z[r, c] = F((k + 0.5) * dx)
    sp = spike_params(tw, xs, ys, dx)
    want = known_answer(xs, ys, spikes, dx)
    assert_same(oracle.calc_mesh_shadows(convert(sp, oracle.ShadowParams), z), want)
    assert_same(ctx.mesh_shadows(z, sp), want)
    n = 46341                                                      # 46341^2 = 2^31 + 4633 cells: the last row's columns >= 41708 lie beyond cell 2^31
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * (1 << 30):
        pytest.skip("needs about 11 GB of free device memory")
    spikes = [(n - 1, 46300, 12), (n - 1, 45000, 40), (n - 1, 41720, 5)]
    assert all((n - 1) * n + c - k >= 1 << 31 for _, c, k in spikes)
    mesh = torch.zeros((n, n), device="cuda")
    for r, c, k in spikes:
        mesh[r, c] = float(F((k + 0.5) * dx))
    m = torch.empty((n, n), dtype=torch.uint8, device="cuda")
    ox, oy = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    ctx.mesh_shadows_launch(mesh, [tw.Light(spike_params(tw, n, n, dx), m, ox, oy)]).poll(True)
    del mesh
    wm, wox, woy = known_answer(n, 1, [(0, c, k) for _, c, k in spikes], dx)
    assert int(m[:-1].count_nonzero()) == 0
    assert np.array_equal(m[-1].cpu().numpy(), wm[0])
    assert np.array_equal(bits(ox.cpu().numpy()), bits(wox)) and np.array_equal(bits(oy.cpu().numpy()), bits(np.full(n, MIN_Z)))


def test_golden_tiles_traced_alone(tw, ctx):
    """Each tile of the reference fixture as a mesh of its own, starting from the fixture's sh_out of its neighbours toward the light (MESH_MIN_Z where
    the tile has none): its mask and sh_out are the fixture's."""
    gs = np.load(os.path.join(GOLD, "shadows.npz"))
    txy = [tuple(int(v) for v in t) for t in gs["tile_xy"]]
    where = {t: i for i, t in enumerate(txy)}
    a = gs["params"]
    zv = gs["tiles"].shape[1]
    for li, lp in enumerate(gs["lights"]):
        sp = tw.ShadowParams()
        sp.x_scene_size, sp.y_scene_size, sp.dx_val, sp.dy_val = float(a[0]), float(a[1]), float(a[2]), float(a[3])
        sp.dx_val_inv, sp.dy_val_inv = 1.0 / np.float32(a[2]), 1.0 / np.float32(a[3])
        sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = int(a[4]), float(a[5]), float(a[6]), 0
        for d in range(3):
            sp.lpos[d] = float(lp[d])
        sx, sy = (-1 if lp[0] < 0 else 1), (-1 if lp[1] < 0 else 1)
        ox, oy = gs["sh_out_x_%d" % li], gs["sh_out_y_%d" % li]
        for t, (x, y) in enumerate(txy):
            ny, nx = where.get((x, y + sy)), where.get((x + sx, y))
            six = ox[ny] if ny is not None else np.full(zv, MIN_Z)
            siy = oy[nx] if nx is not None else np.full(zv, MIN_Z)
            got = ctx.mesh_shadows(gs["tiles"][t], sp, six, siy)
            assert_same(got, (gs["smask_%d" % li][t], ox[t], oy[t]))


# ---- tw_gen_mesh_launch_shadows against scene.gen_mesh -> tw_mesh_shadows ----
def sun_moon(scene, cfg, zmin=0.0, zmax=0.0):
    return [scene.mesh_shadow_params(cfg, (3.0, -2.0, 1.2), zmin, zmax), scene.mesh_shadow_params(cfg, (-1.5, -4.0, 0.6), zmin, zmax),
            scene.mesh_shadow_params(cfg, (0.0, 5.0, 0.3), zmin, zmax, no_shadow=True)]


def check_job(tw, scene, ctx, cfg, iters, mesh=None):
    zmax_est = cfg.zmax_est
    want, zw, _ = scene.gen_mesh(ctx, cfg, erosion_iters=iters)
    steps_w = ctx.last_erosion_steps if iters else 0
    shadows_w = [ctx.mesh_shadows(want, sp) for sp in sun_moon(scene, cfg, zw["zmin"], zw["zmax"])]
    cfg.zmax_est = zmax_est
    job, _ = scene.gen_mesh_async(ctx, cfg, iters, mesh=mesh)
    plain, z0 = job.poll(True)
    plain = host(plain).copy()
    steps0 = ctx.last_erosion_steps
    cfg.zmax_est = zmax_est
    job, _ = scene.gen_mesh_async(ctx, cfg, iters, mesh=mesh, lights=sun_moon(scene, cfg, -123.0, 456.0))  # their zmin / zmax are replaced
    got, z, shadows = job.poll(True)
    assert np.array_equal(bits(host(got)), bits(want)) and np.array_equal(bits(plain), bits(want))
    assert z == z0 and all(F(z[k]) == F(zw[k]) for k in zw)
    assert ctx.last_erosion_steps == steps0 == steps_w == z["erosion_moves"]
    for g, w in zip(shadows, shadows_w):
        assert_same(g, w)
    return z


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_job_equals_chain_modes(tw, scene, ctx, mode):
    for glaciate, iters in ((1, 700), (0, 300)):
        cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=3 + mode, glaciate=glaciate, hmap=HM_CFG, water_h_off=0.05, relh_adj_tex=0.02)
        check_job(tw, scene, ctx, cfg, iters)
    cfg = scene.SceneConfig(mesh_size=(256, 128, 1), scene_size=(8.0, 4.0, 4.0), mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=9, hmap=HM_CFG)
    check_job(tw, scene, ctx, cfg, 500)


@pytest.mark.parametrize("size,iters", [(130, 5000), (512, 3000), (1024, 20000), (2048, 4000)])
def test_job_equals_chain_erosion_paths(tw, scene, ctx, size, iters):
    cfg = scene.SceneConfig(mesh_size=(size, size, 1), scene_size=(size / 32.0, size / 32.0, 4.0), mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG)
    assert check_job(tw, scene, ctx, cfg, iters)["erosion_moves"] > iters


def test_job_flat_mesh_and_buffers(tw, scene, ctx):
    import torch
    cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_seed=5, glaciate=0)
    sp = np.array(cfg.sine_params(), F).reshape(-1, 5)
    sp[:, 0] = 0.0
    ctx.set_sine_params(sp)
    hp, ep = cfg.height_params(), cfg.erosion_params()
    prev = (0.25, 0.75, -0.125)
    args = (cfg.mesh_size[:2], hp, ep, 400, 3, -4, float(cfg.dx_val), float(cfg.dy_val), cfg.scene_size[:2])
    want, zw = ctx.gen_mesh_launch(*args, prev=prev).poll(True)
    got, z, sh = ctx.gen_mesh_launch(*args, prev=prev, lights=sun_moon(scene, cfg)).poll(True)
    assert np.array_equal(bits(got), bits(want)) and z == zw
    for g, s in zip(sh, sun_moon(scene, cfg, z["zmin"], z["zmax"])):
        assert_same(g, ctx.mesh_shadows(want, s))
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=4, hmap=HM_CFG)
    MX, MY = cfg.mesh_size[:2]
    for mesh in (torch.empty((MY, MX), device="cuda"), torch.empty((MY, MX)).pin_memory()):
        check_job(tw, scene, ctx, cfg, 600, mesh=mesh)
    want, zw, _ = scene.gen_mesh(ctx, cfg, erosion_iters=600)      # device and pinned outputs
    lights = [tw.Light(s, torch.empty((MY, MX), dtype=torch.uint8, device="cuda"), torch.empty(MX).pin_memory(), torch.empty(MY, device="cuda"))
              for s in sun_moon(scene, cfg)]
    _, _, sh = scene.gen_mesh_async(ctx, cfg, 600, lights=lights)[0].poll(True)
    for g, s in zip(sh, sun_moon(scene, cfg, zw["zmin"], zw["zmax"])):
        assert_same(g, ctx.mesh_shadows(want, s))


def test_job_on_shared_context_beside_a_tile_job(tw, scene):
    import torch
    root = tw.Context(0)
    try:
        s = root.shared()
        cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_freq_filter=1, mesh_seed=6, hmap=HM_CFG)
        want, zw, _ = scene.gen_mesh(root, cfg, erosion_iters=1500)
        shadows_w = [root.mesh_shadows(want, sp) for sp in sun_moon(scene, cfg, zw["zmin"], zw["zmax"])]
        hp, ep = cfg.height_params(), cfg.erosion_params()
        org = np.array([[x * 256, y * 256] for y in range(4) for x in range(4)], np.int32)
        zt = torch.empty((16, 258, 258), device="cuda")
        root.create_tiles_launch(org, (128, 128), float(cfg.dx_val), float(cfg.dy_val), 258, hp, 1000, ep, -1.0, zt)
        job = s.gen_mesh_launch(cfg.mesh_size[:2], hp, ep, 1500, 0, 0, float(cfg.dx_val), float(cfg.dy_val), cfg.scene_size[:2], cfg.water_h_off,
                                cfg.water_h_off_rel, mesh=torch.empty((128, 128)).pin_memory(), lights=sun_moon(scene, cfg))
        got, z, sh = job.poll(True)
        assert root.create_tiles_poll(True)
        assert np.array_equal(bits(host(got)), bits(want))
        for g, w in zip(sh, shadows_w):
            assert_same(g, w)
        mjob = s.mesh_shadows_launch(torch.from_numpy(want).cuda(), sun_moon(scene, cfg, zw["zmin"], zw["zmax"]))
        root.create_tiles_launch(org, (128, 128), float(cfg.dx_val), float(cfg.dy_val), 258, hp, 1000, ep, -1.0, zt)
        for g, w in zip(mjob.poll(True), shadows_w):
            assert_same(g, w)
        assert root.create_tiles_poll(True)
    finally:
        root.close()


def test_cancel(tw, scene, ctx):
    cfg = scene.SceneConfig(mesh_size=(2048, 2048, 1), scene_size=(64.0, 64.0, 4.0), mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG)
    job, _ = scene.gen_mesh_async(ctx, cfg, 2000000, lights=sun_moon(scene, cfg))
    ctx.cancel()
    with pytest.raises(tw.TwCanceled):
        job.poll(True)
    z = terrain(2048, 2048, 1)
    sp = shadow_params(tw, 2048, 2048, (3.0, 1.0, 0.4), -2.0, 2.0)
    job = ctx.mesh_shadows_launch(z, [sp] * 8)
    ctx.cancel()
    try:
        job.poll(True)                                             # the rays may all have started before the cancel landed
    except tw.TwCanceled:
        pass
    small = scene.SceneConfig(mesh_gen_mode=2, mesh_freq_filter=1, mesh_seed=8, hmap=HM_CFG)
    check_job(tw, scene, ctx, small, 800)                          # the next job on the context is unaffected


def test_gen_mesh_refusals(tw, scene):
    root = tw.Context(0)
    try:
        cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_seed=2)
        root.set_sine_params(cfg.sine_params())
        hp, ep = cfg.height_params(), cfg.erosion_params()
        info = tw.GenMeshInfo()
        ref = lambda v: C.cast(C.pointer(v), C.c_void_p)  # noqa: E731

        def status(MX=128, MY=128, nlights=1, lights=True, smask=True, align=0):
            import torch
            mesh = np.zeros((MY, MX), F)
            dm = torch.empty(MX * MY + 8, dtype=torch.uint8, device="cuda")
            m = C.c_void_p(dm.data_ptr() + align) if smask else None
            arr = (tw.TileLight * 1)(tw.TileLight(scene.mesh_shadow_params(cfg, (1.0, 1.0, 1.0)), None, None, m, None, None))
            a = tw.GenMeshJobArgs(MX, MY, 0, 0, float(cfg.dx_val), float(cfg.dy_val), 4.0, 4.0, ref(hp), 100, ref(ep), 0.0, 0.0, 0.0, 0.0, 0.0,
                                  tw._ptr(mesh), ref(info))
            before = root.launch_count
            rc = tw.lib.tw_gen_mesh_launch_shadows(root._h, C.byref(a), nlights, C.cast(arr, C.c_void_p) if lights else None)
            assert root.launch_count == before and root.create_tiles_poll(False)
            return rc
        ARG = tw.TW_ERR_ARG
        assert status(lights=False) == ARG
        assert status(smask=False) == ARG
        assert status(align=2) == ARG
        assert status(MX=1, MY=128) == ARG and status(MX=128, MY=1) == ARG
        assert tw.lib.tw_gen_mesh_launch_shadows(None, None, 0, None) == ARG
        check_job(tw, scene, root, cfg, 300)
    finally:
        root.close()
