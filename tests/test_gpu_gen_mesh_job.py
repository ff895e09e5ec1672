"""GPU: the ground-mode mesh as one asynchronous job (tw_gen_mesh_launch, Context.gen_mesh_launch, scene.gen_mesh_async), bit for bit against the golden
fixtures of the reference's gen_mesh() and against the synchronous chain scene.gen_mesh: every gen mode and shape, with and without glaciation, a custom
glaciation exponent, scroll offsets, a flat mesh, the whole-map, single-walk and speculative erosion paths, device / pinned / pageable meshes, a shared
context beside a tile job, tw_cancel, and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

from cases import HM_CFG

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = np.float32
ZKEYS = ("zmin", "zmax", "zmax_est", "zbottom", "ztop", "water_plane_z")


def same(a, b):
    a, b = np.ascontiguousarray(a, F).ravel(), np.ascontiguousarray(b, F).ravel()
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def zsame(got, want):
    return all(F(got[k]).view(np.uint32) == F(want[k]).view(np.uint32) for k in ZKEYS)


def host(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else t


def job_and_chain(ctx, scene, cfg, iters, xoff2=0, yoff2=0, mesh=None):
    """(job mesh, job info, job steps), (chain mesh, chain info, chain steps) for the same arguments; the chain is scene.gen_mesh."""
    zmax_est = cfg.zmax_est
    want, zw, sp = scene.gen_mesh(ctx, cfg, erosion_iters=iters, xoff2=xoff2, yoff2=yoff2)
    steps_w = ctx.last_erosion_steps if iters else 0
    cfg.zmax_est = zmax_est                                    # the job ignores it; restore it so both start from the same configuration
    job, sp2 = scene.gen_mesh_async(ctx, cfg, iters, xoff2, yoff2, mesh=mesh)
    assert same(sp, sp2)
    got, z = job.poll(True)
    return (host(got), z, ctx.last_erosion_steps), (want, zw, steps_w)


def check(ctx, scene, cfg, iters, xoff2=0, yoff2=0, mesh=None):
    (got, z, steps), (want, zw, steps_w) = job_and_chain(ctx, scene, cfg, iters, xoff2, yoff2, mesh)
    assert same(got, want)
    assert zsame(z, zw)
    assert steps == steps_w == z["erosion_moves"]
    return z


@pytest.mark.parametrize("name", ["gm_cfg1", "gm_cfg1_eroded", "gm_simplex"])
def test_job_matches_reference_golden(tw, scene, ctx, name):
    h = np.load(os.path.join(GOLD, "height.npz"))
    mode, seed, ff, iters, mhs, smag, sfreq, sbias = h[name + "_args"]
    hmap = dict(sine_mag=float(smag), sine_freq=float(sfreq), sine_bias=float(sbias)) if smag else {}
    cfg = scene.SceneConfig(mesh_gen_mode=int(mode), mesh_freq_filter=int(ff), mesh_seed=int(seed), mesh_height=float(mhs), hmap=hmap)
    cfg.clip_hd1 = lambda: 0.5           # the fixture was generated with clip_hd1 = 0.5, relh_adj_tex = 0
    job, _ = scene.gen_mesh_async(ctx, cfg, int(iters))
    mesh, z = job.poll(True)
    assert same(mesh, h[name])
    assert same(np.array([z[k] for k in ZKEYS], F), h[name + "_zvals"])


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("shape", [0, 1, 2])
def test_job_equals_chain_modes_shapes(tw, scene, ctx, mode, shape):
    for glaciate, exp, iters in ((1, 0.0, 700), (0, 0.0, 300), (1, 2.2, 0)):
        cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_gen_shape=shape, mesh_freq_filter=1, mesh_seed=3 + mode, glaciate=glaciate, custom_glaciate_exp=exp,
                                hmap=HM_CFG, water_h_off=0.05, water_h_off_rel=-0.03, relh_adj_tex=0.02)
        check(ctx, scene, cfg, iters)


def test_job_equals_chain_offsets_and_custom_exponent(tw, scene, ctx):
    for mode, seed, xoff2, yoff2, exp in ((0, 6, 37, -512, 0.0), (2, 9, -1000, 250, 1.7), (4, 2, 4096, -77, 2.5)):
        cfg = scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=seed, custom_glaciate_exp=exp,
                                hmap=dict(HM_CFG, volcano_width=300.0, volcano_height=2.0))
        check(ctx, scene, cfg, 500, xoff2, yoff2)


def test_flat_mesh_keeps_the_previous_values(tw, scene, ctx):
    """All sine magnitudes 0: estimate_zminmax returns before set_zvals (tw3d::gen_mesh's flat branch). The chain here is the adapter's, step by step."""
    for glaciate, iters in ((0, 400), (1, 400)):
        cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_seed=5, glaciate=glaciate)
        sp = np.array(cfg.sine_params(), F).reshape(-1, 5)
        sp[:, 0] = 0.0
        ctx.set_sine_params(sp)
        hp, ep = cfg.height_params(), cfg.erosion_params()
        prev = (0.25, 0.75, -0.125)
        job = ctx.gen_mesh_launch(cfg.mesh_size[:2], hp, ep, iters, 3, -4, float(cfg.dx_val), float(cfg.dy_val), cfg.scene_size[:2], prev=prev)
        got, z = job.poll(True)
        steps = ctx.last_erosion_steps
        MX, MY = cfg.mesh_size[:2]
        mesh, (zmin, zmax) = ctx.heightgen_2d(tw.Grid2D(float(3 - MX // 2), float(-4 - MY // 2), float(cfg.dx_val), float(cfg.dy_val), MX, MY), hp,
                                              enable_glaciate=0, want_minmax=True)
        zmin, zmax = F(zmin), F(zmax)
        assert zmin == zmax
        zmax_est = F(float(-zmin if zmax < -zmin else zmax) + 1.0E-6)
        zb, zt, wpz = (F(v) for v in prev)
        hp.zmax_est = float(zmax_est)
        if glaciate:
            zb, zt = ctx.glaciate_mesh(mesh, 3, -4, (MX, MY), hp)
        ctx.erode(mesh, float(zb), iters, tw.ErosionParams(ep.erode_amount, float(wpz), ep.half_dxy, float(zmin), float(zmax), ep.relh_adj_tex, ep.clip_hd1))
        assert same(got, mesh) and steps == ctx.last_erosion_steps == z["erosion_moves"]
        assert zsame(z, dict(zmin=zmin, zmax=zmax, zmax_est=zmax_est, zbottom=zb, ztop=zt, water_plane_z=wpz))


@pytest.mark.parametrize("size,iters", [(130, 5000), (512, 3000), (1024, 20000), (2048, 4000)])
def test_job_equals_chain_erosion_paths(tw, scene, ctx, size, iters):
    """130^2: the whole map in shared memory (and the cancellable walk); 512^2: the one-warp walk; 1024^2 and 2048^2: M_SPEC's rounds."""
    cfg = scene.SceneConfig(mesh_size=(size, size, 1), scene_size=(size / 32.0, size / 32.0, 4.0), mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG)
    z = check(ctx, scene, cfg, iters)
    assert z["erosion_moves"] > iters


@pytest.mark.parametrize("kind", ["device", "pinned", "pageable_tensor"])
def test_job_outputs(tw, scene, ctx, kind):
    import torch
    cfg = scene.SceneConfig(mesh_gen_mode=1, mesh_freq_filter=1, mesh_seed=4, hmap=HM_CFG)
    MX, MY = cfg.mesh_size[:2]
    mesh = {"device": lambda: torch.full((MY, MX), float("nan"), device="cuda"),
            "pinned": lambda: torch.full((MY, MX), float("nan")).pin_memory(),
            "pageable_tensor": lambda: torch.full((MY, MX), float("nan"))}[kind]()
    check(ctx, scene, cfg, 600, mesh=mesh)


def test_shared_context_beside_a_tile_job(tw, scene):
    import torch
    root = tw.Context(0)
    try:
        s = root.shared()
        cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_freq_filter=1, mesh_seed=6, hmap=HM_CFG)
        want, zw, sp = scene.gen_mesh(root, cfg, erosion_iters=1500)
        steps_w = root.last_erosion_steps
        hp, ep = cfg.height_params(), cfg.erosion_params()
        org = np.array([[x * 256, y * 256] for y in range(4) for x in range(4)], np.int32)
        zt = torch.empty((16, 258, 258), device="cuda")
        root.create_tiles_launch(org, (128, 128), float(cfg.dx_val), float(cfg.dy_val), 258, hp, 1000, ep, -1.0, zt)
        mesh = torch.empty((128, 128)).pin_memory()
        job = s.gen_mesh_launch(cfg.mesh_size[:2], hp, ep, 1500, 0, 0, float(cfg.dx_val), float(cfg.dy_val), cfg.scene_size[:2],
                                cfg.water_h_off, cfg.water_h_off_rel, mesh=mesh)
        got, z = job.poll(True)
        assert root.create_tiles_poll(True)
        assert same(host(got), want) and zsame(z, zw) and s.last_erosion_steps == steps_w
        ref = torch.empty_like(zt)
        root.create_tiles_launch(org, (128, 128), float(cfg.dx_val), float(cfg.dy_val), 258, hp, 1000, ep, -1.0, ref)
        assert root.create_tiles_poll(True)
        assert torch.equal(zt, ref)
    finally:
        root.close()


def test_cancel_stops_a_long_erosion(tw, scene, ctx):
    cfg = scene.SceneConfig(mesh_size=(2048, 2048, 1), scene_size=(64.0, 64.0, 4.0), mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG)
    job, _ = scene.gen_mesh_async(ctx, cfg, 2000000)
    ctx.cancel()
    with pytest.raises(tw.TwCanceled):
        job.poll(True)
    assert ctx.last_erosion_steps == 0
    small = scene.SceneConfig(mesh_gen_mode=2, mesh_freq_filter=1, mesh_seed=8, hmap=HM_CFG)
    check(ctx, scene, small, 800)                              # the next job on the context is unaffected


def test_refusals_enqueue_nothing(tw, scene):
    root = tw.Context(0)
    try:
        s = root.shared()
        cfg = scene.SceneConfig(mesh_gen_mode=0, mesh_seed=2)
        hp, ep = cfg.height_params(), cfg.erosion_params()
        mesh = np.zeros((128, 128), F)
        info = tw.GenMeshInfo()

        def status(c, MX=128, MY=128, hp_=hp, ep_=ep, mesh_=mesh):
            ref = lambda v: C.cast(C.pointer(v), C.c_void_p) if v is not None else None  # noqa: E731
            a = tw.GenMeshJobArgs(MX, MY, 0, 0, float(cfg.dx_val), float(cfg.dy_val), 4.0, 4.0, ref(hp_), 100, ref(ep_), 0.0, 0.0, 0.0, 0.0, 0.0,
                                  tw._ptr(mesh_), C.cast(C.pointer(info), C.c_void_p))
            before = c.launch_count
            rc = tw.lib.tw_gen_mesh_launch(c._h, C.byref(a))
            assert c.launch_count == before and c.create_tiles_poll(False)
            return rc
        ARG, STATE = tw.TW_ERR_ARG, tw.TW_ERR_STATE
        for c in (root, s):
            assert status(c) == STATE                                              # sine mode without the sine params
        root.set_sine_params(cfg.sine_params())
        assert tw.lib.tw_gen_mesh_launch(root._h, None) == ARG
        assert tw.lib.tw_gen_mesh_launch(None, None) == ARG
        hp_bad = cfg.height_params()
        hp_bad.start_eval_sin = 91
        hp_mode = cfg.height_params()
        hp_mode.gen_mode = 7
        for c in (root, s):
            assert status(c, hp_=None) == ARG
            assert status(c, ep_=None) == ARG
            assert status(c, mesh_=None) == ARG
            assert status(c, MX=0) == ARG
            assert status(c, MY=-1) == ARG
            assert status(c, MY=65536) == ARG
            assert status(c, hp_=hp_bad) == ARG
            assert status(c, hp_=hp_mode) == ARG
        for c in (root, s):                                                        # the next job gives the normal result
            job = c.gen_mesh_launch(cfg.mesh_size[:2], hp, ep, 300, 0, 0, float(cfg.dx_val), float(cfg.dy_val), cfg.scene_size[:2])
            got, z = job.poll(True)
            want, zw, _ = scene.gen_mesh(root, cfg, erosion_iters=300, sine_rng=None)
            assert same(got, want) and zsame(z, zw)
    finally:
        root.close()
