"""GPU: shared contexts (tw_create_shared, Context.shared()) - several asynchronous jobs in flight on one device, each context with its own stream, scratch
and pending job, all reading the parent's tables. Every output and erosion step count must equal the parent's blocking call bit for bit; a launch on one
context must not complete another's job; the parent's table setters complete the shared jobs first and the next shared job sees the new tables."""
import ctypes as C
import time

import numpy as np
import pytest

from test_gpu_tiles_shading import S, ZV, ITERS, _host, _origins, _weights_case
from test_gpu_tiles_shadows import SUN, MOON, _light, _grid
from cases import HM_CFG

pytestmark = pytest.mark.gpu


def _cfg(scene, mode, seed=1):
    return scene.SceneConfig(mesh_gen_mode=mode, mesh_freq_filter=1, mesh_seed=seed, hmap=HM_CFG, zmax_est=2.3, mesh_size=(S, S, 1), scene_size=(0.5, 0.5, 4.0))


def _parent(tw, scene, mode, img_n=512):
    """A parent context with the mode's sine params and a terrain image (tw_proc_gen_heightmap) set, and a mirror-edge sampler for the image."""
    P = tw.Context(0)
    cfg = _cfg(scene, mode)
    P.set_sine_params(cfg.sine_params())
    hp, ep = cfg.height_params(), cfg.erosion_params()
    dx, dy = float(cfg.dx_val), float(cfg.dy_val)
    img, hs = _image(tw, P, hp, ep, dx, dy, img_n)
    P.set_heightmap(img)
    return P, cfg, hp, ep, dx, dy, img, hs


def _image(tw, P, hp, ep, dx, dy, n, m=None):
    m = m or n
    data16, info, _ = P.proc_gen_heightmap(n, m, dx, dy, hp, 0, ep)
    hs = tw.HmapSampler(n, m, 2, 1.0, float(np.float32(0.0008) * np.float32(hp.mesh_height_scale)), info.mesh_file_scale, info.mesh_file_tz, hp.mesh_scale_z_inv)
    return data16.reshape(m, n, 2), hs


def _snap(outs):
    """The bytes of every output of a completed job."""
    r = []
    for o in outs:
        if o is None:
            r.append(None)
        elif hasattr(o, "cpu") or isinstance(o, np.ndarray):
            r.append(np.ascontiguousarray(_host(o)).tobytes())
        elif isinstance(o, C.Array) or isinstance(o, C.Structure):
            r.append(bytes(o))
        else:
            raise TypeError(type(o))
    return r


def _kinds(tw, torch, cfg, hp, ep, dx, dy, hs, where):
    """Every kind of asynchronous job: launch(c) enqueues it on context c and returns its output buffers."""
    origins = _origins(3)
    nt, wpz_max, hd = len(origins), float(ep.water_plane_z), 0.5 * (dx + dy)
    txy = _grid(3)
    wp, corners = _weights_case(tw, np.array([ep.zmin, ep.zmax], np.float32), S, dx, dy, nt)

    def buf(shape, dt):
        return torch.empty(shape, dtype=dt, device="cuda") if where == "device" else torch.empty(shape, dtype=dt).pin_memory()

    def base():
        return (buf((nt, ZV, ZV), torch.float32), buf((nt, ZV - 1, ZV - 1, 4), torch.uint8), np.empty((nt, 2), np.float32), (tw.TileBounds * nt)(),
                np.empty(nt, np.float32))

    def tiles(c, **kw):
        z, n, mm, b, mnz = base()
        extra = []
        if kw.pop("shading", False):
            extra = [buf((nt, ZV - 1, ZV - 1), torch.uint8) if "hmap" not in kw else None, buf((nt, ZV - 1, ZV - 1, 4), torch.uint8), buf((nt,), torch.uint8)]
            kw.update(ao=extra[0], weights=extra[1], has_any_grass=extra[2], half_dxy=hd, wp=wp, tile_params=corners)
        if kw.pop("shadows", False):
            lights = [tw.Light(_light(tw, ep, dx, dy, lp), buf((nt, ZV, ZV), torch.uint8), buf((nt, ZV), torch.float32), buf((nt, ZV), torch.float32)) for lp in (SUN, MOON)]
            kw.update(tile_xy=txy, lights=lights)
            extra = [x for L in lights for x in (L.smask, L.sh_out_x, L.sh_out_y)]
        c.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, mm=mm, bounds=b, normals=n, min_normal_z=mnz, wpz_max=wpz_max, size=S, **kw)
        return [z, n, mm, b, mnz] + extra

    def grid(c):
        g = cfg.heightmap_grid(700, 300)
        out, mm = buf((300, 700), torch.float32), tw.MinMax()
        c.heightgen_2d_launch(g, hp, 1, 0, out, mm)
        return [out, mm]

    return {"grid": grid, "tiles": tiles, "ex": lambda c: tiles(c, shading=True), "shadows": lambda c: tiles(c, shadows=True),
            "hmap": lambda c: tiles(c, hmap=hs, shading=True)}


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("mode", [0, 1, 4])
def test_all_job_kinds_in_flight_at_once(tw, scene, where, mode):
    import torch
    P, cfg, hp, ep, dx, dy, img, hs = _parent(tw, scene, mode)
    try:
        kinds = _kinds(tw, torch, cfg, hp, ep, dx, dy, hs, where)
        exp = {}
        for k, launch in kinds.items():                      # the parent's blocking calls
            outs = launch(P)
            assert P.create_tiles_poll(wait=True)
            exp[k] = (_snap(outs), P.last_erosion_steps)
        shared = {k: P.shared() for k in kinds}
        outs = {k: kinds[k](shared[k]) for k in kinds}        # every kind in flight on its own shared context ...
        outs_p = kinds["ex"](P)                               # ... and one on the parent
        launches = {k: s.launch_count for k, s in shared.items()}
        for k, s in shared.items():
            assert s.create_tiles_poll(wait=True)
        assert P.create_tiles_poll(wait=True)
        for k, s in shared.items():
            assert _snap(outs[k]) == exp[k][0], k
            if k != "grid":
                assert s.last_erosion_steps == exp[k][1], k
            assert s.launch_count == launches[k] > 0, k       # its own launch count
        assert _snap(outs_p) == exp["ex"][0] and P.last_erosion_steps == exp["ex"][1]
        assert exp["tiles"][1] > 0
    finally:
        P.close()


def test_one_launch_does_not_complete_another(tw, scene, beq):
    """A heavy job on A (64 tiles of 258^2, 1000 droplets each, mode 4) is still running right after a small job's launch on B returns."""
    import torch
    P = tw.Context(0)
    try:
        cfg = scene.SceneConfig(mesh_gen_mode=4, mesh_freq_filter=1, mesh_seed=1, hmap=HM_CFG, zmax_est=2.3, mesh_size=(256, 256, 1))
        hp, ep = cfg.height_params(), cfg.erosion_params()
        dx, dy = float(cfg.dx_val), float(cfg.dy_val)
        nt, zv = 64, 258
        origins = np.array([((t % 8) * 256, (t // 8) * 256) for t in range(nt)], np.int32)
        small = [(tx * 256 * 3 - 2000, ty * 256 * 3 + 700) for ty in range(3) for tx in range(3)]
        exp = torch.empty((nt, zv, zv), dtype=torch.float32, device="cuda")
        _, exp_mm = P.create_zvals_batch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, out=exp, want_minmax=True)
        steps = P.last_erosion_steps
        exp_s, exp_smm = P.create_zvals_batch(small, cfg.mesh_size, dx, dy, 34, hp, 1000, ep, ep.zmin, want_minmax=True)
        steps_s = P.last_erosion_steps
        A, B = P.shared(), P.shared()
        zs, smm = torch.empty((9, 34, 34), dtype=torch.float32).pin_memory(), np.empty((9, 2), np.float32)
        B.create_tiles_launch(small, cfg.mesh_size, dx, dy, 34, hp, 1000, ep, ep.zmin, zs, mm=smm)   # B's scratch and staging exist before A runs
        assert B.create_tiles_poll(wait=True)
        z, mm = torch.empty_like(exp), np.empty((nt, 2), np.float32)
        A.create_tiles_launch(origins, cfg.mesh_size, dx, dy, zv, hp, 1000, ep, ep.zmin, z, mm=mm)
        t0 = time.perf_counter()
        B.create_tiles_launch(small, cfg.mesh_size, dx, dy, 34, hp, 1000, ep, ep.zmin, zs, mm=smm)
        t_b = time.perf_counter() - t0
        a_running = not A.create_tiles_poll(wait=False)
        assert B.create_tiles_poll(wait=True)
        b_done = time.perf_counter() - t0
        a_running_after_b = not A.create_tiles_poll(wait=False)
        assert A.create_tiles_poll(wait=True)
        print("B's launch blocked the host for %.3f ms, B ready after %.2f ms; A still running then: %s; A ready after %.1f ms"
              % (1e3 * t_b, 1e3 * b_done, a_running_after_b, 1e3 * (time.perf_counter() - t0)))
        assert a_running
        assert torch.equal(z.view(torch.int32), exp.view(torch.int32)) and beq(mm, exp_mm) == 0 and A.last_erosion_steps == steps
        assert beq(_host(zs), exp_s) == 0 and beq(smm, exp_smm) == 0 and B.last_erosion_steps == steps_s
    finally:
        P.close()


def test_table_changes_complete_shared_jobs(tw, scene, beq):
    """tw_set_sine_params, tw_set_sin_table and tw_set_heightmap (an image of another size) on the parent while a shared job is pending: the job is complete
    when the call returns, with the old tables' result, and the shared context's next job equals the parent's blocking result under the new tables."""
    import torch
    P, cfg, hp, ep, dx, dy, img, hs = _parent(tw, scene, 0)
    try:
        B = P.shared()
        origins = _origins(4)
        nt = len(origins)

        def blocking(**kw):
            z = np.empty((nt, ZV, ZV), np.float32)
            P.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, kw.pop("hp", hp), ITERS, ep, ep.zmin, z, **kw)
            assert P.create_tiles_poll(wait=True)
            return z, P.last_erosion_steps

        def check(change, exp_old, new_kw, **kw):
            z = torch.empty((nt, ZV, ZV), dtype=torch.float32).pin_memory()
            B.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, **kw)
            change()
            assert tw.lib.tw_create_tiles_poll(B._h, 0) == tw.TW_OK                   # completed by the parent's setter
            assert beq(z.numpy(), exp_old[0]) == 0 and B.last_erosion_steps == exp_old[1]
            exp_new = blocking(**dict(kw, **new_kw))
            assert beq(exp_new[0], exp_old[0]) > 0                                    # the new table changes the result
            B.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, ITERS, ep, ep.zmin, z, **dict(kw, **new_kw))
            assert B.create_tiles_poll(wait=True)
            assert beq(z.numpy(), exp_new[0]) == 0 and B.last_erosion_steps == exp_new[1]
            return exp_new
        old = blocking()
        old = check(lambda: P.set_sine_params(_cfg(scene, 0, seed=2).sine_params()), old, {})
        tab = tw.build_sin_table() * np.float32(0.75)
        check(lambda: P._check(tw.lib.tw_set_sin_table(P._h, tw._ptr(tab))), old, {})
        img_b, hs_b = _image(tw, P, hp, ep, dx, dy, 384, 320)
        check(lambda: P.set_heightmap(img_b), blocking(hmap=hs), {"hmap": hs_b}, hmap=hs)
    finally:
        P.close()


def test_refusals(tw, scene, beq):
    P, cfg, hp, ep, dx, dy, img, hs = _parent(tw, scene, 0)
    try:
        L = tw.lib
        B = P.shared()
        g = cfg.heightmap_grid(128, 96)
        before = P.heightgen_2d(g, hp)
        origins = _origins(2)
        z0 = np.empty((4, ZV, ZV), np.float32)
        P.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 0, None, 0.0, z0, hmap=hs)
        assert P.create_tiles_poll(wait=True)
        sp2 = np.ascontiguousarray(_cfg(scene, 0, seed=3).sine_params(), np.float32)
        tab = tw.build_sin_table() * np.float32(0.5)
        other = np.zeros((40, 30, 2), np.uint8)
        assert L.tw_set_sine_params(B._h, tw._ptr(sp2)) == tw.TW_ERR_ARG
        assert L.tw_set_sin_table(B._h, tw._ptr(tab)) == tw.TW_ERR_ARG
        assert L.tw_set_sin_table(B._h, None) == tw.TW_ERR_ARG
        assert L.tw_set_heightmap(B._h, tw._ptr(other), 30, 40) == tw.TW_ERR_ARG
        assert L.tw_set_heightmap(B._h, None, 0, 0) == tw.TW_ERR_ARG
        assert L.tw_last_error(B._h)
        assert beq(P.heightgen_2d(g, hp), before) == 0 and beq(B.heightgen_2d(g, hp), before) == 0    # the parent's tables as they were
        z1 = np.empty_like(z0)
        B.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 0, None, 0.0, z1, hmap=hs)     # and its image
        assert B.create_tiles_poll(wait=True) and beq(z1, z0) == 0
        h = C.c_void_p()
        assert L.tw_create_shared(B._h, C.byref(h)) == tw.TW_ERR_ARG and h.value is None              # one level only
        with pytest.raises(tw.TwError):
            B.shared()
        Q = tw.Context(0)                                    # a parent without a heightmap or sine params
        try:
            R = Q.shared()
            with pytest.raises(tw.TwError) as e:
                R.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, None, 0, None, 0.0, z1, hmap=hs)
            assert e.value.status == tw.TW_ERR_STATE
            with pytest.raises(tw.TwError) as e:
                R.heightgen_2d(g, hp)                         # sine mode before tw_set_sine_params
            assert e.value.status == tw.TW_ERR_STATE
            Q.set_sine_params(cfg.sine_params())             # set on the parent: the shared context sees it at its next call
            assert beq(R.heightgen_2d(g, hp), before) == 0
        finally:
            Q.close()
    finally:
        P.close()


def test_lifetime(tw, scene, beq):
    """Destroying a shared context with a pending job leaves complete outputs, the small per-tile results included; destroying the parent destroys its
    live shared contexts the same way."""
    import torch
    P, cfg, hp, ep, dx, dy, img, hs = _parent(tw, scene, 4)
    origins = _origins(5)
    nt = len(origins)
    exp_z, exp_mm = P.create_zvals_batch(origins, cfg.mesh_size, dx, dy, ZV, hp, 1000, ep, ep.zmin, want_minmax=True)

    def launch(c):
        z, mm = torch.empty((nt, ZV, ZV), dtype=torch.float32).pin_memory(), np.full((nt, 2), np.nan, np.float32)
        c.create_tiles_launch(origins, cfg.mesh_size, dx, dy, ZV, hp, 1000, ep, ep.zmin, z, mm=mm)
        return z, mm
    B = P.shared()
    z, mm = launch(B)
    B.close()
    assert B._h is None and B not in P._shared
    assert beq(z.numpy(), exp_z) == 0 and beq(mm, exp_mm) == 0
    jobs = [launch(s) for s in (P.shared(), P.shared(), P.shared())]
    kids = list(P._shared)
    P.close()
    assert all(s._h is None for s in kids)
    for z, mm in jobs:
        assert beq(z.numpy(), exp_z) == 0 and beq(mm, exp_mm) == 0
