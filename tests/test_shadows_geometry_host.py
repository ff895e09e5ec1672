"""CPU: the mesh-shadow oracle's geometry checked in float64 against the shadow a single raised cell must cast on a flat tile, on square and non-square
cells, equal and unequal scene sizes, lights in every quadrant, on every axis and exact diagonal, and grazing and steep suns; and the plan's edge cases (light
straight overhead above and below zmin, at exactly zmin, no_shadow).

A spike of height h at cell (x0, y0) of a tile at z = 0 shadows the cells behind it along the light's shadow direction while the running height
h + (pt - spike)[dim] * dir.z / dir[dim] stays above 0, where dim is the axis with the larger |dir| component in world units (x on an exact diagonal). So
the shadow ends exactly ceil(L / d_dim) - 1 index steps along dim from the spike, L = h |dir[dim]| / |dir.z|, d_dim = dx_val or dy_val. A dx / dy or
x_scene_size / y_scene_size mix-up anywhere in the tracer changes that count (by 1.5x for the 32 x 48 cells), which the reference pin would not notice when
the reference objects are absent and the GPU parity tests would not notice when the oracle shares the mistake. tests/test_gpu_shadows_geometry.py runs the
same check on the GPU's output."""
import math

import numpy as np
import pytest
from scipy import ndimage

MIN_Z = np.float32(-1.0e6)      # TW_MESH_MIN_Z
ZV = 65                         # the spike tile's size

# name -> (mesh_size, scene_size): square cells with equal and unequal scene sizes, and 32 x 48-style cells both ways round (dx > dy and dx < dy)
GEOMS = {
    "sq": ((32, 32, 1), (4.0, 4.0, 4.0)),
    "sq_xs!=ys": ((32, 48, 1), (4.0, 6.0, 4.0)),
    "dx>dy": ((32, 48, 1), (4.0, 4.0, 4.0)),
    "dx>dy_xs!=ys": ((32, 48, 1), (4.0, 3.0, 4.0)),
    "dx<dy": ((48, 32, 1), (4.0, 4.0, 4.0)),
    "dx<dy_xs!=ys": ((48, 32, 1), (3.0, 4.0, 4.0)),
}
# one light per quadrant, both signs of each axis, the four exact diagonals (|x| == |y|), a grazing sun (z / |xy| = 0.02) and a steep one (|xy| = 1e-3)
LIGHTS = {
    "q++": (3.0, 2.0, 0.6), "q-+": (-2.0, 3.0, 0.5), "q--": (-3.0, -1.5, 0.7), "q+-": (1.5, -3.0, 0.4),
    "+x": (4.0, 0.0, 1.0), "-x": (-4.0, 0.0, 1.0), "+y": (0.0, 4.0, 1.0), "-y": (0.0, -4.0, 1.0),
    "d++": (2.0, 2.0, 0.8), "d-+": (-2.0, 2.0, 0.8), "d--": (-2.0, -2.0, 0.8), "d+-": (2.0, -2.0, 0.8),
    "grazing": (3.0, 2.0, 0.02 * math.sqrt(13.0)), "steep": (8.0e-4, -6.0e-4, 5.0),
}
K_RUN = 6.4                     # L / d_dim of the spikes: the shadow ends 6 steps along dim from the spike, well inside the tile


def geometry(scene, gname):
    """(mesh_size, scene_size, dx_val, dy_val) from scene.SceneConfig, as the reference computes them (set_scene_constants)."""
    mesh, size = GEOMS[gname]
    cfg = scene.SceneConfig(mesh_size=mesh, scene_size=size)
    return mesh, size, float(cfg.dx_val), float(cfg.dy_val)


def shadow_params(cls, scene, gname, lp, zmin, zmax, no_shadow=0):
    """A ShadowParams of class cls (the oracle's or the product's) for geometry gname and light lp."""
    mesh, size, dx, dy = geometry(scene, gname)
    sp = cls()
    sp.x_scene_size, sp.y_scene_size = size[0], size[1]
    sp.dx_val, sp.dy_val, sp.dx_val_inv, sp.dy_val_inv = dx, dy, 1.0 / np.float32(dx), 1.0 / np.float32(dy)
    sp.xy_sum_size, sp.zmin, sp.zmax, sp.no_shadow = mesh[0] + mesh[1], zmin, zmax, no_shadow
    for d in range(3):
        sp.lpos[d] = lp[d]
    return sp


def direction(lp):
    """float64 shadow direction -lpos / |lpos| and dim (1 = y when |dir.y| > |dir.x|; x on an exact diagonal, as the reference breaks the tie)."""
    d = -np.asarray(lp, np.float64) / np.linalg.norm(np.asarray(lp, np.float64))
    return d, int(abs(d[0]) < abs(d[1]))


def spike_case(scene, gname, lname):
    """(height h, L / d_dim, first spike cell (x0, y0)) for one geometry and light: the spike sits upstream of the tile's centre so that its shadow runs
    toward the centre, K_RUN steps along dim (the grazing sun's runs off the tile)."""
    _, _, dx, dy = geometry(scene, gname)
    d, dim = direction(LIGHTS[lname])
    dd = (dx, dy)[dim]
    h = 1.0 if lname == "grazing" else K_RUN * dd * abs(d[2]) / abs(d[dim])
    k = h * abs(d[dim]) / abs(d[2]) / dd
    u = np.array([d[0] / dx, d[1] / dy])            # the shadow direction in index steps
    u /= np.abs(u).max()
    back = 24 if lname == "grazing" else 10
    x0, y0 = (int(round(ZV // 2 - back * u[0])), int(round(ZV // 2 - back * u[1])))
    return h, k, (x0, y0)


def spike_tile(h, at):
    z = np.zeros((ZV, ZV), np.float32)
    z[at[1], at[0]] = np.float32(h)
    return z


def check_spike(scene, gname, lname, h, k, at, mask, ox, oy):
    """The analytic shadow of the spike (module docstring) against one tile's mask and outgoing heights; returns the number of shadowed cells."""
    _, _, dx, dy = geometry(scene, gname)
    d, dim = direction(LIGHTS[lname])
    sh = mask == 2
    assert not (mask & ~np.uint8(2)).any()
    ys, xs = np.nonzero(sh)
    assert len(xs) > 0, "no shadow"
    assert not sh[at[1], at[0]]
    rel = np.stack([xs - at[0], ys - at[1]], 1).astype(np.float64)
    # every shadowed cell lies on the side of the spike away from the light
    assert ((rel[:, 0] * dx * d[0] + rel[:, 1] * dy * d[1]) > 0.0).all()
    # one 8-connected region with the spike, starting next to it
    lab, nlab = ndimage.label(sh | (np.arange(ZV)[:, None] == at[1]) & (np.arange(ZV)[None, :] == at[0]), structure=np.ones((3, 3)))
    assert nlab == 1
    assert (np.abs(rel).max(1) == 1).any()
    # within 1.5 cells of the line through the spike, in index coordinates
    u = np.array([d[0] / dx, d[1] / dy])
    u /= np.linalg.norm(u)
    assert (np.abs(rel[:, 0] * u[1] - rel[:, 1] * u[0]) <= 1.5).all()
    far = int(np.abs(rel[:, dim]).max())
    if lname == "grazing":      # the run leaves the tile toward -x / -y, and the outgoing edges carry it
        edge_x, edge_y = sh[:, 0], sh[0, :]
        assert edge_x.any() or edge_y.any()
        assert (oy[edge_x] > MIN_Z).all() and (ox[edge_y] > MIN_Z).all()
    else:
        assert abs(k - round(k)) > 1e-3
        assert far == math.ceil(k) - 1, (far, k)
        # The run ends inside the tile, so nothing leaves it - except on an axis, where a ray's walk stays on the row (column) it ends on and every
        # shadowed cell is its last in y (x): sh_out_x (sh_out_y) holds exactly the shadowed columns (rows).
        ax, ay = lname in ("+x", "-x"), lname in ("+y", "-y")
        assert np.array_equal(ox > MIN_Z, sh.any(0) if ax else np.zeros(ZV, bool))
        assert np.array_equal(oy > MIN_Z, sh.any(1) if ay else np.zeros(ZV, bool))
    return int(sh.sum())


def trace_spike(oracle, scene, gname, lname):
    """The oracle's shadow of the spike: (h, k, spike cell, smask, sh_out_x, sh_out_y). A spike that no ray walks through is moved by one cell."""
    h, k, at = spike_case(scene, gname, lname)
    for off in ((0, 0), (1, 0), (0, 1), (1, 1)):
        a = (at[0] + off[0], at[1] + off[1])
        sp = shadow_params(oracle.ShadowParams, scene, gname, LIGHTS[lname], -1.0, h + 1.0)
        m, ox, oy = oracle.calc_mesh_shadows(sp, spike_tile(h, a))
        if (m == 2).any():
            return h, k, a, m, ox, oy
    raise AssertionError("no ray walks through the spike near %s" % (at,))


@pytest.mark.parametrize("lname", list(LIGHTS))
@pytest.mark.parametrize("gname", list(GEOMS))
def test_spike_shadow_is_analytic(oracle, scene, gname, lname):
    h, k, at, m, ox, oy = trace_spike(oracle, scene, gname, lname)
    n = check_spike(scene, gname, lname, h, k, at, m, ox, oy)
    assert n >= (2 if lname != "grazing" else 10)


@pytest.mark.parametrize("gname", ["sq", "dx>dy_xs!=ys"])
def test_dx_dy_swap_changes_the_run(scene, gname):
    """The check is sensitive to the cell size on dim: with dx and dy swapped the run would end elsewhere on the non-square cells."""
    _, _, dx, dy = geometry(scene, gname)
    for lname in ("q++", "+x", "-y", "d--", "steep"):
        h, k, _ = spike_case(scene, gname, lname)
        d, dim = direction(LIGHTS[lname])
        swapped = h * abs(d[dim]) / abs(d[2]) / (dy, dx)[dim]
        assert (math.ceil(swapped) == math.ceil(k)) == (dx == dy), lname


def test_plan_edges(oracle, scene):
    """lpos = (0, 0, z): below zmin everything is in shadow, above it nothing is traced; a light exactly at zmin is traced and not all in shadow;
    no_shadow leaves everything lit, even for a light below zmin."""
    h, _, at = spike_case(scene, "dx>dy", "q++")
    z = spike_tile(h, at)
    zmin, zmax = -1.0, h + 1.0

    def run(lp, no_shadow=0):
        return oracle.calc_mesh_shadows(shadow_params(oracle.ShadowParams, scene, "dx>dy", lp, zmin, zmax, no_shadow), z)
    m, ox, oy = run((0.0, 0.0, zmin - 0.5))
    assert (m == 2).all() and (ox == MIN_Z).all() and (oy == MIN_Z).all()
    for zl in (zmin + 0.5, 5.0, zmin):
        m, ox, oy = run((0.0, 0.0, zl))
        assert not m.any() and (ox == MIN_Z).all() and (oy == MIN_Z).all()
    m, _, _ = run((3.0, 2.0, zmin))                     # below the horizon: traced, the spike shadows what lies behind it to the tile's edge
    assert 0 < (m == 2).sum() < m.size
    for lp in ((3.0, 2.0, 0.6), (0.0, 0.0, zmin - 0.5), (3.0, 2.0, zmin - 0.5)):
        m, ox, oy = run(lp, no_shadow=1)
        assert not m.any() and (ox == MIN_Z).all() and (oy == MIN_Z).all()
