"""3dworld_b200 - H100-native terrain hot path of fegennari/3DWorld (height generation, droplet erosion, voxel density).

The product is the C-ABI shared library lib3dworld_b200.so (hand-written sm_90a CUDA, include/tw3d.h); the C++ adapter with the
reference's own class/function signatures is host/tw3d_adapter.h. This Python module is only the thin ctypes binding that tests and
bench.py drive the library through. There is no CPU fallback: importing works anywhere (so the ABI can be inspected), but creating a
Context without a CUDA device raises, and a missing library raises at import.

Import with importlib (the package name starts with a digit):  tw = importlib.import_module("3dworld_b200")
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib3dworld_b200.so")

MGEN_SINE, MGEN_SIMPLEX, MGEN_PERLIN, MGEN_SIMPLEX_GPU, MGEN_DWARP_GPU = range(5)
TW_OK, TW_ERR_NO_DEVICE, TW_ERR_CUDA, TW_ERR_ARG, TW_ERR_STATE, TW_ERR_NOT_READY = 0, -1, -2, -3, -4, -5
PQ_SIN_TERMS, PQ_SIN_TERMS_SCALED, PQ_EXACT_ZVAL = 0, 1, 2   # tw_point_query.kind


class TwError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("tw3d status %d: %s" % (status, msg))
        self.status = status


# ---- POD mirrors of include/tw3d.h ----
class HmapParams(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("plat_bot", "plat_h", "plat_s", "plat_max", "crat_h", "crat_s", "crack_lo", "crack_hi",
                                         "crack_d", "sine_mag", "sine_freq", "sine_bias", "volcano_width", "volcano_height")]


class HeightParams(C.Structure):
    _fields_ = [("gen_mode", C.c_int), ("gen_shape", C.c_int), ("start_eval_sin", C.c_int), ("glaciate", C.c_int),
                ("mesh_scale", C.c_float), ("mesh_scale_z_inv", C.c_float), ("dx_val_inv", C.c_float), ("dy_val_inv", C.c_float),
                ("mesh_height", C.c_float), ("mesh_height_scale", C.c_float), ("zmax_est", C.c_float),
                ("custom_glaciate_exp", C.c_float), ("rx", C.c_float), ("ry", C.c_float), ("hmap", HmapParams)]


class Grid2D(C.Structure):
    _fields_ = [("x0", C.c_float), ("y0", C.c_float), ("dx", C.c_float), ("dy", C.c_float), ("nx", C.c_uint32), ("ny", C.c_uint32)]


class MinMax(C.Structure):
    _fields_ = [("zmin", C.c_float), ("zmax", C.c_float)]


class ErosionParams(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("erode_amount", "water_plane_z", "half_dxy", "zmin", "zmax", "relh_adj_tex", "clip_hd1")]


class VoxelParams(C.Structure):
    _fields_ = [("nx", C.c_uint32), ("ny", C.c_uint32), ("nz", C.c_uint32),
                ("lo_pos", C.c_float * 3), ("vsz", C.c_float * 3), ("offset", C.c_float * 3),
                ("mag", C.c_float), ("freq", C.c_float), ("gen_mode", C.c_int), ("normalize_to_1", C.c_int),
                ("rseed1", C.c_int), ("rseed2", C.c_int), ("octaves", C.c_int), ("rx", C.c_float), ("ry", C.c_float),
                ("zscale", C.c_float), ("atten_mode", C.c_int), ("atten_val", C.c_float), ("atten_inner_radius", C.c_float)]


class VoxelPostParams(C.Structure):
    _fields_ = [("nx", C.c_uint32), ("ny", C.c_uint32), ("nz", C.c_uint32), ("lo_pos", C.c_float * 3), ("vsz", C.c_float * 3), ("isolevel", C.c_float),
                ("invert", C.c_int), ("make_closed_surface", C.c_int), ("remove_unconnected", C.c_int), ("keep_at_edge", C.c_int), ("centre_seed", C.c_int),
                ("skip_under_mesh", C.c_int)]


class WeightParams(C.Structure):
    """tw_weight_params (include/tw3d.h): the terrain weights texture's tables and scene scalars."""
    _fields_ = [("h_dirt", C.c_float * 5), ("tex_class", C.c_int * 5), ("class_ix", C.c_int * 5), ("sthresh", (C.c_float * 2) * 2), ("zmin", C.c_float), ("zmax", C.c_float),
                ("relh_adj_tex", C.c_float), ("water_level", C.c_float), ("noise_scale", C.c_float), ("vnz_scale", C.c_float), ("vegetation", C.c_float), ("snow_to_rock", C.c_int),
                ("dx_val", C.c_float), ("dy_val", C.c_float), ("dxdy", C.c_float), ("xy_mult", C.c_float)]


class ShadowParams(C.Structure):
    _fields_ = [("lpos", C.c_float * 3), ("x_scene_size", C.c_float), ("y_scene_size", C.c_float), ("dx_val", C.c_float), ("dy_val", C.c_float), ("dx_val_inv", C.c_float),
                ("dy_val_inv", C.c_float), ("xy_sum_size", C.c_int), ("zmin", C.c_float), ("zmax", C.c_float), ("no_shadow", C.c_int)]


class TileBounds(C.Structure):
    _fields_ = [("sub_zmin", C.c_float * 16), ("sub_zmax", C.c_float * 16), ("mzmin", C.c_float), ("mzmax", C.c_float), ("mesh_dz", C.c_float),
                ("radius", C.c_float), ("wx1", C.c_int32), ("wy1", C.c_int32), ("wx2", C.c_int32), ("wy2", C.c_int32)]


class TileOutputs(C.Structure):
    """tw_tile_outputs (include/tw3d.h): where tw_create_tiles_launch puts each requested per-tile product (NULL = not requested)."""
    _fields_ = [("zvals", C.c_void_p), ("mm", C.c_void_p), ("bounds", C.c_void_p), ("normals_rgba", C.c_void_p), ("min_normal_z", C.c_void_p)]


class TileShading(C.Structure):
    """tw_tile_shading (include/tw3d.h): the AO map and terrain weights texture tw_create_tiles_launch_ex adds to the tile job (NULL = not requested)."""
    _fields_ = [("half_dxy", C.c_float), ("wp", C.c_void_p), ("tile_params", C.c_void_p), ("ao", C.c_void_p), ("weights", C.c_void_p), ("has_any_grass", C.c_void_p)]


class TileLight(C.Structure):
    """tw_tile_light (include/tw3d.h): one light's mesh shadows in the tile job (smask required; sh_in_* / sh_out_* optional)."""
    _fields_ = [("sp", ShadowParams), ("sh_in_x", C.c_void_p), ("sh_in_y", C.c_void_p), ("smask", C.c_void_p), ("sh_out_x", C.c_void_p), ("sh_out_y", C.c_void_p)]


class TileShadows(C.Structure):
    """tw_tile_shadows (include/tw3d.h): the tiles' grid coordinates and the lights whose mesh shadows tw_create_tiles_launch_shadows adds to the job."""
    _fields_ = [("tile_xy", C.c_void_p), ("nlights", C.c_uint32), ("lights", C.c_void_p)]


class PointQuery(C.Structure):
    _fields_ = [("kind", C.c_int), ("xy_scale", C.c_float), ("mesh_x_size", C.c_int), ("mesh_y_size", C.c_int), ("x_scene_size", C.c_float),
                ("y_scene_size", C.c_float), ("xoff2", C.c_int), ("yoff2", C.c_int), ("no_xyoff", C.c_int)]


class HmapSampler(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("edge_mode", C.c_int), ("mesh_scale", C.c_float), ("h_scale", C.c_float),
                ("mesh_file_scale", C.c_float), ("mesh_file_tz", C.c_float), ("mesh_scale_z_inv", C.c_float)]


class HeightmapInfo(C.Structure):
    _fields_ = [("min_z", C.c_float), ("max_z", C.c_float), ("val_mult", C.c_float), ("val_add", C.c_float), ("mesh_file_scale", C.c_float),
                ("mesh_file_tz", C.c_float), ("erosion_moves", C.c_uint64)]


class Rng(C.Structure):
    _fields_ = [("rseed1", C.c_int64), ("rseed2", C.c_int64)]


def hmap_params(**kw):
    """hmap_params_t with the reference defaults (src/mesh.h:85-88)."""
    h = HmapParams(1000.0, 0, 0, 0, 1000.0, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    for k, v in kw.items():
        setattr(h, k, v)
    return h


# every symbol include/tw3d.h declares (tests check the library exports exactly these)
ABI_SYMBOLS = ["tw_abi_version", "tw_create", "tw_destroy", "tw_last_error", "tw_sync", "tw_stream", "tw_launch_count",
               "tw_build_sin_table", "tw_compute_scale", "tw_gen_sine_params", "tw_gen_rx_ry", "tw_noise3d_gen_sines",
               "tw_water_z_height", "tw_set_sin_table", "tw_set_sine_params", "tw_heightgen_2d", "tw_heightgen_2d_launch",
               "tw_heightgen_2d_poll", "tw_heightgen_tiles", "tw_create_zvals_batch", "tw_create_tiles_launch", "tw_create_tiles_launch_ex", "tw_create_tiles_poll", "tw_tile_bounds_batch", "tw_tile_normals_batch", "tw_tile_ao_batch", "tw_create_zvals_ao_batch", "tw_glaciate_mesh", "tw_eval_points", "tw_erode", "tw_erode_parallel", "tw_erode_tiles", "tw_last_erosion_steps", "tw_voxel_fill",
               "tw_heightmap_from_floats_u16", "tw_heightmap_to_floats_u16", "tw_proc_gen_heightmap", "tw_heightmap_sample_tiles", "tw_set_heightmap", "tw_create_tiles_launch_hmap", "tw_minmax_f32",
               "tw_multi_create", "tw_multi_destroy", "tw_multi_size", "tw_multi_ctx", "tw_multi_last_error", "tw_multi_set_sine_params", "tw_multi_range",
               "tw_multi_alloc_host", "tw_multi_free_host", "tw_create_zvals_sharded", "tw_heightgen_2d_sharded", "tw_dist_unique_id", "tw_dist_init",
               "tw_dist_allreduce_minmax", "tw_dist_finalize", "tw_bind_thread_to_device", "tw_erode_sweeps", "tw_erode_sweeps_banded", "tw_erode_sweeps_sharded", "tw_voxel_outside", "tw_voxel_remove_unconnected", "tw_voxel_triangles", "tw_tile_shadows_batch", "tw_tile_shadows_batch_ex", "tw_create_tiles_launch_shadows", "tw_tile_weights_batch", "tw_gen_tex_height_tables"]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError("3dworld_b200: %s is missing - build it with `python 3dworld_b200/build.py` (or __graft_entry__.build()); "
                          "there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, fp = C.c_void_p, C.POINTER(C.c_float)
    L.tw_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.tw_destroy.argtypes = [vp]
    L.tw_destroy.restype = None
    L.tw_last_error.argtypes = [vp]
    L.tw_last_error.restype = C.c_char_p
    L.tw_sync.argtypes = [vp]
    L.tw_stream.argtypes = [vp]
    L.tw_stream.restype = vp
    L.tw_launch_count.argtypes = [vp]
    L.tw_launch_count.restype = C.c_uint64
    L.tw_build_sin_table.argtypes = [vp]
    L.tw_build_sin_table.restype = None
    L.tw_compute_scale.argtypes = [C.c_float, C.c_int]
    L.tw_gen_sine_params.argtypes = [C.POINTER(Rng), C.c_float, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int,
                                     C.c_float, C.c_float, C.c_float, C.c_float, vp]
    L.tw_gen_sine_params.restype = None
    L.tw_gen_rx_ry.argtypes = [C.c_int, C.c_int, C.c_int, fp, fp]
    L.tw_gen_rx_ry.restype = None
    L.tw_noise3d_gen_sines.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, vp]
    L.tw_noise3d_gen_sines.restype = None
    L.tw_water_z_height.argtypes = [C.c_float, C.c_int, C.c_float, C.c_float, C.c_float]
    L.tw_water_z_height.restype = C.c_float
    L.tw_set_sin_table.argtypes = [vp, vp]
    L.tw_set_sine_params.argtypes = [vp, vp]
    hg = [vp, C.POINTER(Grid2D), C.POINTER(HeightParams), C.c_int, C.c_int, vp, C.POINTER(MinMax)]
    L.tw_heightgen_2d.argtypes = hg
    L.tw_heightgen_2d_launch.argtypes = hg
    L.tw_heightgen_2d_poll.argtypes = [vp, C.c_int]
    L.tw_heightgen_tiles.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), vp, vp]
    L.tw_create_zvals_batch.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.c_uint32,
                                        C.POINTER(ErosionParams), C.c_float, vp, vp]
    L.tw_create_tiles_launch.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.c_uint32,
                                         C.POINTER(ErosionParams), C.c_float, C.c_float, C.c_uint32, C.POINTER(TileOutputs)]
    L.tw_create_tiles_launch_ex.argtypes = L.tw_create_tiles_launch.argtypes + [C.POINTER(TileShading)]
    L.tw_create_tiles_launch_shadows.argtypes = L.tw_create_tiles_launch_ex.argtypes + [C.POINTER(TileShadows)]
    L.tw_create_tiles_launch_hmap.argtypes = [vp, C.POINTER(HmapSampler)] + L.tw_create_tiles_launch_shadows.argtypes[1:]
    L.tw_create_tiles_poll.argtypes = [vp, C.c_int]
    L.tw_tile_bounds_batch.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_uint32, vp]
    L.tw_glaciate_mesh.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(HeightParams), C.POINTER(MinMax)]
    L.tw_erode.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams)]
    L.tw_tile_normals_batch.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_float, C.c_float, vp, vp]
    L.tw_tile_ao_batch.argtypes = [vp, vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.c_float, vp]
    L.tw_create_zvals_ao_batch.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.c_uint32,
                                           C.POINTER(ErosionParams), C.c_float, C.c_float, vp, vp, vp]
    L.tw_heightmap_sample_tiles.argtypes = [vp, vp, C.POINTER(HmapSampler), vp, C.c_uint32, C.c_uint32, vp]
    L.tw_set_heightmap.argtypes = [vp, vp, C.c_int, C.c_int]
    L.tw_eval_points.argtypes = [vp, vp, C.c_size_t, C.POINTER(HeightParams), C.POINTER(PointQuery), vp]
    L.tw_erode_parallel.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams), C.c_uint32]
    L.tw_erode_tiles.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, vp, C.c_float, C.c_uint32, C.POINTER(ErosionParams)]
    L.tw_last_erosion_steps.argtypes = [vp]
    L.tw_last_erosion_steps.restype = C.c_uint64
    L.tw_voxel_fill.argtypes = [vp, C.POINTER(VoxelParams), vp, vp]
    L.tw_heightmap_from_floats_u16.argtypes = [vp, vp, C.c_size_t, C.c_float, C.c_float, vp]
    L.tw_heightmap_to_floats_u16.argtypes = [vp, vp, C.c_size_t, C.c_float, C.c_float, vp]
    L.tw_proc_gen_heightmap.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.POINTER(HeightParams), C.c_uint32, C.POINTER(ErosionParams), vp, vp,
                                        C.POINTER(HeightmapInfo)]
    L.tw_minmax_f32.argtypes = [vp, vp, C.c_size_t, C.POINTER(MinMax)]
    # multi-GPU
    L.tw_multi_create.argtypes = [vp, C.c_int, C.POINTER(vp)]
    L.tw_multi_destroy.argtypes = [vp]
    L.tw_multi_destroy.restype = None
    L.tw_multi_size.argtypes = [vp]
    L.tw_multi_ctx.argtypes = [vp, C.c_int]
    L.tw_multi_ctx.restype = vp
    L.tw_multi_last_error.argtypes = [vp]
    L.tw_multi_last_error.restype = C.c_char_p
    L.tw_multi_set_sine_params.argtypes = [vp, vp]
    L.tw_multi_range.argtypes = [C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.tw_multi_range.restype = None
    L.tw_multi_alloc_host.argtypes = [vp, C.c_int, C.c_size_t, C.POINTER(vp)]
    L.tw_multi_free_host.argtypes = [vp, vp]
    L.tw_multi_free_host.restype = None
    L.tw_create_zvals_sharded.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.c_uint32,
                                          C.POINTER(ErosionParams), C.c_float, vp, vp, C.POINTER(MinMax)]
    L.tw_heightgen_2d_sharded.argtypes = [vp, C.POINTER(Grid2D), C.POINTER(HeightParams), C.c_int, vp, C.POINTER(MinMax)]
    L.tw_erode_sweeps.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams), C.c_uint32, C.c_int, C.POINTER(C.c_uint64)]
    L.tw_erode_sweeps_banded.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams), C.c_uint32, C.c_int, C.POINTER(C.c_uint64)]
    L.tw_erode_sweeps_sharded.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams), C.c_uint32, C.c_int, C.POINTER(C.c_uint64)]
    L.tw_voxel_outside.argtypes = [vp, vp, C.POINTER(VoxelPostParams), vp, vp]
    L.tw_voxel_remove_unconnected.argtypes = [vp, vp, vp, C.POINTER(VoxelPostParams), C.POINTER(C.c_uint64)]
    L.tw_voxel_triangles.argtypes = [vp, vp, vp, C.POINTER(VoxelPostParams), vp, vp, vp, vp, C.c_uint64, C.POINTER(C.c_uint64)]
    L.tw_tile_shadows_batch.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.POINTER(ShadowParams), vp, vp, vp]
    L.tw_tile_shadows_batch_ex.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.POINTER(ShadowParams), vp, vp, vp, vp, vp]
    L.tw_tile_weights_batch.argtypes = [vp, vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.c_uint32, C.POINTER(HeightParams), C.POINTER(WeightParams), vp, vp, vp]
    L.tw_gen_tex_height_tables.argtypes = [C.c_float, C.c_float, C.c_float, vp, vp, vp]
    L.tw_gen_tex_height_tables.restype = None
    L.tw_dist_unique_id.argtypes = [vp]
    L.tw_dist_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.tw_dist_allreduce_minmax.argtypes = [vp, C.POINTER(MinMax)]
    L.tw_dist_finalize.argtypes = [vp]
    L.tw_dist_finalize.restype = None
    L.tw_bind_thread_to_device.argtypes = [C.c_int]
    return L


lib = _load()


def _ptr(a):
    """Raw address of a numpy array (host) or a torch tensor (host or CUDA)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        assert a.is_contiguous()
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


def _edge(a):
    """An optional incoming shadow edge: a CUDA tensor as it is, anything else as a contiguous float32 numpy array."""
    return a if a is None or hasattr(a, "data_ptr") else np.ascontiguousarray(a, np.float32)


class Light:
    """One light of Context.create_tiles_launch(lights=...): its ShadowParams, the required smask [nt, zv, zv] uint8 and the optional sh_out_x, sh_out_y,
    sh_in_x, sh_in_y ([nt, zv] float32), numpy arrays (pinned for a launch that does not block) or CUDA tensors."""

    def __init__(self, sp, smask, sh_out_x=None, sh_out_y=None, sh_in_x=None, sh_in_y=None):
        self.sp, self.smask, self.sh_out_x, self.sh_out_y, self.sh_in_x, self.sh_in_y = sp, smask, sh_out_x, sh_out_y, sh_in_x, sh_in_y


# ---- host-side helpers (no GPU needed) ----
def build_sin_table():
    t = np.empty(65536, np.float32)
    lib.tw_build_sin_table(_ptr(t))
    return t


def compute_scale(mesh_scale, mesh_freq_filter):
    return lib.tw_compute_scale(mesh_scale, mesh_freq_filter)


def gen_sine_params(scaled_height, mesh=(128, 128), scene=(4.0, 4.0), seed=0, rgen_index=0, mode=0, rng=None,
                    start_mag=0.02, start_freq=240.0, mag_mult=2.0, freq_mult=0.5):
    rng = rng if rng is not None else Rng(1, 1)
    out = np.empty((90, 5), np.float32)
    lib.tw_gen_sine_params(C.byref(rng), scaled_height, mesh[0], mesh[1], scene[0], scene[1], seed, rgen_index, mode,
                           start_mag, start_freq, mag_mult, freq_mult, _ptr(out))
    return out


def gen_rx_ry(seed, rgen_index, mode):
    rx, ry = C.c_float(), C.c_float()
    lib.tw_gen_rx_ry(seed, rgen_index, mode, C.byref(rx), C.byref(ry))
    return rx.value, ry.value


def noise3d_gen_sines(rs1, rs2, mag, freq):
    out = np.empty(420, np.float32)
    lib.tw_noise3d_gen_sines(rs1, rs2, mag, freq, _ptr(out))
    return out


def water_z_height(zmax_est, glaciate=1, custom_glaciate_exp=0.0, water_h_off=0.0, water_h_off_rel=0.0):
    return lib.tw_water_z_height(zmax_est, glaciate, custom_glaciate_exp, water_h_off, water_h_off_rel)


def multi_range(n, ndev, i):
    a, b = C.c_uint32(), C.c_uint32()
    lib.tw_multi_range(n, ndev, i, C.byref(a), C.byref(b))
    return a.value, b.value


def dist_unique_id():
    """128-byte NCCL id for Context.dist_init (rank 0 makes it, every rank receives it out of band, e.g. a torch.distributed broadcast)."""
    buf = C.create_string_buffer(128)
    rc = lib.tw_dist_unique_id(buf)
    if rc != TW_OK:
        raise TwError(rc, "tw_dist_unique_id: libnccl.so.2 not loadable")
    return buf.raw


def bind_thread_to_device(device):
    return lib.tw_bind_thread_to_device(int(device)) == TW_OK


class Multi:
    """tw_multi: one process driving several GPUs (one tw_ctx + worker thread per device, NCCL z-range reduction inside the library)."""

    def __init__(self, devices):
        devs = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        rc = lib.tw_multi_create(C.cast(devs, C.c_void_p), len(devices), C.byref(h))
        if rc != TW_OK:
            raise TwError(rc, "tw_multi_create failed")
        self._h, self.n, self.devices = h, len(devices), list(devices)

    def close(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.tw_multi_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != TW_OK:
            raise TwError(rc, lib.tw_multi_last_error(self._h).decode())

    def set_sine_params(self, sp):
        sp = np.ascontiguousarray(sp, np.float32)
        self._check(lib.tw_multi_set_sine_params(self._h, _ptr(sp)))

    def alloc_host(self, i, shape, dtype=np.float32):
        """numpy view of pinned host memory on device i's NUMA node (freed with free_host)."""
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = C.c_void_p()
        self._check(lib.tw_multi_alloc_host(self._h, i, n, C.byref(p)))
        arr = np.frombuffer((C.c_char * n).from_address(p.value), dtype=dtype).reshape(shape)
        return arr, p

    def free_host(self, p):
        lib.tw_multi_free_host(self._h, p)

    def _bands(self, outs):
        assert len(outs) == self.n
        return (C.c_void_p * self.n)(*[_ptr(o).value for o in outs])

    def create_zvals_sharded(self, origins_xy, mesh_size, dx, dy, zvsize, hp, erosion_iters, ep, min_zval, out_bands, want_minmax=False):
        """out_bands: one array / CUDA tensor per device for its band of tiles (multi_range). Returns (per-tile min/max or None, global (zmin, zmax))."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        mm = np.empty((nt, 2), np.float32) if want_minmax else None
        zr = MinMax()
        self._check(lib.tw_create_zvals_sharded(self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zvsize, C.byref(hp), erosion_iters, C.byref(ep), min_zval,
                                                C.cast(self._bands(out_bands), C.c_void_p), _ptr(mm), C.byref(zr)))
        return mm, (zr.zmin, zr.zmax)

    def erode_sweeps_sharded(self, bands, xsize, ysize, min_zval, num_iters, ep, sweep, halo):
        """Coherent batched erosion of one map held as row bands (in place; one band per device: numpy arrays or that device's CUDA tensors)."""
        moves = C.c_uint64()
        self._check(lib.tw_erode_sweeps_sharded(self._h, C.cast(self._bands(bands), C.c_void_p), xsize, ysize, min_zval, num_iters, C.byref(ep), sweep, halo, C.byref(moves)))
        return moves.value

    def heightgen_2d_sharded(self, grid, hp, out_bands, enable_glaciate=1):
        zr = MinMax()
        self._check(lib.tw_heightgen_2d_sharded(self._h, C.byref(grid), C.byref(hp), int(enable_glaciate), C.cast(self._bands(out_bands), C.c_void_p), C.byref(zr)))
        return zr.zmin, zr.zmax


class Context:
    """One tw_ctx (device + stream + uploaded tables). All compute goes through the C ABI."""

    def __init__(self, device=0, sin_table=None):
        h = C.c_void_p()
        rc = lib.tw_create(device, C.byref(h))
        if rc != TW_OK:
            raise TwError(rc, "tw_create failed (no CUDA device? this library has no CPU fallback)")
        self._h = h
        self.device = device
        self._check(lib.tw_set_sin_table(self._h, _ptr(sin_table)))

    def close(self):
        if getattr(self, "_h", None) and lib is not None:   # lib can already be gone at interpreter shutdown
            lib.tw_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != TW_OK:
            raise TwError(rc, lib.tw_last_error(self._h).decode())

    @property
    def stream(self):
        return lib.tw_stream(self._h)

    @property
    def launch_count(self):
        return int(lib.tw_launch_count(self._h))

    def sync(self):
        self._check(lib.tw_sync(self._h))

    # one process per GPU: the library's own NCCL communicator for the z-range reduction
    def dist_init(self, nranks, rank, unique_id):
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self._check(lib.tw_dist_init(self._h, nranks, rank, buf))

    def dist_allreduce_minmax(self, zmin, zmax):
        mm = MinMax(zmin, zmax)
        self._check(lib.tw_dist_allreduce_minmax(self._h, C.byref(mm)))
        return mm.zmin, mm.zmax

    def set_sine_params(self, sp):
        sp = np.ascontiguousarray(sp, np.float32)
        assert sp.size == 450
        self._check(lib.tw_set_sine_params(self._h, _ptr(sp)))

    def heightgen_2d(self, grid, hp, enable_glaciate=1, min_start_sin=0, out=None, want_minmax=False):
        if out is None:
            out = np.empty((grid.ny, grid.nx), np.float32)
        mm = MinMax() if want_minmax else None
        self._check(lib.tw_heightgen_2d(self._h, C.byref(grid), C.byref(hp), int(enable_glaciate), int(min_start_sin), _ptr(out),
                                        C.byref(mm) if mm else None))
        return (out, (mm.zmin, mm.zmax)) if want_minmax else out

    def heightgen_2d_launch(self, grid, hp, enable_glaciate, min_start_sin, out, mm=None):
        self._check(lib.tw_heightgen_2d_launch(self._h, C.byref(grid), C.byref(hp), int(enable_glaciate), int(min_start_sin), _ptr(out),
                                               C.byref(mm) if mm is not None else None))

    def heightgen_2d_poll(self, wait=False):
        rc = lib.tw_heightgen_2d_poll(self._h, int(wait))
        if rc == TW_ERR_NOT_READY:
            return False
        self._check(rc)
        return True

    def heightgen_tiles(self, origins_xy, mesh_size, dx, dy, zvsize, hp, out=None, want_minmax=False):
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        if out is None:
            out = np.empty((nt, zvsize, zvsize), np.float32)
        mm = np.empty((nt, 2), np.float32) if want_minmax else None
        self._check(lib.tw_heightgen_tiles(self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zvsize, C.byref(hp), _ptr(out), _ptr(mm)))
        return (out, mm) if want_minmax else out

    def create_zvals_batch(self, origins_xy, mesh_size, dx, dy, zvsize, hp, erosion_iters, ep, min_zval, out=None, want_minmax=False):
        """Fused height fill + per-tile erosion (tile_t::create_zvals for a batch of tiles)."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        if out is None:
            out = np.empty((nt, zvsize, zvsize), np.float32)
        mm = np.empty((nt, 2), np.float32) if want_minmax else None
        self._check(lib.tw_create_zvals_batch(self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zvsize, C.byref(hp), erosion_iters,
                                              C.byref(ep), min_zval, _ptr(out), _ptr(mm)))
        return (out, mm) if want_minmax else out

    def create_tiles_launch(self, origins_xy, mesh_size, dx, dy, zvsize, hp, erosion_iters, ep, min_zval, zvals, mm=None, bounds=None, normals=None,
                            min_normal_z=None, wpz_max=0.0, size=0, ao=None, weights=None, has_any_grass=None, half_dxy=None, wp=None, tile_params=None,
                            tile_xy=None, lights=None, hmap=None):
        """tw_create_tiles_launch(_ex): a frame's new tiles (heights, erosion, z range, sub-block bounds, normal map, and on request the AO map and the
        terrain weights texture) enqueued without waiting for the GPU. hmap (HmapSampler) takes the heights from the image of set_heightmap instead of the
        height function (tw_create_tiles_launch_hmap): hp may then be None unless weights is given, and ao is refused.
        zvals [nt, zv, zv] float32, normals [nt, zv-1, zv-1, 4] uint8, ao [nt, zv-1, zv-1] uint8 and weights [nt, zv-1, zv-1, 4] uint8: numpy arrays
        (pinned for a launch that does not block) or CUDA tensors; mm [nt, 2] float32, bounds (TileBounds * nt) and min_normal_z [nt] float32 are host
        arrays that the completing create_tiles_poll fills, has_any_grass [nt] uint8 is either. weights needs wp (WeightParams) and tile_params
        ([nt, 8] float32, host or CUDA); ao takes the ray step half_dxy. In GPU gen modes (3/4) requesting ao makes the zvals those of
        create_zvals_ao_batch (see tw3d.h). lights adds the mesh shadows of these tiles (tw_create_tiles_launch_shadows): a list of Light records or
        (ShadowParams, smask, sh_out_x, sh_out_y, sh_in_x, sh_in_y) tuples - smask [nt, zv, zv] uint8 required, the rest [nt, zv] float32 or None - and
        needs tile_xy [nt, 2] (x1/size, y1/size). The origins, tile_xy, host tile_params and host sh_in rows are copied during the launch; the outputs and
        device inputs are kept referenced here until the job completes."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        outs = TileOutputs(_ptr(zvals), _ptr(mm), C.cast(bounds, C.c_void_p) if bounds is not None else None, _ptr(normals), _ptr(min_normal_z))
        args = [self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zvsize, C.byref(hp) if hp is not None else None, erosion_iters,
                C.byref(ep) if ep is not None else None,
                min_zval, wpz_max, size, C.byref(outs)]
        shading = None
        if ao is not None and half_dxy is None:
            raise ValueError("create_tiles_launch: ao needs half_dxy (the ray's z step, HALF_DXY)")
        if ao is not None or weights is not None or has_any_grass is not None:
            if tile_params is not None and not hasattr(tile_params, "data_ptr"):
                tile_params = np.ascontiguousarray(tile_params, np.float32)
            shading = TileShading(0.0 if half_dxy is None else half_dxy, C.cast(C.pointer(wp), C.c_void_p) if wp is not None else None, _ptr(tile_params),
                                  _ptr(ao), _ptr(weights), _ptr(has_any_grass))
        shadows, keep = None, []
        if lights is not None:
            if tile_xy is None:
                raise ValueError("create_tiles_launch: lights need tile_xy (the tiles' grid coordinates)")
            tile_xy = np.ascontiguousarray(tile_xy, np.int32).reshape(-1, 2)
            recs = [lt if isinstance(lt, Light) else Light(*lt) for lt in lights]
            keep = [[r.smask, r.sh_out_x, r.sh_out_y, _edge(r.sh_in_x), _edge(r.sh_in_y)] for r in recs]
            arr = (TileLight * max(1, len(recs)))()
            for i, (r, k) in enumerate(zip(recs, keep)):
                arr[i] = TileLight(r.sp, _ptr(k[3]), _ptr(k[4]), _ptr(k[0]), _ptr(k[1]), _ptr(k[2]))
            shadows = TileShadows(_ptr(tile_xy), len(recs), C.cast(arr, C.c_void_p))
            keep.append(arr)
        if hmap is not None:
            self._check(lib.tw_create_tiles_launch_hmap(args[0], C.byref(hmap), *args[1:], C.byref(shading) if shading is not None else None,
                                                        C.byref(shadows) if shadows is not None else None))
        elif shadows is not None:
            self._check(lib.tw_create_tiles_launch_shadows(*args, C.byref(shading) if shading is not None else None, C.byref(shadows)))
        elif shading is not None:
            self._check(lib.tw_create_tiles_launch_ex(*args, C.byref(shading)))
        else:
            self._check(lib.tw_create_tiles_launch(*args))
        self._tiles_job = (zvals, mm, bounds, normals, min_normal_z, ao, weights, has_any_grass, wp, tile_params, shading, tile_xy, keep, shadows)

    def create_tiles_poll(self, wait=False):
        """True once the job of create_tiles_launch (or any pending job of this context) is complete, False while it runs (wait=False)."""
        rc = lib.tw_create_tiles_poll(self._h, int(wait))
        if rc == TW_ERR_NOT_READY:
            return False
        self._tiles_job = None
        self._check(rc)
        return True

    def tile_bounds(self, tiles, wpz_max, dx_val, dy_val, size):
        """Tail of tile_t::create_zvals: returns a numpy structured view of ntiles tw_tile_bounds."""
        nt, zv = tiles.shape[0], tiles.shape[1]
        out = (TileBounds * nt)()
        self._check(lib.tw_tile_bounds_batch(self._h, _ptr(tiles), nt, zv, wpz_max, dx_val, dy_val, size, C.cast(out, C.c_void_p)))
        return out

    def heightmap_sample_tiles(self, data16, hs, origins_xy, zvsize, out=None):
        """Heightmap-texture mode of tile_t::create_zvals: get_clamped_height over tiles; data16 = uint8 [h, w, 2] (numpy or CUDA tensor)."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        if out is None:
            out = np.empty((nt, zvsize, zvsize), np.float32)
        self._check(lib.tw_heightmap_sample_tiles(self._h, _ptr(data16), C.byref(hs), _ptr(org), nt, zvsize, _ptr(out)))
        return out

    def set_heightmap(self, data16):
        """tw_set_heightmap: the image create_tiles_launch(hmap=...) samples, copied to device memory this context owns; data16 = uint8 [h, w, 2]
        (numpy or CUDA tensor), None releases it."""
        if data16 is None:
            self._check(lib.tw_set_heightmap(self._h, None, 0, 0))
            return
        if not hasattr(data16, "data_ptr"):
            data16 = np.ascontiguousarray(data16, np.uint8)
        if len(data16.shape) != 3 or data16.shape[2] != 2:
            raise ValueError("set_heightmap: data16 must have shape [h, w, 2]")
        self._check(lib.tw_set_heightmap(self._h, _ptr(data16), int(data16.shape[1]), int(data16.shape[0])))

    def tile_normals(self, tiles, dx_val, dy_val, out=None):
        """tile_t::upload_normal_texture for a batch: returns (rgba [nt, stride, stride, 4] uint8, min_normal_z [nt])."""
        nt, zv = int(tiles.shape[0]), int(tiles.shape[1])
        if out is None:
            out = np.empty((nt, zv - 1, zv - 1, 4), np.uint8)
        mnz = np.empty(nt, np.float32)
        self._check(lib.tw_tile_normals_batch(self._h, _ptr(tiles), nt, zv, dx_val, dy_val, _ptr(out), _ptr(mnz)))
        return out, mnz

    def tile_ao(self, tiles, origins_xy, mesh_size, dx, dy, hp, half_dxy, out=None):
        """tile_t::calc_mesh_ao_lighting for a batch: ao [nt, stride, stride] uint8 (context heights generated internally)."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt, zv = int(tiles.shape[0]), int(tiles.shape[1])
        if out is None:
            out = np.empty((nt, zv - 1, zv - 1), np.uint8)
        self._check(lib.tw_tile_ao_batch(self._h, _ptr(tiles), _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zv, C.byref(hp), half_dxy, _ptr(out)))
        return out

    def create_zvals_ao_batch(self, origins_xy, mesh_size, dx, dy, zvsize, hp, erosion_iters, ep, min_zval, half_dxy, out=None, ao=None, want_minmax=False):
        """tile_t::create_zvals + calc_mesh_ao_lighting (enable_tiled_mesh_ao) for a batch: returns (zvals, ao[, minmax])."""
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        if out is None:
            out = np.empty((nt, zvsize, zvsize), np.float32)
        if ao is None:
            ao = np.empty((nt, zvsize - 1, zvsize - 1), np.uint8)
        mm = np.empty((nt, 2), np.float32) if want_minmax else None
        self._check(lib.tw_create_zvals_ao_batch(self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zvsize, C.byref(hp), erosion_iters,
                                                 C.byref(ep), min_zval, half_dxy, _ptr(out), _ptr(ao), _ptr(mm)))
        return (out, ao, mm) if want_minmax else (out, ao)

    def glaciate_mesh(self, mesh, xoff2, yoff2, mesh_size, hp):
        """glaciate() of the ground-mode mesh, in place; returns (zbottom, ztop)."""
        ny, nx = mesh.shape
        mm = MinMax()
        self._check(lib.tw_glaciate_mesh(self._h, _ptr(mesh), nx, ny, xoff2, yoff2, mesh_size[0], mesh_size[1], C.byref(hp), C.byref(mm)))
        return mm.zmin, mm.zmax

    def eval_points(self, xy, hp, pq, out=None):
        """Batched eval_mesh_sin_terms / eval_mesh_sin_terms_scaled / get_exact_zval (PQ_* kinds); xy = [n, 2] numpy array or CUDA tensor."""
        n = int(xy.shape[0])
        if out is None:
            out = np.empty(n, np.float32)
        self._check(lib.tw_eval_points(self._h, _ptr(xy), n, C.byref(hp), C.byref(pq), _ptr(out)))
        return out

    def erode(self, h, min_zval, num_iters, ep):
        """In place on h (numpy [ys, xs] or CUDA tensor)."""
        ys, xs = h.shape
        self._check(lib.tw_erode(self._h, _ptr(h), xs, ys, min_zval, num_iters, C.byref(ep)))
        return h

    def erode_parallel(self, h, min_zval, num_iters, ep, num_threads=0):
        """The reference's OpenMP mode (src/erosion.cpp:66): num_threads droplets walk h concurrently; order-dependent result, 1 == erode()."""
        ys, xs = h.shape
        self._check(lib.tw_erode_parallel(self._h, _ptr(h), xs, ys, min_zval, num_iters, C.byref(ep), num_threads))
        return h

    def erode_sweeps(self, h, min_zval, num_iters, ep, sweep, halo):
        """The coherent batched erosion on one device (see tw_erode_sweeps); in place, returns the droplet moves."""
        ys, xs = h.shape
        moves = C.c_uint64()
        self._check(lib.tw_erode_sweeps(self._h, _ptr(h), xs, ys, min_zval, num_iters, C.byref(ep), sweep, halo, C.byref(moves)))
        return moves.value

    def erode_sweeps_banded(self, bands, xsize, ysize, min_zval, num_iters, ep, sweep, halo):
        """tw_erode_sweeps_banded: the multi-GPU band decomposition with all bands on this device (in place; bands = row bands as multi_range deals them)."""
        moves = C.c_uint64()
        ptrs = (C.c_void_p * len(bands))(*[_ptr(b).value for b in bands])
        self._check(lib.tw_erode_sweeps_banded(self._h, C.cast(ptrs, C.c_void_p), len(bands), xsize, ysize, min_zval, num_iters, C.byref(ep), sweep, halo, C.byref(moves)))
        return moves.value

    def erode_tiles(self, tiles, num_iters, ep, min_zvals=None, min_zval_all=0.0):
        nt, ys, xs = tiles.shape
        mz = None if min_zvals is None else np.ascontiguousarray(min_zvals, np.float32)
        self._check(lib.tw_erode_tiles(self._h, _ptr(tiles), nt, xs, ys, _ptr(mz), min_zval_all, num_iters, C.byref(ep)))
        return tiles

    @property
    def last_erosion_steps(self):
        return int(lib.tw_last_erosion_steps(self._h))

    def voxel_fill(self, vp, rdata=None, out=None):
        if out is None:
            out = np.empty((vp.ny, vp.nx, vp.nz), np.float32)
        rd = None if rdata is None else np.ascontiguousarray(rdata, np.float32)
        self._check(lib.tw_voxel_fill(self._h, C.byref(vp), _ptr(rd), _ptr(out)))
        return out

    def tile_shadows(self, tiles, tile_xy, sp, out=None, sh_in_x=None, sh_in_y=None):
        """calc_mesh_shadows for a batch of tiles with neighbour chaining: returns (smask [nt, zv, zv] uint8, sh_out_x [nt, zv], sh_out_y [nt, zv]).
        sh_in_x / sh_in_y ([nt, zv] float32, numpy or CUDA): incoming heights from neighbours outside the batch (tw_tile_shadows_batch_ex)."""
        nt, zv = int(tiles.shape[0]), int(tiles.shape[1])
        txy = np.ascontiguousarray(tile_xy, np.int32).reshape(-1, 2)
        if out is None:
            out = np.empty((nt, zv, zv), np.uint8)
        ox, oy = np.empty((nt, zv), np.float32), np.empty((nt, zv), np.float32)
        if sh_in_x is None and sh_in_y is None:
            self._check(lib.tw_tile_shadows_batch(self._h, _ptr(tiles), _ptr(txy), nt, zv, C.byref(sp), _ptr(out), _ptr(ox), _ptr(oy)))
        else:
            ix, iy = _edge(sh_in_x), _edge(sh_in_y)
            self._check(lib.tw_tile_shadows_batch_ex(self._h, _ptr(tiles), _ptr(txy), nt, zv, C.byref(sp), _ptr(ix), _ptr(iy), _ptr(out), _ptr(ox), _ptr(oy)))
        return out, ox, oy

    def tile_weights(self, tiles, origins_xy, mesh_size, dx, dy, hp, wp, tile_params, out=None, want_grass_flags=True):
        """tile_t::create_texture's terrain part for a batch of tiles (tw_tile_weights_batch): returns (rgba [nt, zv-1, zv-1, 4] uint8, has_any_grass [nt] uint8 or None)."""
        nt, zv = int(tiles.shape[0]), int(tiles.shape[1])
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        tp = tile_params if hasattr(tile_params, "data_ptr") else np.ascontiguousarray(tile_params, np.float32).reshape(nt, 8)
        if out is None:
            out = np.empty((nt, zv - 1, zv - 1, 4), np.uint8)
        flags = np.empty(nt, np.uint8) if want_grass_flags else None
        self._check(lib.tw_tile_weights_batch(self._h, _ptr(tiles), _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, zv, C.byref(hp), C.byref(wp), _ptr(tp), _ptr(out), _ptr(flags)))
        return out, flags

    # ---- voxel post-processing (N3) ----
    def voxel_outside(self, vals, vpp, zix_xy=None, out=None):
        """determine_voxels_outside: flag byte per voxel (vals / out: numpy [ny, nx, nz] or CUDA tensors)."""
        if out is None:
            out = np.empty((vpp.ny, vpp.nx, vpp.nz), np.uint8)
        z = None if zix_xy is None else (zix_xy if hasattr(zix_xy, "data_ptr") else np.ascontiguousarray(zix_xy, np.uint32))
        self._check(lib.tw_voxel_outside(self._h, _ptr(vals), C.byref(vpp), _ptr(z), _ptr(out)))
        return out

    def voxel_remove_unconnected(self, vals, outside, vpp):
        """remove_unconnected_outside (+ remove_interior_holes): in place on vals and outside; returns the number of voxels flipped."""
        ch = C.c_uint64()
        self._check(lib.tw_voxel_remove_unconnected(self._h, _ptr(vals), _ptr(outside), C.byref(vpp), C.byref(ch)))
        return ch.value

    def voxel_triangles(self, vals, outside, vpp, tables, out=None):
        """Marching cubes over the grid: unwelded triangle soup [ntris, 3, 3] in the reference's emission order (out: optional CUDA tensor, truncated to its capacity)."""
        e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
        n = C.c_uint64()
        if out is None:
            self._check(lib.tw_voxel_triangles(self._h, _ptr(vals), _ptr(outside), C.byref(vpp), _ptr(e), _ptr(t), _ptr(v), None, 0, C.byref(n)))
            out = np.empty((n.value, 3, 3), np.float32)
            if n.value == 0:
                return out
        cap = int(out.shape[0])
        self._check(lib.tw_voxel_triangles(self._h, _ptr(vals), _ptr(outside), C.byref(vpp), _ptr(e), _ptr(t), _ptr(v), _ptr(out), cap, C.byref(n)))
        return out if isinstance(out, np.ndarray) else (out, n.value)

    def from_floats_u16(self, vals, val_mult, val_add, out=None):
        n = int(np.prod(vals.shape))
        if out is None:
            out = np.empty(2 * n, np.uint8)
        self._check(lib.tw_heightmap_from_floats_u16(self._h, _ptr(vals), n, val_mult, val_add, _ptr(out)))
        return out

    def to_floats_u16(self, data, val_mult, val_add, out=None):
        n = int(np.prod(data.shape)) // 2
        if out is None:
            out = np.empty(n, np.float32)
        self._check(lib.tw_heightmap_to_floats_u16(self._h, _ptr(data), n, val_mult, val_add, _ptr(out)))
        return out

    def proc_gen_heightmap(self, width, height, dx_val, dy_val, hp, erosion_iters, ep, data16=None, vals=None):
        """heightmap_t::proc_gen in one call; returns (16-bit image bytes, info, vals or None)."""
        if data16 is None:
            data16 = np.empty(2 * width * height, np.uint8)
        info = HeightmapInfo()
        self._check(lib.tw_proc_gen_heightmap(self._h, width, height, dx_val, dy_val, C.byref(hp), erosion_iters, C.byref(ep), _ptr(data16), _ptr(vals), C.byref(info)))
        return data16, info, vals

    def minmax(self, vals):
        mm = MinMax()
        self._check(lib.tw_minmax_f32(self._h, _ptr(vals), int(np.prod(vals.shape)), C.byref(mm)))
        return mm.zmin, mm.zmax


def gen_tex_height_tables(water_h_off_rel=0.0, temperature=20.0, glaciate_exp=3.0):
    """init_terrain_mesh + gen_tex_height_tables on the host (tw_gen_tex_height_tables): (h_dirt[5], tex_class[5], clip_hd1)."""
    h, ids, clip = (C.c_float * 5)(), (C.c_int * 5)(), C.c_float()
    lib.tw_gen_tex_height_tables(water_h_off_rel, temperature, glaciate_exp, C.cast(h, C.c_void_p), C.cast(ids, C.c_void_p), C.cast(C.byref(clip), C.c_void_p))
    return [float(v) for v in h], [int(v) for v in ids], float(clip.value)

