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
TW_OK, TW_ERR_NO_DEVICE, TW_ERR_CUDA, TW_ERR_ARG, TW_ERR_STATE, TW_ERR_NOT_READY, TW_ERR_CANCELED = 0, -1, -2, -3, -4, -5, -6
TW_EROSION_SERIAL, TW_EROSION_OPENMP, TW_EROSION_SWEEPS = 0, 1, 2
PQ_SIN_TERMS, PQ_SIN_TERMS_SCALED, PQ_EXACT_ZVAL, PQ_HMAP = 0, 1, 2, 3   # tw_point_query.kind (PQ_HMAP: tw_points_launch only)


class TwError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("tw3d status %d: %s" % (status, msg))
        self.status = status


class TwCanceled(TwError):
    """A poll completed a job that Context.cancel() cut short (TW_ERR_CANCELED): the job's outputs are unspecified."""


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


class VoxelBuild(C.Structure):
    """tw_voxel_build (include/tw3d.h): one asynchronous voxel build - optional fill, outside flags, remove_unconnected and marching cubes."""
    _fields_ = [("fill", C.c_void_p), ("rdata420", C.c_void_p), ("post", C.c_void_p), ("zix_xy", C.c_void_p), ("edge_table256", C.c_void_p),
                ("tri_table256x16", C.c_void_p), ("edge_to_vals12x2", C.c_void_p), ("vals", C.c_void_p), ("outside", C.c_void_p), ("tris", C.c_void_p),
                ("capacity", C.c_uint64), ("ntris", C.c_void_p), ("changed", C.c_void_p)]


class VoxelMesh(C.Structure):
    """tw_voxel_mesh (include/tw3d.h): the welded mesh's outputs - vertices, triangle indices, and the host counts."""
    _fields_ = [("verts", C.c_void_p), ("vcapacity", C.c_uint64), ("indices", C.c_void_p), ("tcapacity", C.c_uint64), ("nverts", C.c_void_p), ("ntris", C.c_void_p)]


class VoxelBlockMesh(C.Structure):
    """tw_voxel_block_mesh (include/tw3d.h): one listed block's vertex and triangle ranges in a voxel model job's outputs."""
    _fields_ = [("block", C.c_uint32), ("pad", C.c_uint32), ("voff", C.c_uint64), ("nverts", C.c_uint64), ("toff", C.c_uint64), ("ntris", C.c_uint64)]


class VoxelBlocksOut(C.Structure):
    """tw_voxel_blocks_out (include/tw3d.h): a voxel model job's mesh buffers, block table and host counts."""
    _fields_ = [("verts", C.c_void_p), ("vcapacity", C.c_uint64), ("indices", C.c_void_p), ("tcapacity", C.c_uint64), ("blocks", C.c_void_p),
                ("nblocks", C.c_void_p), ("nverts", C.c_void_p), ("ntris", C.c_void_p), ("changed", C.c_void_p)]


class VoxelChanges(C.Structure):
    """tw_voxel_changes (include/tw3d.h): the voxels an edit changed - index, value and flags buffers, their capacity, and the host count."""
    _fields_ = [("index", C.c_void_p), ("vals", C.c_void_p), ("outside", C.c_void_p), ("capacity", C.c_uint64), ("nchanged", C.c_void_p)]


class VoxelModelBuild(C.Structure):
    """tw_voxel_model_build (include/tw3d.h): one model of tw_voxel_model_build_batch_launch and the arguments of its tw_voxel_model_build_launch_on."""
    _fields_ = [("model", C.c_void_p), ("fill", C.c_void_p), ("rdata420", C.c_void_p), ("vals", C.c_void_p), ("out", C.c_void_p)]


class VoxelModelEdit(C.Structure):
    """tw_voxel_model_edit (include/tw3d.h): one model of tw_voxel_model_edit_batch_launch and the arguments of its tw_voxel_model_edit_launch_on."""
    _fields_ = [("model", C.c_void_p), ("boxes", C.c_void_p), ("nboxes", C.c_uint32), ("values", C.c_void_p), ("out", C.c_void_p), ("ch", C.c_void_p)]


class VoxelBox(C.Structure):
    """tw_voxel_box (include/tw3d.h): the voxels [x, x+w) x [y, y+h) x [z, z+d)."""
    _fields_ = [(n, C.c_uint32) for n in ("x", "y", "z", "w", "h", "d")]


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


class TileSetLight(C.Structure):
    """tw_tile_set_light (include/tw3d.h): one light of a tile set relight (smask required; sh_out_* optional)."""
    _fields_ = [("sp", ShadowParams), ("smask", C.c_void_p), ("sh_out_x", C.c_void_p), ("sh_out_y", C.c_void_p)]


class TileSetRequest(C.Structure):
    """tw_tile_set_request (include/tw3d.h): the resident tiles a relight outputs, its lights, and the optional host recomputed flags."""
    _fields_ = [("tile_xy", C.c_void_p), ("n", C.c_uint32), ("nlights", C.c_uint32), ("lights", C.c_void_p), ("recomputed", C.c_void_p)]


class TileSetFrame(C.Structure):
    """tw_tile_set_frame (include/tw3d.h): a frame launch's removes, the new tiles' grid coordinates, the optional heightmap sampler and relight request."""
    _fields_ = [("remove_xy", C.c_void_p), ("nremove", C.c_uint32), ("tile_xy", C.c_void_p), ("hs", C.c_void_p), ("relight", C.c_void_p)]


class PointQuery(C.Structure):
    _fields_ = [("kind", C.c_int), ("xy_scale", C.c_float), ("mesh_x_size", C.c_int), ("mesh_y_size", C.c_int), ("x_scene_size", C.c_float),
                ("y_scene_size", C.c_float), ("xoff2", C.c_int), ("yoff2", C.c_int), ("no_xyoff", C.c_int)]


class HmapSampler(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("edge_mode", C.c_int), ("mesh_scale", C.c_float), ("h_scale", C.c_float),
                ("mesh_file_scale", C.c_float), ("mesh_file_tz", C.c_float), ("mesh_scale_z_inv", C.c_float)]


class PointsJobArgs(C.Structure):
    """tw_points_job (include/tw3d.h): the points, the query and, for PQ_HMAP, the heightmap sampler of one tw_points_launch, and where the heights go."""
    _fields_ = [("xy", C.c_void_p), ("n", C.c_size_t), ("p", C.c_void_p), ("q", C.c_void_p), ("hs", C.c_void_p), ("out", C.c_void_p)]


class HmapRect(C.Structure):
    """tw_hmap_rect (include/tw3d.h): texels [x, x + w) x [y, y + h) of the heightmap image."""
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("w", C.c_int), ("h", C.c_int)]


class HmapReadArgs(C.Structure):
    """tw_hmap_read (include/tw3d.h): the rects of one tw_read_heightmap_launch and where their texels go (texel (x, y) -> dst16 + y*dst_pitch + 2*x)."""
    _fields_ = [("rects", C.c_void_p), ("nrects", C.c_uint32), ("dst16", C.c_void_p), ("dst_pitch", C.c_size_t)]


class HeightmapInfo(C.Structure):
    _fields_ = [("min_z", C.c_float), ("max_z", C.c_float), ("val_mult", C.c_float), ("val_add", C.c_float), ("mesh_file_scale", C.c_float),
                ("mesh_file_tz", C.c_float), ("erosion_moves", C.c_uint64)]


class HeightmapOutputs(C.Structure):
    """tw_heightmap_outputs (include/tw3d.h): where tw_proc_gen_heightmap_launch puts the image, the eroded heights and the info, and whether the image
    becomes the context's set_heightmap image."""
    _fields_ = [("data16", C.c_void_p), ("vals", C.c_void_p), ("info", C.c_void_p), ("set_image", C.c_int)]


class ErosionJobArgs(C.Structure):
    """tw_erosion_job (include/tw3d.h): the map tw_erode_launch erodes (a float map, or the context's set_heightmap image when heightmap is NULL) and how."""
    _fields_ = [("heightmap", C.c_void_p), ("xsize", C.c_int), ("ysize", C.c_int), ("min_zval", C.c_float), ("val_mult", C.c_float), ("val_add", C.c_float),
                ("num_iters", C.c_uint32), ("ep", C.c_void_p), ("mode", C.c_int), ("num_threads", C.c_uint32), ("vals", C.c_void_p)]


class GenMeshInfo(C.Structure):
    """tw_gen_mesh_info (include/tw3d.h): the z globals gen_mesh leaves and the erosion's droplet moves, filled by the poll that completes the job."""
    _fields_ = [(n, C.c_float) for n in ("zmin", "zmax", "zmax_est", "zbottom", "ztop", "water_plane_z")] + [("erosion_moves", C.c_uint64)]


class GenMeshJobArgs(C.Structure):
    """tw_gen_mesh_job (include/tw3d.h): the arguments of one tw_gen_mesh_launch."""
    _fields_ = [("mesh_x_size", C.c_int), ("mesh_y_size", C.c_int), ("xoff2", C.c_int), ("yoff2", C.c_int), ("dx_val", C.c_float), ("dy_val", C.c_float),
                ("x_scene_size", C.c_float), ("y_scene_size", C.c_float), ("p", C.c_void_p), ("erosion_iters", C.c_uint32), ("ep", C.c_void_p),
                ("water_h_off", C.c_float), ("water_h_off_rel", C.c_float), ("prev_zbottom", C.c_float), ("prev_ztop", C.c_float),
                ("prev_water_plane_z", C.c_float), ("mesh", C.c_void_p), ("info", C.c_void_p)]


class MeshShadowsJobArgs(C.Structure):
    """tw_mesh_shadows_job (include/tw3d.h): one mesh and the lights tw_mesh_shadows_launch traces over it."""
    _fields_ = [("mesh", C.c_void_p), ("xsize", C.c_int), ("ysize", C.c_int), ("nlights", C.c_uint32), ("lights", C.c_void_p)]


class SweepParams(C.Structure):
    """tw_sweep_params (include/tw3d.h): tw_erode_sweeps' sweep and halo for tw_erode_launch_ex's TW_EROSION_SWEEPS mode."""
    _fields_ = [("sweep", C.c_uint32), ("halo", C.c_int)]


class Rng(C.Structure):
    _fields_ = [("rseed1", C.c_int64), ("rseed2", C.c_int64)]


def hmap_params(**kw):
    """hmap_params_t with the reference defaults (src/mesh.h:85-88)."""
    h = HmapParams(1000.0, 0, 0, 0, 1000.0, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    for k, v in kw.items():
        setattr(h, k, v)
    return h


# every symbol include/tw3d.h declares (tests check the library exports exactly these)
ABI_SYMBOLS = ["tw_abi_version", "tw_create", "tw_create_shared", "tw_destroy", "tw_last_error", "tw_sync", "tw_stream", "tw_launch_count",
               "tw_dwarp_window_launches",
               "tw_build_sin_table", "tw_compute_scale", "tw_gen_sine_params", "tw_gen_rx_ry", "tw_noise3d_gen_sines",
               "tw_water_z_height", "tw_set_sin_table", "tw_set_sine_params", "tw_heightgen_2d", "tw_heightgen_2d_launch",
               "tw_heightgen_2d_poll", "tw_heightgen_tiles", "tw_create_zvals_batch", "tw_create_tiles_launch", "tw_create_tiles_launch_ex", "tw_create_tiles_poll", "tw_tile_bounds_batch", "tw_tile_normals_batch", "tw_tile_ao_batch", "tw_create_zvals_ao_batch", "tw_glaciate_mesh", "tw_eval_points", "tw_erode", "tw_erode_parallel", "tw_erode_tiles", "tw_last_erosion_steps", "tw_voxel_fill",
               "tw_heightmap_from_floats_u16", "tw_heightmap_to_floats_u16", "tw_proc_gen_heightmap", "tw_heightmap_sample_tiles", "tw_set_heightmap", "tw_create_tiles_launch_hmap", "tw_minmax_f32",
               "tw_multi_create", "tw_multi_destroy", "tw_multi_size", "tw_multi_ctx", "tw_multi_last_error", "tw_multi_set_sine_params", "tw_multi_range",
               "tw_multi_alloc_host", "tw_multi_free_host", "tw_create_zvals_sharded", "tw_heightgen_2d_sharded", "tw_dist_unique_id", "tw_dist_init",
               "tw_dist_allreduce_minmax", "tw_dist_finalize", "tw_bind_thread_to_device", "tw_erode_sweeps", "tw_erode_sweeps_banded", "tw_erode_sweeps_sharded", "tw_voxel_outside", "tw_voxel_remove_unconnected", "tw_voxel_triangles", "tw_tile_shadows_batch", "tw_tile_shadows_batch_ex", "tw_create_tiles_launch_shadows", "tw_tile_weights_batch", "tw_gen_tex_height_tables",
               "tw_tile_set_create", "tw_tile_set_destroy", "tw_tile_set_put", "tw_tile_set_remove", "tw_tile_set_stale", "tw_tile_set_shadows_launch",
               "tw_tile_set_create_tiles_launch", "tw_tile_set_stale_after", "tw_voxel_build_launch",
               "tw_proc_gen_heightmap_launch", "tw_erode_launch", "tw_cancel", "tw_erode_launch_ex",
               "tw_update_heightmap", "tw_hmap_tiles_touched", "tw_voxel_mesh_welded", "tw_voxel_build_launch_ex",
               "tw_voxel_model_create", "tw_voxel_model_destroy", "tw_voxel_model_build_launch", "tw_voxel_model_edit_launch", "tw_voxel_model_read",
               "tw_voxel_model_edit_launch_ex", "tw_voxel_model_build_launch_on", "tw_voxel_model_edit_launch_on", "tw_voxel_model_read_launch",
               "tw_points_launch", "tw_gen_mesh_launch", "tw_mesh_shadows", "tw_mesh_shadows_launch", "tw_gen_mesh_launch_shadows",
               "tw_read_heightmap_launch", "tw_read_heightmap", "tw_voxel_build_batch_launch",
               "tw_voxel_model_build_batch_launch", "tw_voxel_model_edit_batch_launch"]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError("3dworld_b200: %s is missing - build it with `python 3dworld_b200/build.py` (or __graft_entry__.build()); "
                          "there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, fp = C.c_void_p, C.POINTER(C.c_float)
    L.tw_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.tw_create_shared.argtypes = [vp, C.POINTER(vp)]
    L.tw_destroy.argtypes = [vp]
    L.tw_destroy.restype = None
    L.tw_last_error.argtypes = [vp]
    L.tw_last_error.restype = C.c_char_p
    L.tw_sync.argtypes = [vp]
    L.tw_stream.argtypes = [vp]
    L.tw_stream.restype = vp
    L.tw_launch_count.argtypes = [vp]
    L.tw_launch_count.restype = C.c_uint64
    L.tw_dwarp_window_launches.argtypes = [vp]
    L.tw_dwarp_window_launches.restype = C.c_uint64
    L.tw_cancel.argtypes = [vp]
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
    L.tw_update_heightmap.argtypes = [vp, vp, C.c_size_t, vp, C.c_uint32]
    L.tw_read_heightmap_launch.argtypes = [vp, C.POINTER(HmapReadArgs)]
    L.tw_read_heightmap.argtypes = [vp, C.POINTER(HmapReadArgs)]
    L.tw_hmap_tiles_touched.argtypes = [C.POINTER(HmapSampler), vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, vp]
    L.tw_eval_points.argtypes = [vp, vp, C.c_size_t, C.POINTER(HeightParams), C.POINTER(PointQuery), vp]
    L.tw_points_launch.argtypes = [vp, C.POINTER(PointsJobArgs)]
    L.tw_gen_mesh_launch.argtypes = [vp, C.POINTER(GenMeshJobArgs)]
    L.tw_gen_mesh_launch_shadows.argtypes = [vp, C.POINTER(GenMeshJobArgs), C.c_uint32, vp]
    L.tw_mesh_shadows.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(ShadowParams), vp, vp, vp, vp, vp]
    L.tw_mesh_shadows_launch.argtypes = [vp, C.POINTER(MeshShadowsJobArgs)]
    L.tw_erode_parallel.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(ErosionParams), C.c_uint32]
    L.tw_erode_launch.argtypes = [vp, C.POINTER(ErosionJobArgs)]
    L.tw_erode_launch_ex.argtypes = [vp, C.POINTER(ErosionJobArgs), C.POINTER(SweepParams)]
    L.tw_erode_tiles.argtypes = [vp, vp, C.c_uint32, C.c_int, C.c_int, vp, C.c_float, C.c_uint32, C.POINTER(ErosionParams)]
    L.tw_last_erosion_steps.argtypes = [vp]
    L.tw_last_erosion_steps.restype = C.c_uint64
    L.tw_voxel_fill.argtypes = [vp, C.POINTER(VoxelParams), vp, vp]
    L.tw_heightmap_from_floats_u16.argtypes = [vp, vp, C.c_size_t, C.c_float, C.c_float, vp]
    L.tw_heightmap_to_floats_u16.argtypes = [vp, vp, C.c_size_t, C.c_float, C.c_float, vp]
    L.tw_proc_gen_heightmap.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.POINTER(HeightParams), C.c_uint32, C.POINTER(ErosionParams), vp, vp,
                                        C.POINTER(HeightmapInfo)]
    L.tw_proc_gen_heightmap_launch.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.POINTER(HeightParams), C.c_uint32, C.POINTER(ErosionParams),
                                               C.POINTER(HeightmapOutputs)]
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
    L.tw_voxel_build_launch.argtypes = [vp, C.POINTER(VoxelBuild)]
    L.tw_voxel_mesh_welded.argtypes = [vp, vp, vp, C.POINTER(VoxelPostParams), vp, vp, vp, C.POINTER(VoxelMesh)]
    L.tw_voxel_build_launch_ex.argtypes = [vp, C.POINTER(VoxelBuild), C.POINTER(VoxelMesh)]
    L.tw_voxel_build_batch_launch.argtypes = [vp, C.POINTER(VoxelBuild), C.POINTER(VoxelMesh), C.c_uint32]
    L.tw_voxel_model_create.argtypes = [vp, C.POINTER(VoxelPostParams), vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.POINTER(vp)]
    L.tw_voxel_model_destroy.argtypes = [vp]
    L.tw_voxel_model_destroy.restype = None
    L.tw_voxel_model_build_launch.argtypes = [vp, C.POINTER(VoxelParams), vp, vp, C.POINTER(VoxelBlocksOut)]
    L.tw_voxel_model_edit_launch.argtypes = [vp, vp, C.c_uint32, vp, C.POINTER(VoxelBlocksOut)]
    L.tw_voxel_model_read.argtypes = [vp, vp, vp, vp]
    L.tw_voxel_model_edit_launch_ex.argtypes = [vp, vp, C.c_uint32, vp, C.POINTER(VoxelBlocksOut), C.POINTER(VoxelChanges)]
    L.tw_voxel_model_build_launch_on.argtypes = [vp] + L.tw_voxel_model_build_launch.argtypes
    L.tw_voxel_model_edit_launch_on.argtypes = [vp] + L.tw_voxel_model_edit_launch_ex.argtypes
    L.tw_voxel_model_read_launch.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, vp]
    L.tw_voxel_model_build_batch_launch.argtypes = [vp, C.POINTER(VoxelModelBuild), C.c_uint32]
    L.tw_voxel_model_edit_batch_launch.argtypes = [vp, C.POINTER(VoxelModelEdit), C.c_uint32]
    L.tw_tile_shadows_batch.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.POINTER(ShadowParams), vp, vp, vp]
    L.tw_tile_shadows_batch_ex.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.POINTER(ShadowParams), vp, vp, vp, vp, vp]
    L.tw_tile_set_create.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(vp)]
    L.tw_tile_set_destroy.argtypes = [vp]
    L.tw_tile_set_destroy.restype = None
    L.tw_tile_set_put.argtypes = [vp, vp, C.c_uint32, vp]
    L.tw_tile_set_remove.argtypes = [vp, vp, C.c_uint32]
    L.tw_tile_set_stale.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(C.c_uint32)]
    L.tw_tile_set_shadows_launch.argtypes = [vp, C.POINTER(TileSetRequest)]
    L.tw_tile_set_create_tiles_launch.argtypes = [vp, vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_float, C.POINTER(HeightParams), C.c_uint32,
                                                  C.POINTER(ErosionParams), C.c_float, C.c_float, C.c_uint32, C.POINTER(TileOutputs), C.POINTER(TileShading),
                                                  C.POINTER(TileSetFrame)]
    L.tw_tile_set_stale_after.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.POINTER(C.c_uint32)]
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


def _rects(rects):
    """[n, 4] (x, y, w, h) as a tw_hmap_rect array (None for n = 0) and n."""
    r = np.ascontiguousarray(rects, np.int32).reshape(-1, 4)
    arr = (HmapRect * max(1, len(r)))()
    C.memmove(arr, r.ctypes.data, r.nbytes)
    return (arr if len(r) else None), len(r)


def hmap_tiles_touched(hs, origins, zvsize, rects):
    """tw_hmap_tiles_touched (host only): uint8 [nt], 1 where some cell of the heightmap tile at origins[t] (x1, y1) reads, under hs (HmapSampler), a texel
    inside one of rects ([n, 4] x, y, w, h) - the live tiles an image edit changes."""
    org = np.ascontiguousarray(origins, np.int32).reshape(-1, 2)
    arr, n = _rects(rects)
    out = np.zeros(len(org), np.uint8)
    rc = lib.tw_hmap_tiles_touched(C.byref(hs), _ptr(org) if len(org) else None, len(org), int(zvsize), arr, n, _ptr(out) if len(org) else None)
    if rc != TW_OK:
        raise TwError(rc, "tw_hmap_tiles_touched: bad argument")
    return out


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


class VoxelBuildJob:
    """The host results of Context.voxel_build_launch, filled by the poll that completes the job."""

    def __init__(self):
        self._ntris, self._changed, self._nverts, self._mesh_ntris = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)

    @property
    def ntris(self):
        return int(self._ntris.value)

    @property
    def nverts(self):
        """Vertices of the welded mesh (a job launched with mesh outputs)."""
        return int(self._nverts.value)

    @property
    def mesh_ntris(self):
        """Triangles of the welded mesh (a job launched with mesh outputs)."""
        return int(self._mesh_ntris.value)

    @property
    def changed(self):
        return int(self._changed.value)


class VoxelBuildBatchJob:
    """The host results of Context.voxel_build_batch_launch, filled by the poll that completes the job: per grid, the welded mesh's nverts / ntris and the
    voxels remove_unconnected flipped (changed)."""

    def __init__(self, n):
        self._counts = (C.c_uint64 * (3 * n))()
        self.n = n

    def _col(self, k):
        return [int(self._counts[3 * i + k]) for i in range(self.n)]

    @property
    def nverts(self):
        return self._col(0)

    @property
    def ntris(self):
        return self._col(1)

    @property
    def changed(self):
        return self._col(2)


class VoxelModelJob:
    """The host results of a VoxelModel job, filled by the poll that completes it: blocks (numpy structured array of the listed blocks' VoxelBlockMesh
    rows: block, voff, nverts, toff, ntris), nverts, ntris and changed; for an edit launched with a change list, nchanged and changes."""

    def __init__(self, nblocks_max):
        self._table = (VoxelBlockMesh * max(nblocks_max, 1))()
        self._nblocks, self._nverts, self._ntris, self._changed = C.c_uint32(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._nchanged, self._change_bufs = C.c_uint64(0), None

    def _changes(self, changes):
        """VoxelChanges of (index, vals, outside) buffers, each None or a CUDA tensor / page-locked buffer; the capacity is index's length."""
        index, vals, outside = changes
        self._change_bufs = (index, vals, outside)
        cap = 0 if index is None else (int(index.numel()) if hasattr(index, "numel") else int(index.size))
        return VoxelChanges(_ptr(index), _ptr(vals), _ptr(outside), cap, C.cast(C.pointer(self._nchanged), C.c_void_p))

    @property
    def nchanged(self):
        """Voxels whose value or flags the edit changed (may exceed the change list's capacity)."""
        return int(self._nchanged.value)

    @property
    def changes(self):
        """(index, vals, outside): the caller's buffers cut to the listed entries, min(capacity, nchanged); None where no buffer was given."""
        index = self._change_bufs[0]
        k = min(self.nchanged, 0 if index is None else (int(index.numel()) if hasattr(index, "numel") else int(index.size)))
        return tuple(None if b is None else b[:k] for b in self._change_bufs)

    def _out(self, verts, indices):
        size = lambda a: 0 if a is None else (int(a.numel()) if hasattr(a, "numel") else int(a.size)) // 3  # noqa: E731
        p = lambda c: C.cast(C.pointer(c), C.c_void_p)  # noqa: E731
        return VoxelBlocksOut(_ptr(verts), size(verts), _ptr(indices), size(indices), C.cast(self._table, C.c_void_p), p(self._nblocks), p(self._nverts),
                              p(self._ntris), p(self._changed))

    @property
    def blocks(self):
        n = int(self._nblocks.value)
        return np.ctypeslib.as_array(self._table)[:n].copy() if n else np.zeros(0, np.ctypeslib.as_array(self._table).dtype)

    @property
    def nverts(self):
        return int(self._nverts.value)

    @property
    def ntris(self):
        return int(self._ntris.value)

    @property
    def changed(self):
        return int(self._changed.value)


class HeightmapJob:
    """The host result of Context.proc_gen_heightmap_launch: info (HeightmapInfo) is filled by the poll that completes the job."""

    def __init__(self):
        self.info = HeightmapInfo()


class ErosionJob:
    """What Context.erode_launch / erode_image_launch return: the buffers the job writes (heightmap, vals), complete once the poll that completes the job
    returns; Context.last_erosion_steps then holds the job's droplet moves."""

    def __init__(self, heightmap=None, vals=None):
        self.heightmap, self.vals = heightmap, vals


class PointsJob:
    """What Context.points_launch returns: poll(wait) completes the job (the context's pending job) and returns out, or None while it runs (wait=False)."""

    def __init__(self, ctx, out):
        self._ctx, self.out = ctx, out

    def poll(self, wait=False):
        return self.out if self._ctx.create_tiles_poll(wait) else None


class HmapReadJob(PointsJob):
    """What Context.read_heightmap_launch returns: poll(wait) completes the job (the context's pending job) and returns out, or None while it runs
    (wait=False)."""


class VoxelReadJob(PointsJob):
    """What VoxelModel.read_launch returns: poll(wait) completes the job (the pending job of the Context it was launched on) and returns (raw, vals,
    outside), or None while it runs (wait=False)."""


class GenMeshJob:
    """What Context.gen_mesh_launch returns: poll(wait) completes the job (the context's pending job) and returns (mesh, info dict with the keys of
    scene.gen_mesh's plus erosion_moves), or None while it runs (wait=False). With lights it returns (mesh, info, shadows), shadows as MeshShadowsJob's."""

    def __init__(self, ctx, mesh, lights=None):
        self._ctx, self.mesh, self.info, self.lights = ctx, mesh, GenMeshInfo(), lights

    def poll(self, wait=False):
        if not self._ctx.create_tiles_poll(wait):
            return None
        info = {n: (int if n == "erosion_moves" else float)(getattr(self.info, n)) for n, _ in GenMeshInfo._fields_}
        if self.lights is None:
            return self.mesh, info
        return self.mesh, info, [(r.smask, r.sh_out_x, r.sh_out_y) for r in self.lights]


class MeshShadowsJob:
    """What Context.mesh_shadows_launch returns: poll(wait) completes the job (the context's pending job) and returns one (smask, sh_out_x, sh_out_y) per
    light, or None while it runs (wait=False)."""

    def __init__(self, ctx, lights):
        self._ctx, self.lights = ctx, lights

    def poll(self, wait=False):
        if not self._ctx.create_tiles_poll(wait):
            return None
        return [(r.smask, r.sh_out_x, r.sh_out_y) for r in self.lights]


def _mesh_lights(lights, xsize, ysize):
    """Light records for a whole xsize x ysize mesh and their TileLight array: each light is a Light, a (ShadowParams, smask, sh_out_x, sh_out_y, sh_in_x,
    sh_in_y) tuple, or a bare ShadowParams, whose smask [ysize, xsize] uint8, sh_out_x [xsize] and sh_out_y [ysize] float32 are new numpy arrays."""
    recs = []
    for lt in lights:
        if isinstance(lt, ShadowParams):
            lt = Light(lt, np.empty((ysize, xsize), np.uint8), np.empty(xsize, np.float32), np.empty(ysize, np.float32))
        elif not isinstance(lt, Light):
            lt = Light(*lt)
        recs.append(Light(lt.sp, lt.smask, lt.sh_out_x, lt.sh_out_y, _edge(lt.sh_in_x), _edge(lt.sh_in_y)))
    arr = (TileLight * max(1, len(recs)))()
    for i, r in enumerate(recs):
        arr[i] = TileLight(r.sp, _ptr(r.sh_in_x), _ptr(r.sh_in_y), _ptr(r.smask), _ptr(r.sh_out_x), _ptr(r.sh_out_y))
    return recs, arr


class Context:
    """One tw_ctx (device + stream + uploaded tables). All compute goes through the C ABI."""

    def __init__(self, device=0, sin_table=None):
        h = C.c_void_p()
        rc = lib.tw_create(device, C.byref(h))
        if rc != TW_OK:
            raise TwError(rc, "tw_create failed (no CUDA device? this library has no CPU fallback)")
        self._h = h
        self.device = device
        self.parent, self._shared, self._sets, self._models = None, [], [], []
        self._check(lib.tw_set_sin_table(self._h, _ptr(sin_table)))

    def shared(self):
        """tw_create_shared: a Context on this one's device that reads this one's tables (sin and direction tables, sine params, LUTs, the set_heightmap
        image) and has its own stream, scratch and pending job, so its asynchronous job runs beside this context's and the other shared ones'. Tables are
        set here only: on the shared Context the setters raise. It keeps a reference to this Context; close() here closes it first."""
        h = C.c_void_p()
        self._check(lib.tw_create_shared(self._h, C.byref(h)))
        s = Context.__new__(Context)
        s._h, s.device, s.parent, s._shared, s._sets, s._models = h, self.device, self, [], [], []
        self._shared.append(s)
        return s

    def tile_set(self, zvsize, nlights):
        """tw_tile_set_create: a TileSet of this context - the live tiles' zvals on the device and each light slot's cached mesh shadows."""
        return TileSet(self, zvsize, nlights)

    def voxel_model(self, vpp, tables, zix_xy=None, bx=32, by=32):
        """tw_voxel_model_create: a VoxelModel of this context - the field of grid vpp kept on the device, meshed per block of bx x by cube columns."""
        return VoxelModel(self, vpp, tables, zix_xy, bx, by)

    def close(self):
        if getattr(self, "_h", None) and lib is not None:   # lib can already be gone at interpreter shutdown
            for s in getattr(self, "_shared", ()):         # tw_destroy(parent) destroys them: their handles must not be destroyed again
                for ts in list(getattr(s, "_sets", ())) + list(getattr(s, "_models", ())):
                    ts._h = None
                s._h = None
            for ts in list(getattr(self, "_sets", ())) + list(getattr(self, "_models", ())):   # and this context's tile sets and voxel models
                ts._h = None
            lib.tw_destroy(self._h)
            if getattr(self, "parent", None) is not None and self in self.parent._shared:
                self.parent._shared.remove(self)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != TW_OK:
            raise (TwCanceled if rc == TW_ERR_CANCELED else TwError)(rc, lib.tw_last_error(self._h).decode())

    def cancel(self):
        """tw_cancel: asks this context's pending job to stop and returns at once. The poll that completes a job cut short raises TwCanceled; a job
        that has already finished, or has nothing left to cut, completes as usual. Raises TwError (TW_ERR_STATE) for a job that touches a TileSet."""
        self._check(lib.tw_cancel(self._h))

    @property
    def stream(self):
        return lib.tw_stream(self._h)

    @property
    def launch_count(self):
        return int(lib.tw_launch_count(self._h))

    @property
    def dwarp_window_launches(self):
        """Of launch_count, the launches of the domain-warp kernel with lattice windows (tw_dwarp_window_launches)"""
        return int(lib.tw_dwarp_window_launches(self._h))

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
        self._tiles_job = None
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
            self._hmap_size = None
            return
        if not hasattr(data16, "data_ptr"):
            data16 = np.ascontiguousarray(data16, np.uint8)
        if len(data16.shape) != 3 or data16.shape[2] != 2:
            raise ValueError("set_heightmap: data16 must have shape [h, w, 2]")
        self._check(lib.tw_set_heightmap(self._h, _ptr(data16), int(data16.shape[1]), int(data16.shape[0])))
        self._hmap_size = (int(data16.shape[1]), int(data16.shape[0]))

    def update_heightmap(self, data16, rects):
        """tw_update_heightmap: texels rects ([n, 4] x, y, w, h) of the set_heightmap image become those of data16 (uint8 [h, w, 2] host array, the whole
        edited image). Returns without completing any job or waiting for the GPU: jobs launched earlier see the old image, later ones the edited one. The
        texels are copied before the call returns, so data16 may change at once."""
        if hasattr(data16, "data_ptr") and data16.is_cuda:
            ptr, pitch = _ptr(data16), 2 * int(data16.shape[1])          # refused by the library: the source is host memory
        else:
            data16 = np.asarray(data16)
            if data16.dtype != np.uint8 or len(data16.shape) != 3 or data16.shape[2] != 2 or data16.strides[1:] != (2, 1):
                raise ValueError("update_heightmap: data16 must be uint8 [h, w, 2] with contiguous rows")
            ptr, pitch = C.c_void_p(data16.ctypes.data), int(data16.strides[0])
        arr, n = _rects(rects)
        self._check(lib.tw_update_heightmap(self._h, ptr, pitch, arr, n))

    def image_size(self):
        """(width, height) of the set_heightmap image this context reads (a shared context: its parent's), as the last set_heightmap or set_image
        heightmap job on the root gave it; None without one."""
        root = self.parent or self
        return getattr(root, "_hmap_size", None)

    def read_heightmap_launch(self, rects=None, out=None):
        """tw_read_heightmap_launch: the set_heightmap image's texels back, as this context's asynchronous job (also on a shared context, which reads its
        parent's image). rects = [n, 4] (x, y, w, h), default the whole image. out = uint8 [rows, cols, 2] with contiguous rows: a numpy array or a torch
        tensor, host (pageable or pinned) or CUDA, whose texel (x, y) is out[y, x] (its row pitch may exceed 2*cols); default a new numpy [h, w, 2] array.
        The job sees every update_heightmap made before the launch and none after it. Returns a HmapReadJob whose poll returns out."""
        size = self.image_size()
        if rects is None:
            if size is None:
                raise TwError(TW_ERR_STATE, "read_heightmap: the context has no heightmap image")
            rects = [(0, 0, size[0], size[1])]
        if out is None:
            if size is None:
                raise TwError(TW_ERR_STATE, "read_heightmap: the context has no heightmap image")
            out = np.zeros((size[1], size[0], 2), np.uint8)
        if hasattr(out, "data_ptr"):
            import torch
            if out.dtype != torch.uint8 or out.dim() != 3 or out.shape[2] != 2 or tuple(out.stride())[1:] != (2, 1):
                raise ValueError("read_heightmap: out must be uint8 [rows, cols, 2] with contiguous rows")
            ptr, pitch = C.c_void_p(out.data_ptr()), int(out.stride(0))
        else:
            if not isinstance(out, np.ndarray) or out.dtype != np.uint8 or out.ndim != 3 or out.shape[2] != 2 or out.strides[1:] != (2, 1):
                raise ValueError("read_heightmap: out must be uint8 [rows, cols, 2] with contiguous rows")
            ptr, pitch = C.c_void_p(out.ctypes.data), int(out.strides[0])
        arr, n = _rects(rects)
        a = HmapReadArgs(C.cast(arr, C.c_void_p) if n else None, n, ptr, pitch)
        self._check(lib.tw_read_heightmap_launch(self._h, C.byref(a)))
        job = HmapReadJob(self, out)
        self._tiles_job = (out, job)
        return job

    def read_heightmap(self, rects=None, out=None):
        """tw_read_heightmap: read_heightmap_launch(rects, out) completed at once; returns out (default the whole image as a new uint8 [h, w, 2] array)."""
        return self.read_heightmap_launch(rects, out).poll(wait=True)

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

    def points_launch(self, xy, hp=None, pq=None, hs=None, out=None):
        """tw_points_launch: eval_points (hp, pq of a PQ_* procedural kind) or, with pq.kind = PQ_HMAP and hs (HmapSampler), the heights of the set_heightmap
        image at cells xy, as this context's asynchronous job. xy = [n, 2] float32 numpy array or torch tensor (host xy is copied during the launch, CUDA xy
        stays referenced until the job completes); out = n floats (numpy array or torch tensor, host or CUDA; default a new numpy array). Returns a PointsJob."""
        n = int(xy.shape[0])
        if out is None:
            out = np.empty(n, np.float32)
        ref = lambda s: C.cast(C.pointer(s), C.c_void_p) if s is not None else None  # noqa: E731
        a = PointsJobArgs(_ptr(xy), n, ref(hp), ref(pq), ref(hs), _ptr(out))
        self._check(lib.tw_points_launch(self._h, C.byref(a)))
        job = PointsJob(self, out)
        self._tiles_job = (xy, out, hp, pq, hs, job)
        return job

    def gen_mesh_launch(self, mesh_size, hp, ep, erosion_iters=0, xoff2=0, yoff2=0, dx_val=None, dy_val=None, scene_size=(4.0, 4.0), water_h_off=0.0,
                        water_h_off_rel=0.0, prev=(0.0, 0.0, 0.0), mesh=None, lights=None):
        """tw_gen_mesh_launch: gen_mesh in ground mode after its sine table (set_sine_params first) as this context's asynchronous job. mesh_size =
        (MESH_X_SIZE, MESH_Y_SIZE); hp (its zmax_est is ignored) and ep (erode_amount, half_dxy, relh_adj_tex, clip_hd1 are read) are copied during the
        launch; dx_val / dy_val default to 1/hp.dx_val_inv, 1/hp.dy_val_inv; scene_size = (X_SCENE_SIZE, Y_SCENE_SIZE); prev = (zbottom, ztop, water_plane_z)
        before the call, which a flat mesh keeps. mesh = [MY, MX] floats (numpy array or torch tensor, host or CUDA; default a new numpy array).
        lights (tw_gen_mesh_launch_shadows): a list of lights as mesh_shadows_launch takes them, traced over the final mesh with the job's own zmin / zmax
        in place of each ShadowParams' (the GenMeshJob's poll then also returns the shadows). Returns a GenMeshJob."""
        MX, MY = int(mesh_size[0]), int(mesh_size[1])
        if mesh is None:
            mesh = np.empty((MY, MX), np.float32)
        dx = float(np.float32(1.0) / np.float32(hp.dx_val_inv)) if dx_val is None else dx_val
        dy = float(np.float32(1.0) / np.float32(hp.dy_val_inv)) if dy_val is None else dy_val
        recs, arr = _mesh_lights(lights, MX, MY) if lights is not None else (None, None)
        job = GenMeshJob(self, mesh, recs)
        a = GenMeshJobArgs(MX, MY, xoff2, yoff2, dx, dy, scene_size[0], scene_size[1], C.cast(C.pointer(hp), C.c_void_p), erosion_iters,
                           C.cast(C.pointer(ep), C.c_void_p), water_h_off, water_h_off_rel, prev[0], prev[1], prev[2], _ptr(mesh),
                           C.cast(C.pointer(job.info), C.c_void_p))
        if lights is None:
            self._check(lib.tw_gen_mesh_launch(self._h, C.byref(a)))
        else:
            self._check(lib.tw_gen_mesh_launch_shadows(self._h, C.byref(a), len(recs), C.cast(arr, C.c_void_p)))
        self._tiles_job = (mesh, job, arr)
        return job

    def mesh_shadows(self, mesh, sp, sh_in_x=None, sh_in_y=None):
        """tw_mesh_shadows: calc_mesh_shadows on the whole mesh [ysize, xsize] (numpy or CUDA) for one light: returns (smask [ysize, xsize] uint8,
        sh_out_x [xsize] float32, sh_out_y [ysize] float32). sh_in_x [xsize] / sh_in_y [ysize] (numpy or CUDA): incoming heights."""
        ysize, xsize = int(mesh.shape[0]), int(mesh.shape[1])
        out, ox, oy = np.empty((ysize, xsize), np.uint8), np.empty(xsize, np.float32), np.empty(ysize, np.float32)
        ix, iy = _edge(sh_in_x), _edge(sh_in_y)
        self._check(lib.tw_mesh_shadows(self._h, _ptr(mesh), xsize, ysize, C.byref(sp), _ptr(ix), _ptr(iy), _ptr(out), _ptr(ox), _ptr(oy)))
        return out, ox, oy

    def mesh_shadows_launch(self, mesh, lights):
        """tw_mesh_shadows_launch: calc_mesh_shadows on the whole mesh [ysize, xsize] (numpy or CUDA) for every light, as this context's asynchronous job.
        lights: Light records, (ShadowParams, smask, sh_out_x, sh_out_y, sh_in_x, sh_in_y) tuples - smask [ysize, xsize] uint8 required, sh_*_x [xsize]
        and sh_*_y [ysize] float32 or None - or bare ShadowParams (outputs allocated here). A host mesh and host sh_in rows are copied during the launch;
        the outputs and device inputs are kept referenced here until the job completes. Returns a MeshShadowsJob."""
        ysize, xsize = int(mesh.shape[0]), int(mesh.shape[1])
        recs, arr = _mesh_lights(lights, xsize, ysize)
        a = MeshShadowsJobArgs(_ptr(mesh), xsize, ysize, len(recs), C.cast(arr, C.c_void_p))
        self._check(lib.tw_mesh_shadows_launch(self._h, C.byref(a)))
        job = MeshShadowsJob(self, recs)
        self._tiles_job = (mesh, job, arr)
        return job

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

    def _erode_launch(self, job, heightmap, xsize, ysize, min_zval, val_mult, val_add, num_iters, ep, num_threads, vals, sweep=None, halo=None):
        if (sweep is None) != (halo is None):
            raise ValueError("sweep and halo select the sweeps mode together")
        sweeps = sweep is not None
        mode = TW_EROSION_SWEEPS if sweeps else TW_EROSION_SERIAL if num_threads is None else TW_EROSION_OPENMP
        a = ErosionJobArgs(_ptr(heightmap), xsize, ysize, min_zval, val_mult, val_add, num_iters, C.cast(C.pointer(ep), C.c_void_p), mode,
                           0 if num_threads is None else num_threads, _ptr(vals))
        sw = SweepParams(sweep, halo) if sweeps else None
        self._check(lib.tw_erode_launch_ex(self._h, C.byref(a), C.byref(sw) if sweeps else None))
        self._tiles_job = job
        return job

    def erode_launch(self, h, min_zval, num_iters, ep, num_threads=None, sweep=None, halo=None):
        """tw_erode_launch on h (numpy [ys, xs] or CUDA tensor, in place) as this context's asynchronous job; create_tiles_poll completes it.
        num_threads=None: the serial order (erode()); an int: the OpenMP mode (erode_parallel(num_threads), 0 = fill the GPU). sweep and halo (both):
        the sweeps mode (erode_sweeps(sweep, halo), tw_erode_launch_ex). h stays referenced until then."""
        ys, xs = h.shape
        return self._erode_launch(ErosionJob(heightmap=h), h, xs, ys, min_zval, 0.0, 0.0, num_iters, ep, num_threads, None, sweep, halo)

    def erode_image_launch(self, val_mult, val_add, num_iters, ep, num_threads=None, vals=None, sweep=None, halo=None):
        """tw_erode_launch on this context's set_heightmap image: unpack with val_mult / val_add, erode down to the image's minimum, pack back, as one
        asynchronous job. vals (optional, w*h floats, numpy array or CUDA tensor) receives the eroded floats before the pack. num_threads, sweep and halo
        as erode_launch."""
        return self._erode_launch(ErosionJob(vals=vals), None, 0, 0, 0.0, val_mult, val_add, num_iters, ep, num_threads, vals, sweep, halo)

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

    def voxel_mesh(self, vals, outside, vpp, tables, verts=None, indices=None):
        """tw_voxel_mesh_welded: create_block's indexed mesh -> (verts [nv, 3] float32, indices [nt, 3] uint32). verts / indices (optional, numpy or torch,
        host or CUDA) are filled up to their sizes and returned with the counts as (verts, indices, nverts, ntris)."""
        e, t, v = (np.ascontiguousarray(tables[0], np.uint32), np.ascontiguousarray(tables[1], np.int32), np.ascontiguousarray(tables[2], np.uint32))
        nv, nt = C.c_uint64(), C.c_uint64()
        given = verts is not None or indices is not None
        if not given:
            m = VoxelMesh(None, 0, None, 0, C.cast(C.pointer(nv), C.c_void_p), C.cast(C.pointer(nt), C.c_void_p))
            self._check(lib.tw_voxel_mesh_welded(self._h, _ptr(vals), _ptr(outside), C.byref(vpp), _ptr(e), _ptr(t), _ptr(v), C.byref(m)))
            verts, indices = np.empty((nv.value, 3), np.float32), np.empty((nt.value, 3), np.uint32)
        size = lambda a: 0 if a is None else (int(a.numel()) if hasattr(a, "numel") else int(a.size)) // 3
        m = VoxelMesh(_ptr(verts), size(verts), _ptr(indices), size(indices), C.cast(C.pointer(nv), C.c_void_p), C.cast(C.pointer(nt), C.c_void_p))
        self._check(lib.tw_voxel_mesh_welded(self._h, _ptr(vals), _ptr(outside), C.byref(vpp), _ptr(e), _ptr(t), _ptr(v), C.byref(m)))
        return (verts, indices, nv.value, nt.value) if given else (verts, indices)

    def voxel_build_launch(self, vpp, vals=None, outside=None, tris=None, fill=None, rdata=None, zix_xy=None, tables=None, capacity=None, mesh=None, soup=True):
        """tw_voxel_build_launch: fill (VoxelParams, optional) -> voxel_outside -> voxel_remove_unconnected -> voxel_triangles as one asynchronous job on
        this context; create_tiles_poll completes it. vals [ny, nx, nz] float32 is the input field without fill, else an optional output; outside
        [ny, nx, nz] uint8 optional output; tris: triangles out, a CUDA tensor or a page-locked numpy / torch buffer of capacity*9 floats (capacity defaults
        to its size // 9). numpy arrays, torch tensors or None. tables (edge_table, tri_table, edge_to_vals) or None = no triangles. Returns a VoxelBuildJob
        whose ntris / changed are valid once the job is complete. The outputs and device inputs stay referenced here until then.
        mesh = (verts, indices): also the welded mesh (tw_voxel_build_launch_ex), into a CUDA tensor or page-locked buffer each (None for none), filled up
        to their sizes; the job's nverts / mesh_ntris are its counts. soup=False with a mesh: no triangle soup (tris must be None)."""
        job = VoxelBuildJob()
        keep = [vals, outside, tris, mesh]
        tabs = (None, None, None)
        if tables is not None:
            tabs = tuple(t if hasattr(t, "data_ptr") else np.ascontiguousarray(t, dt) for t, dt in zip(tables, (np.uint32, np.int32, np.uint32)))
        z = None if zix_xy is None else (zix_xy if hasattr(zix_xy, "data_ptr") else np.ascontiguousarray(zix_xy, np.uint32))
        rd = None if rdata is None else np.ascontiguousarray(rdata, np.float32)
        if capacity is None:
            capacity = 0 if tris is None else (int(tris.numel()) if hasattr(tris, "numel") else int(tris.size)) // 9
        b = VoxelBuild(C.cast(C.pointer(fill), C.c_void_p) if fill is not None else None, _ptr(rd), C.cast(C.pointer(vpp), C.c_void_p), _ptr(z),
                       _ptr(tabs[0]), _ptr(tabs[1]), _ptr(tabs[2]), _ptr(vals), _ptr(outside), _ptr(tris), int(capacity),
                       C.cast(C.pointer(job._ntris), C.c_void_p) if tables is not None and (soup or mesh is None) else None,
                       C.cast(C.pointer(job._changed), C.c_void_p))
        if mesh is None:
            self._check(lib.tw_voxel_build_launch(self._h, C.byref(b)))
        else:
            size = lambda a: 0 if a is None else (int(a.numel()) if hasattr(a, "numel") else int(a.size)) // 3
            m = VoxelMesh(_ptr(mesh[0]), size(mesh[0]), _ptr(mesh[1]), size(mesh[1]), C.cast(C.pointer(job._nverts), C.c_void_p),
                          C.cast(C.pointer(job._mesh_ntris), C.c_void_p))
            self._check(lib.tw_voxel_build_launch_ex(self._h, C.byref(b), C.byref(m)))
        self._tiles_job = (keep, tabs, z, job)
        return job

    def voxel_build_batch_launch(self, grids, tables):
        """tw_voxel_build_batch_launch: many small grids (nx*ny*nz <= 2^18 each) built in one asynchronous job, each exactly as voxel_build_launch with
        mesh=(verts, indices) and soup=False would build it alone; create_tiles_poll completes it. grids: a list of dicts with the keys of voxel_build_launch -
        vpp (required), vals, outside, fill, rdata, zix_xy - and mesh = (verts, indices) (each a CUDA tensor, a page-locked buffer or None). tables (edge_table,
        tri_table, edge_to_vals) are shared by every grid. Returns a VoxelBuildBatchJob whose per-grid nverts / ntris / changed are valid once the job is
        complete. The outputs and device inputs stay referenced here until then."""
        n = len(grids)
        job = VoxelBuildBatchJob(max(n, 1))
        tabs = tuple(t if hasattr(t, "data_ptr") else np.ascontiguousarray(t, dt) for t, dt in zip(tables, (np.uint32, np.int32, np.uint32)))
        bs, ms, keep = (VoxelBuild * max(n, 1))(), (VoxelMesh * max(n, 1))(), [tabs]
        size = lambda a: 0 if a is None else (int(a.numel()) if hasattr(a, "numel") else int(a.size)) // 3
        base = C.addressof(job._counts)
        for i, g in enumerate(grids):
            z = g.get("zix_xy")
            z = None if z is None else (z if hasattr(z, "data_ptr") else np.ascontiguousarray(z, np.uint32))
            rd = None if g.get("rdata") is None else np.ascontiguousarray(g["rdata"], np.float32)
            vpp, fill = g["vpp"], g.get("fill")
            verts, indices = g.get("mesh", (None, None))
            keep.append((g, z, rd))
            bs[i] = VoxelBuild(C.cast(C.pointer(fill), C.c_void_p) if fill is not None else None, _ptr(rd), C.cast(C.pointer(vpp), C.c_void_p), _ptr(z),
                               _ptr(tabs[0]), _ptr(tabs[1]), _ptr(tabs[2]), _ptr(g.get("vals")), _ptr(g.get("outside")), None, 0, None, base + (24 * i + 16))
            ms[i] = VoxelMesh(_ptr(verts), size(verts), _ptr(indices), size(indices), base + 24 * i, base + (24 * i + 8))
        self._check(lib.tw_voxel_build_batch_launch(self._h, bs, ms, n))
        self._tiles_job = (keep, job)
        return job

    def voxel_model_build_batch_launch(self, builds):
        """tw_voxel_model_build_batch_launch: many small VoxelModels (nx*ny*nz <= 2^18 each) built in one asynchronous job on this Context, each exactly as
        its build_launch(ctx=self) would build it alone; create_tiles_poll completes it. builds: a list of dicts with the keys model (required) and fill,
        vals, rdata, verts, indices as VoxelModel.build_launch takes them. Returns one VoxelModelJob per entry, filled once the job is complete; the buffers
        stay referenced here until then."""
        n = len(builds)
        es, jobs, keep = (VoxelModelBuild * max(n, 1))(), [], []
        for i, b in enumerate(builds):
            m = b["model"]
            job = VoxelModelJob(m.nblocks)
            out = job._out(b.get("verts"), b.get("indices"))
            rd = None if b.get("rdata") is None else np.ascontiguousarray(b["rdata"], np.float32)
            fill = b.get("fill")
            keep.append((b, out, rd))
            es[i] = VoxelModelBuild(m._h, C.cast(C.pointer(fill), C.c_void_p) if fill is not None else None, _ptr(rd), _ptr(b.get("vals")),
                                    C.cast(C.pointer(out), C.c_void_p))
            jobs.append(job)
        self._check(lib.tw_voxel_model_build_batch_launch(self._h, es, n))
        self._tiles_job = (keep, jobs)
        return jobs

    def voxel_model_edit_batch_launch(self, edits):
        """tw_voxel_model_edit_batch_launch: edits of many small VoxelModels in one asynchronous job on this Context, each exactly as its
        edit_launch(ctx=self) would edit it alone; create_tiles_poll completes it. edits: a list of dicts with the keys model (required) and boxes, values,
        verts, indices, changes as VoxelModel.edit_launch takes them (boxes absent or empty: no change). Returns one VoxelModelJob per entry."""
        n = len(edits)
        es, jobs, keep = (VoxelModelEdit * max(n, 1))(), [], []
        for i, e in enumerate(edits):
            m, boxes = e["model"], e.get("boxes")
            boxes = [] if boxes is None else boxes
            b = (VoxelBox * max(len(boxes), 1))(*[VoxelBox(*[int(v) for v in t]) for t in boxes])
            vals = np.ascontiguousarray(e.get("values", np.zeros(0, np.float32)), np.float32).ravel()
            job = VoxelModelJob(m.nblocks)
            out = job._out(e.get("verts"), e.get("indices"))
            ch = None if e.get("changes") is None else job._changes(e["changes"])
            keep.append((e, b, vals, out, ch))
            es[i] = VoxelModelEdit(m._h, C.cast(b, C.c_void_p) if len(boxes) else None, len(boxes), _ptr(vals) if len(boxes) else None, C.cast(C.pointer(out), C.c_void_p),
                                   C.cast(C.pointer(ch), C.c_void_p) if ch is not None else None)
            jobs.append(job)
        self._check(lib.tw_voxel_model_edit_batch_launch(self._h, es, n))
        self._tiles_job = (keep, jobs)
        return jobs

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

    def proc_gen_heightmap_launch(self, width, height, dx_val, dy_val, hp, erosion_iters, ep, data16=None, vals=None, set_image=False):
        """tw_proc_gen_heightmap_launch: proc_gen_heightmap as one asynchronous job on this context; create_tiles_poll completes it. data16 (2*w*h bytes)
        and vals (w*h floats) are optional outputs - numpy arrays or CUDA tensors - but data16 or set_image is required; set_image makes the image this
        context's set_heightmap image once the job completes. Returns a HeightmapJob whose info is valid then. The outputs stay referenced here until then."""
        job = HeightmapJob()
        o = HeightmapOutputs(_ptr(data16), _ptr(vals), C.cast(C.pointer(job.info), C.c_void_p), 1 if set_image else 0)
        self._check(lib.tw_proc_gen_heightmap_launch(self._h, width, height, dx_val, dy_val, C.byref(hp), erosion_iters, C.byref(ep), C.byref(o)))
        if set_image:
            self._hmap_size = (int(width), int(height))
        self._tiles_job = (data16, vals, job)
        return job

    def minmax(self, vals):
        mm = MinMax()
        self._check(lib.tw_minmax_f32(self._h, _ptr(vals), int(np.prod(vals.shape)), C.byref(mm)))
        return mm.zmin, mm.zmax


class VoxelModel:
    """tw_voxel_model (include/tw3d.h): a voxel grid's raw field, outside flags and post-processed field kept on the device, meshed per block of bx x by
    cube columns. build_launch, edit_launch and read_launch are asynchronous jobs, completed by create_tiles_poll of the Context they run on; they cannot be
    cancelled. They run on the model's Context by default, or on ctx: its parent or a shared Context of that parent, so several strokes and reads are in
    flight at once, ordered on the device in launch order. Context.close() destroys the model with the context."""

    def __init__(self, ctx, vpp, tables, zix_xy, bx, by):
        self.tables = tuple(np.ascontiguousarray(t, dt) for t, dt in zip(tables, (np.uint32, np.int32, np.uint32)))
        z = None if zix_xy is None else (zix_xy if hasattr(zix_xy, "data_ptr") else np.ascontiguousarray(zix_xy, np.uint32))
        h = C.c_void_p()
        ctx._check(lib.tw_voxel_model_create(ctx._h, C.byref(vpp), _ptr(self.tables[0]), _ptr(self.tables[1]), _ptr(self.tables[2]), _ptr(z), int(bx), int(by),
                                             C.byref(h)))
        self._h, self.ctx, self.vpp, self.bx, self.by = h, ctx, vpp, int(bx), int(by)
        self.nbx, self.nby = (max(int(vpp.nx) - 1, 0) + self.bx - 1) // self.bx, (max(int(vpp.ny) - 1, 0) + self.by - 1) // self.by
        ctx._models.append(self)

    @property
    def nblocks(self):
        return self.nbx * self.nby

    def close(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.tw_voxel_model_destroy(self._h)
            if self in self.ctx._models:
                self.ctx._models.remove(self)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def build_launch(self, fill=None, vals=None, rdata=None, verts=None, indices=None, ctx=None):
        """tw_voxel_model_build_launch(_on): the raw field from fill (VoxelParams) or vals (numpy or CUDA tensor, [ny, nx, nz] float32), its flags and
        remove_unconnected, and every block's mesh into verts / indices (CUDA tensors or page-locked buffers, filled up to their sizes). Runs on ctx (default
        the model's Context). Returns a VoxelModelJob."""
        c = self.ctx if ctx is None else ctx
        job = VoxelModelJob(self.nblocks)
        rd = None if rdata is None else np.ascontiguousarray(rdata, np.float32)
        out = job._out(verts, indices)
        c._check(lib.tw_voxel_model_build_launch_on(c._h, self._h, C.byref(fill) if fill is not None else None, _ptr(rd), _ptr(vals), C.byref(out)))
        c._tiles_job = (vals, verts, indices, job)
        return job

    def edit_launch(self, boxes, values, verts=None, indices=None, changes=None, ctx=None):
        """tw_voxel_model_edit_launch(_on): boxes = (x, y, z, w, h, d) tuples, values = their new raw values one box after another, each in the grid's
        order (z fastest, then x, then y), copied during the launch. Re-meshes the blocks the edit changed; returns a VoxelModelJob listing them.
        changes = (index, vals, outside) (tw_voxel_model_edit_launch_ex): buffers for the list of the voxels the edit changed, each None or a CUDA tensor /
        page-locked buffer (uint32, float32, uint8) of the list's capacity; the job's nchanged and changes hold the list once it completes. Runs on ctx
        (default the model's Context)."""
        c = self.ctx if ctx is None else ctx
        b = (VoxelBox * max(len(boxes), 1))(*[VoxelBox(*[int(v) for v in t]) for t in boxes])
        vals = np.ascontiguousarray(values, np.float32).ravel()
        job = VoxelModelJob(self.nblocks)
        out = job._out(verts, indices)
        ch = None if changes is None else job._changes(changes)
        c._check(lib.tw_voxel_model_edit_launch_on(c._h, self._h, C.cast(b, C.c_void_p) if len(boxes) else None, len(boxes), _ptr(vals) if len(boxes) else None,
                                                   C.byref(out), C.byref(ch) if ch is not None else None))
        c._tiles_job = (verts, indices, changes, job)
        return job

    def read_launch(self, boxes=None, raw=None, vals=None, outside=None, ctx=None):
        """tw_voxel_model_read_launch: (raw field, field after remove_unconnected, its flags) as they are after every job launched on the model before
        this call, on any Context, as a job on ctx (default the model's Context). boxes = None: the whole grid, as new [ny, nx, nz] numpy arrays by default;
        else (x, y, z, w, h, d) tuples whose voxels are packed one box after another as edit_launch's values, as new flat numpy arrays by default. Each of
        raw / vals / outside may be given (numpy, page-locked or CUDA, float32 / float32 / uint8 of that size) or False to skip it; a numpy destination is
        staged in ctx's pinned staging, which grows to its size. Returns a VoxelReadJob."""
        c = self.ctx if ctx is None else ctx
        if boxes is None:
            shape, b, nb = (int(self.vpp.ny), int(self.vpp.nx), int(self.vpp.nz)), None, 0
        else:
            shape, nb = (sum(int(t[3]) * int(t[4]) * int(t[5]) for t in boxes),), len(boxes)
            b = (VoxelBox * max(nb, 1))(*[VoxelBox(*[int(v) for v in t]) for t in boxes])
        outs = [np.empty(shape, dt) if a is None else (None if a is False else a) for a, dt in ((raw, np.float32), (vals, np.float32), (outside, np.uint8))]
        c._check(lib.tw_voxel_model_read_launch(c._h, self._h, C.cast(b, C.c_void_p) if b is not None else None, nb, *[_ptr(a) for a in outs]))
        job = VoxelReadJob(c, tuple(outs))
        c._tiles_job = (b, outs, job)
        return job

    def read(self, raw=None, vals=None, outside=None):
        """tw_voxel_model_read (completes the pending job): (raw field, field after remove_unconnected, its flags), [ny, nx, nz] numpy arrays unless given."""
        shape = (int(self.vpp.ny), int(self.vpp.nx), int(self.vpp.nz))
        raw = np.empty(shape, np.float32) if raw is None else raw
        vals = np.empty(shape, np.float32) if vals is None else vals
        outside = np.empty(shape, np.uint8) if outside is None else outside
        self.ctx._check(lib.tw_voxel_model_read(self._h, _ptr(raw), _ptr(vals), _ptr(outside)))
        self.ctx._tiles_job = None
        return raw, vals, outside


class TileSet:
    """tw_tile_set (include/tw3d.h): resident tiles keyed by their grid coordinates (x1/size, y1/size), with per light slot the mesh shadows each tile was
    last computed with. A relight (shadows_launch) is the context's asynchronous job, completed by Context.create_tiles_poll; its outputs equal
    tw_tile_shadows_batch_ex over all resident tiles, bit for bit. Context.close() destroys the set with the context."""

    def __init__(self, ctx, zvsize, nlights):
        h = C.c_void_p()
        ctx._check(lib.tw_tile_set_create(ctx._h, int(zvsize), int(nlights), C.byref(h)))
        self._h, self.ctx, self.zvsize, self.nlights = h, ctx, int(zvsize), int(nlights)
        ctx._sets.append(self)

    def close(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.tw_tile_set_destroy(self._h)
            if self in self.ctx._sets:
                self.ctx._sets.remove(self)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _xy(tile_xy):
        return np.ascontiguousarray(tile_xy, np.int32).reshape(-1, 2)

    def put(self, tile_xy, zvals):
        """Inserts or replaces tiles: zvals [n, zv, zv] float32, numpy or CUDA tensor (read before the call returns)."""
        txy = self._xy(tile_xy)
        if not hasattr(zvals, "data_ptr"):
            zvals = np.ascontiguousarray(zvals, np.float32)
        self.ctx._check(lib.tw_tile_set_put(self._h, _ptr(txy), len(txy), _ptr(zvals)))

    def remove(self, tile_xy):
        txy = self._xy(tile_xy)
        self.ctx._check(lib.tw_tile_set_remove(self._h, _ptr(txy), len(txy)))

    def stale(self, sps):
        """The resident tiles a relight of every tile with these ShadowParams (light l = slot l) would recompute: [k, 2] int32 in (x, y) order."""
        arr = (ShadowParams * len(sps))(*sps)
        k = C.c_uint32()
        self.ctx._check(lib.tw_tile_set_stale(self._h, C.cast(arr, C.c_void_p), len(sps), None, 0, C.byref(k)))
        out = np.empty((k.value, 2), np.int32)
        if k.value:
            self.ctx._check(lib.tw_tile_set_stale(self._h, C.cast(arr, C.c_void_p), len(sps), _ptr(out), k.value, C.byref(k)))
        return out

    def shadows_launch(self, tile_xy, lights):
        """tw_tile_set_shadows_launch: enqueues the relight of the resident tiles tile_xy [n, 2] and returns the host recomputed flags [n] uint8 (1 = this job
        computes the tile for at least one light). lights: Light records or (ShadowParams, smask, sh_out_x, sh_out_y) tuples - smask [n, zv, zv] uint8
        required, sh_out_* [n, zv] float32 or None - numpy arrays (pinned for a launch that does not block) or CUDA tensors, kept referenced here until
        Context.create_tiles_poll completes the job."""
        txy = self._xy(tile_xy)
        recs = [lt if isinstance(lt, Light) else Light(*lt) for lt in lights]
        if any(r.sh_in_x is not None or r.sh_in_y is not None for r in recs):
            raise ValueError("shadows_launch: a tile set takes its incoming rows from its own tiles (no sh_in)")
        arr = (TileSetLight * max(1, len(recs)))()
        for i, r in enumerate(recs):
            arr[i] = TileSetLight(r.sp, _ptr(r.smask), _ptr(r.sh_out_x), _ptr(r.sh_out_y))
        recomputed = np.zeros(len(txy), np.uint8)
        req = TileSetRequest(_ptr(txy), len(txy), len(recs), C.cast(arr, C.c_void_p), _ptr(recomputed))
        self.ctx._check(lib.tw_tile_set_shadows_launch(self._h, C.byref(req)))
        self.ctx._tiles_job = ([(r.smask, r.sh_out_x, r.sh_out_y) for r in recs], arr)
        return recomputed

    def stale_after(self, sps, remove_xy=None, put_xy=None):
        """tw_tile_set_stale_after: what stale(sps) would return after remove(remove_xy) and put(put_xy), without changing the set - the tiles to name in
        a frame's relight (create_tiles_launch(relight_xy=...))."""
        arr = (ShadowParams * len(sps))(*sps)
        rem = self._xy(remove_xy if remove_xy is not None else np.empty((0, 2)))
        put = self._xy(put_xy if put_xy is not None else np.empty((0, 2)))
        k = C.c_uint32()
        args = [self._h, C.cast(arr, C.c_void_p), len(sps), _ptr(rem) if len(rem) else None, len(rem), _ptr(put) if len(put) else None, len(put)]
        self.ctx._check(lib.tw_tile_set_stale_after(*args, None, 0, C.byref(k)))
        out = np.empty((k.value, 2), np.int32)
        if k.value:
            self.ctx._check(lib.tw_tile_set_stale_after(*args, _ptr(out), k.value, C.byref(k)))
        return out

    def create_tiles_launch(self, origins_xy, mesh_size, dx, dy, hp, erosion_iters, ep, min_zval, tile_xy, zvals=None, mm=None, bounds=None, normals=None,
                            min_normal_z=None, wpz_max=0.0, size=0, ao=None, weights=None, has_any_grass=None, half_dxy=None, wp=None, tile_params=None,
                            remove_xy=None, relight_xy=None, lights=None, hmap=None, ctx=None):
        """tw_tile_set_create_tiles_launch: one frame in one asynchronous job - remove remove_xy, create the tiles of origins_xy (grid coordinates tile_xy
        [nt, 2]) as Context.create_tiles_launch would, put them into this set, and relight relight_xy with lights (Light records or (ShadowParams, smask,
        sh_out_x, sh_out_y) tuples sized for relight_xy, as shadows_launch). The job runs on ctx: this set's Context (None), its parent or a shared Context of
        that parent, so frames on several shared Contexts are in flight at once; ctx.create_tiles_poll completes it. zvals may be None (the zvals then stay in
        the set only); the other outputs are those of Context.create_tiles_launch. Returns the relight's recomputed flags [len(relight_xy)] uint8, or None
        without lights."""
        c = self.ctx if ctx is None else ctx
        org = np.ascontiguousarray(origins_xy, np.int32).reshape(-1, 2)
        nt = org.shape[0]
        txy = self._xy(tile_xy)
        outs = TileOutputs(_ptr(zvals), _ptr(mm), C.cast(bounds, C.c_void_p) if bounds is not None else None, _ptr(normals), _ptr(min_normal_z))
        shading = None
        if ao is not None and half_dxy is None:
            raise ValueError("create_tiles_launch: ao needs half_dxy (the ray's z step, HALF_DXY)")
        if ao is not None or weights is not None or has_any_grass is not None:
            if tile_params is not None and not hasattr(tile_params, "data_ptr"):
                tile_params = np.ascontiguousarray(tile_params, np.float32)
            shading = TileShading(0.0 if half_dxy is None else half_dxy, C.cast(C.pointer(wp), C.c_void_p) if wp is not None else None, _ptr(tile_params),
                                  _ptr(ao), _ptr(weights), _ptr(has_any_grass))
        rem = self._xy(remove_xy) if remove_xy is not None else None
        req, arr, recs, recomputed = None, None, [], None
        if (lights is None) != (relight_xy is None):
            raise ValueError("create_tiles_launch: a relight needs both relight_xy (the resident tiles to relight) and lights")
        if lights is not None:
            rxy = self._xy(relight_xy)
            recs = [lt if isinstance(lt, Light) else Light(*lt) for lt in lights]
            if any(r.sh_in_x is not None or r.sh_in_y is not None for r in recs):
                raise ValueError("create_tiles_launch: a tile set takes its incoming rows from its own tiles (no sh_in)")
            arr = (TileSetLight * max(1, len(recs)))()
            for i, r in enumerate(recs):
                arr[i] = TileSetLight(r.sp, _ptr(r.smask), _ptr(r.sh_out_x), _ptr(r.sh_out_y))
            recomputed = np.zeros(len(rxy), np.uint8)
            req = TileSetRequest(_ptr(rxy), len(rxy), len(recs), C.cast(arr, C.c_void_p), _ptr(recomputed))
        frame = TileSetFrame(_ptr(rem), 0 if rem is None else len(rem), _ptr(txy), C.cast(C.pointer(hmap), C.c_void_p) if hmap is not None else None,
                             C.cast(C.pointer(req), C.c_void_p) if req is not None else None)
        c._check(lib.tw_tile_set_create_tiles_launch(c._h, self._h, _ptr(org), nt, mesh_size[0], mesh_size[1], dx, dy, C.byref(hp) if hp is not None else None,
                                                     erosion_iters, C.byref(ep) if ep is not None else None, min_zval, wpz_max, size, C.byref(outs),
                                                     C.byref(shading) if shading is not None else None, C.byref(frame)))
        c._tiles_job = (zvals, mm, bounds, normals, min_normal_z, ao, weights, has_any_grass, wp, tile_params, shading,
                        [(r.smask, r.sh_out_x, r.sh_out_y) for r in recs], arr, req, frame)
        return recomputed


def gen_tex_height_tables(water_h_off_rel=0.0, temperature=20.0, glaciate_exp=3.0):
    """init_terrain_mesh + gen_tex_height_tables on the host (tw_gen_tex_height_tables): (h_dirt[5], tex_class[5], clip_hd1)."""
    h, ids, clip = (C.c_float * 5)(), (C.c_int * 5)(), C.c_float()
    lib.tw_gen_tex_height_tables(water_h_off_rel, temperature, glaciate_exp, C.cast(h, C.c_void_p), C.cast(ids, C.c_void_p), C.cast(C.byref(clip), C.c_void_p))
    return [float(v) for v in h], [int(v) for v in ids], float(clip.value)

