/* tw3d.h - C ABI of the H100-native terrain hot path (drop-in for fegennari/3DWorld's procedural height / erosion / voxel-density path).
 *
 * The reference has no FFI layer: its boundary is a C++ class + free-function surface (SURVEY.md section 8b). Every entry point below
 * names the reference interface it replaces (file:line relative to the reference root). A C++ adapter that re-exposes the exact reference
 * signatures (mesh_xy_grid_cache_t, apply_erosion, noise_gen_3d, voxel_manager::create_procedural) on top of this ABI lives in
 * 3dworld_b200/host/tw3d_adapter.h; INTEGRATION.md shows the binding a 3DWorld maintainer would add.
 *
 * Conventions: plain pointers and sizes only; every function returns 0 (TW_OK) or a negative tw_status (no assert()/exit() as in the
 * reference); data pointers may be HOST or DEVICE pointers (detected with cudaPointerGetAttributes) - host buffers are staged through
 * pinned memory inside the call; all arithmetic is fp32 with the reference's rounding sequence (no FMA contraction where it could change a
 * result), so outputs are bit-identical to the reference CPU path built with its makefile flags (-O3, no -march).
 * There is NO CPU fallback: without a CUDA device tw_create fails with TW_ERR_NO_DEVICE.
 */
#ifndef TW3D_H
#define TW3D_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TW_ABI_VERSION 1

#if defined(__GNUC__)
#define TW_API __attribute__((visibility("default")))
#else
#define TW_API
#endif

typedef enum tw_status {
	TW_OK = 0,
	TW_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product path refuses to run (no CPU fallback) */
	TW_ERR_CUDA      = -2,   /* a CUDA runtime call failed; see tw_last_error() */
	TW_ERR_ARG       = -3,   /* invalid argument (the reference would assert) */
	TW_ERR_STATE     = -4,   /* tables not set (tw_set_sin_table / tw_set_sine_params) */
	TW_ERR_NOT_READY = -5    /* tw_heightgen_2d_poll / tw_create_tiles_poll: result not available yet (mirrors build_arrays() returning 0 with no_wait) */
} tw_status;

/* mesh_gen_mode values, src/3DWorld.h:1399 */
enum { TW_MGEN_SINE = 0, TW_MGEN_SIMPLEX = 1, TW_MGEN_PERLIN = 2, TW_MGEN_SIMPLEX_GPU = 3, TW_MGEN_DWARP_GPU = 4 };

#define TW_F_TABLE_SIZE   90      /* NUM_FREQ_COMP*N_RAND_SIN2, src/mesh_gen.cpp:14,16,30 */
#define TW_SIN_TABLE_SIZE 65536   /* 2*TSIZE, src/sinf.h:8 */
#define TW_N3D_RDATA      420     /* SINE_DATA_SIZE, src/upsurface.h:14-16 */
#define TW_N3D_SINES      60      /* TOT_NUM_SINES */

typedef struct tw_ctx tw_ctx;   /* one per (thread, device): owns a CUDA stream, the uploaded tables and scratch buffers */

/* hmap_params_t, src/mesh.h:85-89 (same field order) */
typedef struct tw_hmap_params {
	float plat_bot, plat_h, plat_s, plat_max, crat_h, crat_s;
	float crack_lo, crack_hi, crack_d, sine_mag, sine_freq, sine_bias, volcano_width, volcano_height;
} tw_hmap_params;

/* Every reference global the height path reads (SURVEY.md section 8b), as one explicit POD. */
typedef struct tw_height_params {
	int   gen_mode;            /* mesh_gen_mode (force_sine_mode => pass TW_MGEN_SINE) */
	int   gen_shape;           /* mesh_gen_shape: 0 linear, 1 billowy, 2 ridged */
	int   start_eval_sin;      /* compute_scale() result, src/mesh_gen.cpp:544-548 (tw_compute_scale) */
	int   glaciate;            /* GLACIATE global: apply_glaciate() is a no-op when 0, src/mesh_gen.cpp:380-385 */
	float mesh_scale;          /* mesh_scale */
	float mesh_scale_z_inv;    /* mesh_scale_z_inv */
	float dx_val_inv, dy_val_inv; /* DX_VAL_INV, DY_VAL_INV, src/matrix_ops.cpp:77-78 */
	float mesh_height;         /* MESH_HEIGHT = 0.1*Z_SCENE_SIZE, src/matrix_ops.cpp:70 */
	float mesh_height_scale;   /* mesh_height_scale */
	float zmax_est;            /* zmax_est; zmax_est2 / zmax_est2_inv are derived exactly as set_zmax_est() does, src/mesh_gen.cpp:162-167 */
	float custom_glaciate_exp; /* custom_glaciate_exp (0 => cube) */
	float rx, ry;              /* gen_rx_ry() result, src/mesh_gen.cpp:581-586 (tw_gen_rx_ry); hoisted out of the per-cell loop */
	tw_hmap_params hmap;       /* hmap_params */
} tw_height_params;

/* mesh_xy_grid_cache_t::build_arrays(x0,y0,dx,dy,nx,ny) arguments, src/mesh_gen.cpp:588 */
typedef struct tw_grid2d {
	float x0, y0, dx, dy;
	uint32_t nx, ny;
} tw_grid2d;

typedef struct tw_minmax { float zmin, zmax; } tw_minmax;

/* The scalars apply_erosion() reads from globals: erode_amount, water_plane_z, HALF_DXY (src/erosion.cpp:11,98) and, through
 * get_bare_ls_tid() (src/Textures.cpp:1284-1287), zmin, zmax, relh_adj_tex, clip_hd1. */
typedef struct tw_erosion_params {
	float erode_amount, water_plane_z, half_dxy, zmin, zmax, relh_adj_tex, clip_hd1;
} tw_erosion_params;

/* what tile_t::create_zvals derives from the finished zvals (src/tiled_mesh.cpp:517-540): sub_zmin/sub_zmax[yy][xx] of the 4x4 sub-blocks
 * (block_size = zvsize/4, inclusive ends), mzmin/mzmax, mesh_dz = max sub-block range, bounding radius, and the bbox (tile-local cell
 * indices) of the cells below wpz_max; wx1 > wx2 when no cell is under water. */
typedef struct tw_tile_bounds {
	float sub_zmin[16], sub_zmax[16];
	float mzmin, mzmax, mesh_dz, radius;
	int32_t wx1, wy1, wx2, wy2;
} tw_tile_bounds;

/* voxel_grid geometry (src/voxels.cpp:91-108) + create_procedural() arguments (src/voxels.cpp:278) */
typedef struct tw_voxel_params {
	uint32_t nx, ny, nz;
	float lo_pos[3], vsz[3], offset[3];
	float mag, freq;
	int   gen_mode;            /* TW_MGEN_SINE, TW_MGEN_SIMPLEX or TW_MGEN_PERLIN (GPU modes 3/4 evaluate the CPU simplex formula) */
	int   normalize_to_1;
	int   rseed1, rseed2;      /* noise_gen_3d seeds (sine mode) */
	int   octaves;             /* max(1, MAX_FREQ_BINS - mesh_freq_filter), src/voxels.cpp:333 (GLM modes) */
	float rx, ry;              /* gen_rx_ry() (GLM modes) */
	float zscale;              /* (invert ? -1 : 1)*z_gradient/(nz-1), src/voxels.cpp:284 */
	/* optional fused attenuation pass (src/voxels.cpp:403-482); atten_mode 0 = none, 1 = top only (atten_top_mode 0), 2 = 5 edges, 3/4/5 = sphere */
	int   atten_mode;
	float atten_val, atten_inner_radius;
} tw_voxel_params;

/* ---- context ----
 * No reference counterpart: the reference keeps this state in process globals (sin_table src/sinf.h:11, sinTable src/mesh_gen.cpp:38,
 * the GL compute shader of mesh_xy_grid_cache_t src/mesh.h:33). One context = one device, one CUDA stream, its scratch buffers and the
 * uploaded tables; not re-entrant (use one per thread). tw_create fails with TW_ERR_NO_DEVICE when there is no GPU - there is no CPU fallback.
 * Every call makes the context's device the calling thread's current CUDA device (cudaSetDevice) and leaves it so.
 * Host output buffers: asynchronous entry points (tw_heightgen_2d_launch, tw_create_tiles_launch) overlap the device->host copy with compute only when
 * the buffer is page-locked (cudaHostAlloc / cudaHostRegister / tw_multi_alloc_host); with pageable memory the copy - and therefore the launch call - blocks.
 * A context has at most one asynchronous job in flight: every other call on it (including the next launch) first completes the pending job, exactly
 * as a poll with wait = 1 would, and either poll function completes whichever job is pending. */
TW_API int  tw_abi_version(void);
TW_API int  tw_create(int device, tw_ctx **out);
TW_API void tw_destroy(tw_ctx *ctx);
TW_API const char *tw_last_error(const tw_ctx *ctx);
TW_API int  tw_sync(tw_ctx *ctx);                         /* cudaStreamSynchronize on the context stream */
TW_API void *tw_stream(tw_ctx *ctx);                      /* the cudaStream_t all work of this context is issued on */
TW_API uint64_t tw_launch_count(const tw_ctx *ctx);       /* kernels launched by this context so far (bench.py gpu_launches) */

/* ---- host-side table generation (bit-exact restatements; tiny, run once) ---- */
/* create_sin_table(), src/mesh_gen.cpp:72-81: tab[i]=sinf(i/sscale), tab[i+32768]=cosf(i/sscale) with the host libm. */
TW_API void tw_build_sin_table(float *tab65536);
/* compute_scale(), src/mesh_gen.cpp:544-548 */
TW_API int  tw_compute_scale(float mesh_scale, int mesh_freq_filter);
/* rand_gen_t state (src/rand_gen.h:29): pass the same object to successive tw_gen_sine_params calls to reproduce the reference's
 * function-static generator (src/mesh_gen.cpp:237). Initial state {1,1}. */
typedef struct tw_rng { int64_t rseed1, rseed2; } tw_rng;
/* gen_rand_sine_table_entries() + apply_mesh_rand_seed(), src/mesh_gen.cpp:213-254 */
TW_API void tw_gen_sine_params(tw_rng *rgen, float scaled_height, int mesh_x_size, int mesh_y_size, float x_scene_size, float y_scene_size,
                        int mesh_seed, int mesh_rgen_index, int mesh_gen_mode, float mesh_start_mag, float mesh_start_freq,
                        float mesh_mag_mult, float mesh_freq_mult, float *sine_params450);
/* gen_rx_ry(), src/mesh_gen.cpp:581-586 */
TW_API void tw_gen_rx_ry(int mesh_seed, int mesh_rgen_index, int mesh_gen_mode, float *rx, float *ry);
/* noise_gen_3d::set_rand_seeds + gen_sines, src/upsurface.cpp:16-38 */
TW_API void tw_noise3d_gen_sines(int rseed1, int rseed2, float mag, float freq, float *rdata420);
/* get_water_z_height(), src/mesh_gen.cpp:507-512 (water_h_off/water_h_off_rel as arguments) */
TW_API float tw_water_z_height(float zmax_est, int glaciate, float custom_glaciate_exp, float water_h_off, float water_h_off_rel);
/* init_terrain_mesh() + gen_tex_height_tables() (src/mesh_gen.cpp:407-431, src/Textures.cpp:1757-1761), host: the height thresholds h_dirt[5] of the ground textures
 * (tex_class[5], optional = TW_TEX_SAND .. TW_TEX_SNOW in the reference's order) and clip_hd1 (optional) = the rock/dirt threshold of tw_erosion_params. glaciate_exp =
 * the reference's global of that name: DEF_GLACIATE_EXP = 3 (or custom_glaciate_exp) once glaciate() has run, 1 without glaciation. */
TW_API void tw_gen_tex_height_tables(float water_h_off_rel, float temperature, float glaciate_exp, float h_dirt[5], int tex_class[5], float *clip_hd1);

/* ---- table upload ---- */
/* sin_table (src/sinf.h:11). tab==NULL: build with tw_build_sin_table. Also builds the 1e6-entry cos/sin direction table used by the
 * erosion random-direction fallback (src/erosion.cpp:84-87) from the host libm so device results match the host bit for bit. */
TW_API int tw_set_sin_table(tw_ctx *ctx, const float *tab65536);
/* sinTable[90][5] (src/mesh_gen.cpp:40) */
TW_API int tw_set_sine_params(tw_ctx *ctx, const float *sine_params450);

/* ---- 2-D height generation: build_arrays + enable_glaciate + eval_index over the whole grid ----
 * Replaces mesh_xy_grid_cache_t::{build_arrays,enable_glaciate,eval_index} (src/mesh.h:39-41, src/mesh_gen.cpp:588-650,754-792) as used by
 * heightmap_t::proc_gen (src/heightmap.cpp:130-151), tile_t::create_zvals (src/tiled_mesh.cpp:467-515) and gen_mesh_sine_table
 * (src/mesh_gen.cpp:201-210); for gen modes 3/4 it is the backend behind run_gpu_simplex/cache_gpu_simplex_vals (src/mesh_gen.cpp:652-695).
 * out[y*nx + x] = eval_index(x, y, min_start_sin); mm (optional, host pointer) receives min/max over the grid (fused reduction). */
TW_API int tw_heightgen_2d(tw_ctx *ctx, const tw_grid2d *grid, const tw_height_params *p, int enable_glaciate, int min_start_sin,
                    float *out, tw_minmax *mm);
/* Asynchronous pair mirroring the reference's no_wait contract (src/mesh_gen.cpp:597-603, src/tiled_mesh.cpp:2393-2402):
 * launch returns immediately; poll returns TW_ERR_NOT_READY until the result (and host copy, if out is a host pointer) is complete. */
TW_API int tw_heightgen_2d_launch(tw_ctx *ctx, const tw_grid2d *grid, const tw_height_params *p, int enable_glaciate, int min_start_sin,
                           float *out, tw_minmax *mm);
TW_API int tw_heightgen_2d_poll(tw_ctx *ctx, int wait);

/* Batched tile form of tile_t::create_zvals' height fill (src/tiled_mesh.cpp:458-464,495-514): tile t covers
 * build_arrays(origins[2t]-mesh_x_size/2, origins[2t+1]-mesh_y_size/2, dx, dy, zvsize, zvsize) with glaciate enabled;
 * out[t*zvsize*zvsize + y*zvsize + x]. origins is a HOST array of ntiles (x1,y1) pairs. mm (optional, host) = ntiles entries. */
TW_API int tw_heightgen_tiles(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                       uint32_t zvsize, const tw_height_params *p, float *out, tw_minmax *mm);

/* Tail of tile_t::create_zvals (src/tiled_mesh.cpp:517-540) for ntiles finished tiles: zvals host or device, out = HOST array of ntiles. */
TW_API int tw_tile_bounds_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, float dx_val, float dy_val,
                         uint32_t size, tw_tile_bounds *out);
/* Per-tile derived fields of a batch of finished tiles (SURVEY.md 8f row N1). zvals: ntiles*zvsize^2 floats, host or device; outputs host or
 * device. stride = zvsize - 1.
 * tw_tile_normals_batch = tile_t::upload_normal_texture (src/tiled_mesh.cpp:865-880) without the GL upload: rgba = ntiles*stride^2*4 bytes,
 *   (unsigned char)(127.0*(n + 1.0)) of get_norm(y*zvsize + x) (src/tiled_mesh.h:281-284), alpha 0; min_normal_z (optional, HOST, ntiles) as the
 *   reference leaves it (starts at 1.0).
 * tw_tile_ao_batch = tile_t::calc_mesh_ao_lighting (src/tiled_mesh.cpp:586-662): ao = ntiles*stride^2 bytes. The context heights around each
 *   tile ((stride + 72)^2 grid at origin (x1 - 36, y1 - 36), setup_height_gen_async, :608) are generated internally with p exactly as
 *   tw_heightgen_tiles would. CPU gen modes (0-2): inside the tile the given zvals are used (:621) and the context's interior is not even
 *   generated. GPU gen modes (p->gen_mode >= TW_MGEN_SIMPLEX_GPU): the reference keeps the un-eroded context of create_zvals in ao_zvals and
 *   tests the rays against it inside the tile too (:479-487,604); only the ray origin is the given (eroded) zval - reproduced here.
 *   origins_xy = tile (x1, y1) pairs as for tw_heightgen_tiles.
 * tw_create_zvals_ao_batch = tile_t::create_zvals + calc_mesh_ao_lighting with enable_tiled_mesh_ao: heights, per-tile erosion and the AO map
 *   of a batch in one call. GPU gen modes: ONE (stride + 72)^2 generation per tile, zvals cut out of it (:505) - 1.4x less noise work than
 *   tw_create_zvals_batch + tw_tile_ao_batch for 128-tiles - and bit-identical to the reference, whose zvals ARE the context's interior there.
 *   CPU gen modes: zvals generated directly (as the reference does), context generated only outside the tile. zvals/ao host or device, mm optional HOST.
 *   Blocks until the result is complete: it is tw_create_tiles_launch_ex (below) with zvals, mm and ao, followed by tw_create_tiles_poll(wait = 1).
 *   So it needs the device memory that job needs, as tw_create_zvals_batch does: host zvals / ao are staged whole on the device (n*zvsize^2*4 +
 *   n*(zvsize-1)^2 bytes) besides about 2 GB of context grids, and in sine mode (gen_mode 0) one batch may hold at most 65535 distinct tile
 *   columns + rows (TW_ERR_ARG beyond). Split larger batches into several calls. */
TW_API int tw_tile_normals_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float dx_val, float dy_val, uint8_t *rgba,
                          float *min_normal_z);
TW_API int tw_tile_ao_batch(tw_ctx *ctx, const float *zvals, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size,
                     float dx, float dy, uint32_t zvsize, const tw_height_params *p, float half_dxy, uint8_t *ao);
TW_API int tw_create_zvals_ao_batch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                     uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                     float half_dxy, float *zvals, uint8_t *ao, tw_minmax *mm);
/* glaciate() of the ground-mode mesh (src/mesh_gen.cpp:388-404): apply_glaciate + apply_mesh_sine(x = j + xoff2 - MESH_X_SIZE/2, ...) per
 * cell, in place (mesh host or device, row-major nx*ny); zbottom_ztop (optional, host) receives min/max of the result. */
TW_API int tw_glaciate_mesh(tw_ctx *ctx, float *mesh, int nx, int ny, int xoff2, int yoff2, int mesh_x_size, int mesh_y_size,
                     const tw_height_params *p, tw_minmax *zbottom_ztop);

/* ---- point queries (SURVEY.md 8a row a9) ----
 * Batched form of the reference's single-point height functions, for callers that place many objects (buildings, scenery, cities):
 *   TW_PQ_SIN_TERMS         float eval_mesh_sin_terms(float xv, float yv)                          src/mesh_gen.cpp:797-805 (raw sine-table sum)
 *   TW_PQ_SIN_TERMS_SCALED  float eval_mesh_sin_terms_scaled(float xval, float yval, float xy_scale) src/mesh_gen.cpp:807-813
 *   TW_PQ_EXACT_ZVAL        float get_exact_zval(float xval, float yval, bool no_xyoff)            src/mesh_gen.cpp:816-847, the procedural
 *                           branch (no landscape file / tiled-terrain heightmap texture): glaciate + hmap sine bias/volcano applied
 * xy = n (x, y) pairs, out = n floats; both host or device. GLACIATE is p->glaciate. */
#define TW_PQ_SIN_TERMS        0
#define TW_PQ_SIN_TERMS_SCALED 1
#define TW_PQ_EXACT_ZVAL       2
typedef struct tw_point_query {
	int   kind;                       /* TW_PQ_* */
	float xy_scale;                   /* TW_PQ_SIN_TERMS_SCALED */
	int   mesh_x_size, mesh_y_size;   /* MESH_X_SIZE, MESH_Y_SIZE (scaled / exact) */
	float x_scene_size, y_scene_size; /* X_SCENE_SIZE, Y_SCENE_SIZE (exact) */
	int   xoff2, yoff2, no_xyoff;     /* current mesh scroll offset, and the no_xyoff argument (exact) */
} tw_point_query;
TW_API int tw_eval_points(tw_ctx *ctx, const float *xy, size_t n, const tw_height_params *p, const tw_point_query *q, float *out);

/* ---- hydraulic erosion ----
 * Replaces apply_erosion(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters) (src/function_registry.h:354,
 * src/erosion.cpp:14-164): in place, row-major x-fastest, droplets applied in the reference's serial order (iter = 0..num_iters-1;
 * this is the OMP_NUM_THREADS=1 order, the only deterministic one - SURVEY.md section 0). Early-out as the reference when
 * num_iters==0 or erode_amount<=0. One big map (>= 2^20 padded cells, >= 64 droplets) is walked speculatively - a window of consecutive droplets in
 * flight, each against the committed map with a private view and a write log, committed strictly in order; droplets whose cells an earlier droplet
 * touched are walked again - which gives the serial result bit for bit at ~4x the speed of walking one droplet after the other (DESIGN.md section 6,
 * M_SPEC; TW_EROSION_MODE=global selects the plain walk). */
TW_API int tw_erode(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p);
/* The reference's MULTI-THREADED mode of the same function: `#pragma omp parallel for schedule(dynamic,1)` over the droplets
 * (src/erosion.cpp:66) lets num_threads droplets walk ONE heightmap at the same time with unsynchronised read-modify-writes, so its result
 * depends on thread timing. Here num_threads droplets are in flight (dynamic,1 assignment through an atomic counter; float atomics, so no
 * update is lost); the result is equally order-dependent, and num_threads == 1 is bit-identical to tw_erode(). num_threads == 0 picks a
 * count that fills the GPU. Use tw_erode() when reproducible output matters, this entry point when the reference would run with OpenMP. */
TW_API int tw_erode_parallel(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                      uint32_t num_threads);
/* The same on ntiles independent heightmaps stored back to back (tile_t::create_zvals semantics, src/tiled_mesh.cpp:515): every tile
 * gets droplets 0..num_iters-1 exactly as a separate apply_erosion() call would. min_zvals: HOST array of ntiles values, or NULL to use
 * min_zval_all for every tile. */
TW_API int tw_erode_tiles(tw_ctx *ctx, float *heightmaps, uint32_t ntiles, int xsize, int ysize, const float *min_zvals, float min_zval_all,
                   uint32_t num_iters, const tw_erosion_params *p);
/* Fused tile pipeline = the height fill AND the per-tile erosion of tile_t::create_zvals (src/tiled_mesh.cpp:467-515) for a batch of tiles:
 * exactly tw_heightgen_tiles followed by tw_erode_tiles(min_zval_all = min_zval) in one call (one upload of the origins, one download of
 * the result, per-tile z range fused). When memory forces several chunks, generation of chunk k+1 is issued on a separate stream and
 * overlaps the droplet walk of chunk k. mm (optional, HOST, ntiles entries) receives
 * the per-tile z range AFTER erosion (mzmin/mzmax). erosion_iters == 0 or erode_amount <= 0 => height fill only.
 * Blocks until the result is complete: it is tw_create_tiles_launch (below) with zvals and mm only, followed by tw_create_tiles_poll(wait = 1). */
TW_API int tw_create_zvals_batch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                          uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float *out, tw_minmax *mm);
/* Asynchronous form of a frame's new tiles (tile_draw_t::update creates them with build_arrays(..., no_wait=1) and collects them on a later frame,
 * src/tiled_mesh.cpp:2367-2417): tw_create_tiles_launch enqueues tw_create_zvals_batch AND the tile tail - tw_tile_bounds_batch(wpz_max, dx, dy, size)
 * and tw_tile_normals_batch(dx, dy) - on the context's streams and returns without waiting for the device; tw_create_tiles_poll(wait = 0) only
 * queries an event and returns TW_ERR_NOT_READY until every requested output is complete (wait = 1 blocks until then); TW_OK when no job is pending.
 * Every output is bit-identical to the three synchronous calls with the same arguments, and tw_last_erosion_steps() after the completing poll equals
 * its value after tw_create_zvals_batch. The sub-block bounds and the normal map of a chunk of tiles are computed on the stream that eroded it, right
 * after its erosion, so they run under the generation and erosion of the other chunks. origins_xy and the parameter structs are copied during the
 * launch (they may be reused as soon as it returns). Outputs must stay valid until the completing poll:
 *   zvals         required, ntiles*zvsize^2 floats, host or device
 *   mm            optional HOST array of ntiles: per-tile z range after erosion (as tw_create_zvals_batch)
 *   bounds        optional HOST array of ntiles (as tw_tile_bounds_batch; needs zvsize >= 4 with 4*(zvsize/4) < zvsize)
 *   normals_rgba  optional, ntiles*(zvsize-1)^2*4 bytes, host or device (as tw_tile_normals_batch)
 *   min_normal_z  optional HOST array of ntiles (needs normals_rgba)
 * The host arrays mm / bounds / min_normal_z are filled by the poll that reports completion. */
typedef struct tw_tile_outputs {
	float          *zvals;
	tw_minmax      *mm;
	tw_tile_bounds *bounds;
	uint8_t        *normals_rgba;
	float          *min_normal_z;
} tw_tile_outputs;
TW_API int tw_create_tiles_launch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                           uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                           float wpz_max, uint32_t size, const tw_tile_outputs *out);
/* The same job with the two other per-tile products the reference makes for every new tile; tw_create_tiles_launch(...) is
 * tw_create_tiles_launch_ex(..., NULL), and tw_create_tiles_poll completes both. shading (optional) adds:
 *   ao             optional, ntiles*(zvsize-1)^2 bytes, host or device: tile_t::calc_mesh_ao_lighting with the ray z step half_dxy, as tw_tile_ao_batch
 *   weights        optional, ntiles*(zvsize-1)^2*4 bytes, host or device: the terrain weights texture of tile_t::create_texture, as tw_tile_weights_batch
 *                  (needs wp, tile_params and tw_set_sine_params; wp is validated and copied during the launch)
 *   has_any_grass  optional, needs weights, ntiles bytes: HOST (filled by the completing poll) or device
 *   tile_params    with weights: ntiles*8 floats as for tw_tile_weights_batch; HOST (copied during the launch) or device (read until the completing poll)
 * Each chunk's AO map and weights texture are computed on the stream that eroded it, after its erosion, like the bounds and the normal map.
 * AO follows the reference's two flows, exactly as tw_create_zvals_ao_batch:
 *   CPU gen modes (0-2): the zvals are generated directly; the (stride + 72)^2 context is generated outside the tile only, and the rays read the
 *     eroded zvals inside the tile. Every output equals the synchronous calls'.
 *   GPU gen modes (3/4): the context is generated once and the zvals are cut from its interior BEFORE erosion; the un-eroded context is the ray
 *     source everywhere, only the ray origin is the eroded zval. So in these modes requesting AO CHANGES THE ZVALS: they equal
 *     tw_create_zvals_ao_batch's, not tw_create_zvals_batch's (the reference does the same). The z range, bounds, normal map and weights are then
 *     derived from those zvals, and tw_last_erosion_steps() after the completing poll equals its value after tw_create_zvals_ao_batch.
 * Errors: TW_ERR_ARG for weights without wp or tile_params, has_any_grass without weights, a tex_class that does not name each class once, or
 * zmax <= zmin; TW_ERR_STATE for weights before tw_set_sine_params. The layout of tw_tile_outputs is unchanged (ABI 1).
 * The per-light mesh shadows of the same tiles join the job through tw_create_tiles_launch_shadows (below, with tw_tile_shadows_batch). */
typedef struct tw_tile_shading {
	float                   half_dxy;      /* HALF_DXY: the AO ray's z step, as tw_tile_ao_batch */
	const struct tw_weight_params *wp;     /* required with weights (declared below) */
	const float            *tile_params;   /* required with weights: ntiles*8 biome corners */
	uint8_t                *ao;            /* optional: ntiles*(zvsize-1)^2 bytes */
	uint8_t                *weights;       /* optional: ntiles*(zvsize-1)^2*4 bytes */
	uint8_t                *has_any_grass; /* optional, needs weights: ntiles bytes */
} tw_tile_shading;
TW_API int tw_create_tiles_launch_ex(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                           uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                           float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading);
TW_API int tw_create_tiles_poll(tw_ctx *ctx, int wait);
/* droplet steps executed by the last tw_erode/tw_erode_tiles call (sum over droplets; for roofline byte accounting) */
TW_API uint64_t tw_last_erosion_steps(const tw_ctx *ctx);

/* ---- 3-D voxel density ----
 * Replaces the fill loop of voxel_manager::create_procedural (src/voxels.cpp:278-346) + noise_gen_3d::{gen_xyz_vals,get_val}
 * (src/upsurface.cpp:41-70); out[z + (x + y*nx)*nz] (src/voxels.h:141-144). rdata420: noise_gen_3d::rdata (sine mode; host pointer;
 * NULL => generated from rseed1/rseed2/mag/freq with tw_noise3d_gen_sines). */
TW_API int tw_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *out);

/* ---- next rows (SURVEY.md section 8f N2): heightmap quantise, fused streaming passes ----
 * heightmap_t::from_floats 16-bit pack (src/heightmap.cpp:205-215, src/Textures.cpp:1889-1893): v=(h-add)*(1/mult);
 * out[2i+1]=trunc(v), out[2i]=trunc(256*(v-trunc(v))). Returns TW_ERR_ARG if any v is outside [0,256) (the reference asserts). */
TW_API int tw_heightmap_from_floats_u16(tw_ctx *ctx, const float *vals, size_t n, float val_mult, float val_add, uint8_t *out2n);
/* heightmap_t::to_floats 16-bit unpack (src/heightmap.cpp:191-203) */
TW_API int tw_heightmap_to_floats_u16(tw_ctx *ctx, const uint8_t *data2n, size_t n, float val_mult, float val_add, float *vals);
/* heightmap_t::proc_gen (src/heightmap.cpp:130-151) in one device-resident call: build_arrays(-0.5*width, -0.5*height, DX_VAL, DY_VAL, width,
 * height, cache_values=1) + enable_glaciate + eval_index over the grid, run_erosion (min_zval = min of the grid, src/heightmap.cpp:153-187),
 * get_heightmap_z_range, set_mesh_height_scales_for_zval_range(min_z, dz/255) (src/mesh_gen.cpp:124-131) and from_floats to 16-bit
 * (src/heightmap.cpp:205-215). run_city_gen is out of scope. data16 (2*width*height bytes) and vals (optional, width*height floats) may be
 * host or device pointers; info (host) receives the z range, the resulting get_mh_texture_mult()/get_mh_texture_add() and the droplet moves. */
typedef struct tw_heightmap_info { float min_z, max_z, val_mult, val_add, mesh_file_scale, mesh_file_tz; uint64_t erosion_moves; } tw_heightmap_info;
TW_API int tw_proc_gen_heightmap(tw_ctx *ctx, uint32_t width, uint32_t height, float dx_val, float dy_val, const tw_height_params *p,
                          uint32_t erosion_iters, const tw_erosion_params *ep, uint8_t *data16, float *vals, tw_heightmap_info *info);
/* Heightmap-texture mode of tile_t::create_zvals (src/tiled_mesh.cpp:498-501; SURVEY.md 8f row N2): every cell of every tile is
 * terrain_hmap_manager_t::get_clamped_height(x1 + x, y1 + y) (src/heightmap.cpp:385-402) of a 16-bit heightmap image -
 *   mesh_scale < 1: bilinear interpolate_height(); otherwise the nearest texel round_fp(mesh_scale*x) (clamp_xy, :309-313);
 *   texel (0,0) of index space is the image centre; outside the image edge_mode applies (clamp_no_scale, :315-341): 0 clamp,
 *   1 "off the texture" => scale_mh_texture_val(0), 2 mirror (the reference's compile-time TEX_EDGE_MODE, src/heightmap.cpp:16);
 *   texel value hi + lo/256 (get_heightmap_value, :74-77), scaled by scale_mh_texture_val (src/mesh_gen.cpp:120):
 *   (READ_MESH_H_SCALE*mesh_height_scale*mesh_file_scale*val + mesh_file_tz)*mesh_scale_z_inv with h_scale = READ_MESH_H_SCALE*mesh_height_scale.
 * data16 = the image in the layout of tw_heightmap_from_floats_u16 (2*width*height bytes), host or device; out = ntiles*zvsize^2 floats. */
typedef struct tw_hmap_sampler {
	int   width, height;       /* image size */
	int   edge_mode;           /* TW_HMAP_EDGE_* */
	float mesh_scale;
	float h_scale, mesh_file_scale, mesh_file_tz, mesh_scale_z_inv;
} tw_hmap_sampler;
#define TW_HMAP_EDGE_CLAMP  0
#define TW_HMAP_EDGE_CLIFF  1
#define TW_HMAP_EDGE_MIRROR 2
TW_API int tw_heightmap_sample_tiles(tw_ctx *ctx, const uint8_t *data16, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles,
                              uint32_t zvsize, float *out);
/* The context's heightmap image for tw_create_tiles_launch_hmap: copies data16 (2*width*height bytes in the layout of tw_heightmap_from_floats_u16, host or
 * device) into device memory the context owns, so a frame's tiles do not upload the image again. Completes a pending job first. data16 == NULL releases the
 * image; width or height <= 0 with an image is TW_ERR_ARG. Changing the map (brushes, a new file) means calling it again; tw_destroy frees the image. */
TW_API int tw_set_heightmap(tw_ctx *ctx, const uint8_t *data16, int width, int height);
/* min/max over a float array (get_heightmap_z_range, src/map_view.cpp:399-407) */
TW_API int tw_minmax_f32(tw_ctx *ctx, const float *vals, size_t n, tw_minmax *mm);


/* ---- voxel post-processing (SURVEY.md 8f row N3): the steps of voxel_model::build after the density fill (src/voxels.cpp:1496-1530), on the device, so
 * the 537 MB field of a 512^3 grid never goes back to the host. Layout everywhere: index z + (x + y*nx)*nz (src/voxels.h:141-144). ---- */
#define TW_VOX_OUTSIDE    0x01   /* outside[] values, src/voxels.cpp:22-24, :748: 0 inside, 1 outside, 2 on the closed-surface edge, 8-bit = under the mesh */
#define TW_VOX_ON_EDGE    0x02
#define TW_VOX_ANCHORED   0x04   /* transient, only during the flood fills */
#define TW_VOX_UNDER_MESH 0x08
typedef struct tw_voxel_post_params {
	uint32_t nx, ny, nz;
	float lo_pos[3], vsz[3];     /* voxel_grid geometry: get_xv(x) = x*vsz.x + lo_pos.x (src/voxels.h:127-129) */
	float isolevel;              /* voxel_params_t::isolevel / invert / make_closed_surface (src/voxels.h:14-37) */
	int   invert, make_closed_surface;
	int   remove_unconnected;    /* params.remove_unconnected: > 0 remove_unconnected_outside(), > 2 also remove_interior_holes() */
	int   keep_at_edge;          /* keep_at_scene_edge == 1 || (== 2 && dynamic_mesh_scroll) */
	int   centre_seed;           /* params.atten_sphere_mode() || !use_mesh: one anchor at the grid centre instead of the voxels under the mesh */
	int   skip_under_mesh;       /* params.remove_under_mesh && (display_mode & 1): cubes whose 4 lower corners are all under the mesh produce no triangles */
} tw_voxel_post_params;
/* determine_voxels_outside + calc_outside_val + val_is_outside (src/voxels.cpp:571-604): outside[i] = ON_EDGE on the grid boundary when make_closed_surface, else
 * (val == isolevel || (val < isolevel) != invert); | UNDER_MESH for z < zix_xy[y*nx + x]. zix_xy (optional, nx*ny uint32, host or device) is the caller's
 * max(0, int((z_min_matrix[ypos][xpos] - lo_pos.z)/vsz.z)) per column (it reads the caller's ground mesh, :596-600); NULL = no voxel is under the mesh.
 * vals / outside: host or device. */
TW_API int tw_voxel_outside(tw_ctx *ctx, const float *vals, const tw_voxel_post_params *vp, const uint32_t *zix_xy, uint8_t *outside);
/* remove_unconnected_outside (+ remove_interior_holes when remove_unconnected > 2), src/voxels.cpp:606-610,739-868: flood fill of the inside voxels from the
 * anchors (voxels under the mesh / the centre voxel / the scene-edge columns), every inside voxel not reached becomes outside (make_voxel_outside:
 * val = isolevel -+ TOLERANCE); then the outside space is flood-filled from the top plane and unreached pockets become inside. The set of reached voxels does
 * not depend on the fill order, so the result is identical to the reference's stack-based fill. vals / outside modified in place (host or device);
 * changed (optional) = number of voxels flipped. */
TW_API int tw_voxel_remove_unconnected(tw_ctx *ctx, float *vals, uint8_t *outside, const tw_voxel_post_params *vp, uint64_t *changed);
/* Marching cubes: voxel_manager::add_triangles_for_voxel at LOD 0 for every cube of the grid in the order of voxel_model::create_block (y, x, z),
 * src/voxels.cpp:485-566,1077-1108, as an UNWELDED triangle soup: tris[t] = 3 vertices x (x, y, z), each cube's vertices interpolated by that cube
 * (interpolate_pt); triangles whose normal is the zero vector are dropped as the reference drops them (:550). The reference additionally welds vertices
 * through a per-block index cache (a vertex on a shared edge keeps the position computed by the first cube that used it - at most 1 ulp from this soup's)
 * and averages normals; both stay with the renderer-side caller. The case tables are the caller's voxel_detail::edge_table[256], tri_table[256][16],
 * edge_to_vals[12][2] (src/marching_cubes.h; Paul Bourke's polygonise tables) - data, passed in like the sin table. tris: capacity*9 floats, host or
 * device (NULL with capacity 0 to only count); ntris = triangles the grid produces (may exceed capacity: nothing is written beyond it). */
TW_API int tw_voxel_triangles(tw_ctx *ctx, const float *vals, const uint8_t *outside, const tw_voxel_post_params *vp, const uint32_t *edge_table256,
                       const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, float *tris, uint64_t capacity, uint64_t *ntris);

/* ---- mesh shadows of tiles (SURVEY.md 8f row N4): calc_mesh_shadows (src/visibility.cpp:411-517) for a batch of tiles with the neighbour chaining of
 * tile_t::calc_shadows_for_light (src/tiled_mesh.cpp:664-692) ---- */
typedef struct tw_shadow_params {
	float lpos[3];                       /* get_light_pos(l) */
	float x_scene_size, y_scene_size;    /* X_SCENE_SIZE, Y_SCENE_SIZE */
	float dx_val, dy_val, dx_val_inv, dy_val_inv;
	int   xy_sum_size;                   /* XY_SUM_SIZE = MESH_X_SIZE + MESH_Y_SIZE (src/matrix_ops.cpp) */
	float zmin, zmax;                    /* the globals the line clip of trace_shadow_path uses (:424) */
	int   no_shadow;                     /* l == LIGHT_MOON && combined_gu (:511) */
} tw_shadow_params;
#define TW_MESH_SHADOW 0x02              /* MESH_SHADOW, src/3DWorld.h:1403 */
#define TW_MESH_MIN_Z  (-1.0E6f)         /* MESH_MIN_Z, src/mesh.h:9: "no incoming shadow height" */
/* smask (ntiles*zvsize^2 bytes) = 0 / MESH_SHADOW per cell as calc_mesh_shadows leaves it; every tile traces 2*zvsize rays from its x edge and 2*zvsize from its
 * y edge toward the light's shadow direction (Bresenham walk, one thread per ray) carrying the running shadow height. tile_xy = the tiles' grid coordinates
 * (x1/size, y1/size): a tile whose neighbour TOWARD the light (x + (lpos.x < 0 ? -1 : 1), resp. y) is in the batch starts its rays from that neighbour's outgoing
 * shadow heights (sh_in = the neighbour's sh_out, :680-686), so the batch is processed in dependency waves. sh_out_x / sh_out_y (optional, ntiles*zvsize floats each,
 * host or device) receive the outgoing heights (MESH_MIN_Z where no shadowed ray left the tile). Where two rays write the same sh_out entry the later ray in the
 * reference's sequential order (run_x rays by y, then run_y rays by x) wins - the reference runs the two loops as OpenMP sections, i.e. with a race; its
 * 1-thread order is reproduced. zvals / smask: host or device. */
TW_API int tw_tile_shadows_batch(tw_ctx *ctx, const float *zvals, const int32_t *tile_xy, uint32_t ntiles, uint32_t zvsize, const tw_shadow_params *sp,
                          uint8_t *smask, float *sh_out_x, float *sh_out_y);
/* The same with incoming shadow heights from tiles OUTSIDE the batch - what calc_shadows_for_light reads from the tile map when a frame's new tiles border
 * existing ones. With sx = (lpos.x < 0 ? -1 : 1), sy = (lpos.y < 0 ? -1 : 1), tile t at (tx, ty):
 *   sh_in_x   optional, ntiles*zvsize floats, host or device: row t = the sh_out_x of its neighbour (tx, ty + sy)
 *   sh_in_y   optional, ntiles*zvsize floats, host or device: row t = the sh_out_y of its neighbour (tx + sx, ty)
 * A caller row is read only where that neighbour is NOT in the batch; an in-batch neighbour's sh_out, computed in this call, always wins. Entries
 * <= TW_MESH_MIN_Z mean "no incoming height". With both NULL the results equal tw_tile_shadows_batch's. Unlike it, this call takes any number of tiles and
 * returns TW_ERR_ARG when tile_xy names a tile twice.
 * What stays the caller's job: when new tiles appear, existing tiles on their far side from the light may need new shadows, because their neighbour toward
 * the light now exists. Which of them to redo is engine policy; redo them with this call, passing the new tiles' sh_out as their sh_in. */
TW_API int tw_tile_shadows_batch_ex(tw_ctx *ctx, const float *zvals, const int32_t *tile_xy, uint32_t ntiles, uint32_t zvsize, const tw_shadow_params *sp,
                          const float *sh_in_x, const float *sh_in_y, uint8_t *smask, float *sh_out_x, float *sh_out_y);
/* Mesh shadows of a frame's new tiles inside the asynchronous tile job: tw_create_tiles_launch_shadows(..., shading, shadows) is tw_create_tiles_launch_ex
 * (..., shading) plus, for every light, the results of tw_tile_shadows_batch_ex on the job's own final zvals (in GPU gen modes with AO: the zvals of
 * tw_create_zvals_ao_batch, as documented above) with the same tile_xy, sp and sh_in - bit for bit. Every other output is the job's without shadows, and
 * tw_create_tiles_launch_ex(...) is tw_create_tiles_launch_shadows(..., NULL). The shadow pass runs after every chunk's erosion (a tile's rays read its
 * neighbours' final heights), light after light; tw_create_tiles_poll completes it with the rest. tile_xy, the lights array, each sp and HOST sh_in rows are
 * copied during the launch; device sh_in rows are read until the completing poll; smask and sh_out_* must stay valid until then (pinned host memory or device
 * memory for a launch that does not block). Errors (TW_ERR_ARG, nothing enqueued): no tile_xy, nlights == 0 or no lights, a light without smask, a device
 * smask that is not 4-byte aligned, a tile named twice in tile_xy, zvsize < 2. */
typedef struct tw_tile_light {
	tw_shadow_params sp;               /* one light: lpos, scene sizes, zmin/zmax, no_shadow (moon with combined_gu) */
	const float *sh_in_x, *sh_in_y;    /* optional: incoming edges from tiles outside the batch, as tw_tile_shadows_batch_ex */
	uint8_t     *smask;                /* required: ntiles*zvsize^2 bytes, host or device (device: 4-byte aligned) */
	float       *sh_out_x, *sh_out_y;  /* optional: ntiles*zvsize floats each, host or device */
} tw_tile_light;
typedef struct tw_tile_shadows {
	const int32_t       *tile_xy;      /* required: (x1/size, y1/size) per tile, caller order */
	uint32_t             nlights;      /* >= 1; the reference has sun and moon */
	const tw_tile_light *lights;
} tw_tile_shadows;
TW_API int tw_create_tiles_launch_shadows(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                          uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows);
/* The asynchronous tile job (tw_create_tiles_launch_shadows, above) with heights from the context's heightmap image instead of the height function: tile t's
 * zvals are get_clamped_height(x1 + x, y1 + y) of the image under hs - exactly what tw_heightmap_sample_tiles returns for the same origins. Everything after
 * that is the job's: erosion when erosion_iters > 0 && erode_amount > 0, per-tile z range, bounds, normal map and min_normal_z, the weights texture with
 * has_any_grass, and the per-light mesh shadows with sh_in. Every output is bit-identical to tw_heightmap_sample_tiles, then tw_erode_tiles(min_zval_all =
 * min_zval) when eroding, then tw_tile_bounds_batch(wpz_max, dx, dy, size), tw_tile_normals_batch(dx, dy), tw_tile_weights_batch(origins, mesh size, dx, dy, p,
 * wp, tile_params) and tw_tile_shadows_batch_ex per light; tw_last_erosion_steps() after the completing poll equals its value after that tw_erode_tiles.
 * Whether heightmap tiles are eroded is the caller's choice (erosion_iters_tt or 0): this library does not pin the reference's (its test harness cannot reach the heightmap branch of create_zvals, see
 * oracle/refbuild/ref_tiled_harness.inc). tw_create_tiles_poll
 * completes the job; the image must not be replaced before then (tw_set_heightmap completes the job first). p is read only by the weights' jitter noise and
 * may be NULL without weights. No tile limit. Not done: the AO map (calc_mesh_ao_lighting reads a (stride + 72)^2 context around the tile, and what the
 * reference reads outside the tile in this mode is not pinned here). Errors, nothing enqueued: TW_ERR_STATE without tw_set_heightmap; TW_ERR_ARG for hs NULL
 * or sized unlike the image, edge_mode outside 0..2, shading->ao, weights without p, and every error of tw_create_tiles_launch_shadows. */
TW_API int tw_create_tiles_launch_hmap(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size,
                          float dx, float dy, uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows);

/* ---- terrain weights texture of tiles (SURVEY.md 8f row N4): tile_t::create_texture (src/tiled_mesh.cpp:1071-1248), the terrain part ----
 * RGBA texel (x, y) of a tile, x, y < stride = zvsize - 1: the weights {sand, dirt, grass, rock} (snow = the rest) of the ground textures from the cell's relative
 * height (get_tids against the h_dirt table, jittered by a high-frequency sine-table noise: build_arrays(x1 - MESH_X_SIZE/2, y1 - MESH_Y_SIZE/2, 80*DX_VAL, 80*DY_VAL,
 * stride, stride, 0, force_sine_mode = 1) / eval_index(x, y, 50)), its slope (steep grass -> dirt / rock, steep snow -> rock), the tile's biome corners (dirt -> sand,
 * grass -> sand) and the water level (no grass under water). NOT here: the texels inside cities / over tunnels / under buildings, the grass-exclusion cubes of bridges, the
 * high-resolution city grass, the grass blocks and the tree-shadow pass (:1113-1138, 1204-1225, 1250-1350) - they read engine state (road networks, building footprints,
 * the tree map); the caller overwrites those texels afterwards, exactly as the reference's loop `continue`s past them. The arithmetic is the reference's, mixed float / double
 * included. tex_class[i] = which ground texture lttex_dirt[i] is, h_dirt[i] = its height threshold (gen_tex_height_tables) - set-up tables, passed in like the sin table. */
enum {TW_TEX_SAND = 0, TW_TEX_DIRT = 1, TW_TEX_GROUND = 2, TW_TEX_ROCK = 3, TW_TEX_SNOW = 4};
typedef struct tw_weight_params {
	float h_dirt[5];          /* h_dirt[] (src/Textures.cpp:1757-1761) */
	int   tex_class[5];       /* lttex_dirt[i].id as TW_TEX_* (each class exactly once: get_texture_ixs asserts it, :1049-1062) */
	int   class_ix[5];        /* filled in by the library: index i of each class */
	float sthresh[2][2];      /* {grass, snow} x {lo, hi} (src/mesh_gen.cpp:44) */
	float zmin, zmax, relh_adj_tex;
	float water_level;        /* get_water_z_height() */
	float noise_scale;        /* ((mesh_gen_shape == 2) ? 2.0 : 1.0)*MESH_NOISE_SCALE*mesh_scale_z, MESH_NOISE_SCALE = 0.003f (:1085-1088) */
	float vnz_scale;          /* (mesh_gen_mode == MGEN_DWARP_GPU) ? SQRT2 : 1.0 (:1092) */
	float vegetation;
	int   snow_to_rock;       /* water_is_lava || DISABLE_WATER == 2 (update_lttex_ix) */
	float dx_val, dy_val, dxdy; /* DX_VAL, DY_VAL, dxdy = DX_VAL*DY_VAL (get_norm_not_normalized) */
	float xy_mult;            /* 1.0/float(size) */
} tw_weight_params;
/* zvals: ntiles*zvsize^2 (host or device); origins_xy: (x1, y1) per tile; p: the scene's height parameters (the noise is force-sine-mode: the context's sine tables from
 * max(p->start_eval_sin, 50) on, shape 0 whatever p->gen_shape says - src/mesh_gen.cpp:592-593); tile_params: ntiles*8 floats = the tile's biome corners params[y][x].grass (4 values) then .dirt (4 values);
 * weights: ntiles*stride^2*4 bytes (host or device); has_any_grass (optional): ntiles bytes. */
TW_API int tw_tile_weights_batch(tw_ctx *ctx, const float *zvals, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                          uint32_t zvsize, const tw_height_params *p, const tw_weight_params *wp, const float *tile_params, uint8_t *weights, uint8_t *has_any_grass);

/* ---------------------------------------------------------------------------------------------------------------------------------------
 * Multi-GPU (SURVEY.md 8e). The reference is one process with OpenMP threads and has no distributed layer; what it has is the tile loop of
 * tile_draw_t::update (src/tiled_mesh.cpp:2367-2417) and the global z range get_heightmap_z_range (src/map_view.cpp:399-407). Tiles and row
 * bands are pure functions of global cell coordinates + seed and every tile is eroded on its own, so the path shards with no data-path
 * collective; the one reduction is the 2-float min/max, done INSIDE the library with ncclAllReduce over NVLink. libnccl.so.2 is loaded at run
 * time (dlopen) only when a multi-GPU entry point is used: the single-GPU library has no NCCL dependency.
 *
 * (1) one process driving all GPUs of the box - what a 3DWorld integration (a single-process engine) would use: */
typedef struct tw_multi tw_multi;  /* one tw_ctx + stream set per device, an NCCL communicator over them (ncclCommInitAll), one host worker thread per device */
TW_API int  tw_multi_create(const int *devices, int ndev, tw_multi **out);   /* devices == NULL: devices 0..ndev-1; tables (tw_set_sin_table) are set up on every device */
TW_API void tw_multi_destroy(tw_multi *m);
TW_API int  tw_multi_size(const tw_multi *m);
TW_API tw_ctx *tw_multi_ctx(tw_multi *m, int i);                              /* the per-device context, for single-device calls */
TW_API const char *tw_multi_last_error(const tw_multi *m);
TW_API int  tw_multi_set_sine_params(tw_multi *m, const float *sine_params450);
/* the partition every sharded call uses: device i owns tiles / rows [n*i/ndev, n*(i+1)/ndev) - contiguous bands */
TW_API void tw_multi_range(uint32_t n, int ndev, int i, uint32_t *begin, uint32_t *end);
/* pinned host memory on the NUMA node of device i's PCIe root (allocated from a thread bound to the GPU's local CPUs): output buffers of the
 * sharded calls should come from here - 8 concurrent device->host streams into memory of the wrong socket cost a third of the end-to-end rate */
TW_API int  tw_multi_alloc_host(tw_multi *m, int i, size_t bytes, void **ptr);
TW_API void tw_multi_free_host(tw_multi *m, void *ptr);
/* tile_t::create_zvals for a batch of tiles dealt out over the devices (tw_create_zvals_batch on each device's band, concurrently).
 * out_bands: ndev pointers, one per band (host or device memory of ANY kind, e.g. from tw_multi_alloc_host, or device i's own memory), band i =
 * tiles tw_multi_range(ntiles, ndev, i); mm (optional, HOST, ntiles); zrange (optional, HOST) = min/max over ALL tiles, reduced with ncclAllReduce. */
TW_API int  tw_create_zvals_sharded(tw_multi *m, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                             uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                             float *const *out_bands, tw_minmax *mm, tw_minmax *zrange);
/* mesh_xy_grid_cache_t::build_arrays + eval_index over ONE nx*ny grid split into ndev row bands (heightmap_t::proc_gen's fill, sharded):
 * band i = rows tw_multi_range(g->ny, ndev, i), out_bands[i] receives rows*nx floats; zrange as above. */
TW_API int  tw_heightgen_2d_sharded(tw_multi *m, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, float *const *out_bands, tw_minmax *zrange);
/* Coherent erosion of ONE heightmap that is too big for / spread over several GPUs (SURVEY.md 8e "optional coherent variant"; the single-grid
 * caller is heightmap_t::run_erosion, src/heightmap.cpp:153-187). The reference's droplet order cannot be kept across devices (every droplet
 * sees all earlier writes), so this is its BATCHED variant, defined independently of the device count: droplets are processed in sweeps of
 * `sweep` droplets; all droplets of a sweep read the map as it was when the sweep began; their deposits / erosions (same per-move arithmetic as
 * src/erosion.cpp:76-152) are accumulated in 64-bit fixed point (2^-40 height units: integer sums do not depend on order) and added to the map
 * after the sweep; a droplet still sees its OWN writes through a private 32x32 view (sweep-start heights + its writes; re-read and re-centred
 * ahead of its heading when it walks out of it - without that feedback a droplet in a pit never fills it); it ends once it is more than
 * halo-36 rows away from its start row (halo >= 44), or when its next position is not a finite number (a NaN of its own making; the reference would go on
 * to read the map's first row there, which a device holding one band does not have). Row bands as tw_multi_range(ysize, ndev, i); each
 * device keeps its band +- halo rows and after every sweep neighbours exchange the deltas of the 2*halo rows around their border in ONE grouped
 * ncclSend/ncclRecv over NVLink (width*2*halo*8 bytes per neighbour). The result is bit-identical for every device count (tw_erode_sweeps ==
 * tw_erode_sweeps_sharded), which is what the parity tests check, next to the CPU oracle of the same algorithm. bands[i]: the band's rows in
 * place (device i's memory or host memory); moves (optional) = droplet moves. */
TW_API int  tw_erode_sweeps(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                     uint32_t sweep, int halo, uint64_t *moves);
/* The same band decomposition on ONE device: nbands row bands (tw_multi_range(ysize, nbands, i)), each with its own halo copy, exchanging the border deltas with
 * device-to-device copies instead of NCCL. Same result as tw_erode_sweeps; exists so that the decomposition for any band count can be checked on a single GPU. */
TW_API int  tw_erode_sweeps_banded(tw_ctx *ctx, float *const *bands, int nbands, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                            uint32_t sweep, int halo, uint64_t *moves);
TW_API int  tw_erode_sweeps_sharded(tw_multi *m, float *const *bands, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                             uint32_t sweep, int halo, uint64_t *moves);
/* (2) one process per GPU (torchrun / mpirun style): rank 0 makes an id, every rank passes it to tw_dist_init on its own context */
TW_API int  tw_dist_unique_id(char id128[128]);
TW_API int  tw_dist_init(tw_ctx *ctx, int nranks, int rank, const char id128[128]);
TW_API int  tw_dist_allreduce_minmax(tw_ctx *ctx, tw_minmax *inout);          /* global z range over all ranks (blocking) */
TW_API void tw_dist_finalize(tw_ctx *ctx);
/* binds the CALLING thread to the CPUs local to `device` (sysfs local_cpulist of its PCI function), so that pinned buffers it allocates next
 * are NUMA-local to that GPU; returns TW_OK or TW_ERR_ARG when the topology is not exposed (then nothing changes) */
TW_API int  tw_bind_thread_to_device(int device);

#ifdef __cplusplus
}
#endif
#endif /* TW3D_H */
