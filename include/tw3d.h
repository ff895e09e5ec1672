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
	TW_ERR_NOT_READY = -5,   /* tw_heightgen_2d_poll / tw_create_tiles_poll: result not available yet (mirrors build_arrays() returning 0 with no_wait) */
	TW_ERR_CANCELED  = -6    /* tw_heightgen_2d_poll / tw_create_tiles_poll: tw_cancel cut the job short; its outputs are unspecified (see tw_cancel) */
} tw_status;

/* mesh_gen_mode values, src/3DWorld.h:1399 */
enum { TW_MGEN_SINE = 0, TW_MGEN_SIMPLEX = 1, TW_MGEN_PERLIN = 2, TW_MGEN_SIMPLEX_GPU = 3, TW_MGEN_DWARP_GPU = 4 };

#define TW_F_TABLE_SIZE   90      /* NUM_FREQ_COMP*N_RAND_SIN2, src/mesh_gen.cpp:14,16,30 */
#define TW_SIN_TABLE_SIZE 65536   /* 2*TSIZE, src/sinf.h:8 */
#define TW_N3D_RDATA      420     /* SINE_DATA_SIZE, src/upsurface.h:14-16 */
#define TW_N3D_SINES      60      /* TOT_NUM_SINES */

typedef struct tw_ctx tw_ctx;   /* one per (thread, device): owns a CUDA stream, the uploaded tables (or reads its parent's: tw_create_shared) and scratch buffers */

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
 * as a poll with wait = 1 would, and either poll function completes whichever job is pending. The rule is per context: to keep several jobs in flight
 * on one device, give each its own shared context (tw_create_shared); a call on one context never completes another context's job, except the three
 * table setters on a parent (below). Deliberate exceptions to "complete the pending job first": tw_cancel and tw_update_heightmap complete no job and
 * never wait for the device.
 * Threads: one thread at a time per context. A parent's tw_set_sin_table, tw_set_sine_params, tw_set_heightmap and tw_update_heightmap must not run while
 * another thread is inside a call on one of its shared contexts (tw_update_heightmap reads the shared contexts' pending-job state). */
TW_API int  tw_abi_version(void);
TW_API int  tw_create(int device, tw_ctx **out);
/* A context on parent's device that uses parent's tables instead of its own: sin table, direction table, sine params, the simplex/Perlin
 * and 3-D noise LUTs, and the tw_set_heightmap image. It has its own streams, scratch, pinned staging, pending job, launch count and
 * erosion step count, so its asynchronous job runs beside the parent's and the other shared contexts' jobs. Every entry point accepts it, with the
 * results the same call on the parent gives, bit for bit.
 * - Tables are set on the parent only: tw_set_sin_table, tw_set_sine_params and tw_set_heightmap on a shared context return TW_ERR_ARG and change
 *   nothing. On the parent they first complete the pending job of every shared context (as a poll with wait = 1 would), then replace the table; the
 *   next call on a shared context uses the new tables. Before the parent has a table, a shared context gets TW_ERR_STATE where the parent would.
 * - The parent's LUTs are built here if absent (one synchronisation of the parent's stream); a shared context never allocates or builds a table.
 * - TW_ERR_ARG for a NULL parent and for a parent that is itself a shared context (one level only).
 * - tw_destroy(shared) completes its job as a poll with wait = 1 would and frees only what it owns. tw_destroy(parent) first destroys the shared
 *   contexts still alive the same way; their handles are invalid afterwards. */
TW_API int  tw_create_shared(tw_ctx *parent, tw_ctx **out);
TW_API void tw_destroy(tw_ctx *ctx);
TW_API const char *tw_last_error(const tw_ctx *ctx);
TW_API int  tw_sync(tw_ctx *ctx);                         /* cudaStreamSynchronize on the context stream */
TW_API void *tw_stream(tw_ctx *ctx);                      /* the cudaStream_t all work of this context is issued on */
TW_API uint64_t tw_launch_count(const tw_ctx *ctx);       /* kernels launched by this context so far (bench.py gpu_launches) */
TW_API uint64_t tw_dwarp_window_launches(const tw_ctx *ctx); /* of those, launches of the domain-warp kernel with lattice windows (one per grid or
                                                            * row band whose windows fit its tables; every other launch of that mode reduces mod 289) */
/* Asks the context's pending asynchronous job to stop, for work the caller no longer wants (a map reloaded or the scene quit while it is eroded, tiles
 * that went out of range, a voxel model replaced while its fills run). Returns at once: it never waits for the device and enqueues nothing on the
 * context's stream. Called by the thread that owns the context, like every other entry point.
 * - TW_OK whether or not a job is pending; with no job, or a job that has already finished, nothing changes. TW_ERR_ARG for a NULL ctx.
 * - TW_ERR_STATE for a job that touches a tile set (tw_tile_set_shadows_launch, tw_tile_set_create_tiles_launch), which keeps running unaffected: a set's
 *   state is committed at launch, in launch order, and frames launched later on other shared contexts already rely on it.
 * - The job stops at its next cancellation point: a droplet walk within its next 8 droplets (tile erosion, the OpenMP mode; on a batch small enough to be
 *   walked all at once, only walks of at least 4096 droplets per map - shorter ones take well under 0.1 s and run to their end), the serial order's
 *   speculative erosion at its next round (a round is at most 64 moves per walker), the TW_EROSION_SWEEPS job after its current sweep, a voxel flood fill
 *   at its next generation, the mesh shadows at their next wave.
 *   What is already enqueued of everything else still runs (generation, the tile tail, marching cubes, the end-of-job copies); a job without a
 *   cancellation point (a tw_heightgen_2d_launch grid, a heightmap job without erosion) completes as if tw_cancel had not been called.
 * - The completing poll (tw_create_tiles_poll / tw_heightgen_2d_poll) returns TW_ERR_CANCELED when a cancellation point acted. Every output of the job is
 *   then unspecified: device and host buffers may be partly written, and the host arrays the poll fills (mm, bounds, info, ntris, ...) are not written.
 *   tw_last_erosion_steps() is 0, and a job that would have set the context's heightmap image (set_image, erosion of the image) leaves the context without
 *   one. Nothing else changes: the next job gives what it gives on a fresh context. Otherwise the poll returns what it would have returned, with every
 *   output bit-identical to the job without tw_cancel.
 * - Every entry point, tw_set_heightmap and tw_destroy still complete the pending job first; calling tw_cancel before them makes that wait short. A job
 *   they complete that was cut short counts as completed, not as an error: the call goes on with its own work (a new map is loaded, the next job is
 *   launched) and returns its own status. Only the two polls report TW_ERR_CANCELED. The same holds for a parent's table setters, which complete the jobs of
 *   its shared contexts. Synchronous calls are not jobs and are never cancelled. */
TW_API int  tw_cancel(tw_ctx *ctx);

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
/* Heights at many points as the context's ASYNCHRONOUS job, so that object placement does not stall the frame: the procedural kinds of tw_eval_points, and
 * TW_PQ_HMAP, the height of the context's tw_set_heightmap image.
 * - TW_PQ_SIN_TERMS .. TW_PQ_EXACT_ZVAL: after the completing poll out equals tw_eval_points(ctx, xy, n, p, q, out) bit for bit (same kernel).
 * - TW_PQ_HMAP: xy holds cells of the heightmap tiles' index space (a tile's cell (x, y) is (x1 + x, y1 + y), tw_create_tiles_launch_hmap); out[i] is
 *   get_clamped_height there under hs, scaled by scale_mh_texture_val, with the expressions of tw_heightmap_sample_tiles: mesh_scale < 1 interpolate_height
 *   at mesh_scale*x with its floor and ceil taps, otherwise the nearest texel round_fp(mesh_scale*x); outside the image clamp_no_scale in hs->edge_mode (cliff:
 *   scale_mh_texture_val(0)). At an integer cell with |mesh_scale*x|, |mesh_scale*y| < 2^30 (every |x|, |y| < 2^24 at a mesh_scale below 64) the result equals,
 *   bit for bit, the tw_heightmap_sample_tiles value of any tile containing the cell. At a fractional cell (an object between cells) the same expressions
 *   take the float directly: the library's extension of the reference's integer-cell function. Scaled coordinates beyond +-2^30, and NaN, are held to
 *   -2^30 .. 2^30. p is not read.
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it (wait = 0 returns TW_ERR_NOT_READY while it runs), every
 *   other entry point and tw_destroy complete it first. On a shared context it runs beside the other contexts' jobs. tw_cancel returns TW_ERR_STATE: the
 *   job is one kernel.
 * - TW_PQ_HMAP sees the image as it was when its launch returned: every tw_update_heightmap made before the launch, none made after it. A later edit waits
 *   on the device only for this job's kernel. While an erosion of the image or a set_image heightmap job is pending the launch returns TW_ERR_STATE, as
 *   tw_create_tiles_launch_hmap does.
 * - Host xy (pageable or page-locked) is copied into the context's pinned staging during the launch, so the caller may reuse it as soon as the call returns;
 *   device xy is read until the completing poll. out is device, page-locked or pageable host memory; pageable out is filled by the completing poll. With
 *   device or page-locked xy and out the launch never waits for the device, except when the context's scratch or staging first has to grow.
 * - Errors, nothing enqueued: TW_ERR_ARG for what tw_eval_points refuses, a NULL job, a NULL q, xy or out with n > 0, TW_PQ_HMAP without hs, hs sized
 *   unlike the image and edge_mode outside 0..2; TW_ERR_STATE without the sin table or (sine mode, TW_PQ_SIN_TERMS) the sine params, and TW_PQ_HMAP
 *   without an image. n == 0 is TW_OK and enqueues nothing. tw_eval_points refuses TW_PQ_HMAP as any other unknown kind. */
#define TW_PQ_HMAP 3
typedef struct tw_points_job {
	const float            *xy;   /* n (x, y) pairs: host (copied during the launch) or device (read until the completing poll) */
	size_t                  n;
	const tw_height_params *p;    /* procedural kinds, as tw_eval_points */
	const tw_point_query   *q;    /* required; q->kind selects TW_PQ_SIN_TERMS .. TW_PQ_EXACT_ZVAL or TW_PQ_HMAP */
	const struct tw_hmap_sampler *hs; /* TW_PQ_HMAP only: required, sized like the context's image (declared below) */
	float                  *out;  /* n floats: device, page-locked or pageable host memory (the last is filled by the completing poll) */
} tw_points_job;
TW_API int tw_points_launch(tw_ctx *ctx, const tw_points_job *job);

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
/* tw_erode / tw_erode_parallel of ONE map as the context's ASYNCHRONOUS job (heightmap_t::run_erosion, src/heightmap.cpp:153-187, without holding the host):
 * everything is enqueued without the host reading anything back (the speculative erosion's rounds end on the device, the step count is staged) and the
 * completing poll reports the result.
 * - heightmap != NULL: xsize*ysize floats eroded in place, device or host. After the completing poll the map and tw_last_erosion_steps() equal
 *   tw_erode(heightmap, xsize, ysize, min_zval, num_iters, ep) bit for bit in TW_EROSION_SERIAL mode, and tw_erode_parallel(..., num_threads) in
 *   TW_EROSION_OPENMP mode (bit for bit with num_threads == 1; order-dependent as that call's result otherwise). The serial order's "made no progress" case
 *   is reported by the poll as TW_ERR_STATE with tw_erode's message.
 * - heightmap == NULL: the context's tw_set_heightmap image (root context only; xsize = ysize = 0, min_zval unused). After a poll that returns TW_OK the image,
 *   vals and tw_last_erosion_steps() equal the synchronous chain tw_heightmap_to_floats_u16(image, val_mult, val_add) -> tw_minmax_f32 -> tw_erode (or
 *   tw_erode_parallel) with min_zval = that minimum (run_erosion's min_zval) -> tw_heightmap_from_floats_u16(val_mult, val_add) back into the image, bit for
 *   bit. The launch first completes every shared context's job; until a poll returns TW_OK the context has no image (a shared context's
 *   tw_create_tiles_launch_hmap gets TW_ERR_STATE; the parent's own completes this job first). A packed value outside [0,256) makes the completing poll
 *   return TW_ERR_ARG with tw_heightmap_from_floats_u16's message; a poll that returns an error leaves the context without an image.
 * - num_iters == 0 or erode_amount <= 0 (src/erosion.cpp:16): the job does no work and reports 0 steps; the image keeps its bytes and vals is not written.
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it (wait = 0 returns TW_ERR_NOT_READY while it runs), every
 *   other entry point and tw_destroy complete it first. On a shared context (float maps only) it runs beside the other contexts' jobs.
 * - The launch never waits for the device, except that copies to or from a PAGEABLE host heightmap / vals block it (see "Host output buffers" above). Every
 *   buffer is reserved before anything is enqueued. heightmap and vals must stay valid until the completing poll.
 * - Errors, nothing enqueued and nothing changed: TW_ERR_ARG for a NULL job or ep, an empty map, sizes or vals given with a float map's counterpart (sizes
 *   with the image, vals with a float map), a bad mode, num_threads != 0 in TW_EROSION_SERIAL mode, the image on a shared context; TW_ERR_STATE for the
 *   image when none is set, and without the sin table when there is work to do. */
#define TW_EROSION_SERIAL 0   /* tw_erode: the reference's serial droplet order */
#define TW_EROSION_OPENMP 1   /* tw_erode_parallel: the reference's `#pragma omp parallel for` mode with num_threads droplets in flight */
typedef struct tw_erosion_job {
	float                    *heightmap;        /* xsize*ysize floats, device or host; NULL: the context's tw_set_heightmap image */
	int                       xsize, ysize;     /* with heightmap; 0 with the image */
	float                     min_zval;         /* with heightmap: the lower clamp, as tw_erode's */
	float                     val_mult, val_add;/* with the image: the unpack's and the pack's scalars (get_mh_texture_mult / _add) */
	uint32_t                  num_iters;
	const tw_erosion_params  *ep;               /* required; copied during the launch */
	int                       mode;             /* TW_EROSION_SERIAL or TW_EROSION_OPENMP (TW_EROSION_SWEEPS: tw_erode_launch_ex) */
	uint32_t                  num_threads;      /* TW_EROSION_OPENMP: as tw_erode_parallel's (0 = fill the GPU); must be 0 otherwise */
	float                    *vals;             /* with the image, optional: the eroded floats before the pack, device or host */
} tw_erosion_job;
TW_API int tw_erode_launch(tw_ctx *ctx, const tw_erosion_job *job);
/* The same with a third mode, TW_EROSION_SWEEPS: tw_erode_sweeps (below) of the one map as the job - deterministic like the serial order and, on a big map
 * with many droplets, far faster. tw_erode_launch(ctx, job) is tw_erode_launch_ex(ctx, job, NULL).
 * - sw is required with TW_EROSION_SWEEPS (TW_ERR_ARG without it) and refused with the other two modes; num_threads must be 0.
 * - heightmap != NULL: after the completing poll the map and tw_last_erosion_steps() equal tw_erode_sweeps(heightmap, xsize, ysize, min_zval, num_iters, ep,
 *   sw->sweep, sw->halo, &moves) bit for bit, with the steps equal to moves (device, pinned or pageable host maps).
 * - heightmap == NULL: as above for the image, with tw_erode_sweeps in the chain (min_zval = the image's minimum); every rule of the image mode holds.
 * - Errors, nothing enqueued: those of tw_erode_launch, and those of tw_erode_sweeps - sw->sweep == 0 or sw->halo < 44 (view + 12) - checked even when
 *   num_iters == 0 or erode_amount <= 0 (the job then does no work and reports 0 steps).
 * - The sweeps run as one graph launch whose loop ends on the device, so a job of thousands of sweeps never fills the launch queue. The device memory is
 *   the context's scratch: (xsize + 8)*(ysize + 8)*12 bytes besides the floats. tw_cancel stops the job after its current sweep. */
#define TW_EROSION_SWEEPS 2   /* tw_erode_sweeps: the coherent batched sweeps (tw_sweep_params) */
typedef struct tw_sweep_params { uint32_t sweep; int halo; } tw_sweep_params; /* tw_erode_sweeps' sweep and halo */
TW_API int tw_erode_launch_ex(tw_ctx *ctx, const tw_erosion_job *job, const tw_sweep_params *sw);
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
/* tw_proc_gen_heightmap as the context's ASYNCHRONOUS job: generation, erosion, the z range, the texture scalars and the pack are enqueued without the host
 * reading anything back (the speculative erosion's rounds end on the device). After the completing poll every output equals tw_proc_gen_heightmap with the same
 * arguments, bit for bit - data16, vals, every field of info and tw_last_erosion_steps(); a value outside [0,256) makes that poll return TW_ERR_ARG with the
 * synchronous call's message, after the outputs are written.
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it (wait = 0 returns TW_ERR_NOT_READY while it runs), every
 *   other entry point and tw_destroy complete it first. On a shared context it runs beside the other contexts' jobs.
 * - The launch never waits for the device, except that copies to PAGEABLE host data16 / vals block it (see "Host output buffers" above). Every buffer is
 *   reserved before anything is enqueued.
 * - set_image = 1 (root context only): the packed image becomes the context's tw_set_heightmap image, written straight into the context's allocation. The
 *   launch first completes every shared context's job and releases the old image; until the completing poll the context has no image (a shared context's
 *   tw_create_tiles_launch_hmap gets TW_ERR_STATE; the parent's own completes this job first). After a poll that returns TW_OK the state equals
 *   tw_set_heightmap(data16, width, height).
 * - Errors, nothing enqueued and nothing changed: TW_ERR_ARG for a NULL p or out, an empty grid, neither data16 nor set_image, set_image on a shared context,
 *   and what tw_proc_gen_heightmap refuses; TW_ERR_STATE without the sin table (or, in sine mode, the sine params). */
typedef struct tw_heightmap_outputs {
	uint8_t           *data16;    /* optional: 2*width*height bytes, device or host (the layout of tw_heightmap_from_floats_u16) */
	float             *vals;      /* optional: width*height floats after erosion, device or host */
	tw_heightmap_info *info;      /* optional HOST: filled by the completing poll */
	int                set_image; /* 1: the packed image becomes the context's tw_set_heightmap image (root context only) */
} tw_heightmap_outputs;
TW_API int tw_proc_gen_heightmap_launch(tw_ctx *ctx, uint32_t width, uint32_t height, float dx_val, float dy_val, const tw_height_params *p,
                                        uint32_t erosion_iters, const tw_erosion_params *ep, const tw_heightmap_outputs *out);
/* gen_mesh() of the ground mode (src/mesh_gen.cpp:257-355) after its sine table, as the context's ASYNCHRONOUS job: the mesh fill (gen_mesh_sine_table,
 * :201-210), calc_zminmax, the 128x128 probe of estimate_zminmax (:447-485), set_zvals (:494-504), glaciate() (:388-404) and apply_erosion(mesh, X, Y,
 * zbottom, erosion_iters) (:443) are enqueued without the host reading anything back: every scalar a step takes from the data (zmax_est, zbottom, the
 * erosion's zmin / zmax / water_plane_z) is derived on the device, and the speculative erosion's rounds end on the device. After the completing poll mesh,
 * every field of info and tw_last_erosion_steps() equal, bit for bit, the synchronous chain tw_heightgen_2d of the mesh -> tw_heightgen_2d of the probe ->
 * the host's zmax_est / set_zvals arithmetic -> tw_glaciate_mesh (p->glaciate) -> tw_erode(min_zval = zbottom) with these arguments (tw3d::gen_mesh).
 * - Run tw_gen_sine_params and tw_set_sine_params first, as gen_mesh does: the job reads the context's tables like every other job.
 * - p->zmax_est is ignored: the job derives it. ep's erode_amount, half_dxy, relh_adj_tex and clip_hd1 are read; its zmin, zmax and water_plane_z are the
 *   ones set_zvals leaves (-zmax_est, zmax_est, get_water_z_height(zmax_est) from water_h_off / water_h_off_rel and p's glaciation). The probe's step is
 *   rm_scale = 1000*XY_SCENE_SIZE/mesh_scale with XY_SCENE_SIZE = 0.5*(x_scene_size + y_scene_size) and p->mesh_scale.
 * - A flat mesh (zmin == zmax) keeps what the reference keeps: estimate_zminmax returns before set_zvals, so zmin / zmax are the measured pair and zbottom,
 *   ztop and water_plane_z are the caller's prev_* values (glaciation still replaces zbottom / ztop). The erosion then takes the per-move rock expression
 *   with zmax - zmin = 0, as tw_erode does.
 * - No erosion (erosion_iters == 0 or erode_amount <= 0, src/erosion.cpp:16): info->erosion_moves and tw_last_erosion_steps() are 0.
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it (wait = 0 returns TW_ERR_NOT_READY while it runs), every
 *   other entry point and tw_destroy complete it first. On a shared context it runs beside the other contexts' jobs. tw_cancel stops the erosion at its
 *   cancellation points (as for tw_erode_launch); the poll then returns TW_ERR_CANCELED and the outputs are unspecified.
 * - mesh is device, page-locked or pageable host memory; pageable mesh is filled by the completing poll. With device or page-locked mesh the launch never
 *   waits for the device, except when the context's scratch or staging first has to grow. Every buffer is reserved before anything is enqueued.
 * - The erosion walks the map in the mode tw_erode picks for it (the serial order's result does not depend on the mode): M_SPEC's speculative rounds from
 *   2^20 padded cells and 64 droplets on. A window that stops making progress makes the poll return TW_ERR_STATE with tw_erode's message.
 * - Errors, nothing enqueued: TW_ERR_ARG for a NULL job, p, ep or mesh, a mesh size <= 0 (or a mesh_y_size above 65535), and what tw_heightgen_2d refuses
 *   for either grid; TW_ERR_STATE without the sin table or, in sine mode, the sine params. */
typedef struct tw_gen_mesh_info {
	float    zmin, zmax, zmax_est, zbottom, ztop, water_plane_z; /* the z globals gen_mesh leaves */
	uint64_t erosion_moves;                                      /* droplet moves of the erosion (tw_last_erosion_steps()) */
} tw_gen_mesh_info;
typedef struct tw_gen_mesh_job {
	int                       mesh_x_size, mesh_y_size;  /* MESH_X_SIZE, MESH_Y_SIZE: the mesh is mesh_y_size rows of mesh_x_size floats */
	int                       xoff2, yoff2;              /* the mesh's scroll offset */
	float                     dx_val, dy_val;            /* DX_VAL, DY_VAL */
	float                     x_scene_size, y_scene_size;/* X_SCENE_SIZE, Y_SCENE_SIZE: the probe's step */
	const tw_height_params   *p;                         /* required, copied during the launch; zmax_est is ignored */
	uint32_t                  erosion_iters;
	const tw_erosion_params  *ep;                        /* required, copied during the launch: erode_amount, half_dxy, relh_adj_tex, clip_hd1 */
	float                     water_h_off, water_h_off_rel;
	float                     prev_zbottom, prev_ztop, prev_water_plane_z; /* zbottom, ztop, water_plane_z before the call: a flat mesh keeps them */
	float                    *mesh;                      /* required: mesh_x_size*mesh_y_size floats, device, page-locked or pageable host memory */
	tw_gen_mesh_info         *info;                      /* optional HOST: filled by the completing poll */
} tw_gen_mesh_job;
TW_API int tw_gen_mesh_launch(tw_ctx *ctx, const tw_gen_mesh_job *job);
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
 * image; width or height <= 0 with an image is TW_ERR_ARG. A new map means calling it again; an edit of the map (a brush stroke, the saved edits re-applied
 * when a map loads) is tw_update_heightmap, which waits for nothing. It first orders after the pending edits, then frees their staging; tw_destroy frees the
 * image. */
TW_API int tw_set_heightmap(tw_ctx *ctx, const uint8_t *data16, int width, int height);
/* A rectangle of the heightmap image: texels [x, x + w) x [y, y + h); image row y is bytes [2*width*y, 2*width*(y + 1)). */
typedef struct tw_hmap_rect { int x, y, w, h; } tw_hmap_rect;
/* Edits the context's tw_set_heightmap image in place: for each rect, texel (x, y) becomes the two bytes at src16 + y*src_pitch + 2*x (an engine passes its
 * whole CPU image, src_pitch = 2*width, after its brush code changed it, with the brush's bounding rect). Rects may overlap; overlapping rects copy the same
 * source bytes, so their order does not matter.
 * What each job sees: every job sees the image as it was when its launch returned - every edit made before the launch, none made after it - on the root
 * context and on every shared context. A job launched before the edit gives, bit for bit, the outputs it gives with the old image; a job launched after it
 * gives the outputs of the same job after tw_set_heightmap(the edited image).
 * It completes no job and never waits for the device (an exception to the rule under "context"). The image has its own stream on the root context: the
 * edit's copy and scatter kernel wait there, on the device, for the image work of the family's pending jobs - the sampling of a heightmap tile job (its
 * erosion, shadows and tile-set tail run on beside the edit), the whole of an image erosion or a set_image job - and jobs that read or write the image
 * wait on the device for the edits made before their launch; jobs that do not touch the image wait for nothing. The image is not double-buffered: a job
 * launched after an edit starts on the device only once the image jobs launched before the edit have sampled it (image erosion, set_image: finished).
 * A job launched before an edit and cancelled after it leaves the edit in place. The staging is kept for later edits (an edit reuses a free buffer that is large
 * enough) and freed by tw_set_heightmap, a set_image launch and tw_destroy: freeing pinned memory would synchronise the device, which this call never does.
 * src16 is host memory (pageable or pinned): the call copies the rects' texels into pinned staging of its own before it returns, so the caller may change
 * its image at once.
 * Errors, nothing enqueued: TW_ERR_ARG for a NULL ctx, a shared context (the image is set on the parent), NULL src16 or rects with nrects > 0, a rect with
 * w <= 0 or h <= 0 or reaching outside the image (no clipping), src_pitch < 2*(x + w) for some rect, and a device src16; TW_ERR_STATE without an image,
 * which includes the time an erosion of the image or a set_image heightmap job is pending. nrects == 0 is TW_OK and does nothing. */
TW_API int tw_update_heightmap(tw_ctx *ctx, const uint8_t *src16, size_t src_pitch, const tw_hmap_rect *rects, uint32_t nrects);
/* Reads the context's image back, the inverse of tw_update_heightmap: for each rect, the two bytes of texel (x, y) go to dst16 + y*dst_pitch + 2*x, so a read
 * of rects followed by tw_update_heightmap of the same rects from the same buffer changes no byte. The whole image is the one rect {0, 0, width, height}
 * with dst_pitch = 2*width. This is how an engine's CPU copy catches up with what the device wrote: an erosion of the image, a set_image heightmap job (with
 * or without data16), before its brushes, its PNG or its saved edits read the CPU copy.
 * - What it sees: the image as it was when the launch returned - every tw_update_heightmap made before the launch, none made after it - on the root context
 *   and on every shared context (a shared context reads its parent's image, as TW_PQ_HMAP points do). On the root the launch first completes the pending
 *   job, as every entry point does, so a read launched after an erosion of the image or a set_image job sees their result; on a shared context while such a
 *   job is pending there is no image (TW_ERR_STATE).
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it. A later edit waits on the device for its first kernel
 *   only. tw_cancel returns TW_ERR_STATE: the job has no cancellation point.
 * - The copies run on tw_update_heightmap's row kernel. dst16 in device memory (2-byte aligned, even dst_pitch: texels are 16-bit words) is written at the
 *   caller's pitch: straight from the image when every row has its image row's phase modulo 16 bytes (a buffer laid out like the image), otherwise through
 *   device staging, with one device copy per phase shift (at most 8) and a second run of the kernel. dst16 in host memory (page-locked or pageable)
 *   receives the rows from the context's pinned staging in the completing poll. Either way the launch never waits for the device, except when the
 *   context's scratch or staging first has to grow, and what it enqueues does not grow with nrects: one row-table copy and one kernel, plus one copy down
 *   for host dst16, or the shift copies and the second kernel for a device dst16 out of phase. dst16 must stay valid until the completing poll.
 * - Errors, nothing enqueued: TW_ERR_ARG for a NULL ctx or r, NULL rects or dst16 with nrects > 0, a rect with w <= 0 or h <= 0 or reaching outside the
 *   image (no clipping), dst_pitch < 2*(x + w) for some rect, a device dst16 at an odd address or with an odd dst_pitch; TW_ERR_STATE without an image.
 *   nrects == 0 is TW_OK and does nothing.
 * tw_read_heightmap is the launch followed by a poll with wait = 1. */
typedef struct tw_hmap_read {
	const tw_hmap_rect *rects;   /* nrects rects of the image, as tw_update_heightmap's */
	uint32_t nrects;
	uint8_t *dst16;              /* texel (x, y) of each rect -> dst16 + y*dst_pitch + 2*x */
	size_t   dst_pitch;          /* >= 2*(x + w) for every rect; 2*width for an engine's whole image */
} tw_hmap_read;
TW_API int tw_read_heightmap_launch(tw_ctx *ctx, const tw_hmap_read *r);
TW_API int tw_read_heightmap(tw_ctx *ctx, const tw_hmap_read *r);
/* Host only, no context: touched[t] = 1 exactly when some cell of tile t (origin origins_xy[2t], origins_xy[2t + 1], zvsize^2 cells), as the heightmap-texture
 * tiles sample it under hs, reads a texel inside one of the rects - the live tiles an edit changes. A texel counts as read even where its bilinear weight is 0;
 * cells that read nothing (off the texture in cliff mode) read no texel. Exact, and O(zvsize) per distinct tile column and row: the sampler's index
 * arithmetic is separable per axis. TW_ERR_ARG for a NULL hs, a width or height <= 0, edge_mode outside 0..2, a NULL array with a nonzero count, or
 * zvsize < 2.
 * The tiles whose AO map (tw_hmap_tile_ao_launch) an edit can change: the AO of tile t reads the texels of its window, cells [x1 - 36, x1 + zvsize + 35) on
 * each axis, so this call with origins (x1 - 36, y1 - 36) and zvsize + 71 (= stride + 72) flags them (the C++ adapter's tw3d::hmap_ao_tiles_touched). That is
 * conservative: texels that only the window's corners read, where no ray goes, count too. */
TW_API int tw_hmap_tiles_touched(const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, uint32_t zvsize, const tw_hmap_rect *rects,
                                 uint32_t nrects, uint8_t *touched);
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
 * not depend on the fill order, so the result is identical to the reference's stack-based fill. vals / outside modified in place (host or device;
 * a device outside must be 4-byte aligned, and is worked on in a padded copy when nx*ny*nz is not a multiple of 4); changed (optional) = number of voxels flipped. */
TW_API int tw_voxel_remove_unconnected(tw_ctx *ctx, float *vals, uint8_t *outside, const tw_voxel_post_params *vp, uint64_t *changed);
/* Marching cubes: voxel_manager::add_triangles_for_voxel at LOD 0 for every cube of the grid in the order of voxel_model::create_block (y, x, z),
 * src/voxels.cpp:485-566,1077-1108, as an UNWELDED triangle soup: tris[t] = 3 vertices x (x, y, z), each cube's vertices interpolated by that cube
 * (interpolate_pt); triangles whose normal is the zero vector are dropped as the reference drops them (:550). The reference additionally welds vertices
 * through a per-block index cache: a vertex on a shared edge keeps the position computed by the first cube that used it. Neighbouring cubes walk a shared
 * edge in opposite directions, so this soup's copy of a vertex can differ from the cached one by up to about two ulps of the edge's endpoint coordinate
 * (many ulps of a coordinate near zero), and welding the soup by position cannot rebuild the reference's mesh: tw_voxel_mesh_welded returns that indexed mesh.
 * Vertex normals stay with the renderer-side caller. The case tables are the caller's voxel_detail::edge_table[256], tri_table[256][16],
 * edge_to_vals[12][2] (src/marching_cubes.h; Paul Bourke's polygonise tables) - data, passed in like the sin table. tris: capacity*9 floats, host or
 * device (NULL with capacity 0 to only count); ntris = triangles the grid produces (may exceed capacity: nothing is written beyond it). */
TW_API int tw_voxel_triangles(tw_ctx *ctx, const float *vals, const uint8_t *outside, const tw_voxel_post_params *vp, const uint32_t *edge_table256,
                       const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, float *tris, uint64_t capacity, uint64_t *ntris);
/* The indexed (welded) mesh of voxel_model::create_block at LOD 0, one block (src/voxels.cpp:495-566,1077-1108): the cubes of tw_voxel_triangles, with
 * one vertex per crossing grid edge. The edge's owner is the first cube containing it in (y, x, z) order that is not skipped (last layer of an axis,
 * skip_under_mesh); its position is the owner's interpolate_pt along its local edge, in its edge_to_vals corner order. Vertices are ordered by owner, then
 * by the owner's local edge 0..11: the creation order of a vertex cache filled for every crossing edge of a cube (vertices that only degenerate triangles
 * use are kept, as the reference keeps them). Triangles: per cube in tri_table order, three vertex indices each, dropped when the normal of their WELDED
 * positions is the zero vector, so their count can differ from the soup's. Flattening indices through verts gives the reference's welded triangles.
 * edge_to_vals must name each of the cube's 12 edges once (Bourke's table does). */
typedef struct tw_voxel_mesh {
	float    *verts;      /* vcapacity*3 floats: x, y, z per vertex (NULL with vcapacity 0) */
	uint64_t  vcapacity;
	uint32_t *indices;    /* tcapacity*3 vertex indices (NULL with tcapacity 0) */
	uint64_t  tcapacity;
	uint64_t *nverts;     /* HOST, required: vertices / triangles of the mesh (may exceed the capacities: nothing is written beyond them) */
	uint64_t *ntris;
} tw_voxel_mesh;
/* Synchronous. vals / outside / tables / verts / indices: host or device. TW_ERR_ARG: NULL arguments, a capacity without its buffer, an empty grid, or
 * 3*nx*ny*nz >= 2^32 (the indices are 32-bit). */
TW_API int tw_voxel_mesh_welded(tw_ctx *ctx, const float *vals, const uint8_t *outside, const tw_voxel_post_params *vp, const uint32_t *edge_table256,
                                const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, const tw_voxel_mesh *out);
/* voxel_manager::create_procedural + voxel_model::build as ONE asynchronous job: the fill (optional), tw_voxel_outside, tw_voxel_remove_unconnected and
 * tw_voxel_triangles enqueued on the context's stream without the host reading anything back in between (the flood fills end on the device). After the
 * completing poll every output is bit-identical to that sequence of synchronous calls on one context: tw_voxel_fill(fill, rdata420) if fill is set, then
 * tw_voxel_outside(zix_xy), tw_voxel_remove_unconnected, tw_voxel_triangles(capacity); nothing of tris beyond min(ntris, capacity) triangles is written.
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it (wait = 0 returns TW_ERR_NOT_READY while it runs), every
 *   other entry point and tw_destroy complete it first. On a shared context it runs beside the other contexts' jobs.
 * - Lifetimes: the struct, *fill, *post, rdata420, host tables and host zix_xy are copied during the launch; vals and device zix_xy / tables are read until the
 *   completing poll; the outputs are written until then.
 * - The launch never waits for the device, except that copies to or from PAGEABLE host vals / outside block it (see "Host output buffers" above).
 * - Errors, nothing enqueued and nothing changed: TW_ERR_ARG for what the four synchronous calls refuse (empty grid, 2^32 voxels or more, the fill's size
 *   limits and gen_mode), a fill grid that differs from post's, vals == NULL without fill, some but not all three tables, tables without ntris,
 *   capacity > 0 without tris, tris in pageable host memory; TW_ERR_STATE where tw_voxel_fill returns it. */
typedef struct tw_voxel_build {
	const tw_voxel_params      *fill;      /* optional: fill vals first, exactly as tw_voxel_fill(fill, rdata420); nx/ny/nz must equal post's */
	const float                *rdata420;  /* optional, sine-mode fill only, as tw_voxel_fill; copied during the launch */
	const tw_voxel_post_params *post;      /* required */
	const uint32_t             *zix_xy;    /* optional, as tw_voxel_outside */
	const uint32_t *edge_table256; const int32_t *tri_table256x16; const uint32_t *edge_to_vals12x2; /* all three, or none = no triangles */
	float    *vals;      /* n floats, host or device: the input field when fill == NULL, else an optional output; after the job = vals after remove_unconnected */
	uint8_t  *outside;   /* optional output: n flag bytes after remove_unconnected, host or device (no alignment requirement) */
	float    *tris;      /* optional: capacity*9 floats, device or page-locked host memory (written by the device through its mapping) */
	uint64_t  capacity;
	uint64_t *ntris;     /* HOST, required with the tables: filled by the completing poll (may exceed capacity) */
	uint64_t *changed;   /* optional HOST: voxels flipped by remove_unconnected, filled by the completing poll */
} tw_voxel_build;
TW_API int tw_voxel_build_launch(tw_ctx *ctx, const tw_voxel_build *b);
/* tw_voxel_build_launch with the welded mesh of tw_voxel_mesh_welded (on the flags and field after remove_unconnected) as well as, or instead of, the
 * soup: mesh == NULL is tw_voxel_build_launch(b). With a mesh, the three tables are required, and b->ntris may be NULL for no soup (b->tris and
 * b->capacity must then be NULL / 0). mesh->verts / indices: device or page-locked host memory, as b->tris; *mesh->nverts / *mesh->ntris are filled by the
 * completing poll, and not on TW_ERR_CANCELED. The mesh struct is copied during the launch. Every rule of tw_voxel_build_launch applies; TW_ERR_ARG also
 * for a mesh without tables or counts, a capacity without its buffer, pageable verts / indices and 3*nx*ny*nz >= 2^32. */
TW_API int tw_voxel_build_launch_ex(tw_ctx *ctx, const tw_voxel_build *b, const tw_voxel_mesh *mesh);
/* Many small grids in ONE asynchronous job - an engine's rock and asteroid models (gen_voxel_rock: atten_to_sphere, centre_seed), at start-up or a frame's
 * worth at a time. After the completing poll grid i's outputs are bit-identical to tw_voxel_build_launch_ex(ctx, &grids[i], &meshes[i]) run alone: vals and
 * outside after remove_unconnected, *changed, the welded mesh's verts / indices up to their capacities and *nverts / *ntris. The job launches the same
 * kernels whatever n is, each over every grid, and floods each grid's remove_unconnected inside one SM's shared memory (DESIGN.md section 4l).
 * - Mesh only: meshes[i] is required for every grid, and there is no triangle soup (grids[i].tris, capacity and ntris must be NULL / 0).
 * - Size limit: nx*ny*nz <= 2^18 (64^3, or 8x8x4096, or 512x512x1) per grid; larger grids belong on tw_voxel_build_launch_ex.
 * - Every grid has its own fill (any gen mode and attenuation) or input vals (host or device), post params and zix_xy; all grids pass the same three
 *   marching-cubes table pointers.
 * - Job rules, lifetimes and memory kinds: those of tw_voxel_build_launch_ex, per grid (the grids and meshes arrays are copied during the launch).
 * - The job has no cancellation point (its grids are small): tw_cancel returns TW_OK and changes nothing, as after a job's last cancellation point.
 * - Errors, nothing enqueued and nothing changed: TW_ERR_ARG for NULL grids or meshes, n == 0, a grid above the limit, tables that differ from grid 0's,
 *   soup fields set, and every refusal of tw_voxel_build_launch_ex for a grid; TW_ERR_STATE where it returns that. tw_last_error names the grid's index.
 *   TW_ERR_CUDA when tw_voxel_batch.cubin, the batch's sm_90a module beside the library, cannot be loaded. */
TW_API int tw_voxel_build_batch_launch(tw_ctx *ctx, const tw_voxel_build *grids, const tw_voxel_mesh *meshes, uint32_t n);

/* ---- resident voxel models: the field kept on the device, edited in place, re-meshed per block ----
 * What voxel_model does with brushes (src/voxels.cpp:2139-2245): it keeps one mesh per block, each with its own vertex cache (create_block, :1077-1108), and an
 * edit re-creates only the blocks it modified. Blocks: with block sizes bx, by >= 1 (in cubes), block (i, j) covers the cubes x in [i*bx, min((i+1)*bx, nx-1)),
 * y in [j*by, min((j+1)*by, ny-1)) and every z; its number is j*nbx + i with nbx = ceil((nx-1)/bx), nby = ceil((ny-1)/by) (y-major, the (y, x, z) cube order of
 * create_block). Each block is welded on its own with the owner rule of tw_voxel_mesh_welded restricted to the block's cubes: an edge's owner is the
 * lowest-index valid cube OF THE BLOCK containing it, vertices are ordered by owner then local edge, indices are local to the block, and triangles whose welded
 * positions give a zero normal are dropped. A vertex on a block face therefore appears once in every block that uses it, as with per-block caches. One block
 * covering the grid (bx >= nx-1, by >= ny-1) gives tw_voxel_mesh_welded's mesh bit for bit. Not confirmed: that this partition is create_block's for more
 * than one block (the reference build pinned here has one block); the caller chooses bx, by to match its own block layout.
 * Outputs of a model job: the meshes of the listed blocks, one after another in ascending block order, in one vertex and one index buffer. */
typedef struct tw_voxel_block_mesh {
	uint32_t block, pad;     /* block number j*nbx + i */
	uint64_t voff, nverts;   /* the block's vertices: verts[voff .. voff + nverts) */
	uint64_t toff, ntris;    /* its triangles: indices[toff .. toff + ntris), local to the block (0 = verts[voff]) */
} tw_voxel_block_mesh;
typedef struct tw_voxel_blocks_out {
	float    *verts;         /* vcapacity*3 floats, device or page-locked host memory (NULL with vcapacity 0) */
	uint64_t  vcapacity;
	uint32_t *indices;       /* tcapacity*3 indices, device or page-locked host memory (NULL with tcapacity 0) */
	uint64_t  tcapacity;
	tw_voxel_block_mesh *blocks; /* HOST, required: room for nbx*nby entries; the listed blocks' ranges, filled by the completing poll */
	uint32_t *nblocks;       /* HOST, required: blocks listed */
	uint64_t *nverts, *ntris;/* HOST, required: totals over the listed blocks (may exceed the capacities: nothing is written beyond them) */
	uint64_t *changed;       /* optional HOST: voxels flipped by remove_unconnected */
} tw_voxel_blocks_out;
/* A box of voxels [x, x+w) x [y, y+h) x [z, z+d) */
typedef struct tw_voxel_box {uint32_t x, y, z, w, h, d;} tw_voxel_box;
typedef struct tw_voxel_model tw_voxel_model;
/* A model of the grid *vp with its marching-cubes tables and zix_xy (optional, as tw_voxel_outside; host or device, copied here). It keeps on the device:
 * the raw field (as the caller gave it or the fill made it), its outside flags, the field and flags after remove_unconnected, and a working copy of those
 * for the edit's comparison: 15 bytes per voxel (about 2 GB at 512^3), plus the blocks' words. While a job runs, the context's scratch also holds the
 * flood's frontiers (8 bytes per voxel with remove_unconnected > 0) and the mesh's per-cube words (4 bytes per cube of the listed blocks' worst case).
 * A model belongs to the context that created it: tw_destroy(ctx) destroys the context's live models before its shared contexts (their handles are invalid
 * after). Its jobs run on that context or, through the _on / read_launch calls, on any context of its family - the parent or a shared context of that
 * parent - so several brush strokes and reads are in flight at once:
 * - A model job is the pending job of the context it was launched on (tw_create_tiles_poll on that context completes it); the launch first completes that
 *   context's earlier job and never waits for a job of another context. Its scratch, pinned staging and kernel launches are the launching context's.
 * - Model state is committed at launch, in launch order. On the device, every model job waits for the model's earlier jobs on any context before it
 *   touches the model, so each job sees exactly the jobs launched before it. tw_voxel_model_read and tw_voxel_model_destroy also wait for them.
 * - Threads: one thread at a time across a model and every context it is used on.
 * Model jobs commit the model's state at launch, so they cannot be cancelled: tw_cancel returns TW_ERR_STATE, as for tile-set jobs.
 * TW_ERR_ARG (nothing allocated): NULL arguments, bx or by == 0, an empty grid or 2^32 voxels or more, 3*(bx+1)*(by+1)*nz >= 2^32 with the block sizes
 * clamped to the grid (the block's indices are 32-bit). */
TW_API int  tw_voxel_model_create(tw_ctx *ctx, const tw_voxel_post_params *vp, const uint32_t *edge_table256, const int32_t *tri_table256x16,
                                  const uint32_t *edge_to_vals12x2, const uint32_t *zix_xy, uint32_t bx, uint32_t by, tw_voxel_model **out);
/* Completes the model's context's pending job and waits for the device work of the model's jobs on every other context, then frees the model. Those jobs
 * stay the pending jobs of their contexts; their polls still complete them (with TW_OK). */
TW_API void tw_voxel_model_destroy(tw_voxel_model *m);
/* The build as the context's asynchronous job: the raw field from fill (as tw_voxel_fill(fill, rdata420)) or from vals (n floats, host or device, read
 * during the job), then tw_voxel_outside, tw_voxel_remove_unconnected, and the mesh of every block, listed in order. The model keeps the results. Rules and
 * lifetimes as tw_voxel_build_launch. TW_ERR_ARG (nothing enqueued): NULL arguments, both or neither of fill and vals, a fill grid that differs, a capacity
 * without its buffer, pageable verts / indices; TW_ERR_STATE where tw_voxel_fill returns it. */
TW_API int  tw_voxel_model_build_launch(tw_voxel_model *m, const tw_voxel_params *fill, const float *rdata420, const float *vals, const tw_voxel_blocks_out *out);
/* tw_voxel_model_build_launch as the pending job of ctx: the model's context, its parent or a shared context of that parent (see the model rules above).
 * tw_voxel_model_build_launch(m, ...) is tw_voxel_model_build_launch_on(m's context, m, ...). TW_ERR_ARG (nothing enqueued) also for a NULL ctx or model and
 * a context of another family or device. */
TW_API int  tw_voxel_model_build_launch_on(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_params *fill, const float *rdata420, const float *vals,
                                           const tw_voxel_blocks_out *out);
/* An edit as the context's asynchronous job, without the host reading anything back before the end:
 *   1. each box's new raw values (values: the boxes' voxels one box after another, each packed in the grid's order - z fastest, then x, then y; host
 *      memory, copied during the launch) go into the raw field; where boxes overlap, the later box's value wins;
 *   2. the raw flags are recomputed inside the boxes (they depend only on the voxel's value, its position and zix_xy);
 *   3. with remove_unconnected > 0, tw_voxel_remove_unconnected runs again on the whole raw field (an edit can disconnect ground far from the box);
 *   4. every block whose cubes read a voxel whose value or flags after step 3 differ from the model's previous ones is marked (a voxel on a block face marks
 *      every block that reads it); the model keeps the new field and flags;
 *   5. the marked blocks - and only those - are meshed, listed in ascending order.
 * After the completing poll the model's field and flags equal tw_voxel_outside then tw_voxel_remove_unconnected on the edited raw field, and the listed blocks'
 * meshes equal a fresh build's. nboxes == 0 (boxes and values may then be NULL) changes nothing and lists no block. TW_ERR_ARG (nothing enqueued): NULL
 * arguments, an empty box or one reaching outside the grid (no clipping), and the output errors of tw_voxel_model_build_launch; TW_ERR_STATE before the
 * model's first build. */
TW_API int  tw_voxel_model_edit_launch(tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values, const tw_voxel_blocks_out *out);
/* The voxels an edit changed, so a copy of the field on the host can follow the model without reading the grid back. A voxel is listed when its value
 * after remove_unconnected (bitwise) or its flags differ between the launch and the completion: exactly the voxels that mark blocks in step 4.
 * After the completing poll *nchanged holds their count, and the first min(capacity, *nchanged) of them are written in ascending index order: the linear
 * index z + (x + y*nx)*nz, and optionally the new value and flags. Patching a copy of tw_voxel_model_read's (vals, outside) taken before the edit with
 * the list gives the read after it, byte for byte, whenever *nchanged <= capacity; otherwise the caller can fall back to a read. */
typedef struct tw_voxel_changes {
	uint32_t *index;     /* capacity entries, device or page-locked host memory (NULL with capacity 0) */
	float    *vals;      /* optional, capacity entries: the field after remove_unconnected at index[i] */
	uint8_t  *outside;   /* optional, capacity entries: its flags at index[i] */
	uint64_t  capacity;
	uint64_t *nchanged;  /* HOST, required: filled by the completing poll; may exceed capacity */
} tw_voxel_changes;
/* tw_voxel_model_edit_launch with the list of changed voxels (ch, optional; copied during the launch). tw_voxel_model_edit_launch(m, ...) is
 * tw_voxel_model_edit_launch_ex(m, ..., NULL). The job keeps one bit per voxel in the context's scratch (n/8 bytes) while it runs. TW_ERR_ARG (nothing
 * enqueued): the errors of tw_voxel_model_edit_launch, a missing nchanged, a capacity without index, vals or outside without index, and pageable buffers.
 * The list's kernels are a module of their own, tw_voxel_changes.cubin, shipped beside the library and loaded by the first edit with a list: TW_ERR_CUDA
 * (nothing enqueued) when it is missing or cannot be loaded. */
TW_API int  tw_voxel_model_edit_launch_ex(tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values, const tw_voxel_blocks_out *out,
                                          const tw_voxel_changes *ch);
/* tw_voxel_model_edit_launch_ex as the pending job of ctx, a context of the model's family (as tw_voxel_model_build_launch_on). tw_voxel_model_edit_launch_ex(m,
 * ...) is tw_voxel_model_edit_launch_on(m's context, m, ...). The change list's bits are in ctx's scratch. */
TW_API int  tw_voxel_model_edit_launch_on(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values,
                                          const tw_voxel_blocks_out *out, const tw_voxel_changes *ch);
/* Synchronous, after completing the pending job of the model's context and waiting for the model's jobs on the other contexts: the raw field, the field
 * after remove_unconnected and its flags (each optional; n elements, host or device). TW_ERR_STATE before the model's first build. */
TW_API int  tw_voxel_model_read(tw_voxel_model *m, float *raw, float *vals, uint8_t *outside);
/* The read as the pending job of ctx, a context of the model's family: what the model holds after every model job launched before this call and none
 * launched after it, on any context. raw (the raw field), vals (the field after remove_unconnected) and outside (its flags) are each optional, in device,
 * page-locked or pageable host memory; pageable ones are filled by the completing poll, the others by the device before it. A pageable destination
 * is staged in the launching context's pinned staging, which grows to the read's size (671 MB for a whole 512^3 read of all three arrays) with a blocking
 * cudaMallocHost the first time and stays allocated for the context's life: read whole grids into page-locked memory (cudaHostRegister the engine's arrays). boxes == NULL (with nboxes 0):
 * the whole grid, n elements in the grid's order; otherwise the boxes' voxels one box after another, each packed as tw_voxel_model_edit_launch's values
 * (z fastest, then x, then y) - one strided copy per box and array, no kernel. The boxes are read during the launch. TW_ERR_ARG (nothing enqueued): a NULL
 * ctx or model, a context of another family or device, NULL boxes with nboxes > 0, an empty box or one reaching outside the grid; TW_ERR_STATE before the
 * model's first build has been launched. */
TW_API int  tw_voxel_model_read_launch(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, float *raw, float *vals, uint8_t *outside);
/* Many small models built, or edited, in ONE asynchronous job - an engine's rock and asteroid models, loaded together or hit by the same frame's brushes.
 * Entry i names a model and the arguments of its single call: after the completing poll each entry gives what tw_voxel_model_build_launch_on(ctx, model,
 * fill, rdata420, vals, out) or tw_voxel_model_edit_launch_on(ctx, model, boxes, nboxes, values, out, ch) would give for that model alone, bit for bit:
 * the raw field, the field and flags after remove_unconnected, the block table, vertices and indices up to their capacities, *nblocks, *nverts, *ntris,
 * *changed, the change list and *nchanged. The job launches the same kernels whatever n is, each over every model, and floods each model's
 * remove_unconnected inside one SM's shared memory, as tw_voxel_build_batch_launch does (DESIGN.md section 4m); each model costs one event wait and one
 * event record, not a launch.
 * - Job and family rules: those of the _on calls. The job is ctx's pending job (tw_create_tiles_poll completes it); every model belongs to ctx's family and
 *   device; the job waits for each model's earlier jobs on any context before it touches that model and orders its later ones. Model state is committed
 *   at launch, so tw_cancel returns TW_ERR_STATE. The entries array, boxes and values are read during the launch.
 * - Size limit: nx*ny*nz <= 2^18 per model; larger models stay on the single calls.
 * - Errors, nothing enqueued and no model changed: TW_ERR_ARG for NULL arrays, n == 0, a NULL model, a model above the limit, a model named twice, a
 *   model of another family or device, and every refusal of the single call for an entry; TW_ERR_STATE for an edit of a model never built, and where
 *   the single call returns it. tw_last_error names the entry's index. TW_ERR_CUDA when tw_voxel_model_batch.cubin or tw_voxel_batch.cubin, the sm_90a
 *   modules beside the library, cannot be loaded. */
typedef struct tw_voxel_model_build {
	tw_voxel_model            *model;     /* required */
	const tw_voxel_params     *fill;      /* exactly one of fill / vals, as tw_voxel_model_build_launch */
	const float               *rdata420;  /* optional, sine fill only */
	const float               *vals;      /* n floats, host or device */
	const tw_voxel_blocks_out *out;       /* required */
} tw_voxel_model_build;
TW_API int tw_voxel_model_build_batch_launch(tw_ctx *ctx, const tw_voxel_model_build *builds, uint32_t n);
typedef struct tw_voxel_model_edit {
	tw_voxel_model            *model;     /* required */
	const tw_voxel_box        *boxes;     /* as tw_voxel_model_edit_launch; nboxes 0 = no change, no block listed */
	uint32_t                   nboxes;
	const float               *values;
	const tw_voxel_blocks_out *out;       /* required */
	const tw_voxel_changes    *ch;        /* optional, as tw_voxel_model_edit_launch_ex */
} tw_voxel_model_edit;
TW_API int tw_voxel_model_edit_batch_launch(tw_ctx *ctx, const tw_voxel_model_edit *edits, uint32_t n);

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
 * When new tiles appear, existing tiles on their far side from the light may need new shadows, because their neighbour toward the light now exists; and when
 * the light moves, every live tile does. A tile set (tw_tile_set_*, below) keeps the live tiles on the device and works out which tiles those are. */
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
 * may be NULL without weights. No tile limit. Not done here: the AO map, which is its own job on the final zvals (tw_hmap_tile_ao_launch, after the tile set
 * section). Errors, nothing enqueued: TW_ERR_STATE without tw_set_heightmap; TW_ERR_ARG for hs NULL
 * or sized unlike the image, edge_mode outside 0..2, shading->ao, weights without p, and every error of tw_create_tiles_launch_shadows. */
TW_API int tw_create_tiles_launch_hmap(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size,
                          float dx, float dy, uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows);

/* ---- mesh shadows of the ground-mode mesh: calc_mesh_shadows (src/visibility.cpp:411-517) on one whole xsize x ysize mesh ----
 * In ground mode the engine calls calc_mesh_shadows(l, light_pos, mesh_height, shadow_mask[l], MESH_X_SIZE, MESH_Y_SIZE) - the whole mesh, no incoming
 * heights - for each light after every regeneration of the mesh and whenever the sun or moon moves (calc_visibility). tw_mesh_shadows is that call, for any
 * xsize x ysize, with the optional incoming and outgoing edges of the tile path:
 *   mesh      xsize*ysize floats (ysize rows of xsize), host or device
 *   sh_in_x   optional, xsize floats: incoming shadow heights along the y edge; sh_in_y optional, ysize floats along the x edge (entries <= TW_MESH_MIN_Z:
 *             no incoming height)
 *   smask     xsize*ysize bytes = 0 / MESH_SHADOW per cell, host or device (device: 4-byte aligned)
 *   sh_out_x  optional, xsize floats; sh_out_y optional, ysize floats: the outgoing heights, MESH_MIN_Z where no shadowed ray wrote one. As in the reference,
 *             only a ray whose clipped end lies on a cell of that edge writes it, and where two rays write one entry the later ray of the sequential order
 *             (2*ysize rays from the x edge by y, then 2*xsize from the y edge by x) wins.
 * sp->zmin / zmax are the globals the line clip reads; lpos.z < zmin shadows every cell. The results equal the reference's function bit for bit (one thread per
 * ray, the same fp32 / double steps). Cell indices are 64-bit: a mesh of more than 2^31 cells is supported. tw_mesh_shadows completes the context's pending
 * job first and blocks until its outputs are written; it is tw_mesh_shadows_launch for one light followed by a waiting poll.
 * Errors (TW_ERR_ARG, nothing enqueued): a NULL mesh, sp or smask, xsize < 2 or ysize < 2, xsize + ysize >= 2^30, a device smask that is not 4-byte aligned. */
TW_API int tw_mesh_shadows(tw_ctx *ctx, const float *mesh, int xsize, int ysize, const tw_shadow_params *sp, const float *sh_in_x, const float *sh_in_y,
                          uint8_t *smask, float *sh_out_x, float *sh_out_y);
/* The same for nlights lights over one mesh as the context's asynchronous job (a relight when the sun or moon moves): every light's results equal its own
 * tw_mesh_shadows call. Each light is a tw_tile_light sized for the mesh: smask xsize*ysize bytes, sh_in_x / sh_out_x xsize floats, sh_in_y / sh_out_y ysize
 * floats. All lights run in one launch of each kernel.
 * - tw_create_tiles_poll / tw_heightgen_2d_poll complete the job (wait = 0 returns TW_ERR_NOT_READY while it runs); every other entry point and tw_destroy
 *   complete it first. On a shared context it runs beside the other contexts' jobs. tw_cancel stops its rays at their cancellation point (the kernel's
 *   entry); the poll then returns TW_ERR_CANCELED and the outputs are unspecified.
 * - The job, the lights array and HOST mesh and sh_in rows are copied during the launch; a device mesh and device sh_in rows are read until the completing
 *   poll. Outputs in device or page-locked memory are written by the device; pageable ones are filled by the completing poll. Every buffer is reserved
 *   before anything is enqueued, and with device or page-locked outputs the launch never waits for the device, except when the context's scratch or staging
 *   first has to grow.
 * - Errors (TW_ERR_ARG, nothing enqueued): those of tw_mesh_shadows for each light, and nlights == 0 or NULL lights. */
typedef struct tw_mesh_shadows_job {
	const float         *mesh;          /* required: xsize*ysize floats, host or device */
	int                  xsize, ysize;  /* MESH_X_SIZE, MESH_Y_SIZE: >= 2 each */
	uint32_t             nlights;       /* >= 1 */
	const tw_tile_light *lights;
} tw_mesh_shadows_job;
TW_API int tw_mesh_shadows_launch(tw_ctx *ctx, const tw_mesh_shadows_job *job);
/* tw_gen_mesh_launch plus one mesh shadow pass per light on the job's final mesh (after glaciation and erosion): mesh, z values and shadows, all on the device
 * in one job. Each light's results equal tw_mesh_shadows_launch on that mesh with the light's sp, except that sp->zmin / zmax are ignored and replaced by
 * the zmin / zmax the job leaves - those tw_gen_mesh_info reports, read on the device. Every other sp field is the caller's (xy_sum_size = mesh_x_size +
 * mesh_y_size in the reference). The contract is that the engine's calc_visibility reads the zmin / zmax gen_mesh leaves; an engine that changes them
 * first uses tw_mesh_shadows_launch with explicit params instead. Lights are sized for the mesh as in tw_mesh_shadows_launch and follow its buffer rules;
 * the mesh, info and tw_last_erosion_steps() are those of tw_gen_mesh_launch, which is tw_gen_mesh_launch_shadows(ctx, job, 0, NULL). Errors (TW_ERR_ARG,
 * nothing enqueued): those of tw_gen_mesh_launch, nlights > 0 with NULL lights, and with lights those of tw_mesh_shadows for each light (a mesh size
 * below 2 x 2, a light without smask, a misaligned device smask). */
TW_API int tw_gen_mesh_launch_shadows(tw_ctx *ctx, const tw_gen_mesh_job *job, uint32_t nlights, const tw_tile_light *lights);

/* ---- tile sets: the live tiles kept on the device, relit with cached, chained mesh shadows ----
 * What tile_draw_t::update does for every live tile when the light moves, and for the existing tiles behind new ones (src/tiled_mesh.cpp:664-692): a tile set
 * holds the zvals of the resident tiles in device memory the set owns, keyed by their grid coordinates (x1/size, y1/size), and per light slot the mesh shadows
 * (smask, sh_out_x, sh_out_y) each tile was last computed with. tw_tile_set_shadows_launch enqueues a relight as the context's asynchronous job:
 *   every output equals tw_tile_shadows_batch_ex on ALL tiles resident at launch time, with no caller rows, bit for bit;
 * the cache only skips tiles whose result cannot have changed. With sx = (lpos.x < 0 ? -1 : 1), sy = (lpos.y < 0 ? -1 : 1), the tiles DOWNSTREAM of (tx, ty)
 * are the resident (tx, ty - sy) and (tx - sx, ty), transitively (the walk stops at a tile that is not resident): exactly the tiles whose incoming rows come
 * from it. A light slot keeps the tw_shadow_params it was last computed with and one valid bit per resident tile:
 *   - a request whose params differ byte for byte from the slot's invalidates the whole slot;
 *   - tw_tile_set_put of a tile invalidates it and its downstream closure in every slot; tw_tile_set_remove invalidates its downstream closure;
 *   - a relight recomputes the invalid requested tiles plus their invalid upstream closure, reading the cached sh_out of valid resident neighbours as
 *     incoming rows and "no incoming height" where a neighbour is not resident.
 * The cache promises equality with the full recompute, not the fewest recomputed tiles: sh_out is written only for light from +x / +y (DESIGN.md §4b), so a
 * closure can recompute tiles whose inputs did not change.
 * A set belongs to its context (a shared context is fine) and follows the context's rules: put, remove, destroy and a new launch complete the context's
 * pending job first, and tw_create_tiles_poll completes the relight. tw_destroy(ctx) destroys the context's live sets first; their handles are invalid after. */
typedef struct tw_tile_set tw_tile_set;
/* zvsize >= 2 and nlights >= 1 (the number of light slots), else TW_ERR_ARG. */
TW_API int  tw_tile_set_create(tw_ctx *ctx, uint32_t zvsize, uint32_t nlights, tw_tile_set **out);
TW_API void tw_tile_set_destroy(tw_tile_set *set);
/* Inserts or replaces n tiles: tile_xy = n (x1/size, y1/size) pairs, zvals = n*zvsize^2 floats, host or device (a tile job's device zvals cost one copy on the
 * device). Returns once zvals has been read. TW_ERR_ARG (nothing changes) for a tile named twice or n == 0. */
TW_API int  tw_tile_set_put(tw_tile_set *set, const int32_t *tile_xy, uint32_t n, const float *zvals);
/* Removes n resident tiles. TW_ERR_ARG (nothing changes) for a tile that is not resident or is named twice. */
TW_API int  tw_tile_set_remove(tw_tile_set *set, const int32_t *tile_xy, uint32_t n);
/* Host only: the resident tiles a relight of every resident tile with these nlights lights (light l = slot l) would recompute for at least one light - the
 * shadow textures the engine has to refresh - in (x, y) order. Writes min(capacity, count) pairs to tile_xy_out (may be NULL with capacity 0); *nstale =
 * count, which may exceed capacity. */
TW_API int  tw_tile_set_stale(tw_tile_set *set, const tw_shadow_params *sps, uint32_t nlights, int32_t *tile_xy_out, uint32_t capacity, uint32_t *nstale);
/* One light of a relight request: all arrays in request order, host or device; smask and sh_out_* must stay valid until the completing poll (pinned host or
 * device memory for a launch that does not block). */
typedef struct tw_tile_set_light {
	tw_shadow_params sp;
	uint8_t *smask;                    /* required: n*zvsize^2 bytes (device: 4-byte aligned) */
	float   *sh_out_x, *sh_out_y;      /* optional: n*zvsize floats each */
} tw_tile_set_light;
typedef struct tw_tile_set_request {
	const int32_t           *tile_xy;     /* required: the n tiles to output, each resident and named once */
	uint32_t                 n;
	uint32_t                 nlights;     /* 1 .. the set's nlights; light l uses slot l */
	const tw_tile_set_light *lights;
	uint8_t                 *recomputed;  /* optional HOST, n bytes, filled before the launch returns: 1 = this job computes tile i for at least one light */
} tw_tile_set_request;
/* Enqueues the relight and returns; tw_create_tiles_poll completes it. The request, its lights array and tile_xy are read during the launch. Errors return
 * TW_ERR_ARG before anything is enqueued or cached state changes. */
TW_API int  tw_tile_set_shadows_launch(tw_tile_set *set, const tw_tile_set_request *req);
/* A frame's new tiles created straight into a set and relit in the same asynchronous job - tile_draw_t::update's per-frame step in one launch:
 *   tw_tile_set_create_tiles_launch(ctx, set, origins_xy, ntiles, ..., out, shading, frame) followed by its completing tw_create_tiles_poll(ctx) gives, bit for
 *   bit, every output and the set state that this sequence gives on a set in the same state, on one context:
 *     tw_tile_set_remove(frame->remove_xy) when nremove > 0; tw_create_tiles_launch_ex (frame->hs == NULL) or tw_create_tiles_launch_hmap(frame->hs) with the
 *     same arguments and zvsize = the set's; a completing poll; tw_tile_set_put(frame->tile_xy, the job's zvals); tw_tile_set_shadows_launch(frame->relight)
 *     when relight != NULL, and its poll.
 *   That covers the job's outputs (zvals, mm, bounds, normals, min_normal_z, AO, weights, has_any_grass), the relight's (smask, sh_out_*, recomputed),
 *   tw_last_erosion_steps() and what tw_tile_set_stale and later relights see. In GPU gen modes with AO the put zvals are the AO flow's, as documented for the job.
 * Arguments: ctx is the set's context or any context of its family (the parent of a shared context, or a shared context of that parent): frames launched on
 * several shared contexts are in flight at once. out and shading are optional, and out->zvals may be NULL (the zvals then live only in the set). The relight
 * may name tiles this launch puts, not tiles it removes; its recomputed flags are filled before the launch returns.
 * Ordering: the host-side set state (residency, slots, valid bits, light params) is committed at launch, in launch order. On the device, generation and erosion
 * never wait for other frames; only the tail that touches the set's slabs (the zvals scatter into the slabs and the relight) waits on the set's event, the last
 * device work on the slabs of any context, and records it again. tw_tile_set_put, tw_tile_set_shadows_launch and tw_tile_set_destroy wait on that event as well.
 * Blocking: the launch returns without waiting for the device, except when the set needs larger slabs: it then first waits for every frame in flight on the
 * set (they hold the old slab pointers) and copies the slabs. Size the set early (a first put or frame with every tile) to avoid it.
 * Errors: the return code tells which state the set is in.
 *   TW_ERR_ARG and TW_ERR_STATE: the set is unchanged. TW_ERR_ARG comes before anything is enqueued for every error of the job, of put, remove and the
 *     relight request, a tile both removed and put, a tile_xy that names a tile twice, a ctx of another family or device, and hs together with shading->ao;
 *     TW_ERR_STATE for the job's missing tables or heightmap image.
 *   TW_ERR_CUDA (whether the launch failed, or completing the context's earlier job reported its failure): the set is left with the removes done, none of
 *     tile_xy resident (a re-put tile is removed too) and every light slot invalid, so later relights recompute what is then resident and still equal the
 *     full recompute. A failure after the set's slabs may have been written is always reported as TW_ERR_CUDA. */
typedef struct tw_tile_set_frame {
	const int32_t              *remove_xy;  /* optional: nremove resident tiles removed first, as tw_tile_set_remove */
	uint32_t                    nremove;
	const int32_t              *tile_xy;    /* required: (x1/size, y1/size) of each new tile, in origins_xy order */
	const tw_hmap_sampler      *hs;         /* NULL: the height function p; else the context's heightmap image, as tw_create_tiles_launch_hmap */
	const tw_tile_set_request  *relight;    /* optional: relight after the put, as tw_tile_set_shadows_launch */
} tw_tile_set_frame;
TW_API int  tw_tile_set_create_tiles_launch(tw_ctx *ctx, tw_tile_set *set, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size,
                          float dx, float dy, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_set_frame *frame);
/* Host only, changes nothing: what tw_tile_set_stale would return after tw_tile_set_remove(remove_xy) (nremove > 0) and tw_tile_set_put(put_xy) (nput > 0) - the
 * tiles to name in a frame's relight request. TW_ERR_ARG for what stale, remove and put refuse, and a tile both removed and put. */
TW_API int  tw_tile_set_stale_after(tw_tile_set *set, const tw_shadow_params *sps, uint32_t nlights, const int32_t *remove_xy, uint32_t nremove,
                          const int32_t *put_xy, uint32_t nput, int32_t *tile_xy_out, uint32_t capacity, uint32_t *nstale);

/* ---- the AO map of heightmap-texture tiles: tile_t::calc_mesh_ao_lighting (src/tiled_mesh.cpp:586-662) in the heightmap-texture mode ----
 * For tile t with origin (x1, y1), zvsize = stride + 1 and final zvals zvals_t (sampled, then eroded when the engine erodes heightmap tiles), ao_t is
 *   czv_t = tw_heightmap_sample_tiles(image, hs, origin (x1 - 36, y1 - 36), zvsize' = stride + 72)   (get_clamped_height over the window)
 *   ao_t  = tile_ao(zvals_t, czv_t, zvsize, half_dxy) with use_ao_zvals = 0                           (tw_tile_ao_batch's kernel, CPU-gen-mode flow)
 * bit for bit: the rays read the tile's own final zvals inside the tile and the image outside it, and start at the final zval. This library defines that AO;
 * it does not pin the reference's heightmap branch (its test harness cannot reach the heightmap branch of create_zvals, see oracle/refbuild/ref_tiled_harness.inc).
 * - The job is the context's pending job: tw_create_tiles_poll / tw_heightgen_2d_poll complete it, and tw_hmap_tile_ao is the launch followed by a poll with
 *   wait = 1. tw_cancel returns TW_ERR_STATE: the job has no cancellation point.
 * - Image: the job sees the image as it was when its launch returned (every tw_update_heightmap made before it, none after it), and a later edit waits on
 *   the device for its kernel only. A shared context reads its parent's image; while the root's erosion of the image or a set_image job is pending there is
 *   no image (TW_ERR_STATE).
 * - Heights: zvals (ntiles*zvsize^2 floats, device, page-locked or pageable host memory, copied during the launch when on the host), or, with zvals == NULL,
 *   the resident tiles of `set` named by tile_xy. The job then waits on the device for the set's earlier work (a frame launched just before on any context
 *   of the family) before it reads the slabs, and orders the set's later work after its reads, as a relight does; ctx may be any context of the set's family.
 * - ao: ntiles*stride^2 bytes, tile t's at t*stride^2, device or host memory (pageable host memory receives it in the completing poll); it must stay
 *   valid until then.
 * - Errors, nothing enqueued: TW_ERR_ARG for a NULL ctx or job, NULL hs, edge_mode outside 0..2, zvsize < 2, both or neither of zvals and set, NULL ao, NULL
 *   origins_xy (or, with set, tile_xy) with ntiles > 0, hs sized unlike the image, and with set: a context of another family or device, zvsize unlike the
 *   set's, a tile of tile_xy that is not resident or is named twice; TW_ERR_STATE without an image. ntiles == 0 is TW_OK and does nothing. */
typedef struct tw_hmap_ao_job {
	const tw_hmap_sampler *hs;       /* sized like the context's image */
	const int32_t *origins_xy;       /* ntiles (x1, y1) pairs, as tw_create_tiles_launch_hmap */
	uint32_t ntiles, zvsize;
	float half_dxy;                  /* HALF_DXY */
	const float *zvals;              /* ntiles*zvsize^2, host or device; NULL => read from set */
	tw_tile_set *set;                /* with zvals == NULL: the resident tiles named by tile_xy */
	const int32_t *tile_xy;          /* ntiles (x1/size, y1/size) keys, required with set */
	uint8_t *ao;                     /* ntiles*stride^2 bytes, host or device */
} tw_hmap_ao_job;
TW_API int tw_hmap_tile_ao_launch(tw_ctx *ctx, const tw_hmap_ao_job *job);  /* the context's pending job */
TW_API int tw_hmap_tile_ao(tw_ctx *ctx, const tw_hmap_ao_job *job);         /* launch + waiting poll */

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
