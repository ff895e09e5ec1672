// tw_internal.h - context object and helpers shared by the CUDA translation units of lib3dworld_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>
#include "../../include/tw3d.h"

// The one asynchronous job a context may have in flight (tw_heightgen_2d_launch or tw_create_tiles_launch). `done` is recorded on ctx->stream
// after everything the job enqueued (the tile pipeline's other streams are joined into ctx->stream first); the small per-tile results are staged
// in ctx->h_pinned at the offsets below and unpacked into the caller's host arrays by the poll that reports completion.
struct tw_async_state {
	bool pending = false;
	bool tiles = false;             // the pending job is a tile job (else a 2-D grid)
	cudaEvent_t done = nullptr;
	float *host_out = nullptr;      // user host buffer (nullptr => result stays on device)
	tw_minmax *host_mm = nullptr;
	uint32_t n_mm = 0;
	// tile job: where the staged results go and what the bounds combination needs
	tw_tile_bounds *host_bounds = nullptr;
	float *host_min_nz = nullptr;
	uint8_t *host_flags = nullptr;  // has_any_grass
	bool steps = false;             // an erosion step counter is staged
	float dx = 0.0f, dy = 0.0f;
	uint32_t size = 0;
	size_t off_steps = 0, off_mm = 0, off_sub = 0, off_min_nz = 0, off_flags = 0; // byte offsets into ctx->h_pinned
};

struct tw_ctx {
	int device = 0;
	unsigned num_sms = 1;   // streaming multiprocessors of `device`: grid sizes and wave counts scale with it
	cudaStream_t stream = nullptr;
	cudaStream_t aux_stream[3] = {nullptr, nullptr, nullptr}; // erosion side of the fused tile pipeline (tw_create_zvals_batch): [0] the heaviest chunk, [1]/[2] alternate
	cudaStream_t heavy_stream[4] = {nullptr, nullptr, nullptr, nullptr}; // fork/join streams of the erosion's latency-mode launch (lane 0: ctx->stream, 1..3: aux_stream[0..2])
	cudaEvent_t  ev_fork[4] = {nullptr, nullptr, nullptr, nullptr}, ev_join[4] = {nullptr, nullptr, nullptr, nullptr};
	const unsigned *tile_perm = nullptr; // set around twi_heightgen by the tile pipeline: output slot of each generated tile
	char err[512] = {0};
	uint64_t launches = 0;
	uint64_t last_erosion_steps = 0;
	// uploaded tables
	float  *d_sin_table = nullptr;     // [65536]  sin_table (src/sinf.h:11)
	void   *d_glm3_lut = nullptr;      // float4[2*291]: simplex(vec3) / perlin(vec3) normalised gradient + permute tables (voxel density)
	void   *d_simplex_lut = nullptr;   // float4 simplex gradient table, simplex hash table, Perlin gradient table (tw_noise2.cuh, tw_heightgen.cu), built on first use
	float2 *d_dir_table = nullptr;     // [1000000] (cosf(a_k), sinf(a_k)), a_k = float(1e-6*k)*TWO_PI, host libm (src/erosion.cpp:85-86)
	float  *d_sine_params = nullptr;   // [450] sinTable
	float   h_sine_params[TW_F_TABLE_SIZE*5];
	bool have_sin = false, have_sine_params = false;
	// growable device scratch
	void  *d_scratch[3] = {nullptr, nullptr, nullptr}; // 0: generic output staging, 1: tables / padded heightmaps, 2: small (minmax, counters, origins)
	size_t scratch_bytes[3] = {0, 0, 0};
	// tw_set_heightmap's 16-bit image (its own allocation: tw_reserve may re-allocate the scratch slots while a tile job still reads the image)
	uint8_t *d_hmap = nullptr;
	int hmap_w = 0, hmap_h = 0;
	// pinned host staging for small results
	void  *h_pinned = nullptr;
	size_t pinned_bytes = 0;
	tw_async_state async;
	void *dist = nullptr;        // tw_dist_state (tw_multi.cu): NCCL communicator of the one-process-per-GPU mode
	unsigned skip_rect[4] = {0, 0, 0, 0}; // x0, y0, w, h of the cells twi_heightgen's paired noise kernels leave unwritten (set around AO context generation only)
};

int  tw_set_error(tw_ctx *ctx, int status, const char *fmt, ...);
int  twi_finish_pending(tw_ctx *ctx);                           // completes the context's pending asynchronous job (if any) before other work reuses its scratch
int  tw_reserve(tw_ctx *ctx, int slot, size_t bytes);           // grow d_scratch[slot]; returns TW_OK / TW_ERR_CUDA
int  tw_reserve_pinned(tw_ctx *ctx, size_t bytes);
bool tw_is_device_ptr(const void *p);

#define TW_CUDA(ctx, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	return tw_set_error((ctx), TW_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } } while (0)
#define TW_LAUNCH_CHECK(ctx) do { (ctx)->launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) { \
	return tw_set_error((ctx), TW_ERR_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); } } while (0)

// ---- constants shared by host and device code (src/3DWorld.h:43,129; src/sinf.h:8-9) ----
#define TW_TSIZE 32768
constexpr float TW_PI_F     = 3.141592654f;
constexpr float TW_TWO_PI_F = (float)(2.0*TW_PI_F);
constexpr float TW_SSCALE   = (float)TW_TSIZE/TW_TWO_PI_F;

// float -> int conversion with the semantics the reference build gets from x86 cvttss2si: truncation toward zero, and the
// "integer indefinite" value INT_MIN for NaN and for anything outside int range (CUDA's cvt would give 0 / saturate instead).
// This matters: a droplet whose state went NaN (SURVEY.md section 7 "NaN hazard") terminates because (int)floor(NaN) == INT_MIN
// makes it "outside" (src/erosion.cpp:93,101), and SINF's table index (src/sinf.h:11) wraps the same way for huge arguments.
__device__ __forceinline__ int tw_x86_f2i(float f) {
	return (f >= -2147483648.0f && f < 2147483648.0f) ? __float2int_rz(f) : (int)0x80000000;
}

// order-preserving float <-> uint encoding for atomicMin/atomicMax reductions
__host__ __device__ inline unsigned tw_f2ord(float f) {
#ifdef __CUDA_ARCH__
	unsigned u = __float_as_uint(f);
#else
	unsigned u; memcpy(&u, &f, 4);
#endif
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ inline float tw_ord2f(unsigned u) {
	u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
	return __uint_as_float(u);
#else
	float f; memcpy(&f, &u, 4); return f;
#endif
}

// entry points implemented in the individual .cu files (called from tw_api.cu)
int twi_heightgen(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin,
                  const float2 *d_tile_origins, uint32_t ntiles, float *d_out, unsigned *d_mm_ord, float *h_out_bands = nullptr);
// h_stage (optional): pinned host staging of twi_sine_tiles_stage_bytes(ntiles) bytes that stays untouched until the enqueued work is done; without it
// the call synchronises ctx->stream after the uploads (its host-side index tables are locals)
int twi_heightgen_sine_tiles(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, const float2 *h_org, uint32_t ntiles,
                             float *d_out, unsigned *d_mm_ord, void *h_stage = nullptr);
size_t twi_sine_tiles_stage_bytes(uint32_t ntiles);
// The same in three steps, for a pipeline that generates the batch chunk by chunk. twi_sine_tiles_plan (host only) finds the batch's distinct tile columns /
// rows and returns the device memory the tables need; twi_sine_tiles_setup uploads the planned batch (staged in h_stage as above, or synchronously read from
// h_org and b until the work is done) and builds the tables in d_mem (nullptr: scratch slot 1); twi_sine_tiles_grid generates batch tiles [t0, t0 + nt) -
// or d_perm[t0 .. t0 + nt) - into consecutive slots of d_out. Setup and grid enqueue on ctx->stream.
#include <vector>
struct twi_sine_batch {
	std::vector<float> uorg; std::vector<uint2> tabs; unsigned nux = 0, nuy = 0; // plan: distinct x then y origins, per-tile table indices
	tw_grid2d g; tw_height_params p; int enable_glaciate, min_start_sin;
	float *Xt, *Yt; const uint2 *d_tabs; const float2 *d_torg;
	size_t xstride, ystride; unsigned xpitch, ypitch;
};
size_t twi_sine_tiles_plan(const tw_grid2d *g, const float2 *h_org, uint32_t ntiles, twi_sine_batch *b);
int twi_sine_tiles_setup(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, const float2 *h_org, uint32_t ntiles,
                         void *d_mem, void *h_stage, twi_sine_batch *b);
int twi_sine_tiles_grid(tw_ctx *ctx, const twi_sine_batch *b, uint32_t t0, uint32_t nt, const unsigned *d_perm, float *d_out, unsigned *d_mm_ord);
int twi_ensure_aux_streams(tw_ctx *ctx);
int twi_erode(tw_ctx *ctx, float *d_maps, uint32_t ntiles, int xsize, int ysize, const float *d_min_zvals, float min_zval_all,
              uint32_t num_iters, const tw_erosion_params *p);
// st: nullptr = ctx->stream; d_perm (optional): launch tile z handles tile d_perm[z] of d_origins and d_out; cstep: tile cell (i, j) samples (x1 + i*cstep, y1 + j*cstep)
int twi_hmap_sample_tiles(tw_ctx *ctx, const uint8_t *d_data16, const tw_hmap_sampler *hs, const void *d_origins, uint32_t ntiles, uint32_t zvsize, float *d_out,
                          cudaStream_t st = nullptr, const unsigned *d_perm = nullptr, uint32_t cstep = 1);
// d_perm (optional): launch tile z handles tile d_perm[z] of d_zvals and of the outputs (the tile pipeline's schedule order)
int twi_tile_normals(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, uint32_t ntiles, uint32_t zvsize, float dx_val, float dy_val, unsigned char *d_rgba, unsigned *d_min_nz_ord,
                     const unsigned *d_perm = nullptr);
int twi_fill_u32(tw_ctx *ctx, cudaStream_t st, unsigned *d_vals, size_t n, unsigned value);
int twi_tile_ao(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, const float *d_czv, uint32_t ntiles, uint32_t zvsize, float half_dxy, bool ctx_inside, unsigned char *d_ao,
                const unsigned *d_perm = nullptr);   // d_czv: context grids in launch order
int twi_tile_cut(tw_ctx *ctx, cudaStream_t st, const float *d_czv, uint32_t ntiles, uint32_t zvsize, float *d_zvals, const unsigned *d_perm = nullptr);
int twi_tile_weights(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, const float *d_rand, uint32_t ntiles, uint32_t zvsize, const float *d_tile_params, const tw_weight_params *W,
                     uint8_t *d_out, uint8_t *d_flags, const unsigned *d_perm = nullptr); // d_rand: jitter grids in launch order
// Mesh shadows of a batch of tiles (tw_shadows.cu) in two steps, so the tile job can run them after its chunks. twi_shadow_plan_make (host only) finds each
// tile's neighbours toward the light, the dependency waves and the light direction; a tile whose neighbour is not in the batch reads the caller's row
// ntiles + t of the edge buffers instead when has_in_x / has_in_y say one exists. It returns false when tile_xy holds a tile twice (the plan is then the one
// tw_tile_shadows_batch has always made: the later entry owns the position). twi_shadow_enqueue runs one light on `st` into buffers reserved by the caller:
//   d_m     ntiles*n^2 bytes, 4-byte aligned        d_keys  2*ntiles*n 64-bit keys
//   d_ox    ntiles*n floats (outputs), then ntiles*n caller rows when has_in_x (resp. d_oy, has_in_y)
//   d_plan  twi_shadow_plan_ints(ntiles) ints of device memory holding twi_shadow_plan_pack's output
// use_graph: more than 32 waves go to the stream as one CUDA graph (for a caller that must not block behind a full launch queue)
struct twi_shadow_dev {
	float xs, ys, dx, dy, dxi, dyi, zmin, zmax; // X/Y_SCENE_SIZE, DX/DY_VAL, their inverses, clip z range
	float dirx, diry, dirz, dist;
	int dim; double dir_ratio;
};
struct twi_shadow_plan {
	std::vector<int> nbx, nby, wave_tiles, wave_start; // wave l = wave_tiles[wave_start[l] .. wave_start[l + 1])
	twi_shadow_dev S;
	bool trace = false, all_shadowed = false;
};
bool   twi_shadow_plan_make(const int32_t *tile_xy, uint32_t ntiles, const tw_shadow_params *sp, bool has_in_x, bool has_in_y, twi_shadow_plan *P);
size_t twi_shadow_plan_ints(uint32_t ntiles);
void   twi_shadow_plan_pack(const twi_shadow_plan &P, int *out); // [wave_tiles | nbx | nby]
int    twi_shadow_enqueue(tw_ctx *ctx, cudaStream_t st, const twi_shadow_plan &P, const float *d_z, uint32_t ntiles, uint32_t n, unsigned char *d_m,
                          unsigned long long *d_keys, float *d_ox, float *d_oy, const int *d_plan, bool use_graph);
int twi_eval_points(tw_ctx *ctx, const float *d_xy, size_t n, const tw_height_params *p, const tw_point_query *q, float *d_out);
int twi_erode_parallel(tw_ctx *ctx, float *d_map, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p, uint32_t num_threads);
size_t   twi_erode_scratch_bytes(const tw_ctx *ctx, uint32_t chunk, int xsize, int ysize);
uint32_t twi_erode_chunk_for(size_t budget, uint32_t ntiles, int xsize, int ysize);
int twi_erode_enqueue(tw_ctx *ctx, cudaStream_t st, int lane, void *scratch, uint32_t capacity, float *maps, uint32_t nt, int xsize, int ysize,
                      const float *d_min_zvals, float min_zval_all, uint32_t num_iters, const tw_erosion_params *p, unsigned long long *d_steps,
                      const unsigned *d_perm = nullptr);
// coherent batched erosion (tw_erode_sweeps*): per-band building blocks, all enqueued on ctx->stream
int twi_sweep_pad(tw_ctx *ctx, const float *U, int u0, int xsize, int ysize, int E0, int rows, float *P);
int twi_sweep_view();
int twi_sweep_walk(tw_ctx *ctx, float *P, long long *D, int xsize, int ysize, int E0, int own0, int own1, int halo_rule, unsigned it0, unsigned it1,
                   const tw_erosion_params *p, unsigned long long *d_steps);
int twi_sweep_add(tw_ctx *ctx, long long *D, const long long *R, size_t n);
int twi_sweep_apply(tw_ctx *ctx, float *P, long long *D, size_t n);
int twi_sweep_unpad(tw_ctx *ctx, const float *P, int E0, int xsize, int y0, int y1, float min_zval, float *out);
int twi_tile_bounds(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, void *d_sub, const unsigned *d_perm = nullptr);
int twi_glaciate_mesh(tw_ctx *ctx, float *d_mesh, int nx, int ny, int xoff2, int yoff2, int MX, int MY, const tw_height_params *p, unsigned *d_mm);
int twi_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *d_out);
int twi_from_floats_u16(tw_ctx *ctx, const float *d_vals, size_t n, float val_mult, float val_add, uint8_t *d_out, unsigned *d_bad);
int twi_to_floats_u16(tw_ctx *ctx, const uint8_t *d_data, size_t n, float val_mult, float val_add, float *d_vals);
int twi_minmax(tw_ctx *ctx, const float *d_vals, size_t n, unsigned *d_mm_ord);
int twi_minmax_tiles(tw_ctx *ctx, cudaStream_t st, const float *d_vals, size_t tile_elems, uint32_t nt, unsigned *d_mm_ord, const unsigned *d_perm = nullptr);
int twi_coarse_work(tw_ctx *ctx, const float *d_coarse, unsigned cells, uint32_t nt, float level, unsigned *d_work);
int twi_gather_origins(tw_ctx *ctx, const void *d_org, const unsigned *d_order, uint32_t nt, void *d_out);
int twi_order_by_work(tw_ctx *ctx, cudaStream_t st, const unsigned *d_work, uint32_t nt, unsigned max_work, unsigned *d_hist256, unsigned *d_order);
int twi_init_minmax(tw_ctx *ctx, unsigned *d_mm_ord, uint32_t n);
