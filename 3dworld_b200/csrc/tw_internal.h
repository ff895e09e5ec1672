// tw_internal.h - context object and helpers shared by the CUDA translation units of lib3dworld_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>
#include <functional>
#include <utility>
#include <vector>
#include "../../include/tw3d.h"

// The one asynchronous job a context may have in flight. Its launch supplies `complete`, which unpacks what that launch staged in ctx->h_pinned into the
// caller's outputs and returns the status of the completed work; it captures by value the destinations and the pinned regions it reads. The poll that sees
// the job done calls it, unless a cancellation point acted. A job is pending while it has a completion (a relight, which stages nothing, has an empty one).
// Only twi_launch_job makes a job pending and only poll_job (tw_api.cu) takes it back.
struct twi_job {
	std::function<int(tw_ctx *)> complete;
	bool cancellable = false;             // tw_cancel may stop it (set by the launch; a job that touches a tile set or a voxel model is not)
	bool reads_image = false;             // it reads or writes the family's heightmap image: its work waits for the edits made before its launch (tw_update_heightmap)
	unsigned seq = 0;                     // the context's number of the job (twi_launch_job), the one tw_cancel names
};

// One edit's staging (tw_update_heightmap): pinned host memory and device memory of `bytes` each, holding [row table | packed texels], reused once `ev` (recorded
// after the edit's scatter kernel) has completed
struct twi_img_stage {void *h = nullptr; void *d = nullptr; size_t bytes = 0; cudaEvent_t ev = nullptr;};
// one row of an edit: w texels from texel src of the staging's packed texels to texel dst of the image (src and dst have the same phase modulo 8 texels)
struct twi_hmap_row {unsigned long long dst, src; unsigned w, pad;};

struct tw_async_state {
	twi_job job;
	cudaEvent_t done = nullptr;           // recorded on ctx->stream after everything the pending job enqueued
	// a job with reads_image: recorded on ctx->stream once the job no longer reads or writes the image, which tw_update_heightmap waits on. A heightmap tile
	// job records it after its last sampling (image_free_set), so its erosion, shadows and tail overlap a later edit; any other image job records it with done.
	cudaEvent_t image_free = nullptr;
	bool image_free_set = false;
};

// The device words behind tw_cancel, one set per context at a fixed address. `job` is the number of the job that runs on ctx->stream (0 between jobs:
// twi_launch_job writes it at the job's start and clears it at its end), `cancel` the number of the last job tw_cancel named. A cancellation point acts
// only when the two are equal and not 0, so a cancel that lands after its job has ended can never stop the next one, nor a synchronous call. A point that
// acts sets `stopped`, which the job's end copies to twi_job_host::stopped for the completing poll. Read as one 64-bit word (twi_job_words_load).
struct twi_job_words {unsigned cancel, job, stopped, pad;};
// Pinned host side: the source of the job-start copy {job, stopped = 0}, the source of tw_cancel's copy, and the staged `stopped`
struct twi_job_host {unsigned start[2]; unsigned cancel; unsigned stopped;};
#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long twi_job_words_load(const twi_job_words *w) { // past L1: the words change while the kernel runs
	unsigned long long v;
	asm volatile("ld.relaxed.gpu.u64 %0, [%1];" : "=l"(v) : "l"(w));
	return v;
}
__device__ __forceinline__ bool twi_job_words_hit(unsigned long long v) {return (unsigned)(v >> 32) != 0u && (unsigned)(v >> 32) == (unsigned)v;}
__device__ __forceinline__ bool twi_cancelled(const twi_job_words *w) {return twi_job_words_hit(twi_job_words_load(w));}
__device__ __forceinline__ void twi_mark_stopped(twi_job_words *w) {*(volatile unsigned *)&w->stopped = 1u;}
#endif

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
	// tw_update_heightmap (root contexts): the image's stream (never ctx->stream, so an edit queued behind one context's long job holds up no other work on
	// that context), the event recorded after the last edit, which image jobs wait on, and the edits' staging buffers
	cudaStream_t img_stream = nullptr;
	cudaEvent_t img_ev = nullptr;
	std::vector<twi_img_stage> img_stage;
	// pinned host staging for small results
	void  *h_pinned = nullptr;
	size_t pinned_bytes = 0;
	tw_async_state async;
	// tw_cancel: the words the cancellation points read, their pinned host side, the stream of tw_cancel's copy (never ctx->stream), the last job number
	twi_job_words *d_job_words = nullptr;
	twi_job_host *h_job = nullptr;
	cudaStream_t cancel_stream = nullptr;
	unsigned job_seq = 0;
	bool cancel_sent = false;               // a tw_cancel copy may still be in flight: the next job start waits for it
	bool in_job = false;                    // set while twi_launch_job enqueues: the droplet walks it enqueues check the words, a synchronous call's do not
	cudaGraphExec_t spec_graph = nullptr;   // the speculative erosion's round loop (tw_erosion.cu), kept while its kernel arguments stay the same
	std::vector<unsigned char> spec_key;    // those arguments
	cudaGraphExec_t sweep_graph = nullptr;  // the sweeps job's loop (twi_erode_sweeps_enqueue), kept the same way
	std::vector<unsigned char> sweep_key;
	void *dist = nullptr;        // tw_dist_state (tw_multi.cu): NCCL communicator of the one-process-per-GPU mode
	unsigned skip_rect[4] = {0, 0, 0, 0}; // x0, y0, w, h of the cells twi_heightgen's paired noise kernels leave unwritten (set around AO context generation only)
	// tw_create_shared: a shared context's tables above (sin / direction tables, sine params, both LUTs, the heightmap image) are its parent's, copied
	// from the parent at the start of every entry point (twi_borrow_tables) and never allocated, built or freed here
	tw_ctx *parent = nullptr;
	std::vector<tw_ctx *> shared; // the parent's live shared contexts
	std::vector<tw_tile_set *> sets; // live tile sets (tw_tileset.cu), destroyed with the context
	std::vector<tw_voxel_model *> models; // live voxel models (tw_voxel_post.cu), destroyed with the context
};

int  tw_set_error(tw_ctx *ctx, int status, const char *fmt, ...);
int  twi_begin(tw_ctx *ctx);                                    // an entry point's prologue: TW_ERR_ARG for a null ctx, else its device made current, its
                                                                // parent's tables borrowed and its pending job completed (twi_finish_pending)
int  twi_finish_pending(tw_ctx *ctx);                           // completes the context's pending asynchronous job (if any) before other work reuses its scratch
void twi_borrow_tables(tw_ctx *ctx);                            // a shared context takes its parent's current tables (no-op on any other context)
int  twi_ensure_simplex_lut(tw_ctx *ctx);                       // builds ctx->d_simplex_lut on ctx->stream if absent (tw_heightgen.cu)
int  twi_ensure_glm3_lut(tw_ctx *ctx);                          // builds ctx->d_glm3_lut on ctx->stream if absent (tw_voxel.cu)
int  tw_reserve(tw_ctx *ctx, int slot, size_t bytes);           // grow d_scratch[slot]; returns TW_OK / TW_ERR_CUDA
int  tw_reserve_pinned(tw_ctx *ctx, size_t bytes);
bool tw_is_device_ptr(const void *p);

// A layout of scratch or pinned staging: regions carved one after another from `base`, each starting on a 256-byte boundary. A layout is written once, as
// code that takes a twi_carve &, and run twice: with base == nullptr it only counts `bytes` (the size to reserve), then on the reserved memory. An absent
// region is written `want ? c.take<T>(n) : nullptr`, never take(0), which returns an address.
struct twi_carve {
	char *base = nullptr; size_t bytes = 0;
	template <typename T> T *take(size_t count) {T *p = base ? (T *)(base + bytes) : nullptr; bytes += (count*sizeof(T) + 255) & ~(size_t)255; return p;}
};
// Counts `layout`, reserves its bytes of scratch slot `slot` (TWI_PINNED: of the pinned staging), then carves it from that memory. Reserve before anything is
// enqueued: tw_reserve synchronises ctx->stream and may re-allocate the slot, so a pointer carved before a later reserve of the same slot is stale after it.
constexpr int TWI_PINNED = -1;
template <typename Layout> int twi_reserve_carve(tw_ctx *ctx, int slot, Layout &&layout) {
	twi_carve c; layout(c);
	int const rc = (slot == TWI_PINNED) ? tw_reserve_pinned(ctx, c.bytes) : tw_reserve(ctx, slot, c.bytes); if (rc) return rc;
	c = twi_carve{(char *)((slot == TWI_PINNED) ? ctx->h_pinned : ctx->d_scratch[slot])}; layout(c);
	return TW_OK;
}
// The fixed words at the start of scratch slot 2 (a layout of slot 2 takes them first): one grid's ordered min/max, the 16-bit packing's count of values out
// of range, the erosion's droplet moves, its droplet counter (tw_erode_parallel) and the speculative erosion's no-progress word
struct twi_slot2_words {unsigned mm[2], bad, pad_; unsigned long long steps; unsigned next, fail;};
inline twi_slot2_words *twi_slot2(tw_ctx *ctx) {return (twi_slot2_words *)ctx->d_scratch[2];}

#define TW_CUDA(ctx, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	return tw_set_error((ctx), TW_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } } while (0)
#define TW_LAUNCH_CHECK(ctx) do { (ctx)->launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) { \
	return tw_set_error((ctx), TW_ERR_CUDA, "%s:%d kernel launch: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); } } while (0)

// The job's number in the device words, on ctx->stream, before its work (twi_job_start sets *seq) / after it: `stopped` to the pinned staging, `job` cleared
int twi_job_start(tw_ctx *ctx, unsigned *seq);
int twi_job_end(tw_ctx *ctx);
// ctx->stream waits (on the device) for every edit of the family's image so far
int twi_wait_image_edits(tw_ctx *ctx);
// Before the root's image is freed or replaced (tw_set_heightmap, a set_image job, tw_destroy): waits for the pending edits (the caller has completed every job
// of the family they could wait for) and frees their staging
int twi_image_settle(tw_ctx *root);
// the scatter kernel of an edit on `st`: nrows rows (d_rows) of packed texels d_data into the image d_img
int twi_hmap_scatter(tw_ctx *ctx, cudaStream_t st, const twi_hmap_row *d_rows, uint32_t nrows, const uint8_t *d_data, uint8_t *d_img);

// Makes `job` the context's pending job (the previous one has been completed): enqueue() puts the job's work on ctx->stream, with every other stream it used
// joined into ctx->stream, between the job's start and end in the device words, and ctx->async.done is recorded behind it. When any step fails, the call
// waits for every stream of the context, so none of the job still runs on the scratch or the pinned staging when the error is returned, and no job is pending.
// A job that reads or writes the image (job.reads_image) first waits on the device for the edits made before its launch.
template <typename Enqueue> int twi_launch_job(tw_ctx *ctx, twi_job job, Enqueue &&enqueue) {
	unsigned seq = 0;
	int rc = job.reads_image ? twi_wait_image_edits(ctx) : TW_OK;
	if (rc == TW_OK) {rc = twi_job_start(ctx, &seq);}
	ctx->async.image_free_set = false;
	if (rc == TW_OK) {ctx->in_job = true; rc = enqueue(); ctx->in_job = false;}
	if (rc == TW_OK) {rc = twi_job_end(ctx);}
	if (rc == TW_OK) {
		cudaError_t e = cudaEventRecord(ctx->async.done, ctx->stream);
		if (e == cudaSuccess && job.reads_image && !ctx->async.image_free_set) e = cudaEventRecord(ctx->async.image_free, ctx->stream);
		if (e != cudaSuccess) rc = tw_set_error(ctx, TW_ERR_CUDA, "recording the job's event: %s", cudaGetErrorString(e));
	}
	if (rc != TW_OK) {
		cudaStreamSynchronize(ctx->stream);
		for (cudaStream_t s : ctx->aux_stream) {if (s) cudaStreamSynchronize(s);}
		for (cudaStream_t s : ctx->heavy_stream) {if (s) cudaStreamSynchronize(s);}
		return rc;
	}
	ctx->async.job = std::move(job);
	ctx->async.job.seq = seq;
	return TW_OK;
}

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
// Work a caller adds to the end of the asynchronous tile job (tw_tile_set_create_tiles_launch: the tile set's put and relight). The job validates its
// arguments, then calls prepare (nothing of the job is enqueued yet), reserves dev_bytes of slot-0 scratch and pin_bytes of pinned staging for the tail
// together with its own (before the erosion budget is taken), and after the chunk join calls enqueue on ctx->stream with the job's caller-order zvals, the
// tail's scratch and its staging; the end-of-job copies and the job's event follow.
struct twi_job_tail {
	size_t dev_bytes = 0, pin_bytes = 0;
	virtual int prepare(tw_ctx *ctx) = 0;
	virtual int enqueue(tw_ctx *ctx, const float *d_zvals, char *d_mem, char *h_mem) = 0;
	virtual ~twi_job_tail() {}
};
// tw_create_tiles_launch_ex (hs == nullptr) or tw_create_tiles_launch_hmap without shadows, with a tail; out->zvals may be NULL with a tail (zvals are then only staged on the device)
int twi_create_tiles_launch(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                            uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval, float wpz_max, uint32_t size,
                            const tw_tile_outputs *out, const tw_tile_shading *shading, twi_job_tail *tail);
int twi_eval_points(tw_ctx *ctx, const float *d_xy, size_t n, const tw_height_params *p, const tw_point_query *q, float *d_out);
// M_SPEC (one big map, the reference's serial droplet order) in parts: whether twi_erode takes it, its scratch, and the enqueue - with host_rounds = false
// one that ends on the device (*d_fail = the rounds run when the window stopped making progress, else 0), with true tw_erode's host-driven rounds
bool   twi_erode_spec_eligible(uint32_t nt, int xsize, int ysize, uint32_t num_iters);
size_t twi_erode_spec_scratch_bytes(int xsize, int ysize);
int    twi_erode_spec_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zvals, float min_zval, uint32_t num_iters,
                              const tw_erosion_params *p, unsigned long long *d_steps, unsigned *d_fail, bool host_rounds);
int twi_erode_parallel(tw_ctx *ctx, float *d_map, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p, uint32_t num_threads);
// tw_erode_parallel in parts: its padded scratch, and the enqueue (lower clamp *d_min_zval, or min_zval when it is nullptr; moves added to *d_steps)
size_t twi_erode_parallel_scratch_bytes(int xsize, int ysize);
int    twi_erode_parallel_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zval, float min_zval, uint32_t num_iters,
                                  const tw_erosion_params *p, uint32_t num_threads, unsigned long long *d_steps, unsigned *d_next);
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
// tw_erode_sweeps of one map in a job (tw_erode_launch_ex): its scratch (padded map, fixed-point deltas, the sweep word), and the enqueue - pad, the sweeps as
// one graph that ends on the device (and at a cancel), unpad with the lower clamp *d_min_zval (nullptr: min_zval); moves added to *d_steps
size_t twi_erode_sweeps_scratch_bytes(int xsize, int ysize);
int    twi_erode_sweeps_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zval, float min_zval, uint32_t num_iters,
                                const tw_erosion_params *p, uint32_t sweep, int halo, unsigned long long *d_steps);
int twi_tile_bounds(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, void *d_sub, const unsigned *d_perm = nullptr);
int twi_glaciate_mesh(tw_ctx *ctx, float *d_mesh, int nx, int ny, int xoff2, int yoff2, int MX, int MY, const tw_height_params *p, unsigned *d_mm);
// the checks of tw_voxel_fill after its null-argument check (TW_ERR_STATE without the sin table, TW_ERR_ARG for a bad gen_mode or size); *tab_bytes = the
// scratch slot 1 bytes twi_voxel_fill uses for this grid (reserve them first and it never re-allocates)
int twi_voxel_fill_check(tw_ctx *ctx, const tw_voxel_params *vp, size_t *tab_bytes);
// h_stage (optional): TW_N3D_RDATA floats of pinned staging left untouched until the enqueued work is done; without it the sine mode synchronises ctx->stream
// after uploading its coefficients (a stack buffer)
int twi_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *d_out, void *h_stage = nullptr);
int twi_from_floats_u16(tw_ctx *ctx, const float *d_vals, size_t n, float val_mult, float val_add, uint8_t *d_out, unsigned *d_bad);
// tw_proc_gen_heightmap's device scalars (tw_streaming.cu): twi_hmap_scales turns the ordered min/max d_mm into a twi_hmap_stage in device memory (the host
// arithmetic of set_mesh_height_scales_for_zval_range and get_mh_texture_mult/add); twi_from_floats_u16_dev packs with that stage's val_add / val_div
struct twi_hmap_stage {float min_z, max_z, val_mult, val_add, mesh_file_scale, mesh_file_tz, val_div; unsigned bad, fail, pad_; unsigned long long steps;};
int twi_hmap_scales(tw_ctx *ctx, const unsigned *d_mm, float mesh_height_scale, float mesh_scale_z_inv, twi_hmap_stage *d_stage);
int twi_from_floats_u16_dev(tw_ctx *ctx, const float *d_vals, size_t n, const twi_hmap_stage *d_stage, uint8_t *d_out);
// *d_min = the minimum of the ordered min/max d_mm as a float (tw_erode_launch's lower clamp of the image, left on the device)
int twi_ord_min(tw_ctx *ctx, const unsigned *d_mm, float *d_min);
// scratch slot 1 bytes twi_heightgen uses for this grid (the sine mode's tables; 0 otherwise)
size_t twi_heightgen_slot1_bytes(const tw_grid2d *g, const tw_height_params *p);
int twi_to_floats_u16(tw_ctx *ctx, const uint8_t *d_data, size_t n, float val_mult, float val_add, float *d_vals);
int twi_minmax(tw_ctx *ctx, const float *d_vals, size_t n, unsigned *d_mm_ord);
int twi_minmax_tiles(tw_ctx *ctx, cudaStream_t st, const float *d_vals, size_t tile_elems, uint32_t nt, unsigned *d_mm_ord, const unsigned *d_perm = nullptr);
int twi_coarse_work(tw_ctx *ctx, const float *d_coarse, unsigned cells, uint32_t nt, float level, unsigned *d_work);
int twi_gather_origins(tw_ctx *ctx, const void *d_org, const unsigned *d_order, uint32_t nt, void *d_out);
int twi_order_by_work(tw_ctx *ctx, cudaStream_t st, const unsigned *d_work, uint32_t nt, unsigned max_work, unsigned *d_hist256, unsigned *d_order);
int twi_init_minmax(tw_ctx *ctx, unsigned *d_mm_ord, uint32_t n);
