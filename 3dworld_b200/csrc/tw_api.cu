// tw_api.cu - the extern "C" boundary (include/tw3d.h): context management, host/device pointer staging, and dispatch to the kernels.
// There is deliberately NO CPU path in this library: without a CUDA device tw_create fails and nothing else can be called.
#include "tw_internal.h"
#include <algorithm>
#include <stdarg.h>
#include <stdlib.h>
#include <new>
#include <vector>
#include <math.h>

extern "C" void twi_build_dir_table(float *cs2x1e6);

int tw_set_error(tw_ctx *ctx, int status, const char *fmt, ...) {
	if (ctx) {
		va_list ap; va_start(ap, fmt);
		vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
		va_end(ap);
	}
	return status;
}

int tw_reserve(tw_ctx *ctx, int slot, size_t bytes) {
	if (ctx->scratch_bytes[slot] >= bytes) return TW_OK;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (ctx->d_scratch[slot]) {TW_CUDA(ctx, cudaFree(ctx->d_scratch[slot])); ctx->d_scratch[slot] = nullptr; ctx->scratch_bytes[slot] = 0;}
	size_t const rounded = (bytes + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
	TW_CUDA(ctx, cudaMalloc(&ctx->d_scratch[slot], rounded));
	ctx->scratch_bytes[slot] = rounded;
	return TW_OK;
}

int tw_reserve_pinned(tw_ctx *ctx, size_t bytes) {
	if (ctx->pinned_bytes >= bytes) return TW_OK;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (ctx->h_pinned) {TW_CUDA(ctx, cudaFreeHost(ctx->h_pinned)); ctx->h_pinned = nullptr; ctx->pinned_bytes = 0;}
	TW_CUDA(ctx, cudaMallocHost(&ctx->h_pinned, bytes));
	ctx->pinned_bytes = bytes;
	return TW_OK;
}

bool tw_is_device_ptr(const void *p) {
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {cudaGetLastError(); return false;}
	return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
}

int twi_ensure_aux_streams(tw_ctx *ctx) {
	if (ctx->aux_stream[0]) return TW_OK;
	int lo = 0, hi = 0; // the latency-bound droplet kernels / band copies get the higher priority
	TW_CUDA(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
	bool const prio = !(getenv("TW_PIPE_NOPRIO"));
	for (int i = 0; i < 3; ++i) {TW_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->aux_stream[i], cudaStreamNonBlocking, prio ? hi : lo));}
	return TW_OK;
}

namespace {

// slot-2 layout (small device scalars)
constexpr size_t OFF_MM = 0, OFF_BAD = 64, OFF_TILES = 4096;

int check_ctx(tw_ctx *ctx) { // NOTE: makes ctx->device the calling thread's current CUDA device and leaves it so (documented in tw3d.h: one context per thread)
	if (!ctx) return TW_ERR_ARG;
	cudaError_t e = cudaSetDevice(ctx->device);
	if (e != cudaSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
	return TW_OK;
}

// what tile_t::create_zvals derives per 4x4 sub-block (tile_bounds_kernel's output, tw_tiles.cu SubBounds)
struct Sub {float zmin, zmax; int wx1, wy1, wx2, wy2;};

void combine_bounds(const Sub *sub, uint32_t ntiles, float dx_val, float dy_val, uint32_t size, tw_tile_bounds *out) {
	for (uint32_t t = 0; t < ntiles; ++t) { // combine the 16 sub-blocks exactly as the reference's loop does (src/tiled_mesh.cpp:517-540)
		tw_tile_bounds &b = out[t];
		b.mzmin = 100.0f; b.mzmax = -100.0f; b.mesh_dz = 0.0f; // FAR_DISTANCE
		b.wx1 = b.wy1 = 2147483647; b.wx2 = b.wy2 = -1;
		for (int k = 0; k < 16; ++k) {
			Sub const &q = sub[(size_t)t*16 + k];
			b.sub_zmin[k] = q.zmin; b.sub_zmax[k] = q.zmax;
			float const range = q.zmax - q.zmin;
			b.mesh_dz = (b.mesh_dz < range) ? range : b.mesh_dz;      // max_eq(mesh_dz, (szmax - szmin))
			b.mzmin = (q.zmin < b.mzmin) ? q.zmin : b.mzmin;          // min(mzmin, szmin)
			b.mzmax = (b.mzmax < q.zmax) ? q.zmax : b.mzmax;          // max(mzmax, szmax)
			if (q.wx1 < b.wx1) b.wx1 = q.wx1; if (q.wy1 < b.wy1) b.wy1 = q.wy1;
			if (q.wx2 > b.wx2) b.wx2 = q.wx2; if (q.wy2 > b.wy2) b.wy2 = q.wy2;
		}
		float const dz = b.mzmax - b.mzmin;
		b.radius = 0.5*sqrtf((dx_val*dx_val + dy_val*dy_val)*size*size + dz*dz); // src/tiled_mesh.cpp:541
	}
}

// Completion of the pending asynchronous job: wait = 0 only queries its event. The call that sees it complete unpacks what the job staged in
// ctx->h_pinned into the caller's host arrays and reports errors of the enqueued work.
int poll_job(tw_ctx *ctx, int wait) {
	tw_async_state &a = ctx->async;
	if (!a.pending) return TW_OK;
	cudaError_t const ev = wait ? cudaEventSynchronize(a.done) : cudaEventQuery(a.done);
	if (ev == cudaErrorNotReady) return TW_ERR_NOT_READY;
	a.pending = false;
	if (ev != cudaSuccess) {a.host_mm = nullptr; a.host_bounds = nullptr; a.host_min_nz = nullptr; a.host_flags = nullptr; return tw_set_error(ctx, TW_ERR_CUDA, "asynchronous job failed: %s", cudaGetErrorString(ev));}
	const char *h = (const char *)ctx->h_pinned;
	if (!a.tiles) {
		if (a.host_mm) {unsigned const *u = (unsigned const *)h; a.host_mm->zmin = tw_ord2f(u[0]); a.host_mm->zmax = tw_ord2f(u[1]);}
	}
	else {
		if (a.steps) {unsigned long long s; memcpy(&s, h + a.off_steps, sizeof(s)); ctx->last_erosion_steps = s;}
		if (a.host_mm) {
			unsigned const *u = (unsigned const *)(h + a.off_mm);
			for (uint32_t i = 0; i < a.n_mm; ++i) {a.host_mm[i].zmin = tw_ord2f(u[2*i]); a.host_mm[i].zmax = tw_ord2f(u[2*i+1]);}
		}
		if (a.host_bounds) {combine_bounds((const Sub *)(h + a.off_sub), a.n_mm, a.dx, a.dy, a.size, a.host_bounds);}
		if (a.host_min_nz) {unsigned const *u = (unsigned const *)(h + a.off_min_nz); for (uint32_t i = 0; i < a.n_mm; ++i) {a.host_min_nz[i] = tw_ord2f(u[i]);}}
		if (a.host_flags) {memcpy(a.host_flags, h + a.off_flags, a.n_mm);}
	}
	a.host_mm = nullptr; a.host_bounds = nullptr; a.host_min_nz = nullptr; a.host_flags = nullptr; a.tiles = false; a.steps = false;
	cudaError_t const e = cudaGetLastError();
	if (e != cudaSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "asynchronous job failed: %s", cudaGetErrorString(e));
	return TW_OK;
}

int finish_pending(tw_ctx *ctx) { // complete an outstanding tw_heightgen_2d_launch / tw_create_tiles_launch before other work reuses the scratch buffers
	return poll_job(ctx, 1);
}

int read_minmax(tw_ctx *ctx, const unsigned *d_mm, tw_minmax *mm, uint32_t n) { // synchronous
	int rc = tw_reserve_pinned(ctx, (size_t)n*2*sizeof(unsigned));
	if (rc) return rc;
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, d_mm, (size_t)n*2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	unsigned const *u = (unsigned const *)ctx->h_pinned;
	for (uint32_t i = 0; i < n; ++i) {mm[i].zmin = tw_ord2f(u[2*i]); mm[i].zmax = tw_ord2f(u[2*i+1]);}
	return TW_OK;
}

int validate_height(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, const float *out) {
	if (!g || !p || !out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (g->nx == 0 || g->ny == 0) return tw_set_error(ctx, TW_ERR_ARG, "nx, ny must be > 0 (reference asserts, src/mesh_gen.cpp:589)");
	if (p->gen_mode < 0 || p->gen_mode > TW_MGEN_DWARP_GPU) return tw_set_error(ctx, TW_ERR_ARG, "bad gen_mode %d", p->gen_mode);
	if (p->start_eval_sin < 0 || p->start_eval_sin > TW_F_TABLE_SIZE) return tw_set_error(ctx, TW_ERR_ARG, "start_eval_sin out of range (src/mesh_gen.cpp:590)");
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	return TW_OK;
}

// copies *wp into W and fills in W.class_ix (tw_tile_weights_batch, tw_create_tiles_launch_ex)
int validate_weights(tw_ctx *ctx, const tw_weight_params *wp, tw_weight_params &W) {
	W = *wp;
	int seen[5] = {0, 0, 0, 0, 0};
	for (int i = 0; i < 5; ++i) {
		if (W.tex_class[i] < 0 || W.tex_class[i] > 4 || seen[W.tex_class[i]]++) return tw_set_error(ctx, TW_ERR_ARG, "tex_class must name each ground texture exactly once (get_texture_ixs asserts it)");
		W.class_ix[W.tex_class[i]] = i;
	}
	if (!(W.zmax > W.zmin)) return tw_set_error(ctx, TW_ERR_ARG, "zmax must exceed zmin");
	return TW_OK;
}

} // namespace

int twi_finish_pending(tw_ctx *ctx) {return finish_pending(ctx);}

extern "C" {

int tw_abi_version(void) {return TW_ABI_VERSION;}

int tw_create(int device, tw_ctx **out) {
	if (!out) return TW_ERR_ARG;
	*out = nullptr;
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {cudaGetLastError(); return TW_ERR_NO_DEVICE;}
	if (device < 0 || device >= ndev) return TW_ERR_ARG;
	if (cudaSetDevice(device) != cudaSuccess) {cudaGetLastError(); return TW_ERR_CUDA;}
	tw_ctx *ctx = new (std::nothrow) tw_ctx();
	if (!ctx) return TW_ERR_CUDA;
	ctx->device = device;
	{int sms = 0; if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) ctx->num_sms = (unsigned)sms; else cudaGetLastError();}
	if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {delete ctx; cudaGetLastError(); return TW_ERR_CUDA;}
	if (cudaEventCreateWithFlags(&ctx->async.done, cudaEventDisableTiming) != cudaSuccess) {cudaStreamDestroy(ctx->stream); delete ctx; cudaGetLastError(); return TW_ERR_CUDA;}
	*out = ctx;
	return TW_OK;
}

void tw_destroy(tw_ctx *ctx) {
	if (!ctx) return;
	if (ctx->dist) tw_dist_finalize(ctx);
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	for (int i = 0; i < 3; ++i) {if (ctx->d_scratch[i]) cudaFree(ctx->d_scratch[i]);}
	if (ctx->d_sin_table) cudaFree(ctx->d_sin_table);
	if (ctx->d_dir_table) cudaFree(ctx->d_dir_table);
	if (ctx->d_simplex_lut) cudaFree(ctx->d_simplex_lut);
	if (ctx->d_glm3_lut) cudaFree(ctx->d_glm3_lut);
	if (ctx->d_sine_params) cudaFree(ctx->d_sine_params);
	if (ctx->d_hmap) cudaFree(ctx->d_hmap);
	if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
	if (ctx->async.done) cudaEventDestroy(ctx->async.done);
	for (int i = 0; i < 3; ++i) {if (ctx->aux_stream[i]) cudaStreamDestroy(ctx->aux_stream[i]);}
	for (int i = 0; i < 4; ++i) {
		if (ctx->heavy_stream[i]) cudaStreamDestroy(ctx->heavy_stream[i]);
		if (ctx->ev_fork[i]) cudaEventDestroy(ctx->ev_fork[i]);
		if (ctx->ev_join[i]) cudaEventDestroy(ctx->ev_join[i]);
	}
	cudaStreamDestroy(ctx->stream);
	delete ctx;
}

const char *tw_last_error(const tw_ctx *ctx) {return ctx ? ctx->err : "null context";}
void *tw_stream(tw_ctx *ctx) {return ctx ? (void *)ctx->stream : nullptr;}
uint64_t tw_launch_count(const tw_ctx *ctx) {return ctx ? ctx->launches : 0;}
uint64_t tw_last_erosion_steps(const tw_ctx *ctx) {return ctx ? ctx->last_erosion_steps : 0;}

int tw_sync(tw_ctx *ctx) {
	int rc = check_ctx(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_set_sin_table(tw_ctx *ctx, const float *tab) {
	int rc = check_ctx(ctx); if (rc) return rc;
	std::vector<float> built;
	if (!tab) {built.resize(TW_SIN_TABLE_SIZE); tw_build_sin_table(built.data()); tab = built.data();}
	if (!ctx->d_sin_table) {TW_CUDA(ctx, cudaMalloc(&ctx->d_sin_table, TW_SIN_TABLE_SIZE*sizeof(float)));}
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_sin_table, tab, TW_SIN_TABLE_SIZE*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	if (!ctx->d_dir_table) {
		std::vector<float> dir(2*1000000);
		twi_build_dir_table(dir.data());
		TW_CUDA(ctx, cudaMalloc(&ctx->d_dir_table, dir.size()*sizeof(float)));
		TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_dir_table, dir.data(), dir.size()*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	ctx->have_sin = true;
	return TW_OK;
}

int tw_set_sine_params(tw_ctx *ctx, const float *sp) {
	int rc = check_ctx(ctx); if (rc) return rc;
	if (!sp) return tw_set_error(ctx, TW_ERR_ARG, "null sine_params");
	if (!ctx->d_sine_params) {TW_CUDA(ctx, cudaMalloc(&ctx->d_sine_params, TW_F_TABLE_SIZE*5*sizeof(float)));}
	memcpy(ctx->h_sine_params, sp, sizeof(ctx->h_sine_params));
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_sine_params, ctx->h_sine_params, sizeof(ctx->h_sine_params), cudaMemcpyHostToDevice, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	ctx->have_sine_params = true;
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ 2-D height
int tw_heightgen_2d_launch(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, float *out, tw_minmax *mm) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	rc = validate_height(ctx, g, p, out); if (rc) return rc;
	size_t const n = (size_t)g->nx*g->ny;
	bool const dev_out = tw_is_device_ptr(out);
	float *d_out = out;
	if (!dev_out) {rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc; d_out = (float *)ctx->d_scratch[0];}
	rc = tw_reserve(ctx, 2, OFF_TILES); if (rc) return rc;
	unsigned *d_mm = mm ? (unsigned *)((char *)ctx->d_scratch[2] + OFF_MM) : nullptr;
	if (d_mm) {rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;}
	if (!dev_out) {rc = twi_ensure_aux_streams(ctx); if (rc) return rc;}
	rc = twi_heightgen(ctx, g, p, enable_glaciate, min_start_sin, nullptr, 1, d_out, d_mm, dev_out ? nullptr : out); // host out: band-wise D2H overlapped with compute
	if (rc) return rc;
	if (mm) {
		rc = tw_reserve_pinned(ctx, 2*sizeof(unsigned)); if (rc) return rc;
		TW_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, d_mm, 2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
	}
	TW_CUDA(ctx, cudaEventRecord(ctx->async.done, ctx->stream));
	ctx->async.pending = true; ctx->async.tiles = false; ctx->async.host_mm = mm; ctx->async.n_mm = mm ? 1 : 0;
	return TW_OK;
}

int tw_heightgen_2d_poll(tw_ctx *ctx, int wait) {
	int rc = check_ctx(ctx); if (rc) return rc;
	return poll_job(ctx, wait);
}

int tw_heightgen_2d(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, float *out, tw_minmax *mm) {
	int rc = tw_heightgen_2d_launch(ctx, g, p, enable_glaciate, min_start_sin, out, mm);
	if (rc) return rc;
	return tw_heightgen_2d_poll(ctx, 1);
}

// tile_t::create_texture, terrain part (include/tw3d.h): the jitter noise grid of every tile (force-sine-mode build_arrays at 80x the cell size, start index >= 50,
// no glaciate) with the batched sine-tile generator, then one thread per texel
int tw_tile_weights_batch(tw_ctx *ctx, const float *zvals, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                          uint32_t zvsize, const tw_height_params *p, const tw_weight_params *wp, const float *tile_params, uint8_t *weights, uint8_t *has_any_grass)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!zvals || !origins_xy || !p || !wp || !tile_params || !weights || ntiles == 0 || zvsize < 3) return tw_set_error(ctx, TW_ERR_ARG, "tw_tile_weights_batch: null argument, no tiles or zvsize < 3");
	tw_weight_params W;
	rc = validate_weights(ctx, wp, W); if (rc) return rc;
	uint32_t const stride = zvsize - 1;
	size_t const zn = (size_t)ntiles*zvsize*zvsize, tn = (size_t)ntiles*stride*stride;
	bool const dev_z = tw_is_device_ptr(zvals), dev_w = tw_is_device_ptr(weights), dev_f = has_any_grass && tw_is_device_ptr(has_any_grass), dev_p = tw_is_device_ptr(tile_params);
	auto al = [](size_t b) {return (b + 255) & ~(size_t)255;};
	rc = tw_reserve(ctx, 0, al(tn*sizeof(float)) + (dev_z ? 0 : al(zn*sizeof(float))) + (dev_w ? 0 : al(tn*4)) + al(ntiles) + (dev_p ? 0 : al((size_t)ntiles*8*sizeof(float))) + 256);
	if (rc) return rc;
	char *q = (char *)ctx->d_scratch[0];
	float *d_rand = (float *)q; q += al(tn*sizeof(float));
	const float *d_z = zvals;
	if (!dev_z) {TW_CUDA(ctx, cudaMemcpyAsync(q, zvals, zn*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_z = (const float *)q; q += al(zn*sizeof(float));}
	uint8_t *d_w = weights;
	if (!dev_w) {d_w = (uint8_t *)q; q += al(tn*4);}
	uint8_t *d_f = dev_f ? has_any_grass : (uint8_t *)q; q += al(ntiles);
	const float *d_p = tile_params;
	if (!dev_p) {TW_CUDA(ctx, cudaMemcpyAsync(q, tile_params, (size_t)ntiles*8*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_p = (const float *)q;}
	if (has_any_grass) {TW_CUDA(ctx, cudaMemsetAsync(d_f, 0, ntiles, ctx->stream));}
	// height_gen.build_arrays((x1 - MESH_X_SIZE/2), (y1 - MESH_Y_SIZE/2), MESH_NOISE_FREQ*DX_VAL, MESH_NOISE_FREQ*DY_VAL, tsize, tsize, 0, 1) (src/tiled_mesh.cpp:1103)
	float const MESH_NOISE_FREQ = 80.0f;
	tw_grid2d g; g.x0 = 0; g.y0 = 0; g.dx = MESH_NOISE_FREQ*dx; g.dy = MESH_NOISE_FREQ*dy; g.nx = stride; g.ny = stride;
	std::vector<float2> org(ntiles);
	for (uint32_t t = 0; t < ntiles; ++t) {
		float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
		org[t] = make_float2(g.dx*x0, g.dy*y0);
	}
	tw_height_params ps = *p;
	ps.gen_mode = TW_MGEN_SINE; ps.gen_shape = 0; // force_sine_mode: gen_mode = MGEN_SINE, gen_shape = 0 (src/mesh_gen.cpp:592-593)
	rc = twi_heightgen_sine_tiles(ctx, &g, &ps, 0, 50, org.data(), ntiles, d_rand, nullptr);
	if (rc) return rc;
	rc = twi_tile_weights(ctx, ctx->stream, d_z, d_rand, ntiles, zvsize, d_p, &W, d_w, has_any_grass ? d_f : nullptr);
	if (rc) return rc;
	if (!dev_w) {TW_CUDA(ctx, cudaMemcpyAsync(weights, d_w, tn*4, cudaMemcpyDeviceToHost, ctx->stream));}
	if (has_any_grass && !dev_f) {TW_CUDA(ctx, cudaMemcpyAsync(has_any_grass, d_f, ntiles, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_heightgen_tiles(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                       uint32_t zvsize, const tw_height_params *p, float *out, tw_minmax *mm)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!origins_xy || ntiles == 0) return tw_set_error(ctx, TW_ERR_ARG, "no tiles");
	tw_grid2d g; g.x0 = 0; g.y0 = 0; g.dx = dx; g.dy = dy; g.nx = zvsize; g.ny = zvsize;
	rc = validate_height(ctx, &g, p, out); if (rc) return rc;
	size_t const tile_elems = (size_t)zvsize*zvsize, n = tile_elems*ntiles;
	bool const dev_out = tw_is_device_ptr(out);
	float *d_out = out;
	if (!dev_out) {rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc; d_out = (float *)ctx->d_scratch[0];}
	size_t const mm_bytes = (size_t)ntiles*2*sizeof(unsigned), org_bytes = (size_t)ntiles*sizeof(float2);
	rc = tw_reserve(ctx, 2, OFF_TILES + mm_bytes + org_bytes); if (rc) return rc;
	unsigned *d_mm = mm ? (unsigned *)((char *)ctx->d_scratch[2] + OFF_TILES) : nullptr;
	float2 *d_org = (float2 *)((char *)ctx->d_scratch[2] + OFF_TILES + mm_bytes);
	if (d_mm) {rc = twi_init_minmax(ctx, d_mm, ntiles); if (rc) return rc;}
	// setup_height_gen_async: build_arrays((x0 - MESH_X_SIZE/2), (y0 - MESH_Y_SIZE/2), dx, dy, ...): int -> float, then mx0 = dx*x0 (src/tiled_mesh.cpp:461, src/mesh_gen.cpp:591)
	if (p->gen_mode != TW_MGEN_SINE) {
		std::vector<float2> org(ntiles);
		for (uint32_t t = 0; t < ntiles; ++t) {
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			org[t] = make_float2(dx*x0, dy*y0);
		}
		TW_CUDA(ctx, cudaMemcpyAsync(d_org, org.data(), org_bytes, cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // org is a local vector
		uint32_t const zmax = 65535;
		for (uint32_t t0 = 0; t0 < ntiles; t0 += zmax) { // gridDim.z limit
			uint32_t const nt = (ntiles - t0 < zmax) ? ntiles - t0 : zmax;
			rc = twi_heightgen(ctx, &g, p, 1, 0, d_org + t0, nt, d_out + (size_t)t0*tile_elems, d_mm ? d_mm + 2*(size_t)t0 : nullptr);
			if (rc) return rc;
		}
	}
	else { // sine tables depend on the tile origin only through its column / row: W + H tables for a W x H block of tiles, one grid launch for the batch
		std::vector<float2> org(ntiles);
		for (uint32_t t = 0; t < ntiles; ++t) {
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			org[t] = make_float2(dx*x0, dy*y0);
		}
		rc = twi_heightgen_sine_tiles(ctx, &g, p, 1, 0, org.data(), ntiles, d_out, d_mm);
		if (rc) return rc;
	}
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(out, d_out, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	if (mm) {rc = read_minmax(ctx, d_mm, mm, ntiles); if (rc) return rc;}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ callers' tails
int tw_tile_bounds_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, float dx_val, float dy_val, uint32_t size, tw_tile_bounds *out) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!zvals || !out || ntiles == 0 || zvsize < 4) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (4*(zvsize/4) >= zvsize) return tw_set_error(ctx, TW_ERR_ARG, "zvsize %u: the last sub-block would end at cell %u (the reference asserts x_end < zvsize, src/tiled_mesh.cpp:520)", zvsize, 4*(zvsize/4));
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	size_t const n = (size_t)ntiles*zvsize*zvsize;
	size_t const sub_bytes = (size_t)ntiles*16*sizeof(Sub);
	const float *d_z = zvals;
	bool const dev = tw_is_device_ptr(zvals);
	rc = tw_reserve(ctx, 0, (dev ? 0 : n*sizeof(float)) + sub_bytes + 256); if (rc) return rc;
	char *s0 = (char *)ctx->d_scratch[0];
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(s0, zvals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_z = (const float *)s0; s0 += (n*sizeof(float) + 255) & ~(size_t)255;}
	rc = twi_tile_bounds(ctx, ctx->stream, d_z, ntiles, zvsize, wpz_max, s0); if (rc) return rc;
	std::vector<Sub> sub((size_t)ntiles*16);
	TW_CUDA(ctx, cudaMemcpyAsync(sub.data(), s0, sub_bytes, cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	combine_bounds(sub.data(), ntiles, dx_val, dy_val, size, out);
	return TW_OK;
}

int tw_glaciate_mesh(tw_ctx *ctx, float *mesh, int nx, int ny, int xoff2, int yoff2, int mesh_x_size, int mesh_y_size, const tw_height_params *p, tw_minmax *zbottom_ztop) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!mesh || !p || nx <= 0 || ny <= 0 || ny > 65535) return tw_set_error(ctx, TW_ERR_ARG, "bad argument");
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	size_t const n = (size_t)nx*ny;
	bool const dev = tw_is_device_ptr(mesh);
	float *d_mesh = mesh;
	if (!dev) {
		rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc;
		d_mesh = (float *)ctx->d_scratch[0];
		TW_CUDA(ctx, cudaMemcpyAsync(d_mesh, mesh, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	}
	rc = tw_reserve(ctx, 2, OFF_TILES); if (rc) return rc;
	unsigned *d_mm = (unsigned *)((char *)ctx->d_scratch[2] + OFF_MM);
	rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
	rc = twi_glaciate_mesh(ctx, d_mesh, nx, ny, xoff2, yoff2, mesh_x_size, mesh_y_size, p, d_mm); if (rc) return rc;
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(mesh, d_mesh, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	if (zbottom_ztop) {return read_minmax(ctx, d_mm, zbottom_ztop, 1);}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ erosion
int tw_erode_tiles(tw_ctx *ctx, float *maps, uint32_t ntiles, int xsize, int ysize, const float *min_zvals, float min_zval_all,
                   uint32_t num_iters, const tw_erosion_params *p)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!maps || !p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (xsize <= 0 || ysize <= 0 || ntiles == 0) return tw_set_error(ctx, TW_ERR_ARG, "empty heightmap");
	if (num_iters == 0 || p->erode_amount <= 0.0) {ctx->last_erosion_steps = 0; return TW_OK;} // src/erosion.cpp:16
	size_t const n = (size_t)xsize*ysize*ntiles;
	bool const dev = tw_is_device_ptr(maps);
	float *d_maps = maps;
	if (!dev) {
		rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc;
		d_maps = (float *)ctx->d_scratch[0];
		TW_CUDA(ctx, cudaMemcpyAsync(d_maps, maps, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	}
	float *d_minz = nullptr;
	if (min_zvals) {
		rc = tw_reserve(ctx, 2, OFF_TILES + (size_t)ntiles*sizeof(float)); if (rc) return rc;
		d_minz = (float *)((char *)ctx->d_scratch[2] + OFF_TILES);
		TW_CUDA(ctx, cudaMemcpyAsync(d_minz, min_zvals, (size_t)ntiles*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	rc = twi_erode(ctx, d_maps, ntiles, xsize, ysize, d_minz, min_zval_all, num_iters, p);
	if (rc) return rc;
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(maps, d_maps, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// The tile pipeline behind tw_create_zvals_batch, tw_create_zvals_ao_batch and tw_create_tiles_launch(_ex, _shadows): enqueues everything and returns
// without waiting for the device; the job completes through poll_job (check_ctx and finish_pending have run). sh (optional): AO map and weights texture;
// shs (optional): per-light mesh shadows. hs: the height source - nullptr = the procedural height function p, else the context's heightmap image under hs
// (tw_create_tiles_launch_hmap, which has checked hs against the image and refused AO); p is then only read by the weights' jitter noise.
static int tiles_launch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy, uint32_t zvsize,
                        const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval, float wpz_max, uint32_t size,
                        const tw_tile_outputs *o, const tw_tile_shading *sh, const tw_tile_shadows *shs, const tw_hmap_sampler *hs)
{
	if (!origins_xy || ntiles == 0 || (!p && !hs) || !o || !o->zvals) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	bool const want_mm = (o->mm != nullptr), want_bounds = (o->bounds != nullptr), want_normals = (o->normals_rgba != nullptr), want_mnz = (o->min_normal_z != nullptr);
	bool const want_ao = (sh && sh->ao), want_w = (sh && sh->weights), want_f = (sh && sh->has_any_grass);
	if (want_mnz && !want_normals) return tw_set_error(ctx, TW_ERR_ARG, "min_normal_z is produced with the normal map: pass normals_rgba too");
	if (want_f && !want_w) return tw_set_error(ctx, TW_ERR_ARG, "has_any_grass is produced with the weights texture: pass weights too");
	if (want_bounds && (zvsize < 4 || 4*(zvsize/4) >= zvsize)) return tw_set_error(ctx, TW_ERR_ARG, "zvsize %u: the last sub-block would end at cell %u (the reference asserts x_end < zvsize, src/tiled_mesh.cpp:520)", zvsize, 4*(zvsize/4));
	if ((want_normals || want_ao) && zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "normals and AO need zvsize >= 2");
	tw_weight_params W;
	if (want_w) {
		if (!sh->wp || !sh->tile_params) return tw_set_error(ctx, TW_ERR_ARG, "the weights texture needs wp and tile_params");
		if (zvsize < 3) return tw_set_error(ctx, TW_ERR_ARG, "the weights texture needs zvsize >= 3");
		int const rc = validate_weights(ctx, sh->wp, W); if (rc) return rc;
	}
	// mesh shadows: the lights and their plans (neighbours, waves, light direction) are taken from the caller's arrays here, during the launch
	uint32_t const nl = shs ? shs->nlights : 0;
	std::vector<tw_tile_light> lights;
	std::vector<twi_shadow_plan> splan;
	std::vector<char> sdev_m, sdev_ix, sdev_iy; // smask / sh_in_x / sh_in_y are device memory
	if (shs) {
		if (!shs->tile_xy || shs->nlights == 0 || !shs->lights) return tw_set_error(ctx, TW_ERR_ARG, "mesh shadows need tile_xy and at least one light");
		if (zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "mesh shadows need zvsize >= 2");
		lights.assign(shs->lights, shs->lights + nl);
		splan.resize(nl); sdev_m.resize(nl); sdev_ix.resize(nl); sdev_iy.resize(nl);
		for (uint32_t l = 0; l < nl; ++l) {
			tw_tile_light const &L = lights[l];
			if (!L.smask) return tw_set_error(ctx, TW_ERR_ARG, "light %u: smask is required", l);
			sdev_m[l] = tw_is_device_ptr(L.smask);
			if (sdev_m[l] && ((size_t)L.smask & 3)) return tw_set_error(ctx, TW_ERR_ARG, "light %u: a device smask must be 4-byte aligned (flag bytes are set with 32-bit atomics)", l);
			sdev_ix[l] = L.sh_in_x && tw_is_device_ptr(L.sh_in_x); sdev_iy[l] = L.sh_in_y && tw_is_device_ptr(L.sh_in_y);
			if (!twi_shadow_plan_make(shs->tile_xy, ntiles, &L.sp, L.sh_in_x != nullptr, L.sh_in_y != nullptr, &splan[l])) return tw_set_error(ctx, TW_ERR_ARG, "tile_xy names a tile twice");
		}
	}
	tw_grid2d g; g.x0 = 0; g.y0 = 0; g.dx = dx; g.dy = dy; g.nx = zvsize; g.ny = zvsize;
	int rc = TW_OK;
	if (!hs) {rc = validate_height(ctx, &g, p, o->zvals); if (rc) return rc;}
	else {
		if (zvsize == 0) return tw_set_error(ctx, TW_ERR_ARG, "zvsize must be > 0");
		if (want_w && !p) return tw_set_error(ctx, TW_ERR_ARG, "the weights texture needs p (its jitter noise is the height function's sine mode)");
		if (want_w && !ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	}
	if (want_w && !ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called (the weights texture's jitter noise is sine mode)");
	bool const erode = (erosion_iters > 0 && ep && ep->erode_amount > 0.0);
	bool const sine = (!hs && p->gen_mode == TW_MGEN_SINE); // sine tables: one batched generation up front (twi_heightgen_sine_tiles), no schedule order
	// AO with a GPU gen mode: the context is generated once and the zvals are cut from it before erosion (src/tiled_mesh.cpp:479-487,505); rays read the un-eroded context
	bool const ctx_mode = want_ao && p->gen_mode >= TW_MGEN_SIMPLEX_GPU;
	uint32_t const stride = zvsize - 1, ray = 36, csz = stride + 2*ray; // AO_RAY_LEN, context_sz (src/tiled_mesh.cpp:43,601)
	size_t const tile_elems = (size_t)zvsize*zvsize, n = tile_elems*ntiles, nrm_elems = (size_t)stride*stride, ctx_elems = (size_t)csz*csz;
	bool const dev_out = tw_is_device_ptr(o->zvals), dev_nrm = want_normals && tw_is_device_ptr(o->normals_rgba);
	bool const dev_ao = want_ao && tw_is_device_ptr(sh->ao), dev_w = want_w && tw_is_device_ptr(sh->weights), dev_f = want_f && tw_is_device_ptr(sh->has_any_grass);
	bool const dev_tp = want_w && tw_is_device_ptr(sh->tile_params);
	auto al = [](size_t b) {return (b + 255) & ~(size_t)255;};
	rc = twi_ensure_aux_streams(ctx); if (rc) return rc;
	// The pipeline. Work per tile is heavy-tailed (ocean tiles: 1000 droplets x 1 move; mountain tiles: 1e5 moves in one serial chain), and a chain
	// cannot be sped up (csrc/tw_erosion.cu, plan_heavy), so the chains must START EARLY: (1) a coarse pre-pass evaluates the height function on an
	// 8x8 sample of every tile (4 M evaluations for 65536 tiles, < 1 ms) and counts the samples above the ocean-stop level - the same predictor the
	// erosion schedule uses, on 64 instead of 70756 cells; (2) the tiles are sorted heaviest first; (3) generation and erosion run chunk by chunk in
	// THAT order: generation of chunk k+1 (main stream) overlaps the droplet walks of chunks <= k (three high-priority streams; chunk 0, which holds
	// every long chain, has one to itself), so the long chains run under the generation of everything else and the last chunk to finish is the
	// lightest one. Each chunk's z range, sub-block bounds, normal map, AO map and weights texture follow its erosion on the same stream. Tiles are
	// generated / eroded in schedule order but stored at their caller-visible index (tile_perm). TW_PIPE_CHUNKS overrides the chunk count (1 = the
	// plain sequence); small batches use one chunk.
	// host-side origins of the context grids ((x1 - AO_RAY_LEN, y1 - AO_RAY_LEN), gen_ao_contexts) and of the jitter grids (80x the cell size, tw_tile_weights_batch)
	float const MESH_NOISE_FREQ = 80.0f;
	tw_grid2d gc = g; gc.nx = csz; gc.ny = csz;
	tw_grid2d gj = g; gj.dx = MESH_NOISE_FREQ*dx; gj.dy = MESH_NOISE_FREQ*dy; gj.nx = stride; gj.ny = stride;
	std::vector<float2> corg(want_ao ? ntiles : 0), jorg(want_w ? ntiles : 0);
	for (uint32_t t = 0; t < ntiles; ++t) {
		float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
		if (want_ao) {corg[t] = make_float2(dx*(float)(origins_xy[2*t] - (int32_t)ray - mesh_x_size/2), dy*(float)(origins_xy[2*t+1] - (int32_t)ray - mesh_y_size/2));}
		if (want_w) {jorg[t] = make_float2(gj.dx*x0, gj.dy*y0);}
	}
	twi_sine_batch sb_ctx, sb_jit; // sine tables of the sine-mode contexts and of the jitter grids: one plan (distinct columns / rows) each
	size_t const ctab_bytes = (want_ao && sine) ? al(twi_sine_tiles_plan(&gc, corg.data(), ntiles, &sb_ctx)) : 0, jtab_bytes = want_w ? al(twi_sine_tiles_plan(&gj, jorg.data(), ntiles, &sb_jit)) : 0;
	// slot 0: device staging of the host-bound arrays [zvals | normal maps | AO maps | weights | has_any_grass], then [tile_params | sine tables | context /
	// jitter grid buffers]. All but the buffers is reserved before the erosion budget is taken, so the budget sees that memory as used.
	size_t const z_bytes = dev_out ? 0 : al(n*sizeof(float)), nrm_bytes = (want_normals && !dev_nrm) ? al(ntiles*nrm_elems*4) : 0;
	size_t const ao_bytes = (want_ao && !dev_ao) ? al(ntiles*nrm_elems) : 0, w_bytes = (want_w && !dev_w) ? al(ntiles*nrm_elems*4) : 0, f_bytes = (want_f && !dev_f) ? al(ntiles) : 0;
	size_t const tp_bytes = (want_w && !dev_tp) ? al((size_t)ntiles*8*sizeof(float)) : 0;
	// mesh shadows, reused light after light: [mask staging (host smask) | 64-bit keys | x edges | y edges (outputs, then caller rows) | plan of every light]
	size_t const edge = (size_t)ntiles*zvsize, plan_bytes = al(twi_shadow_plan_ints(ntiles)*sizeof(int));
	bool sh_host_m = false, sh_in_x = false, sh_in_y = false;
	for (uint32_t l = 0; l < nl; ++l) {sh_host_m |= !sdev_m[l]; sh_in_x |= (lights[l].sh_in_x != nullptr); sh_in_y |= (lights[l].sh_in_y != nullptr);}
	size_t const shm_bytes = sh_host_m ? al(n + 4) : 0, shk_bytes = nl ? al(2*edge*sizeof(unsigned long long)) : 0;
	size_t const shx_bytes = nl ? al((sh_in_x ? 2 : 1)*edge*sizeof(float)) : 0, shy_bytes = nl ? al((sh_in_y ? 2 : 1)*edge*sizeof(float)) : 0;
	size_t const sh_bytes = shm_bytes + shk_bytes + shx_bytes + shy_bytes + nl*plan_bytes;
	size_t const fixed_bytes = z_bytes + nrm_bytes + ao_bytes + w_bytes + f_bytes + tp_bytes + ctab_bytes + jtab_bytes + sh_bytes;
	if (fixed_bytes) {rc = tw_reserve(ctx, 0, fixed_bytes); if (rc) return rc;}
	// AO context grids and weights jitter grids are per chunk (schedule order): written on the main stream, read on the chunk's erosion stream. The buffers
	// hold about 2 GB of context grids (or jitter grids without AO) in all, the bound tw_tile_ao_batch keeps; a chunk holds at most a third of that. When
	// the batch needs more chunks than buffers, chunk 0 (every long droplet chain) keeps its buffer and the later chunks take turns in the others: before the
	// main stream rewrites one it waits for the stream that last read it, which is never chunk 0's. Batches with one buffer per chunk never wait.
	size_t const RING = (size_t)2 << 30, ring_tile = (want_ao ? ctx_elems*sizeof(float) : 0) + (want_w ? nrm_elems*sizeof(float) : 0);
	size_t const bound_tile = want_ao ? ctx_elems*sizeof(float) : nrm_elems*sizeof(float);
	size_t const ring_max = ring_tile ? std::min((RING/bound_tile)*ring_tile, (size_t)ntiles*ring_tile) + 2*65536 : 0; // what the buffers can take, for the erosion budget
	uint32_t nchunks = 0, chunk = 0;
	size_t sbytes = 0;
	if (erode) {
		size_t free_b = 0, total_b = 0;
		TW_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
		size_t budget = (free_b + ctx->scratch_bytes[1] - std::min(free_b, ring_max))/3/3;
		if (budget < ((size_t)512 << 20)) budget = (size_t)512 << 20;
		// A few chunks let generation overlap the long droplet chains; when the batch saturates the machine anyway, generation and erosion compete for the same
		// issue slots and extra chunks only add overhead. tools/bench_pipeline_chunks.py on one H100, 258^2 tiles, 1000 droplets, heaviest-first: 8192 tiles
		// 0.159 / 0.147 / 0.139 / 0.148 s with 1 / 2 / 4 / 8 chunks; 16384 tiles 0.255 / 0.251 / 0.256 / 0.257 s; 65536 tiles 1.01 s with any of them
		uint32_t want_chunks = (ntiles < 4096) ? 1 : ((ntiles <= 24576) ? 4 : 2);
		if (const char *e = getenv("TW_PIPE_CHUNKS")) {int const v = atoi(e); if (v >= 1 && v <= 64) want_chunks = (uint32_t)v;}
		chunk = (ntiles + want_chunks - 1)/want_chunks;
		uint32_t const cap = twi_erode_chunk_for(budget, chunk, (int)zvsize, (int)zvsize);
		nchunks = (ntiles + cap - 1)/cap;
		chunk = (ntiles + nchunks - 1)/nchunks; // balanced
	}
	else { // height fill only: chunks bounded by the tile kernels' gridDim limit
		nchunks = (ntiles + 65534)/65535;
		chunk = (ntiles + nchunks - 1)/nchunks;
	}
	if (ring_tile) {
		uint32_t const cap = (uint32_t)std::max<size_t>(1, std::min<size_t>(65535, (RING/3)/bound_tile));
		if (chunk > cap) {nchunks = (ntiles + cap - 1)/cap; chunk = (ntiles + nchunks - 1)/nchunks;}
	}
	bool const reorder = (erode && nchunks > 1 && !sine && !getenv("TW_PIPE_NO_REORDER"));
	int const nes = (nchunks > 2) ? 3 : (int)nchunks; // aux streams / erosion scratch buffers
	uint32_t const nbuf = ring_tile ? (uint32_t)std::min<size_t>(nchunks, std::max<size_t>(3, RING/((size_t)chunk*bound_tile))) : 0;
	size_t const cz_bytes = want_ao ? al((size_t)chunk*ctx_elems*sizeof(float)) : 0, rand_bytes = want_w ? al((size_t)chunk*nrm_elems*sizeof(float)) : 0;
	size_t const ring_bytes = nbuf*(cz_bytes + rand_bytes);
	if (ring_bytes) {rc = tw_reserve(ctx, 0, fixed_bytes + ring_bytes); if (rc) return rc;}
	char *s0 = (char *)ctx->d_scratch[0];
	float *d_out = dev_out ? o->zvals : (float *)s0; s0 += z_bytes;
	unsigned char *d_rgba = !want_normals ? nullptr : (dev_nrm ? o->normals_rgba : (unsigned char *)s0); s0 += nrm_bytes;
	uint8_t *d_ao = !want_ao ? nullptr : (dev_ao ? sh->ao : (uint8_t *)s0); s0 += ao_bytes;
	uint8_t *d_w = !want_w ? nullptr : (dev_w ? sh->weights : (uint8_t *)s0); s0 += w_bytes;
	uint8_t *d_f = !want_f ? nullptr : (dev_f ? sh->has_any_grass : (uint8_t *)s0); s0 += f_bytes;
	const float *d_tp = !want_w ? nullptr : (dev_tp ? sh->tile_params : (const float *)s0); s0 += tp_bytes;
	char *d_ctab = s0; s0 += ctab_bytes;
	char *d_jtab = s0; s0 += jtab_bytes;
	unsigned char *d_shm = (unsigned char *)s0; s0 += shm_bytes;
	unsigned long long *d_shk = (unsigned long long *)s0; s0 += shk_bytes;
	float *d_shx = (float *)s0; s0 += shx_bytes;
	float *d_shy = (float *)s0; s0 += shy_bytes;
	char *d_shp = s0; s0 += nl*plan_bytes;
	char *d_ring = s0;
	if (erode) {
		sbytes = al(twi_erode_scratch_bytes(ctx, chunk, (int)zvsize, (int)zvsize));
		rc = tw_reserve(ctx, 1, sbytes*nes); if (rc) return rc; // before the sine tables claim the same slot: it is never re-allocated under the erosion
	}
	// slot 2: [small scalars | per-tile min/max | origins | sorted origins | work | order | hist(256) | coarse samples | sub-block bounds | min_normal_z |
	// context origins | sorted context origins]
	bool const ctx_org = want_ao && !sine; // the paired noise kernels read the context origins from the device
	uint32_t const CS = 8, cstep = (zvsize >= CS) ? zvsize/CS : 1;
	size_t const mm_bytes = al((size_t)ntiles*2*sizeof(unsigned)), org_bytes = al((size_t)ntiles*sizeof(float2));
	size_t const u_bytes = al((size_t)ntiles*sizeof(unsigned)), coarse_bytes = reorder ? al((size_t)ntiles*CS*CS*sizeof(float)) : 0;
	size_t const sub_bytes = want_bounds ? al((size_t)ntiles*16*sizeof(Sub)) : 0, mnz_bytes = want_mnz ? u_bytes : 0, corg_bytes = ctx_org ? org_bytes : 0;
	rc = tw_reserve(ctx, 2, OFF_TILES + mm_bytes + 2*org_bytes + 2*u_bytes + 1024 + coarse_bytes + sub_bytes + mnz_bytes + 2*corg_bytes); if (rc) return rc;
	char *s2 = (char *)ctx->d_scratch[2] + OFF_TILES;
	unsigned *d_mm = (unsigned *)s2; s2 += mm_bytes;
	float2 *d_org = (float2 *)s2; s2 += org_bytes;
	float2 *d_org_sorted = (float2 *)s2; s2 += org_bytes;
	unsigned *d_work = (unsigned *)s2; s2 += u_bytes;
	unsigned *d_order = (unsigned *)s2; s2 += u_bytes;
	unsigned *d_hist = (unsigned *)s2; s2 += 1024;
	float *d_coarse = (float *)s2; s2 += coarse_bytes;
	Sub *d_sub = (Sub *)s2; s2 += sub_bytes;
	unsigned *d_mnz = want_mnz ? (unsigned *)s2 : nullptr; s2 += mnz_bytes;
	float2 *d_corg = (float2 *)s2; s2 += corg_bytes;
	float2 *d_corg_sorted = (float2 *)s2;
	unsigned long long *d_steps = (unsigned long long *)((char *)ctx->d_scratch[2] + 2048);
	// pinned staging: inputs [origins | sine-mode index tables | context origins or their sine tables | jitter sine tables | tile_params | per light: shadow plan,
	// host sh_in_x, host sh_in_y], then the small results [steps | min/max | sub-block bounds | min_normal_z | has_any_grass] that the completing poll unpacks.
	// Every sine batch has its own region, and the caller's origins, tile_params, tile_xy and host sh_in rows may be reused as soon as this function returns.
	size_t const in_org = al((size_t)ntiles*sizeof(float2)), in_sine = sine ? al(twi_sine_tiles_stage_bytes(ntiles)) : 0;
	size_t const in_ctx = !want_ao ? 0 : (sine ? al(twi_sine_tiles_stage_bytes(ntiles)) : in_org), in_jit = want_w ? al(twi_sine_tiles_stage_bytes(ntiles)) : 0;
	size_t const in_tp = tp_bytes, off_ctx = in_org + in_sine, off_jit = off_ctx + in_ctx, off_tp = off_jit + in_jit, off_sh = off_tp + in_tp;
	std::vector<size_t> off_six(nl), off_siy(nl);
	size_t in_sh = nl*plan_bytes;
	for (uint32_t l = 0; l < nl; ++l) {
		off_six[l] = off_sh + in_sh; in_sh += (lights[l].sh_in_x && !sdev_ix[l]) ? al(edge*sizeof(float)) : 0;
		off_siy[l] = off_sh + in_sh; in_sh += (lights[l].sh_in_y && !sdev_iy[l]) ? al(edge*sizeof(float)) : 0;
	}
	size_t const off_steps = off_sh + in_sh, off_mm = off_steps + 256, off_sub = off_mm + (want_mm ? mm_bytes : 0), off_mnz = off_sub + sub_bytes, off_f = off_mnz + mnz_bytes;
	rc = tw_reserve_pinned(ctx, off_f + (want_f ? al(ntiles) : 0)); if (rc) return rc;
	char *h_stage = (char *)ctx->h_pinned;
	float2 *h_org = (float2 *)h_stage;
	if (hs) {memcpy(h_stage, origins_xy, (size_t)ntiles*2*sizeof(int32_t));} // the sampler reads the int (x1, y1) origins (d_org then holds int2)
	else {
		for (uint32_t t = 0; t < ntiles; ++t) { // build_arrays((x1 - MESH_X_SIZE/2), (y1 - MESH_Y_SIZE/2), ...): int -> float, mx0 = dx*x0 (src/tiled_mesh.cpp:461, src/mesh_gen.cpp:591)
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			h_org[t] = make_float2(dx*x0, dy*y0);
		}
	}
	if (!sine) {TW_CUDA(ctx, cudaMemcpyAsync(d_org, h_org, (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));}
	if (ctx_org) {
		memcpy(h_stage + off_ctx, corg.data(), (size_t)ntiles*sizeof(float2));
		TW_CUDA(ctx, cudaMemcpyAsync(d_corg, h_stage + off_ctx, (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
	}
	if (tp_bytes) {
		memcpy(h_stage + off_tp, sh->tile_params, (size_t)ntiles*8*sizeof(float));
		TW_CUDA(ctx, cudaMemcpyAsync((void *)d_tp, h_stage + off_tp, (size_t)ntiles*8*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	}
	for (uint32_t l = 0; l < nl; ++l) { // the plans go up now; host sh_in rows wait in the staging until their light's pass copies them into the edge buffers
		twi_shadow_plan_pack(splan[l], (int *)(h_stage + off_sh + l*plan_bytes));
		TW_CUDA(ctx, cudaMemcpyAsync(d_shp + l*plan_bytes, h_stage + off_sh + l*plan_bytes, twi_shadow_plan_ints(ntiles)*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
		if (lights[l].sh_in_x && !sdev_ix[l]) {memcpy(h_stage + off_six[l], lights[l].sh_in_x, edge*sizeof(float));}
		if (lights[l].sh_in_y && !sdev_iy[l]) {memcpy(h_stage + off_siy[l], lights[l].sh_in_y, edge*sizeof(float));}
	}
	if (want_f) {TW_CUDA(ctx, cudaMemsetAsync(d_f, 0, ntiles, ctx->stream));}
	if (erode) {TW_CUDA(ctx, cudaMemsetAsync(d_steps, 0, sizeof(unsigned long long), ctx->stream));} // the aux streams see it through the chunk events
	if (want_mnz) {rc = twi_fill_u32(ctx, ctx->stream, d_mnz, ntiles, tw_f2ord(1.0f)); if (rc) return rc;} // min_normal_z = 1.0, src/tiled_mesh.cpp:868
	const float2 *d_gen_org = d_org, *d_gen_corg = d_corg;
	const unsigned *d_perm = nullptr;
	if (reorder) { // (1) + (2): coarse estimate, heaviest-first order of the WHOLE batch
		if (hs) {rc = twi_hmap_sample_tiles(ctx, ctx->d_hmap, hs, d_org, ntiles, CS, d_coarse, ctx->stream, nullptr, cstep); if (rc) return rc;}
		else {
			tw_grid2d gcs = g; gcs.dx = dx*(float)cstep; gcs.dy = dy*(float)cstep; gcs.nx = CS; gcs.ny = CS;
			for (uint32_t t0 = 0; t0 < ntiles; t0 += 65535) {
				uint32_t const nt = (ntiles - t0 < 65535) ? ntiles - t0 : 65535;
				rc = twi_heightgen(ctx, &gcs, p, 1, 0, d_org + t0, nt, d_coarse + (size_t)t0*CS*CS, nullptr); if (rc) return rc;
			}
		}
		rc = twi_coarse_work(ctx, d_coarse, CS*CS, ntiles, ep->water_plane_z - ep->half_dxy, d_work); if (rc) return rc;
		TW_CUDA(ctx, cudaMemsetAsync(d_hist, 0, 1024, ctx->stream));
		rc = twi_order_by_work(ctx, ctx->stream, d_work, ntiles, CS*CS, d_hist, d_order); if (rc) return rc;
		if (!hs) {rc = twi_gather_origins(ctx, d_org, d_order, ntiles, d_org_sorted); if (rc) return rc;} // the sampler reads its origins through the permutation
		if (ctx_org) {rc = twi_gather_origins(ctx, d_corg, d_order, ntiles, d_corg_sorted); if (rc) return rc; d_gen_corg = d_corg_sorted;}
		d_gen_org = d_org_sorted; d_perm = d_order;
	}
	if (sine) {rc = twi_heightgen_sine_tiles(ctx, &g, p, 1, 0, h_org, ntiles, d_out, nullptr, h_stage + in_org); if (rc) return rc;}
	if (want_ao && sine) {rc = twi_sine_tiles_setup(ctx, &gc, p, 1, 0, corg.data(), ntiles, d_ctab, h_stage + off_ctx, &sb_ctx); if (rc) return rc;}
	if (want_w) { // force_sine_mode: gen_mode = MGEN_SINE, gen_shape = 0 (src/mesh_gen.cpp:592-593); no glaciate, start index >= 50 (src/tiled_mesh.cpp:1103)
		tw_height_params ps = *p;
		ps.gen_mode = TW_MGEN_SINE; ps.gen_shape = 0;
		rc = twi_sine_tiles_setup(ctx, &gj, &ps, 0, 50, jorg.data(), ntiles, d_jtab, h_stage + off_jit, &sb_jit); if (rc) return rc;
	}
	auto chain = [](cudaStream_t from, cudaStream_t to) -> bool { // `to` waits for what `from` has enqueued so far
		cudaEvent_t ev = nullptr;
		bool const ok = (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess && cudaEventRecord(ev, from) == cudaSuccess && cudaStreamWaitEvent(to, ev, 0) == cudaSuccess);
		if (ev) cudaEventDestroy(ev); // released once the device has passed it
		return ok;
	};
	std::vector<cudaEvent_t> ring_ev(nbuf, nullptr); // recorded on the stream that last read each buffer
	bool used[3] = {false, false, false};
	int status = TW_OK;
	for (uint32_t k = 0; k < nchunks && status == TW_OK; ++k) {
		uint32_t const t0 = k*chunk, nt = (ntiles - t0 < chunk) ? (ntiles - t0) : chunk;
		// schedule slots [t0, t0 + nt): with a permutation every kernel addresses `d_out` (and the per-tile results) through it; without, the chunk is a contiguous slice
		float *maps = d_perm ? d_out : d_out + (size_t)t0*tile_elems;
		size_t const r0 = d_perm ? 0 : t0; // first result slot the chunk's kernels address directly
		const unsigned *perm_k = d_perm ? d_perm + t0 : nullptr;
		uint32_t const b = (k < nbuf) ? k : 1 + (k - 1) % (nbuf - 1); // buffer 0 stays chunk 0's
		float *d_cz = (float *)(d_ring + b*(cz_bytes + rand_bytes)), *d_rand = (float *)(d_ring + b*(cz_bytes + rand_bytes) + cz_bytes);
		bool const reuse = (nbuf && ring_ev[b]); // the main stream waits right before its first write into the buffer
		if (ctx_mode && reuse && cudaStreamWaitEvent(ctx->stream, ring_ev[b], 0) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
		if (ctx_mode) { // contexts in schedule order, zvals cut from their interiors into the caller-visible slots
			status = twi_heightgen(ctx, &gc, p, 1, 0, d_gen_corg + t0, nt, d_cz, nullptr); if (status) break;
			status = twi_tile_cut(ctx, ctx->stream, d_cz, nt, zvsize, maps, perm_k); if (status) break;
		}
		else if (hs) {status = twi_hmap_sample_tiles(ctx, ctx->d_hmap, hs, d_perm ? (const void *)d_org : (const void *)(d_org + t0), nt, zvsize, maps, ctx->stream, perm_k); if (status) break;}
		else if (!sine) {
			ctx->tile_perm = perm_k;
			status = twi_heightgen(ctx, &g, p, 1, 0, d_gen_org + t0, nt, maps, nullptr);           // generation on ctx->stream
			ctx->tile_perm = nullptr;
			if (status) break;
		}
		int const lane = (nes < 3) ? (int)(k % nes) : ((k == 0) ? 0 : 1 + (int)((k - 1) & 1)); // the heaviest chunk keeps a stream (and a scratch buffer) to itself
		cudaStream_t const es = ctx->aux_stream[lane];
		if (!chain(ctx->stream, es)) {status = tw_set_error(ctx, TW_ERR_CUDA, "chunk event"); break;}
		used[lane] = true;
		if (erode) {status = twi_erode_enqueue(ctx, es, 1 + lane, (char *)ctx->d_scratch[1] + (size_t)lane*sbytes, chunk, maps, nt, (int)zvsize, (int)zvsize, nullptr, min_zval, erosion_iters, ep, d_steps, perm_k); if (status) break;}
		// the rest of the chunk's main-stream work runs under its erosion: CPU-mode contexts (outside the tile only) and jitter grids
		if (!ctx_mode && reuse && cudaStreamWaitEvent(ctx->stream, ring_ev[b], 0) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
		if (want_ao && !ctx_mode) {
			if (sine) {status = twi_sine_tiles_grid(ctx, &sb_ctx, t0, nt, nullptr, d_cz, nullptr);}
			else {
				ctx->skip_rect[0] = ctx->skip_rect[1] = ray; ctx->skip_rect[2] = ctx->skip_rect[3] = zvsize;
				status = twi_heightgen(ctx, &gc, p, 1, 0, d_gen_corg + t0, nt, d_cz, nullptr);
				ctx->skip_rect[0] = ctx->skip_rect[1] = ctx->skip_rect[2] = ctx->skip_rect[3] = 0;
			}
			if (status) break;
		}
		if (want_w) {status = twi_sine_tiles_grid(ctx, &sb_jit, t0, nt, d_perm, d_rand, nullptr); if (status) break;}
		if (want_mm) {status = twi_minmax_tiles(ctx, es, maps, tile_elems, nt, d_mm + 2*r0, perm_k); if (status) break;}
		if (want_bounds) {status = twi_tile_bounds(ctx, es, maps, nt, zvsize, wpz_max, d_sub + 16*r0, perm_k); if (status) break;}
		if (want_normals) {status = twi_tile_normals(ctx, es, maps, nt, zvsize, dx, dy, d_rgba + r0*nrm_elems*4, d_mnz ? d_mnz + r0 : nullptr, perm_k); if (status) break;}
		if (((want_ao && !ctx_mode) || want_w) && !chain(ctx->stream, es)) {status = tw_set_error(ctx, TW_ERR_CUDA, "chunk event"); break;}
		if (want_ao) {status = twi_tile_ao(ctx, es, maps, d_cz, nt, zvsize, sh->half_dxy, ctx_mode, d_ao + r0*nrm_elems, perm_k); if (status) break;}
		if (want_w) {status = twi_tile_weights(ctx, es, maps, d_rand, nt, zvsize, d_tp + r0*8, &W, d_w + r0*nrm_elems*4, d_f ? d_f + r0 : nullptr, perm_k); if (status) break;}
		if (nbuf) {
			if (!ring_ev[b] && cudaEventCreateWithFlags(&ring_ev[b], cudaEventDisableTiming) != cudaSuccess) {ring_ev[b] = nullptr; status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
			if (cudaEventRecord(ring_ev[b], es) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
		}
		if (!dev_out && !d_perm && cudaMemcpyAsync(o->zvals + (size_t)t0*tile_elems, maps, (size_t)nt*tile_elems*sizeof(float), cudaMemcpyDeviceToHost, es) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "D2H");}
	}
	ctx->tile_perm = nullptr;
	ctx->skip_rect[0] = ctx->skip_rect[1] = ctx->skip_rect[2] = ctx->skip_rect[3] = 0;
	for (cudaEvent_t ev : ring_ev) {if (ev) cudaEventDestroy(ev);} // every wait on them is enqueued
	for (int l = 0; l < 3; ++l) { // join: ctx->stream (and so the job's event) follows everything the chunks enqueued
		if (used[l] && !chain(ctx->aux_stream[l], ctx->stream) && status == TW_OK) status = tw_set_error(ctx, TW_ERR_CUDA, "join event");
	}
	if (status) { // nothing may still run on the scratch buffers when the error is returned
		cudaStreamSynchronize(ctx->stream);
		for (int l = 0; l < 3; ++l) {cudaStreamSynchronize(ctx->aux_stream[l]);}
		return status;
	}
	// mesh shadows on ctx->stream, light after light through the same buffers: every tile's neighbours have their final heights once the chunks are joined
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_light const &L = lights[l];
		unsigned char *d_m = sdev_m[l] ? L.smask : d_shm;
		if (L.sh_in_x) {TW_CUDA(ctx, cudaMemcpyAsync(d_shx + edge, sdev_ix[l] ? (const void *)L.sh_in_x : h_stage + off_six[l], edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		if (L.sh_in_y) {TW_CUDA(ctx, cudaMemcpyAsync(d_shy + edge, sdev_iy[l] ? (const void *)L.sh_in_y : h_stage + off_siy[l], edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		rc = twi_shadow_enqueue(ctx, ctx->stream, splan[l], d_out, ntiles, zvsize, d_m, d_shk, d_shx, d_shy, (const int *)(d_shp + l*plan_bytes), true); if (rc) return rc;
		if (!sdev_m[l]) {TW_CUDA(ctx, cudaMemcpyAsync(L.smask, d_m, n, cudaMemcpyDeviceToHost, ctx->stream));}
		if (L.sh_out_x) {TW_CUDA(ctx, cudaMemcpyAsync(L.sh_out_x, d_shx, edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		if (L.sh_out_y) {TW_CUDA(ctx, cudaMemcpyAsync(L.sh_out_y, d_shy, edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
	}
	// every host-bound result is copied once, at the end: the schedule order scatters a chunk over the whole batch
	if (!dev_out && d_perm) {TW_CUDA(ctx, cudaMemcpyAsync(o->zvals, d_out, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_normals && !dev_nrm) {TW_CUDA(ctx, cudaMemcpyAsync(o->normals_rgba, d_rgba, (size_t)ntiles*nrm_elems*4, cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_ao && !dev_ao) {TW_CUDA(ctx, cudaMemcpyAsync(sh->ao, d_ao, (size_t)ntiles*nrm_elems, cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_w && !dev_w) {TW_CUDA(ctx, cudaMemcpyAsync(sh->weights, d_w, (size_t)ntiles*nrm_elems*4, cudaMemcpyDeviceToHost, ctx->stream));}
	if (erode) {TW_CUDA(ctx, cudaMemcpyAsync(h_stage + off_steps, d_steps, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_mm) {TW_CUDA(ctx, cudaMemcpyAsync(h_stage + off_mm, d_mm, (size_t)ntiles*2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_bounds) {TW_CUDA(ctx, cudaMemcpyAsync(h_stage + off_sub, d_sub, (size_t)ntiles*16*sizeof(Sub), cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_mnz) {TW_CUDA(ctx, cudaMemcpyAsync(h_stage + off_mnz, d_mnz, (size_t)ntiles*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
	if (want_f && !dev_f) {TW_CUDA(ctx, cudaMemcpyAsync(h_stage + off_f, d_f, ntiles, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaEventRecord(ctx->async.done, ctx->stream));
	tw_async_state &a = ctx->async;
	a.pending = true; a.tiles = true; a.steps = erode; a.n_mm = ntiles;
	a.host_mm = o->mm; a.host_bounds = o->bounds; a.host_min_nz = o->min_normal_z; a.host_flags = (want_f && !dev_f) ? sh->has_any_grass : nullptr;
	a.dx = dx; a.dy = dy; a.size = size;
	a.off_steps = off_steps; a.off_mm = off_mm; a.off_sub = off_sub; a.off_min_nz = off_mnz; a.off_flags = off_f;
	return TW_OK;
}

int tw_create_tiles_launch_shadows(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                   uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                                   float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	ctx->last_erosion_steps = 0;
	return tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, shadows, nullptr);
}

int tw_set_heightmap(tw_ctx *ctx, const uint8_t *data16, int width, int height) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (data16 && (width <= 0 || height <= 0)) return tw_set_error(ctx, TW_ERR_ARG, "heightmap size %d x %d", width, height);
	size_t const bytes = (size_t)2*width*height, had = (size_t)2*ctx->hmap_w*ctx->hmap_h;
	if (ctx->d_hmap && (!data16 || bytes != had)) {TW_CUDA(ctx, cudaFree(ctx->d_hmap)); ctx->d_hmap = nullptr;}
	ctx->hmap_w = ctx->hmap_h = 0;
	if (!data16) return TW_OK;
	if (!ctx->d_hmap) {TW_CUDA(ctx, cudaMalloc(&ctx->d_hmap, bytes));}
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_hmap, data16, bytes, cudaMemcpyDefault, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // data16 is the caller's buffer
	ctx->hmap_w = width; ctx->hmap_h = height;
	return TW_OK;
}

int tw_create_tiles_launch_hmap(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                                float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!ctx->hmap_w) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_heightmap() has not been called");
	if (!hs) return tw_set_error(ctx, TW_ERR_ARG, "null heightmap sampler");
	if (hs->width != ctx->hmap_w || hs->height != ctx->hmap_h) return tw_set_error(ctx, TW_ERR_ARG, "sampler size %d x %d differs from the heightmap's %d x %d", hs->width, hs->height, ctx->hmap_w, ctx->hmap_h);
	if (hs->edge_mode < 0 || hs->edge_mode > 2) return tw_set_error(ctx, TW_ERR_ARG, "bad edge_mode %d", hs->edge_mode);
	if (shading && shading->ao) return tw_set_error(ctx, TW_ERR_ARG, "the AO map is not available for heightmap tiles (its context outside the tile is not defined in this mode)");
	ctx->last_erosion_steps = 0;
	return tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, shadows, hs);
}

int tw_create_tiles_launch_ex(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                              uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                              float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading)
{
	return tw_create_tiles_launch_shadows(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, nullptr);
}

int tw_create_tiles_launch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                           uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                           float wpz_max, uint32_t size, const tw_tile_outputs *out)
{
	return tw_create_tiles_launch_ex(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, nullptr);
}

int tw_create_tiles_poll(tw_ctx *ctx, int wait) {
	int rc = check_ctx(ctx); if (rc) return rc;
	return poll_job(ctx, wait);
}

int tw_create_zvals_batch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                          uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                          float *out, tw_minmax *mm)
{
	tw_tile_outputs o;
	memset(&o, 0, sizeof(o));
	o.zvals = out; o.mm = mm;
	int rc = tw_create_tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, 0.0f, 0, &o);
	if (rc) return rc;
	return poll_job(ctx, 1);
}

int tw_heightmap_sample_tiles(tw_ctx *ctx, const uint8_t *data16, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, uint32_t zvsize, float *out) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!data16 || !hs || !origins_xy || !out || ntiles == 0 || zvsize == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (hs->width <= 0 || hs->height <= 0 || hs->edge_mode < 0 || hs->edge_mode > 2) return tw_set_error(ctx, TW_ERR_ARG, "bad heightmap sampler");
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	size_t const img_bytes = ((size_t)2*hs->width*hs->height + 255) & ~(size_t)255, org_bytes = ((size_t)ntiles*8 + 255) & ~(size_t)255;
	size_t const out_bytes = (size_t)ntiles*zvsize*zvsize*sizeof(float);
	bool const dev_img = tw_is_device_ptr(data16), dev_out = tw_is_device_ptr(out);
	rc = tw_reserve(ctx, 0, org_bytes + (dev_img ? 0 : img_bytes) + (dev_out ? 0 : out_bytes) + 256); if (rc) return rc;
	char *sp = (char *)ctx->d_scratch[0];
	void *d_org = sp; sp += org_bytes;
	TW_CUDA(ctx, cudaMemcpyAsync(d_org, origins_xy, (size_t)ntiles*8, cudaMemcpyHostToDevice, ctx->stream));
	const uint8_t *d_img = data16;
	if (!dev_img) {TW_CUDA(ctx, cudaMemcpyAsync(sp, data16, (size_t)2*hs->width*hs->height, cudaMemcpyHostToDevice, ctx->stream)); d_img = (const uint8_t *)sp; sp += img_bytes;}
	float *d_out = dev_out ? out : (float *)sp;
	rc = twi_hmap_sample_tiles(ctx, d_img, hs, d_org, ntiles, zvsize, d_out); if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // origins_xy is the caller's buffer
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ per-tile normals and ambient occlusion (N1)
int tw_tile_normals_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float dx_val, float dy_val, uint8_t *rgba, float *min_normal_z) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!zvals || !rgba || ntiles == 0 || zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	size_t const n = (size_t)ntiles*zvsize*zvsize, stride = zvsize - 1, out_bytes = (size_t)ntiles*stride*stride*4;
	bool const dev_in = tw_is_device_ptr(zvals), dev_out = tw_is_device_ptr(rgba);
	size_t const in_bytes = (n*sizeof(float) + 255) & ~(size_t)255, mn_bytes = ((size_t)ntiles*sizeof(unsigned) + 255) & ~(size_t)255;
	rc = tw_reserve(ctx, 0, (dev_in ? 0 : in_bytes) + (dev_out ? 0 : out_bytes) + mn_bytes + 256); if (rc) return rc;
	char *sp = (char *)ctx->d_scratch[0];
	unsigned *d_mn = (unsigned *)sp; sp += mn_bytes;
	const float *d_z = zvals;
	if (!dev_in) {TW_CUDA(ctx, cudaMemcpyAsync(sp, zvals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_z = (const float *)sp; sp += in_bytes;}
	unsigned char *d_rgba = dev_out ? rgba : (unsigned char *)sp;
	{
		std::vector<unsigned> init(ntiles, tw_f2ord(1.0f)); // min_normal_z = 1.0, src/tiled_mesh.cpp:868
		TW_CUDA(ctx, cudaMemcpyAsync(d_mn, init.data(), ntiles*sizeof(unsigned), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	rc = twi_tile_normals(ctx, ctx->stream, d_z, ntiles, zvsize, dx_val, dy_val, d_rgba, d_mn); if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(rgba, d_rgba, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
	std::vector<unsigned> mn(ntiles);
	if (min_normal_z) {TW_CUDA(ctx, cudaMemcpyAsync(mn.data(), d_mn, ntiles*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (min_normal_z) {for (uint32_t t = 0; t < ntiles; ++t) {min_normal_z[t] = tw_ord2f(mn[t]);}}
	return TW_OK;
}

// context grids of `nt` tiles at (x1 - AO_RAY_LEN, y1 - AO_RAY_LEN) into d_cz; skip_inside: leave the zvsize^2 interior unwritten (never read)
static int gen_ao_contexts(tw_ctx *ctx, const int32_t *origins_xy, uint32_t nt, int mesh_x_size, int mesh_y_size, float dx, float dy, uint32_t zvsize,
                           const tw_height_params *p, bool skip_inside, std::vector<int32_t> &org, float *d_cz)
{
	uint32_t const ray = 36, csz = zvsize - 1 + 2*ray; // AO_RAY_LEN, context_sz (src/tiled_mesh.cpp:43,601)
	for (uint32_t t = 0; t < nt; ++t) {org[2*t] = origins_xy[2*t] - (int32_t)ray; org[2*t + 1] = origins_xy[2*t + 1] - (int32_t)ray;}
	if (skip_inside) {ctx->skip_rect[0] = ctx->skip_rect[1] = ray; ctx->skip_rect[2] = ctx->skip_rect[3] = zvsize;}
	int const rc = tw_heightgen_tiles(ctx, org.data(), nt, mesh_x_size, mesh_y_size, dx, dy, csz, p, d_cz, nullptr); // device output: scratch slot 0 is not touched
	ctx->skip_rect[0] = ctx->skip_rect[1] = ctx->skip_rect[2] = ctx->skip_rect[3] = 0;
	return rc;
}

int tw_tile_ao_batch(tw_ctx *ctx, const float *zvals, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size,
                     float dx, float dy, uint32_t zvsize, const tw_height_params *p, float half_dxy, uint8_t *ao)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!zvals || !origins_xy || !p || !ao || ntiles == 0 || zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	uint32_t const ray = 36, stride = zvsize - 1, csz = stride + 2*ray; // AO_RAY_LEN, context_sz (src/tiled_mesh.cpp:43,601)
	size_t const tile_elems = (size_t)zvsize*zvsize, ctx_elems = (size_t)csz*csz, ao_elems = (size_t)stride*stride;
	bool const dev_in = tw_is_device_ptr(zvals), dev_out = tw_is_device_ptr(ao);
	bool const ctx_inside = (p->gen_mode >= TW_MGEN_SIMPLEX_GPU); // use_ao_zvals: the rays test the un-eroded context inside the tile too (src/tiled_mesh.cpp:604)
	// chunk of tiles whose context grids fit in ~2 GB
	uint32_t chunk = (uint32_t)std::min<size_t>(ntiles, std::max<size_t>(1, ((size_t)2 << 30)/(ctx_elems*sizeof(float))));
	if (chunk > 65535) chunk = 65535;
	size_t const in_bytes = ((size_t)chunk*tile_elems*sizeof(float) + 255) & ~(size_t)255, cz_bytes = ((size_t)chunk*ctx_elems*sizeof(float) + 255) & ~(size_t)255;
	size_t const ao_bytes = ((size_t)chunk*ao_elems + 255) & ~(size_t)255;
	rc = tw_reserve(ctx, 0, (dev_in ? 0 : in_bytes) + cz_bytes + (dev_out ? 0 : ao_bytes) + 256); if (rc) return rc;
	std::vector<int32_t> org(2*(size_t)chunk);
	for (uint32_t t0 = 0; t0 < ntiles; t0 += chunk) {
		uint32_t const nt = (ntiles - t0 < chunk) ? ntiles - t0 : chunk;
		char *sp = (char *)ctx->d_scratch[0];
		float *d_cz = (float *)sp; sp += cz_bytes;
		const float *d_z = zvals + (size_t)t0*tile_elems;
		if (!dev_in) {TW_CUDA(ctx, cudaMemcpyAsync(sp, d_z, (size_t)nt*tile_elems*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_z = (const float *)sp; sp += in_bytes;}
		unsigned char *d_ao = dev_out ? ao + (size_t)t0*ao_elems : (unsigned char *)sp;
		rc = gen_ao_contexts(ctx, origins_xy + 2*(size_t)t0, nt, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, !ctx_inside, org, d_cz);
		if (rc) return rc;
		rc = twi_tile_ao(ctx, ctx->stream, d_z, d_cz, nt, zvsize, half_dxy, ctx_inside, d_ao); if (rc) return rc;
		if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(ao + (size_t)t0*ao_elems, d_ao, (size_t)nt*ao_elems, cudaMemcpyDeviceToHost, ctx->stream));}
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	return TW_OK;
}

int tw_create_zvals_ao_batch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                             uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                             float half_dxy, float *zvals, uint8_t *ao, tw_minmax *mm)
{
	if (!ao) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	tw_tile_outputs o;
	memset(&o, 0, sizeof(o));
	o.zvals = zvals; o.mm = mm;
	tw_tile_shading sh;
	memset(&sh, 0, sizeof(sh));
	sh.half_dxy = half_dxy; sh.ao = ao;
	int rc = tw_create_tiles_launch_ex(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, 0.0f, 0, &o, &sh);
	if (rc) return rc;
	return poll_job(ctx, 1);
}

// ------------------------------------------------------------------------------------------------ point queries
int tw_eval_points(tw_ctx *ctx, const float *xy, size_t n, const tw_height_params *p, const tw_point_query *q, float *out) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!xy || !p || !q || !out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (n == 0) return TW_OK;
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	bool const dev_in = tw_is_device_ptr(xy), dev_out = tw_is_device_ptr(out);
	size_t const in_bytes = (2*n*sizeof(float) + 255) & ~(size_t)255, out_bytes = n*sizeof(float);
	size_t const need = (dev_in ? 0 : in_bytes) + (dev_out ? 0 : out_bytes);
	if (need) {rc = tw_reserve(ctx, 0, need); if (rc) return rc;}
	const float *d_xy = xy; float *d_out = out;
	char *sp = (char *)ctx->d_scratch[0];
	if (!dev_in) {
		d_xy = (const float *)sp; sp += in_bytes;
		TW_CUDA(ctx, cudaMemcpyAsync((void *)d_xy, xy, 2*n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	}
	if (!dev_out) {d_out = (float *)sp;}
	rc = twi_eval_points(ctx, d_xy, n, p, q, d_out);
	if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_erode(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p) {
	return tw_erode_tiles(ctx, heightmap, 1, xsize, ysize, nullptr, min_zval, num_iters, p);
}

int tw_erode_parallel(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p, uint32_t num_threads) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!heightmap || !p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (xsize <= 0 || ysize <= 0) return tw_set_error(ctx, TW_ERR_ARG, "empty heightmap");
	if (num_iters == 0 || p->erode_amount <= 0.0) {ctx->last_erosion_steps = 0; return TW_OK;} // src/erosion.cpp:16
	size_t const n = (size_t)xsize*ysize;
	bool const dev = tw_is_device_ptr(heightmap);
	float *d_map = heightmap;
	if (!dev) {
		rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc;
		d_map = (float *)ctx->d_scratch[0];
		TW_CUDA(ctx, cudaMemcpyAsync(d_map, heightmap, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	}
	rc = twi_erode_parallel(ctx, d_map, xsize, ysize, min_zval, num_iters, p, num_threads);
	if (rc) return rc;
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(heightmap, d_map, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ voxels
int tw_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *out) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!vp || !out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	if (vp->gen_mode < 0 || vp->gen_mode > TW_MGEN_DWARP_GPU) return tw_set_error(ctx, TW_ERR_ARG, "bad gen_mode");
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	bool const dev_out = tw_is_device_ptr(out);
	float *d_out = out;
	if (!dev_out) {rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc; d_out = (float *)ctx->d_scratch[0];}
	rc = twi_voxel_fill(ctx, vp, rdata420, d_out);
	if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(out, d_out, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ streaming passes
int tw_heightmap_from_floats_u16(tw_ctx *ctx, const float *vals, size_t n, float val_mult, float val_add, uint8_t *out2n) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!vals || !out2n || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	bool const dev_in = tw_is_device_ptr(vals), dev_out = tw_is_device_ptr(out2n);
	size_t const in_bytes = n*sizeof(float), out_bytes = 2*n;
	size_t const need = (dev_in ? 0 : in_bytes) + (dev_out ? 0 : out_bytes);
	if (need) {rc = tw_reserve(ctx, 0, need + 256); if (rc) return rc;}
	rc = tw_reserve(ctx, 2, OFF_TILES); if (rc) return rc;
	const float *d_in = vals; uint8_t *d_out = out2n;
	char *s = (char *)ctx->d_scratch[0];
	if (!dev_in) {d_in = (const float *)s; TW_CUDA(ctx, cudaMemcpyAsync(s, vals, in_bytes, cudaMemcpyHostToDevice, ctx->stream)); s += (in_bytes + 255) & ~(size_t)255;}
	if (!dev_out) {d_out = (uint8_t *)s;}
	unsigned *d_bad = (unsigned *)((char *)ctx->d_scratch[2] + OFF_BAD);
	TW_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(unsigned), ctx->stream));
	rc = twi_from_floats_u16(ctx, d_in, n, val_mult, val_add, d_out, d_bad);
	if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(out2n, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
	unsigned bad = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (bad) return tw_set_error(ctx, TW_ERR_ARG, "from_floats: value outside [0,256) (the reference asserts, src/heightmap.cpp:211)");
	return TW_OK;
}

int tw_heightmap_to_floats_u16(tw_ctx *ctx, const uint8_t *data2n, size_t n, float val_mult, float val_add, float *vals) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!vals || !data2n || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	bool const dev_in = tw_is_device_ptr(data2n), dev_out = tw_is_device_ptr(vals);
	size_t const in_bytes = 2*n, out_bytes = n*sizeof(float);
	size_t const need = (dev_in ? 0 : in_bytes) + (dev_out ? 0 : out_bytes);
	if (need) {rc = tw_reserve(ctx, 0, need + 256); if (rc) return rc;}
	const uint8_t *d_in = data2n; float *d_out = vals;
	char *s = (char *)ctx->d_scratch[0];
	if (!dev_out) {d_out = (float *)s; s += (out_bytes + 255) & ~(size_t)255;}
	if (!dev_in) {d_in = (const uint8_t *)s; TW_CUDA(ctx, cudaMemcpyAsync(s, data2n, in_bytes, cudaMemcpyHostToDevice, ctx->stream));}
	rc = twi_to_floats_u16(ctx, d_in, n, val_mult, val_add, d_out);
	if (rc) return rc;
	if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(vals, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_proc_gen_heightmap(tw_ctx *ctx, uint32_t width, uint32_t height, float dx_val, float dy_val, const tw_height_params *p,
                          uint32_t erosion_iters, const tw_erosion_params *ep, uint8_t *data16, float *vals, tw_heightmap_info *info)
{
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!p || !data16 || width == 0 || height == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	tw_grid2d g; g.x0 = -0.5*width; g.y0 = -0.5*height; g.dx = dx_val; g.dy = dy_val; g.nx = width; g.ny = height; // src/heightmap.cpp:135
	size_t const n = (size_t)width*height;
	bool const vals_dev = (vals && tw_is_device_ptr(vals)), out_dev = tw_is_device_ptr(data16);
	// slot 0: [vals (if not given on the device)] [u16 image (if not given on the device)]
	size_t const vbytes = (n*sizeof(float) + 255) & ~(size_t)255;
	rc = tw_reserve(ctx, 0, (vals_dev ? 0 : vbytes) + (out_dev ? 0 : 2*n) + 256); if (rc) return rc;
	char *s0 = (char *)ctx->d_scratch[0];
	float *d_vals = vals_dev ? vals : (float *)s0;
	if (!vals_dev) {s0 += vbytes;}
	uint8_t *d_img = out_dev ? data16 : (uint8_t *)s0;
	rc = validate_height(ctx, &g, p, d_vals); if (rc) return rc;
	rc = tw_reserve(ctx, 2, OFF_TILES); if (rc) return rc;
	unsigned *d_mm = (unsigned *)((char *)ctx->d_scratch[2] + OFF_MM);
	tw_minmax mm;
	rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
	rc = twi_heightgen(ctx, &g, p, 1, 0, nullptr, 1, d_vals, d_mm); if (rc) return rc;
	rc = read_minmax(ctx, d_mm, &mm, 1); if (rc) return rc;
	uint64_t moves = 0;
	if (erosion_iters > 0 && ep && ep->erode_amount > 0.0) { // run_erosion: min_zval = min over vals (src/heightmap.cpp:155-156)
		rc = twi_erode(ctx, d_vals, 1, (int)width, (int)height, nullptr, mm.zmin, erosion_iters, ep); if (rc) return rc;
		moves = ctx->last_erosion_steps;
		rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
		rc = twi_minmax(ctx, d_vals, n, d_mm); if (rc) return rc;
		rc = read_minmax(ctx, d_mm, &mm, 1); if (rc) return rc; // get_heightmap_z_range
	}
	float const min_z = mm.zmin, max_z = mm.zmax;
	float const TOLERANCE = 1.0E-12, READ_MESH_H_SCALE = 0.0008; // src/3DWorld.h:50, src/mesh_gen.cpp:22
	float const dzr = max_z - min_z, dz = (TOLERANCE < dzr) ? dzr : TOLERANCE; // max(TOLERANCE, (max_z - min_z))
	float const dz255 = dz/255.0;                                             // set_mesh_height_scales_for_zval_range(min_z, dz/255.0)
	float const mesh_file_scale = dz255/(READ_MESH_H_SCALE*p->mesh_height_scale*p->mesh_scale_z_inv);
	float const mesh_file_tz    = min_z/p->mesh_scale_z_inv;
	float const val_mult = READ_MESH_H_SCALE*p->mesh_height_scale*mesh_file_scale*p->mesh_scale_z_inv; // get_mh_texture_mult()
	float const val_add  = mesh_file_tz*p->mesh_scale_z_inv;                                             // get_mh_texture_add()
	unsigned *d_bad = (unsigned *)((char *)ctx->d_scratch[2] + OFF_BAD);
	TW_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(unsigned), ctx->stream));
	rc = twi_from_floats_u16(ctx, d_vals, n, val_mult, val_add, d_img, d_bad); if (rc) return rc;
	if (!out_dev) {TW_CUDA(ctx, cudaMemcpyAsync(data16, d_img, 2*n, cudaMemcpyDeviceToHost, ctx->stream));}
	if (vals && !vals_dev) {TW_CUDA(ctx, cudaMemcpyAsync(vals, d_vals, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	unsigned bad = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	ctx->last_erosion_steps = moves;
	if (info) {info->min_z = min_z; info->max_z = max_z; info->val_mult = val_mult; info->val_add = val_add; info->mesh_file_scale = mesh_file_scale; info->mesh_file_tz = mesh_file_tz; info->erosion_moves = moves;}
	if (bad) return tw_set_error(ctx, TW_ERR_ARG, "from_floats: value outside [0,256) (the reference asserts, src/heightmap.cpp:211)");
	return TW_OK;
}

int tw_minmax_f32(tw_ctx *ctx, const float *vals, size_t n, tw_minmax *mm) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (!vals || !mm || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	const float *d_in = vals;
	if (!tw_is_device_ptr(vals)) {
		rc = tw_reserve(ctx, 0, n*sizeof(float)); if (rc) return rc;
		TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_scratch[0], vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		d_in = (const float *)ctx->d_scratch[0];
	}
	rc = tw_reserve(ctx, 2, OFF_TILES); if (rc) return rc;
	unsigned *d_mm = (unsigned *)((char *)ctx->d_scratch[2] + OFF_MM);
	rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
	rc = twi_minmax(ctx, d_in, n, d_mm); if (rc) return rc;
	return read_minmax(ctx, d_mm, mm, 1);
}

} // extern "C"
