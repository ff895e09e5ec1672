// tw_api.cu - the extern "C" boundary (include/tw3d.h): context management, host/device pointer staging, and dispatch to the kernels.
// There is deliberately NO CPU path in this library: without a CUDA device tw_create fails and nothing else can be called.
#include "tw_internal.h"
#include "tw_hmap_ao.h"
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

bool twi_is_page_locked(const void *p) {
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {cudaGetLastError(); return false;}
	return a.type == cudaMemoryTypeHost;
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

int check_ctx(tw_ctx *ctx) { // NOTE: makes ctx->device the calling thread's current CUDA device and leaves it so (documented in tw3d.h: one context per thread);
                             // a shared context takes its parent's current tables
	if (!ctx) return TW_ERR_ARG;
	cudaError_t e = cudaSetDevice(ctx->device);
	if (e != cudaSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
	twi_borrow_tables(ctx);
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

// n ordered min/max pairs u into mm
void unpack_minmax(const unsigned *u, uint32_t n, tw_minmax *mm) {
	for (uint32_t i = 0; i < n; ++i) {mm[i].zmin = tw_ord2f(u[2*i]); mm[i].zmax = tw_ord2f(u[2*i+1]);}
}

// The completion of a job that stages a twi_hmap_stage at h (tw_proc_gen_heightmap_launch; tw_erode_launch_ex, which fills only its min_z, bad, fail and
// steps and has no info), in tw_proc_gen_heightmap's order: the step count and info even when the pack fails, and the image (image_w > 0: the packed image
// becomes (again) the context's tw_set_heightmap image) only when everything succeeded
auto hmap_completion(const twi_hmap_stage *h, tw_heightmap_info *info, int image_w, int image_h) {
	return [h, info, image_w, image_h](tw_ctx *ctx) -> int {
		twi_hmap_stage const st = *h;
		if (st.fail) {ctx->last_erosion_steps = 0; return tw_set_error(ctx, TW_ERR_STATE, "speculative erosion made no progress (%u rounds)", st.fail);}
		ctx->last_erosion_steps = st.steps;
		if (info) {
			info->min_z = st.min_z; info->max_z = st.max_z; info->val_mult = st.val_mult; info->val_add = st.val_add;
			info->mesh_file_scale = st.mesh_file_scale; info->mesh_file_tz = st.mesh_file_tz; info->erosion_moves = st.steps;
		}
		if (st.bad) return tw_set_error(ctx, TW_ERR_ARG, "from_floats: value outside [0,256) (the reference asserts, src/heightmap.cpp:211)");
		if (image_w) {ctx->hmap_w = image_w; ctx->hmap_h = image_h;}
		return TW_OK;
	};
}

// Completion of the pending asynchronous job: wait = 0 only queries its event. The call that sees it complete runs the job's completion, which unpacks
// what the job staged in ctx->h_pinned into the caller's host arrays, and reports errors of the enqueued work.
int poll_job(tw_ctx *ctx, int wait) {
	tw_async_state &a = ctx->async;
	if (!a.job.complete) return TW_OK;
	cudaError_t const ev = wait ? cudaEventSynchronize(a.done) : cudaEventQuery(a.done);
	if (ev == cudaErrorNotReady) return TW_ERR_NOT_READY;
	twi_job const j = std::exchange(a.job, twi_job()); // no job is pending from here on, whether it failed or not
	if (ev != cudaSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "asynchronous job failed: %s", cudaGetErrorString(ev));
	int status; // of the completed work (a heightmap job's pack or erosion)
	if (ctx->h_job->stopped) { // a cancellation point acted (tw_cancel): nothing is unpacked, and an image the job would have set stays unset
		ctx->last_erosion_steps = 0;
		status = tw_set_error(ctx, TW_ERR_CANCELED, "the job was cancelled (tw_cancel)");
	}
	else status = j.complete(ctx);
	cudaError_t const e = cudaGetLastError();
	if (e != cudaSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "asynchronous job failed: %s", cudaGetErrorString(e));
	return status;
}

// Completes the pending job before other work reuses the scratch buffers. A job cut short by tw_cancel completes here without an error: the caller threw
// its outputs away and the entry point goes on with its own work; only the explicit polls report TW_ERR_CANCELED.
int finish_pending(tw_ctx *ctx) {
	int const rc = poll_job(ctx, 1);
	if (rc == TW_ERR_CANCELED) {ctx->err[0] = 0; return TW_OK;}
	return rc;
}

// tw_set_sin_table / tw_set_sine_params / tw_set_heightmap: refused on a shared context; on a parent, the job of every shared context completes first,
// because it may still read the tables about to be replaced
int begin_table_change(tw_ctx *ctx) {
	if (ctx->parent) return tw_set_error(ctx, TW_ERR_ARG, "tables are set on the parent context, not on a shared one");
	for (tw_ctx *s : ctx->shared) {
		int const rc = finish_pending(s);
		if (rc) return tw_set_error(ctx, rc, "a shared context's job failed: %s", s->err);
	}
	return TW_OK;
}

// a context with its own stream and completion event on `device` (the caller has made it current)
tw_ctx *new_ctx(int device) {
	tw_ctx *ctx = new (std::nothrow) tw_ctx();
	if (!ctx) return nullptr;
	ctx->device = device;
	{int sms = 0; if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) ctx->num_sms = (unsigned)sms; else cudaGetLastError();}
	if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {delete ctx; cudaGetLastError(); return nullptr;}
	if (cudaEventCreateWithFlags(&ctx->async.done, cudaEventDisableTiming) != cudaSuccess) {cudaStreamDestroy(ctx->stream); delete ctx; cudaGetLastError(); return nullptr;}
	bool const ok = (cudaEventCreateWithFlags(&ctx->async.image_free, cudaEventDisableTiming) == cudaSuccess &&
	                 cudaStreamCreateWithFlags(&ctx->cancel_stream, cudaStreamNonBlocking) == cudaSuccess
	                 && cudaMalloc(&ctx->d_job_words, sizeof(twi_job_words)) == cudaSuccess && cudaMemset(ctx->d_job_words, 0, sizeof(twi_job_words)) == cudaSuccess
	                 && cudaMallocHost(&ctx->h_job, sizeof(twi_job_host)) == cudaSuccess);
	if (!ok) {tw_destroy(ctx); cudaGetLastError(); return nullptr;}
	memset(ctx->h_job, 0, sizeof(twi_job_host));
	return ctx;
}

int read_minmax(tw_ctx *ctx, const unsigned *d_mm, tw_minmax *mm, uint32_t n) { // synchronous
	int rc = tw_reserve_pinned(ctx, (size_t)n*2*sizeof(unsigned));
	if (rc) return rc;
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, d_mm, (size_t)n*2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	unpack_minmax((const unsigned *)ctx->h_pinned, n, mm);
	return TW_OK;
}

int validate_gen(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p) { // the grid and height params of a generation
	if (!g || !p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (g->nx == 0 || g->ny == 0) return tw_set_error(ctx, TW_ERR_ARG, "nx, ny must be > 0 (reference asserts, src/mesh_gen.cpp:589)");
	if (p->gen_mode < 0 || p->gen_mode > TW_MGEN_DWARP_GPU) return tw_set_error(ctx, TW_ERR_ARG, "bad gen_mode %d", p->gen_mode);
	if (p->start_eval_sin < 0 || p->start_eval_sin > TW_F_TABLE_SIZE) return tw_set_error(ctx, TW_ERR_ARG, "start_eval_sin out of range (src/mesh_gen.cpp:590)");
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	return TW_OK;
}

int validate_height(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, const float *out) {
	if (!out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	return validate_gen(ctx, g, p);
}

// tw_create_tiles_launch_hmap's checks of the sampler against the context's image (after twi_begin)
int validate_hmap(tw_ctx *ctx, const tw_hmap_sampler *hs, const tw_tile_shading *shading) {
	if (!ctx->hmap_w) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_heightmap() has not been called");
	if (!hs) return tw_set_error(ctx, TW_ERR_ARG, "null heightmap sampler");
	if (hs->width != ctx->hmap_w || hs->height != ctx->hmap_h) return tw_set_error(ctx, TW_ERR_ARG, "sampler size %d x %d differs from the heightmap's %d x %d", hs->width, hs->height, ctx->hmap_w, ctx->hmap_h);
	if (hs->edge_mode < 0 || hs->edge_mode > 2) return tw_set_error(ctx, TW_ERR_ARG, "bad edge_mode %d", hs->edge_mode);
	if (shading && shading->ao) return tw_set_error(ctx, TW_ERR_ARG, "the AO map is not available for heightmap tiles (its context outside the tile is not defined in this mode)");
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

// The rects of an edit or a read of the context's image (tw_update_heightmap, tw_read_heightmap_launch): TW_ERR_ARG unless every rect lies inside the image
// and pitch >= 2*(x + w); *nrows = their rows, *texels = the packed staging's texels (each row may start up to 7 texels on, to keep its phase)
int check_hmap_rects(tw_ctx *ctx, const tw_hmap_rect *rects, uint32_t nrects, size_t pitch, const char *pitch_name, size_t *nrows, size_t *texels) {
	int const W = ctx->hmap_w, H = ctx->hmap_h;
	*nrows = *texels = 0;
	for (uint32_t r = 0; r < nrects; ++r) {
		tw_hmap_rect const &R = rects[r];
		if (R.w <= 0 || R.h <= 0 || R.x < 0 || R.y < 0 || R.x > W - R.w || R.y > H - R.h)
			return tw_set_error(ctx, TW_ERR_ARG, "rect %u (%d, %d, %d x %d) is empty or reaches outside the %d x %d image", r, R.x, R.y, R.w, R.h, W, H);
		if (pitch < (size_t)2*((size_t)R.x + (size_t)R.w)) return tw_set_error(ctx, TW_ERR_ARG, "%s %zu < 2*(x + w) for rect %u", pitch_name, pitch, r);
		*nrows += (size_t)R.h; *texels += (size_t)R.w*R.h + 7*(size_t)R.h;
	}
	if (*nrows > 0xffffffffu) return tw_set_error(ctx, TW_ERR_ARG, "too many rows in one call");
	return TW_OK;
}

// Each row of the rects in order: row(rect, y, img), where img = y*width + x is the row's first texel in the image
template <typename Row> void for_hmap_rows(size_t width, const tw_hmap_rect *rects, uint32_t nrects, Row &&row) {
	for (uint32_t r = 0; r < nrects; ++r) {
		for (int y = rects[r].y; y < rects[r].y + rects[r].h; ++y) {row(rects[r], y, (size_t)y*width + (size_t)rects[r].x);}
	}
}

// The next row of w texels of packed staging whose next free texel is `at`: its first texel, placed at the phase of texel `phase_of` modulo 8 texels (16 bytes)
inline size_t pack_hmap_row(size_t &at, size_t phase_of, unsigned w) {size_t const p = at + ((phase_of - at) & 7); at = p + w; return p;}

inline void set_hmap_row(twi_hmap_row &row, size_t dst, size_t src, int w) {row.dst = dst; row.src = src; row.w = (unsigned)w; row.pad = 0;}

} // namespace

int twi_begin(tw_ctx *ctx) {int const rc = check_ctx(ctx); return rc ? rc : finish_pending(ctx);}
int twi_finish_pending(tw_ctx *ctx) {twi_borrow_tables(ctx); return finish_pending(ctx);}

int twi_job_start(tw_ctx *ctx, unsigned *seq) {
	if (ctx->cancel_sent) { // the copy of an earlier tw_cancel lands before this job's number is written (it names an older job either way)
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->cancel_stream));
		ctx->cancel_sent = false;
	}
	if (++ctx->job_seq == 0) ctx->job_seq = 1; // 0 means "no job"
	*seq = ctx->job_seq;
	// the previous job has completed, so its copy out of h_job->start is done
	ctx->h_job->start[0] = ctx->job_seq; ctx->h_job->start[1] = 0u;
	TW_CUDA(ctx, cudaMemcpyAsync(&ctx->d_job_words->job, ctx->h_job->start, 2*sizeof(unsigned), cudaMemcpyHostToDevice, ctx->stream));
	return TW_OK;
}

int twi_job_end(tw_ctx *ctx) {
	TW_CUDA(ctx, cudaMemcpyAsync(&ctx->h_job->stopped, &ctx->d_job_words->stopped, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaMemsetAsync(&ctx->d_job_words->job, 0, sizeof(unsigned), ctx->stream));
	return TW_OK;
}

int twi_wait_image_edits(tw_ctx *ctx) {
	tw_ctx const *root = ctx->parent ? ctx->parent : ctx;
	if (root->img_ev) {TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, root->img_ev, 0));}
	return TW_OK;
}

int twi_image_settle(tw_ctx *root) {
	if (root->img_stream) {TW_CUDA(root, cudaStreamSynchronize(root->img_stream));}
	for (twi_img_stage &g : root->img_stage) {
		if (g.h) cudaFreeHost(g.h);
		if (g.d) cudaFree(g.d);
		if (g.ev) cudaEventDestroy(g.ev);
	}
	root->img_stage.clear();
	return TW_OK;
}

void twi_borrow_tables(tw_ctx *ctx) {
	tw_ctx const *p = ctx->parent;
	if (!p) return;
	ctx->d_sin_table = p->d_sin_table; ctx->d_dir_table = p->d_dir_table; ctx->have_sin = p->have_sin;
	ctx->d_sine_params = p->d_sine_params; ctx->have_sine_params = p->have_sine_params;
	memcpy(ctx->h_sine_params, p->h_sine_params, sizeof(ctx->h_sine_params));
	ctx->d_simplex_lut = p->d_simplex_lut; ctx->d_glm3_lut = p->d_glm3_lut;
	ctx->d_hmap = p->d_hmap; ctx->hmap_w = p->hmap_w; ctx->hmap_h = p->hmap_h;
}

extern "C" {

int tw_abi_version(void) {return TW_ABI_VERSION;}

int tw_create(int device, tw_ctx **out) {
	if (!out) return TW_ERR_ARG;
	*out = nullptr;
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {cudaGetLastError(); return TW_ERR_NO_DEVICE;}
	if (device < 0 || device >= ndev) return TW_ERR_ARG;
	if (cudaSetDevice(device) != cudaSuccess) {cudaGetLastError(); return TW_ERR_CUDA;}
	tw_ctx *ctx = new_ctx(device);
	if (!ctx) return TW_ERR_CUDA;
	*out = ctx;
	return TW_OK;
}

int tw_create_shared(tw_ctx *parent, tw_ctx **out) {
	if (!out) return tw_set_error(parent, TW_ERR_ARG, "null out");
	*out = nullptr;
	if (!parent) return TW_ERR_ARG;
	if (parent->parent) return tw_set_error(parent, TW_ERR_ARG, "a shared context cannot be the parent of another");
	int rc = check_ctx(parent); if (rc) return rc;
	// the parent's LUTs are built once, here: the shared context only ever reads them, on its own stream, once the parent's stream has passed them
	rc = twi_ensure_simplex_lut(parent); if (rc) return rc;
	rc = twi_ensure_glm3_lut(parent); if (rc) return rc;
	TW_CUDA(parent, cudaStreamSynchronize(parent->stream));
	tw_ctx *ctx = new_ctx(parent->device);
	if (!ctx) return tw_set_error(parent, TW_ERR_CUDA, "tw_create_shared: no memory for the context, its stream or its event");
	try {parent->shared.push_back(ctx);} catch (...) {tw_destroy(ctx); return tw_set_error(parent, TW_ERR_CUDA, "tw_create_shared: out of host memory");}
	ctx->parent = parent;
	twi_borrow_tables(ctx);
	*out = ctx;
	return TW_OK;
}

void tw_destroy(tw_ctx *ctx) {
	if (!ctx) return;
	while (!ctx->sets.empty()) tw_tile_set_destroy(ctx->sets.back()); // each completes the pending job and removes itself from the list
	while (!ctx->models.empty()) tw_voxel_model_destroy(ctx->models.back()); // the same
	while (!ctx->shared.empty()) tw_destroy(ctx->shared.back()); // each removes itself from the list
	if (ctx->dist) tw_dist_finalize(ctx);
	cudaSetDevice(ctx->device);
	finish_pending(ctx); // the job completes as a poll with wait = 1 would
	tw_ctx *const parent = ctx->parent;
	if (parent) { // the tables are the parent's
		parent->shared.erase(std::find(parent->shared.begin(), parent->shared.end(), ctx));
		ctx->d_sin_table = nullptr; ctx->d_dir_table = nullptr; ctx->d_simplex_lut = nullptr; ctx->d_glm3_lut = nullptr; ctx->d_sine_params = nullptr; ctx->d_hmap = nullptr;
	}
	cudaStreamSynchronize(ctx->stream);
	twi_image_settle(ctx); // the edits of the image: every job they could wait for has completed
	if (ctx->img_ev) cudaEventDestroy(ctx->img_ev);
	if (ctx->img_stream) cudaStreamDestroy(ctx->img_stream);
	if (ctx->cancel_stream) {cudaStreamSynchronize(ctx->cancel_stream); cudaStreamDestroy(ctx->cancel_stream);}
	if (ctx->d_job_words) cudaFree(ctx->d_job_words);
	if (ctx->h_job) cudaFreeHost(ctx->h_job);
	if (ctx->spec_graph) cudaGraphExecDestroy(ctx->spec_graph);
	if (ctx->sweep_graph) cudaGraphExecDestroy(ctx->sweep_graph);
	for (int i = 0; i < 3; ++i) {if (ctx->d_scratch[i]) cudaFree(ctx->d_scratch[i]);}
	if (ctx->d_sin_table) cudaFree(ctx->d_sin_table);
	if (ctx->d_dir_table) cudaFree(ctx->d_dir_table);
	if (ctx->d_simplex_lut) cudaFree(ctx->d_simplex_lut);
	if (ctx->d_glm3_lut) cudaFree(ctx->d_glm3_lut);
	if (ctx->d_sine_params) cudaFree(ctx->d_sine_params);
	if (ctx->d_hmap) cudaFree(ctx->d_hmap);
	if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
	if (ctx->async.done) cudaEventDestroy(ctx->async.done);
	if (ctx->async.image_free) cudaEventDestroy(ctx->async.image_free);
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
uint64_t tw_dwarp_window_launches(const tw_ctx *ctx) {return ctx ? ctx->dwarp_win_launches : 0;}
uint64_t tw_last_erosion_steps(const tw_ctx *ctx) {return ctx ? ctx->last_erosion_steps : 0;}

// "cancel job k" into the device words, by a copy on the context's cancel stream: nothing waits, nothing goes to ctx->stream
int tw_cancel(tw_ctx *ctx) {
	int rc = check_ctx(ctx); if (rc) return rc;
	twi_job const &j = ctx->async.job;
	if (!j.complete) return TW_OK;
	if (!j.cancellable) return tw_set_error(ctx, TW_ERR_STATE, "the pending job cannot be cancelled: a job that touches a tile set or a voxel model committed its state at "
	                                                           "its launch, and a points job, a heightmap read or a heightmap AO job has no cancellation point");
	ctx->h_job->cancel = j.seq;
	TW_CUDA(ctx, cudaMemcpyAsync(&ctx->d_job_words->cancel, &ctx->h_job->cancel, sizeof(unsigned), cudaMemcpyHostToDevice, ctx->cancel_stream));
	ctx->cancel_sent = true;
	return TW_OK;
}

int tw_sync(tw_ctx *ctx) {
	int rc = check_ctx(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_set_sin_table(tw_ctx *ctx, const float *tab) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = begin_table_change(ctx); if (rc) return rc;
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
	rc = begin_table_change(ctx); if (rc) return rc;
	if (!ctx->d_sine_params) {TW_CUDA(ctx, cudaMalloc(&ctx->d_sine_params, TW_F_TABLE_SIZE*5*sizeof(float)));}
	memcpy(ctx->h_sine_params, sp, sizeof(ctx->h_sine_params));
	TW_CUDA(ctx, cudaMemcpyAsync(ctx->d_sine_params, ctx->h_sine_params, sizeof(ctx->h_sine_params), cudaMemcpyHostToDevice, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	ctx->have_sine_params = true;
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ 2-D height
int tw_heightgen_2d_launch(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, float *out, tw_minmax *mm) {
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate_height(ctx, g, p, out); if (rc) return rc;
	size_t const n = (size_t)g->nx*g->ny;
	twi_user<float> o(out, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {o.take(c);}); if (rc) return rc;
	rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words)); if (rc) return rc;
	if (mm) {rc = tw_reserve_pinned(ctx, 2*sizeof(unsigned)); if (rc) return rc;}
	if (!o.dev) {rc = twi_ensure_aux_streams(ctx); if (rc) return rc;}
	unsigned *d_mm = mm ? twi_slot2(ctx)->mm : nullptr, *h_mm = (unsigned *)ctx->h_pinned;
	twi_job pending;
	pending.cancellable = true;
	pending.complete = [mm, h_mm](tw_ctx *) -> int {if (mm) {unpack_minmax(h_mm, 1, mm);} return TW_OK;};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		if (d_mm) {rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;}
		rc = twi_heightgen(ctx, g, p, enable_glaciate, min_start_sin, nullptr, 1, o.d, d_mm, o.dev ? nullptr : out); // host out: band-wise D2H overlapped with compute
		if (rc) return rc;
		if (mm) {TW_CUDA(ctx, cudaMemcpyAsync(h_mm, d_mm, 2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
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
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!zvals || !origins_xy || !p || !wp || !tile_params || !weights || ntiles == 0 || zvsize < 3) return tw_set_error(ctx, TW_ERR_ARG, "tw_tile_weights_batch: null argument, no tiles or zvsize < 3");
	tw_weight_params W;
	rc = validate_weights(ctx, wp, W); if (rc) return rc;
	uint32_t const stride = zvsize - 1;
	size_t const zn = (size_t)ntiles*zvsize*zvsize, tn = (size_t)ntiles*stride*stride;
	twi_user<const float> z(zvals, zn), tp(tile_params, (size_t)ntiles*8);
	twi_user<uint8_t> w(weights, tn*4), f(has_any_grass, ntiles);
	float *d_rand;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {d_rand = c.take<float>(tn); z.take(c); w.take(c); f.take(c); tp.take(c);}); if (rc) return rc;
	rc = z.in(ctx); if (rc) return rc;
	rc = tp.in(ctx); if (rc) return rc;
	if (has_any_grass) {TW_CUDA(ctx, cudaMemsetAsync(f.d, 0, ntiles, ctx->stream));}
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
	rc = twi_tile_weights(ctx, ctx->stream, z.d, d_rand, ntiles, zvsize, tp.d, &W, w.d, has_any_grass ? f.d : nullptr);
	if (rc) return rc;
	rc = w.out(ctx); if (rc) return rc;
	rc = f.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

int tw_heightgen_tiles(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                       uint32_t zvsize, const tw_height_params *p, float *out, tw_minmax *mm)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!origins_xy || ntiles == 0) return tw_set_error(ctx, TW_ERR_ARG, "no tiles");
	tw_grid2d g; g.x0 = 0; g.y0 = 0; g.dx = dx; g.dy = dy; g.nx = zvsize; g.ny = zvsize;
	rc = validate_height(ctx, &g, p, out); if (rc) return rc;
	size_t const tile_elems = (size_t)zvsize*zvsize, n = tile_elems*ntiles;
	twi_user<float> o(out, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {o.take(c);}); if (rc) return rc;
	unsigned *d_mm = nullptr; float2 *d_org;
	rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {c.take<twi_slot2_words>(1); if (mm) {d_mm = c.take<unsigned>((size_t)ntiles*2);} d_org = c.take<float2>(ntiles);});
	if (rc) return rc;
	if (d_mm) {rc = twi_init_minmax(ctx, d_mm, ntiles); if (rc) return rc;}
	// setup_height_gen_async: build_arrays((x0 - MESH_X_SIZE/2), (y0 - MESH_Y_SIZE/2), dx, dy, ...): int -> float, then mx0 = dx*x0 (src/tiled_mesh.cpp:461, src/mesh_gen.cpp:591)
	if (p->gen_mode != TW_MGEN_SINE) {
		std::vector<float2> org(ntiles);
		for (uint32_t t = 0; t < ntiles; ++t) {
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			org[t] = make_float2(dx*x0, dy*y0);
		}
		TW_CUDA(ctx, cudaMemcpyAsync(d_org, org.data(), (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // org is a local vector
		uint32_t const zmax = 65535;
		for (uint32_t t0 = 0; t0 < ntiles; t0 += zmax) { // gridDim.z limit
			uint32_t const nt = (ntiles - t0 < zmax) ? ntiles - t0 : zmax;
			rc = twi_heightgen(ctx, &g, p, 1, 0, d_org + t0, nt, o.d + (size_t)t0*tile_elems, d_mm ? d_mm + 2*(size_t)t0 : nullptr);
			if (rc) return rc;
		}
	}
	else { // sine tables depend on the tile origin only through its column / row: W + H tables for a W x H block of tiles, one grid launch for the batch
		std::vector<float2> org(ntiles);
		for (uint32_t t = 0; t < ntiles; ++t) {
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			org[t] = make_float2(dx*x0, dy*y0);
		}
		rc = twi_heightgen_sine_tiles(ctx, &g, p, 1, 0, org.data(), ntiles, o.d, d_mm);
		if (rc) return rc;
	}
	rc = o.out(ctx); if (rc) return rc;
	if (mm) {rc = read_minmax(ctx, d_mm, mm, ntiles); if (rc) return rc;}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ callers' tails
int tw_tile_bounds_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, float dx_val, float dy_val, uint32_t size, tw_tile_bounds *out) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!zvals || !out || ntiles == 0 || zvsize < 4) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (4*(zvsize/4) >= zvsize) return tw_set_error(ctx, TW_ERR_ARG, "zvsize %u: the last sub-block would end at cell %u (the reference asserts x_end < zvsize, src/tiled_mesh.cpp:520)", zvsize, 4*(zvsize/4));
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	size_t const n = (size_t)ntiles*zvsize*zvsize;
	twi_user<const float> z(zvals, n);
	Sub *d_sub;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {z.take(c); d_sub = c.take<Sub>((size_t)ntiles*16);}); if (rc) return rc;
	rc = z.in(ctx); if (rc) return rc;
	rc = twi_tile_bounds(ctx, ctx->stream, z.d, ntiles, zvsize, wpz_max, d_sub); if (rc) return rc;
	std::vector<Sub> sub((size_t)ntiles*16);
	TW_CUDA(ctx, cudaMemcpyAsync(sub.data(), d_sub, sub.size()*sizeof(Sub), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	combine_bounds(sub.data(), ntiles, dx_val, dy_val, size, out);
	return TW_OK;
}

int tw_glaciate_mesh(tw_ctx *ctx, float *mesh, int nx, int ny, int xoff2, int yoff2, int mesh_x_size, int mesh_y_size, const tw_height_params *p, tw_minmax *zbottom_ztop) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!mesh || !p || nx <= 0 || ny <= 0 || ny > 65535) return tw_set_error(ctx, TW_ERR_ARG, "bad argument");
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	size_t const n = (size_t)nx*ny;
	twi_user<float> m(mesh, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {m.take(c);}); if (rc) return rc;
	rc = m.in(ctx); if (rc) return rc;
	rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words)); if (rc) return rc;
	unsigned *d_mm = twi_slot2(ctx)->mm;
	rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
	rc = twi_glaciate_mesh(ctx, m.d, nx, ny, xoff2, yoff2, mesh_x_size, mesh_y_size, p, d_mm); if (rc) return rc;
	rc = m.out(ctx); if (rc) return rc;
	if (zbottom_ztop) {return read_minmax(ctx, d_mm, zbottom_ztop, 1);}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ erosion
int tw_erode_tiles(tw_ctx *ctx, float *maps, uint32_t ntiles, int xsize, int ysize, const float *min_zvals, float min_zval_all,
                   uint32_t num_iters, const tw_erosion_params *p)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!maps || !p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (xsize <= 0 || ysize <= 0 || ntiles == 0) return tw_set_error(ctx, TW_ERR_ARG, "empty heightmap");
	if (num_iters == 0 || p->erode_amount <= 0.0) {ctx->last_erosion_steps = 0; return TW_OK;} // src/erosion.cpp:16
	size_t const n = (size_t)xsize*ysize*ntiles;
	twi_user<float> m(maps, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {m.take(c);}); if (rc) return rc;
	rc = m.in(ctx); if (rc) return rc;
	float *d_minz = nullptr;
	if (min_zvals) {
		rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {c.take<twi_slot2_words>(1); d_minz = c.take<float>(ntiles);}); if (rc) return rc;
		TW_CUDA(ctx, cudaMemcpyAsync(d_minz, min_zvals, (size_t)ntiles*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	rc = twi_erode(ctx, m.d, ntiles, xsize, ysize, d_minz, min_zval_all, num_iters, p);
	if (rc) return rc;
	rc = m.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// The tile pipeline behind tw_create_zvals_batch, tw_create_zvals_ao_batch and tw_create_tiles_launch(_ex, _shadows): enqueues everything and returns
// without waiting for the device; the job completes through poll_job (twi_begin has run). sh (optional): AO map and weights texture;
// shs (optional): per-light mesh shadows. hs: the height source - nullptr = the procedural height function p, else the context's heightmap image under hs
// (tw_create_tiles_launch_hmap, which has checked hs against the image and refused AO); p is then only read by the weights' jitter noise.
// tail (optional, twi_job_tail): work appended after the chunk join; with it o->zvals may be NULL.
static int tiles_launch(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy, uint32_t zvsize,
                        const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval, float wpz_max, uint32_t size,
                        const tw_tile_outputs *o, const tw_tile_shading *sh, const tw_tile_shadows *shs, const tw_hmap_sampler *hs, twi_job_tail *tail = nullptr)
{
	if (!origins_xy || ntiles == 0 || (!p && !hs) || !o || (!o->zvals && !tail)) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
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
	if (!hs) {rc = validate_gen(ctx, &g, p); if (rc) return rc;}
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
	bool const dev_out = o->zvals && tw_is_device_ptr(o->zvals), host_out = o->zvals && !dev_out, dev_f = want_f && tw_is_device_ptr(sh->has_any_grass);
	twi_user<uint8_t> nrm(o->normals_rgba, ntiles*nrm_elems*4), ao(want_ao ? sh->ao : nullptr, ntiles*nrm_elems), wt(want_w ? sh->weights : nullptr, ntiles*nrm_elems*4);
	twi_user<const float> tp(want_w ? sh->tile_params : nullptr, (size_t)ntiles*8);
	if (tail) {rc = tail->prepare(ctx); if (rc) return rc;}
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
	size_t const ctab_bytes = (want_ao && sine) ? twi_sine_tiles_plan(&gc, corg.data(), ntiles, &sb_ctx) : 0, jtab_bytes = want_w ? twi_sine_tiles_plan(&gj, jorg.data(), ntiles, &sb_jit) : 0;
	// slot 0: device staging of the host-bound arrays [zvals | normal maps | AO maps | weights | has_any_grass], then [tile_params | sine tables | mesh shadows |
	// tail], then the ring of context / jitter grid buffers. All but the ring is reserved before the erosion budget is taken, so the budget sees that memory as
	// used. Mesh shadows, reused light after light: [mask staging (host smask) | 64-bit keys | x edges | y edges (outputs, then caller rows) | plan of every light].
	size_t const edge = (size_t)ntiles*zvsize;
	bool sh_host_m = false, sh_in_x = false, sh_in_y = false;
	for (uint32_t l = 0; l < nl; ++l) {sh_host_m |= !sdev_m[l]; sh_in_x |= (lights[l].sh_in_x != nullptr); sh_in_y |= (lights[l].sh_in_y != nullptr);}
	float *d_out = dev_out ? o->zvals : nullptr, *d_shx = nullptr, *d_shy = nullptr;
	unsigned char *d_shm = nullptr;
	uint8_t *d_f = dev_f ? sh->has_any_grass : nullptr;
	char *d_ctab = nullptr, *d_jtab = nullptr, *d_tail = nullptr;
	unsigned long long *d_shk = nullptr;
	std::vector<int *> d_shp(nl);
	auto slot0 = [&](twi_carve &c) {
		if (!dev_out) {d_out = c.take<float>(n);} if (want_normals) {nrm.take(c);}
		if (want_ao) {ao.take(c);} if (want_w) {wt.take(c);}
		if (want_f && !dev_f) {d_f = c.take<uint8_t>(ntiles);} if (want_w) {tp.take(c);}
		if (want_ao && sine) {d_ctab = c.take<char>(ctab_bytes);} if (want_w) {d_jtab = c.take<char>(jtab_bytes);} if (sh_host_m) {d_shm = c.take<unsigned char>(n + 4);}
		if (nl) {d_shk = c.take<unsigned long long>(2*edge); d_shx = c.take<float>((sh_in_x ? 2 : 1)*edge); d_shy = c.take<float>((sh_in_y ? 2 : 1)*edge);}
		for (uint32_t l = 0; l < nl; ++l) {d_shp[l] = c.take<int>(twi_shadow_plan_ints(ntiles));} if (tail) {d_tail = c.take<char>(tail->dev_bytes);}
	};
	twi_carve fixed; slot0(fixed);
	rc = tw_reserve(ctx, 0, fixed.bytes); if (rc) return rc;
	// AO context grids and weights jitter grids are per chunk (schedule order): written on the main stream, read on the chunk's erosion stream. The buffers
	// hold about 2 GB of context grids (or jitter grids without AO) in all, the bound tw_tile_ao_batch keeps; a chunk holds at most a third of that. When
	// the batch needs more chunks than buffers, chunk 0 (every long droplet chain) keeps its buffer and the later chunks take turns in the others: before the
	// main stream rewrites one it waits for the stream that last read it, which is never chunk 0's. Batches with one buffer per chunk never wait.
	size_t const RING = (size_t)2 << 30, ring_tile = (want_ao ? ctx_elems*sizeof(float) : 0) + (want_w ? nrm_elems*sizeof(float) : 0);
	size_t const bound_tile = want_ao ? ctx_elems*sizeof(float) : nrm_elems*sizeof(float);
	size_t const ring_max = ring_tile ? std::min((RING/bound_tile)*ring_tile, (size_t)ntiles*ring_tile) + 2*65536 : 0; // what the buffers can take, for the erosion budget
	uint32_t nchunks = 0, chunk = 0;
	size_t sbytes = 0; // one erosion lane's scratch (a multiple of 256 bytes): lane l's is at l*sbytes in slot 1
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
	std::vector<float *> ring_cz(nbuf), ring_rand(nbuf);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		slot0(c);
		for (uint32_t b = 0; b < nbuf; ++b) {ring_cz[b] = want_ao ? c.take<float>((size_t)chunk*ctx_elems) : nullptr; ring_rand[b] = want_w ? c.take<float>((size_t)chunk*nrm_elems) : nullptr;}
	}); if (rc) return rc;
	if (erode) {
		sbytes = twi_erode_scratch_bytes(ctx, chunk, (int)zvsize, (int)zvsize);
		rc = tw_reserve(ctx, 1, sbytes*nes); if (rc) return rc; // before the sine tables claim the same slot: it is never re-allocated under the erosion
	}
	// slot 2: [fixed words | per-tile min/max | origins | sorted origins | work | order | hist(256) | coarse samples | sub-block bounds | min_normal_z |
	// context origins | sorted context origins]
	bool const ctx_org = want_ao && !sine; // the paired noise kernels read the context origins from the device
	uint32_t const CS = 8, cstep = (zvsize >= CS) ? zvsize/CS : 1;
	twi_slot2_words *words;
	unsigned *d_mm, *d_work, *d_order, *d_hist, *d_mnz = nullptr;
	float2 *d_org, *d_org_sorted, *d_corg = nullptr, *d_corg_sorted = nullptr;
	float *d_coarse = nullptr;
	Sub *d_sub = nullptr;
	rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {
		words = c.take<twi_slot2_words>(1); d_mm = c.take<unsigned>((size_t)ntiles*2); d_org = c.take<float2>(ntiles); d_org_sorted = c.take<float2>(ntiles);
		d_work = c.take<unsigned>(ntiles); d_order = c.take<unsigned>(ntiles); d_hist = c.take<unsigned>(256);
		if (reorder) {d_coarse = c.take<float>((size_t)ntiles*CS*CS);} if (want_bounds) {d_sub = c.take<Sub>((size_t)ntiles*16);}
		if (want_mnz) {d_mnz = c.take<unsigned>(ntiles);} if (ctx_org) {d_corg = c.take<float2>(ntiles); d_corg_sorted = c.take<float2>(ntiles);}
	}); if (rc) return rc;
	unsigned long long *d_steps = &words->steps;
	// pinned staging: inputs [origins | sine-mode index tables | context origins or their sine tables | jitter sine tables | tile_params | per light: shadow plan,
	// host sh_in_x, host sh_in_y], then the small results [steps | min/max | sub-block bounds | min_normal_z | has_any_grass] that the completing poll unpacks.
	// Every sine batch has its own region, and the caller's origins, tile_params, tile_xy and host sh_in rows may be reused as soon as this function returns.
	float2 *h_org;
	char *h_sine = nullptr, *h_ctx = nullptr, *h_jit = nullptr, *h_tail = nullptr;
	std::vector<int *> h_shp(nl);
	std::vector<float *> h_six(nl), h_siy(nl);
	unsigned long long *h_steps;
	unsigned *h_mm = nullptr, *h_mnz = nullptr;
	Sub *h_sub = nullptr;
	uint8_t *h_f = nullptr;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		h_org = c.take<float2>(ntiles);
		if (sine) {h_sine = c.take<char>(twi_sine_tiles_stage_bytes(ntiles));}
		if (want_ao) {h_ctx = c.take<char>(sine ? twi_sine_tiles_stage_bytes(ntiles) : ntiles*sizeof(float2));}
		if (want_w) {h_jit = c.take<char>(twi_sine_tiles_stage_bytes(ntiles));}
		tp.take_pinned(c);
		for (uint32_t l = 0; l < nl; ++l) {h_shp[l] = c.take<int>(twi_shadow_plan_ints(ntiles));}
		for (uint32_t l = 0; l < nl; ++l) {
			h_six[l] = (lights[l].sh_in_x && !sdev_ix[l]) ? c.take<float>(edge) : nullptr; h_siy[l] = (lights[l].sh_in_y && !sdev_iy[l]) ? c.take<float>(edge) : nullptr;
		}
		h_steps = c.take<unsigned long long>(1);
		if (want_mm) {h_mm = c.take<unsigned>((size_t)ntiles*2);}
		if (want_bounds) {h_sub = c.take<Sub>((size_t)ntiles*16);}
		if (want_mnz) {h_mnz = c.take<unsigned>(ntiles);}
		if (want_f) {h_f = c.take<uint8_t>(ntiles);}
		if (tail) {h_tail = c.take<char>(tail->pin_bytes);}
	}); if (rc) return rc;
	if (hs) {memcpy(h_org, origins_xy, (size_t)ntiles*2*sizeof(int32_t));} // the sampler reads the int (x1, y1) origins (d_org then holds int2)
	else {
		for (uint32_t t = 0; t < ntiles; ++t) { // build_arrays((x1 - MESH_X_SIZE/2), (y1 - MESH_Y_SIZE/2), ...): int -> float, mx0 = dx*x0 (src/tiled_mesh.cpp:461, src/mesh_gen.cpp:591)
			float const x0 = (float)(origins_xy[2*t] - mesh_x_size/2), y0 = (float)(origins_xy[2*t+1] - mesh_y_size/2);
			h_org[t] = make_float2(dx*x0, dy*y0);
		}
	}
	twi_job pending;
	pending.cancellable = (tail == nullptr); // a tail commits a tile set's state
	pending.reads_image = (hs != nullptr);
	pending.complete = [erode, ntiles, dx, dy, size, h_steps, h_mm, h_sub, h_mnz, h_f, mm = o->mm, bounds = o->bounds, min_nz = o->min_normal_z,
	                    flags = (want_f && !dev_f) ? sh->has_any_grass : nullptr](tw_ctx *c) -> int {
		if (erode) {c->last_erosion_steps = *h_steps;}
		if (mm) {unpack_minmax(h_mm, ntiles, mm);}
		if (bounds) {combine_bounds(h_sub, ntiles, dx, dy, size, bounds);}
		if (min_nz) {for (uint32_t i = 0; i < ntiles; ++i) {min_nz[i] = tw_ord2f(h_mnz[i]);}}
		if (flags) {memcpy(flags, h_f, ntiles);}
		return TW_OK;
	};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		if (!sine) {TW_CUDA(ctx, cudaMemcpyAsync(d_org, h_org, (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));}
		if (ctx_org) {
			memcpy(h_ctx, corg.data(), (size_t)ntiles*sizeof(float2));
			TW_CUDA(ctx, cudaMemcpyAsync(d_corg, h_ctx, (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
		}
		rc = tp.in(ctx); if (rc) return rc;
		for (uint32_t l = 0; l < nl; ++l) { // the plans go up now; host sh_in rows wait in the staging until their light's pass copies them into the edge buffers
			twi_shadow_plan_pack(splan[l], h_shp[l]);
			TW_CUDA(ctx, cudaMemcpyAsync(d_shp[l], h_shp[l], twi_shadow_plan_ints(ntiles)*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
			if (h_six[l]) {memcpy(h_six[l], lights[l].sh_in_x, edge*sizeof(float));}
			if (h_siy[l]) {memcpy(h_siy[l], lights[l].sh_in_y, edge*sizeof(float));}
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
		if (sine) {rc = twi_heightgen_sine_tiles(ctx, &g, p, 1, 0, h_org, ntiles, d_out, nullptr, h_sine); if (rc) return rc;}
		if (want_ao && sine) {rc = twi_sine_tiles_setup(ctx, &gc, p, 1, 0, corg.data(), ntiles, d_ctab, h_ctx, &sb_ctx); if (rc) return rc;}
		if (want_w) { // force_sine_mode: gen_mode = MGEN_SINE, gen_shape = 0 (src/mesh_gen.cpp:592-593); no glaciate, start index >= 50 (src/tiled_mesh.cpp:1103)
			tw_height_params ps = *p;
			ps.gen_mode = TW_MGEN_SINE; ps.gen_shape = 0;
			rc = twi_sine_tiles_setup(ctx, &gj, &ps, 0, 50, jorg.data(), ntiles, d_jtab, h_jit, &sb_jit); if (rc) return rc;
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
			float *d_cz = nbuf ? ring_cz[b] : nullptr, *d_rand = nbuf ? ring_rand[b] : nullptr;
			bool const reuse = (nbuf && ring_ev[b]); // the main stream waits right before its first write into the buffer
			if (ctx_mode && reuse && cudaStreamWaitEvent(ctx->stream, ring_ev[b], 0) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
			if (ctx_mode) { // contexts in schedule order, zvals cut from their interiors into the caller-visible slots
				status = twi_heightgen(ctx, &gc, p, 1, 0, d_gen_corg + t0, nt, d_cz, nullptr); if (status) break;
				status = twi_tile_cut(ctx, ctx->stream, d_cz, nt, zvsize, maps, perm_k); if (status) break;
			}
			else if (hs) {
				status = twi_hmap_sample_tiles(ctx, ctx->d_hmap, hs, d_perm ? (const void *)d_org : (const void *)(d_org + t0), nt, zvsize, maps, ctx->stream, perm_k);
				if (status) break;
				// every read of the image so far (the coarse pass, the chunks' sampling) is on ctx->stream, ahead of the chunk's erosion, part of which a small
				// batch forks onto ctx->stream: after the last chunk this marks the image free (tw_update_heightmap)
				if (cudaEventRecord(ctx->async.image_free, ctx->stream) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "image event"); break;}
				ctx->async.image_free_set = true;
			}
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
			if (want_normals) {status = twi_tile_normals(ctx, es, maps, nt, zvsize, dx, dy, nrm.d + r0*nrm_elems*4, d_mnz ? d_mnz + r0 : nullptr, perm_k); if (status) break;}
			if (((want_ao && !ctx_mode) || want_w) && !chain(ctx->stream, es)) {status = tw_set_error(ctx, TW_ERR_CUDA, "chunk event"); break;}
			if (want_ao) {status = twi_tile_ao(ctx, es, maps, d_cz, nt, zvsize, sh->half_dxy, ctx_mode, ao.d + r0*nrm_elems, perm_k); if (status) break;}
			if (want_w) {status = twi_tile_weights(ctx, es, maps, d_rand, nt, zvsize, tp.d + r0*8, &W, wt.d + r0*nrm_elems*4, d_f ? d_f + r0 : nullptr, perm_k); if (status) break;}
			if (nbuf) {
				if (!ring_ev[b] && cudaEventCreateWithFlags(&ring_ev[b], cudaEventDisableTiming) != cudaSuccess) {ring_ev[b] = nullptr; status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
				if (cudaEventRecord(ring_ev[b], es) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "ring event"); break;}
			}
			if (host_out && !d_perm && cudaMemcpyAsync(o->zvals + (size_t)t0*tile_elems, maps, (size_t)nt*tile_elems*sizeof(float), cudaMemcpyDeviceToHost, es) != cudaSuccess) {status = tw_set_error(ctx, TW_ERR_CUDA, "D2H");}
		}
		ctx->tile_perm = nullptr;
		ctx->skip_rect[0] = ctx->skip_rect[1] = ctx->skip_rect[2] = ctx->skip_rect[3] = 0;
		for (cudaEvent_t ev : ring_ev) {if (ev) cudaEventDestroy(ev);} // every wait on them is enqueued
		for (int l = 0; l < 3; ++l) { // join: ctx->stream (and so the job's event) follows everything the chunks enqueued
			if (used[l] && !chain(ctx->aux_stream[l], ctx->stream) && status == TW_OK) status = tw_set_error(ctx, TW_ERR_CUDA, "join event");
		}
		if (status) return status;
		// mesh shadows on ctx->stream, light after light through the same buffers: every tile's neighbours have their final heights once the chunks are joined
		for (uint32_t l = 0; l < nl; ++l) {
			tw_tile_light const &L = lights[l];
			unsigned char *d_m = sdev_m[l] ? L.smask : d_shm;
			if (L.sh_in_x) {TW_CUDA(ctx, cudaMemcpyAsync(d_shx + edge, sdev_ix[l] ? (const void *)L.sh_in_x : h_six[l], edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
			if (L.sh_in_y) {TW_CUDA(ctx, cudaMemcpyAsync(d_shy + edge, sdev_iy[l] ? (const void *)L.sh_in_y : h_siy[l], edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
			rc = twi_shadow_enqueue(ctx, ctx->stream, splan[l], d_out, ntiles, zvsize, d_m, d_shk, d_shx, d_shy, d_shp[l], true); if (rc) return rc;
			if (!sdev_m[l]) {TW_CUDA(ctx, cudaMemcpyAsync(L.smask, d_m, n, cudaMemcpyDeviceToHost, ctx->stream));}
			if (L.sh_out_x) {TW_CUDA(ctx, cudaMemcpyAsync(L.sh_out_x, d_shx, edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
			if (L.sh_out_y) {TW_CUDA(ctx, cudaMemcpyAsync(L.sh_out_y, d_shy, edge*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		}
		if (tail) {rc = tail->enqueue(ctx, d_out, d_tail, h_tail); if (rc) return rc;} // the tail's work reads the final zvals
		// every host-bound result is copied once, at the end: the schedule order scatters a chunk over the whole batch
		if (host_out && d_perm) {TW_CUDA(ctx, cudaMemcpyAsync(o->zvals, d_out, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
		rc = nrm.out(ctx); if (rc) return rc;
		rc = ao.out(ctx); if (rc) return rc;
		rc = wt.out(ctx); if (rc) return rc;
		if (erode) {TW_CUDA(ctx, cudaMemcpyAsync(h_steps, d_steps, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));}
		if (want_mm) {TW_CUDA(ctx, cudaMemcpyAsync(h_mm, d_mm, (size_t)ntiles*2*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
		if (want_bounds) {TW_CUDA(ctx, cudaMemcpyAsync(h_sub, d_sub, (size_t)ntiles*16*sizeof(Sub), cudaMemcpyDeviceToHost, ctx->stream));}
		if (want_mnz) {TW_CUDA(ctx, cudaMemcpyAsync(h_mnz, d_mnz, (size_t)ntiles*sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));}
		if (want_f && !dev_f) {TW_CUDA(ctx, cudaMemcpyAsync(h_f, d_f, ntiles, cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
}

int tw_create_tiles_launch_shadows(tw_ctx *ctx, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                   uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                                   float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	ctx->last_erosion_steps = 0;
	return tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, shadows, nullptr);
}

int tw_set_heightmap(tw_ctx *ctx, const uint8_t *data16, int width, int height) {
	int rc = check_ctx(ctx); if (rc) return rc;
	rc = begin_table_change(ctx); if (rc) return rc;
	rc = finish_pending(ctx); if (rc) return rc;
	if (data16 && (width <= 0 || height <= 0)) return tw_set_error(ctx, TW_ERR_ARG, "heightmap size %d x %d", width, height);
	rc = twi_image_settle(ctx); if (rc) return rc;
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

// An edit of the image: the rects' texels packed into pinned staging (row by row, each at its destination's phase modulo 16 bytes), then on the image stream,
// behind the pending image jobs of the family, one copy of [row table | texels] to the device and one scatter kernel. Completes no job, never waits.
int tw_update_heightmap(tw_ctx *ctx, const uint8_t *src16, size_t src_pitch, const tw_hmap_rect *rects, uint32_t nrects) {
	int rc = check_ctx(ctx); if (rc) return rc;
	if (ctx->parent) return tw_set_error(ctx, TW_ERR_ARG, "the heightmap image is set on the parent context, not on a shared one");
	if (nrects && (!src16 || !rects)) return tw_set_error(ctx, TW_ERR_ARG, "null src16 or rects");
	if (nrects == 0) return TW_OK;
	if (!ctx->hmap_w) return tw_set_error(ctx, TW_ERR_STATE, "the context has no heightmap image (tw_set_heightmap, or a job that sets it is pending)");
	size_t nrows, texels;
	rc = check_hmap_rects(ctx, rects, nrects, src_pitch, "src_pitch", &nrows, &texels); if (rc) return rc;
	if (tw_is_device_ptr(src16)) return tw_set_error(ctx, TW_ERR_ARG, "src16 must be host memory");
	twi_carve rows_region;
	rows_region.take<twi_hmap_row>(nrows);
	size_t const rows_bytes = rows_region.bytes, need = rows_bytes + 2*texels;
	if (!ctx->img_stream) {
		TW_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->img_stream, cudaStreamNonBlocking));
		TW_CUDA(ctx, cudaEventCreateWithFlags(&ctx->img_ev, cudaEventDisableTiming));
	}
	// staging: the smallest free buffer that fits (free = its edit has completed on the device); otherwise a new one. Nothing here waits for an edit.
	twi_img_stage *g = nullptr;
	for (twi_img_stage &e : ctx->img_stage) {
		if (e.bytes < need || (g && g->bytes <= e.bytes)) continue;
		cudaError_t const q = cudaEventQuery(e.ev);
		if (q == cudaSuccess) g = &e;
		else if (q != cudaErrorNotReady) return tw_set_error(ctx, TW_ERR_CUDA, "an earlier heightmap edit failed: %s", cudaGetErrorString(q));
	}
	if (!g) {
		twi_img_stage e;
		e.bytes = std::max<size_t>((size_t)1 << 16, need);
		cudaError_t err = cudaMallocHost(&e.h, e.bytes);
		if (err == cudaSuccess) err = cudaMalloc(&e.d, e.bytes);
		if (err == cudaSuccess) err = cudaEventCreateWithFlags(&e.ev, cudaEventDisableTiming);
		if (err == cudaSuccess) {try {ctx->img_stage.push_back(e);} catch (...) {err = cudaErrorMemoryAllocation;}}
		if (err != cudaSuccess) {
			if (e.h) cudaFreeHost(e.h);
			if (e.d) cudaFree(e.d);
			if (e.ev) cudaEventDestroy(e.ev);
			cudaGetLastError();
			return tw_set_error(ctx, TW_ERR_CUDA, "heightmap edit staging of %zu bytes: %s", e.bytes, cudaGetErrorString(err));
		}
		g = &ctx->img_stage.back();
	}
	twi_hmap_row *rows = (twi_hmap_row *)g->h;
	uint8_t *data = (uint8_t *)g->h + rows_bytes;
	size_t k = 0, at = 0; // row, next free texel of the packed data
	for_hmap_rows((size_t)ctx->hmap_w, rects, nrects, [&](tw_hmap_rect const &R, int y, size_t img) {
		size_t const packed = pack_hmap_row(at, img, (unsigned)R.w);
		memcpy(data + 2*packed, src16 + (size_t)y*src_pitch + 2*(size_t)R.x, 2*(size_t)R.w);
		set_hmap_row(rows[k++], img, packed, R.w);
	});
	// behind the image work of the family's pending jobs that read or write the image: a heightmap tile job's sampling, the whole of an image erosion or a
	// set_image job (a job that does not complete before its poll is still pending)
	std::vector<tw_ctx *> family(1, ctx);
	family.insert(family.end(), ctx->shared.begin(), ctx->shared.end());
	for (tw_ctx *c : family) {
		if (c->async.job.complete && c->async.job.reads_image) {TW_CUDA(ctx, cudaStreamWaitEvent(ctx->img_stream, c->async.image_free, 0));}
	}
	TW_CUDA(ctx, cudaMemcpyAsync(g->d, g->h, rows_bytes + 2*at, cudaMemcpyHostToDevice, ctx->img_stream));
	rc = twi_hmap_scatter(ctx, ctx->img_stream, (const twi_hmap_row *)g->d, (uint32_t)nrows, (const uint8_t *)g->d + rows_bytes, ctx->d_hmap); if (rc) return rc;
	TW_CUDA(ctx, cudaEventRecord(g->ev, ctx->img_stream));
	TW_CUDA(ctx, cudaEventRecord(ctx->img_ev, ctx->img_stream));
	return TW_OK;
}

// A read of the image, the inverse of an edit, as the context's job, on the edit's kernel run the other way (a row copy between two buffers whose rows share
// their phase modulo 16 bytes). The row tables go up from the pinned staging in one copy. A device dst16 whose rows all have their image rows' phase is
// written by one kernel straight from the image. Otherwise the kernel packs the rows into device staging, each at its image phase:
//   host dst16: one copy brings the staging down to the pinned staging, and the completion moves each row to dst16;
//   device dst16: the rows are packed in groups by their phase shift d (0..7 texels), one copy per group moves it d texels on into a second staging, where
//                 each row has its destination's phase, and a second run of the kernel writes the rows to dst16.
// So the work enqueued does not grow with the number of rects. The image is free for later edits after the first kernel.
// Slot 0: [row tables | staging | second staging (device dst16 out of phase)]; pinned staging: [row tables | staging (host dst16)].
int tw_read_heightmap_launch(tw_ctx *ctx, const tw_hmap_read *r) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!r) return tw_set_error(ctx, TW_ERR_ARG, "null read");
	uint32_t const nrects = r->nrects;
	if (nrects && (!r->rects || !r->dst16)) return tw_set_error(ctx, TW_ERR_ARG, "null rects or dst16");
	if (nrects == 0) return TW_OK;
	if (!ctx->hmap_w) return tw_set_error(ctx, TW_ERR_STATE, "the context has no heightmap image (tw_set_heightmap, or a job that sets it is pending)");
	size_t nrows, texels;
	rc = check_hmap_rects(ctx, r->rects, nrects, r->dst_pitch, "dst_pitch", &nrows, &texels); if (rc) return rc;
	uint8_t *const dst16 = r->dst16;
	size_t const pitch = r->dst_pitch, W = (size_t)ctx->hmap_w;
	bool const dev = tw_is_device_ptr(dst16);
	if (dev && ((reinterpret_cast<uintptr_t>(dst16) | pitch) & 1)) return tw_set_error(ctx, TW_ERR_ARG, "a device dst16 must be 2-byte aligned and dst_pitch even: its texels are 16-bit words");
	// a device dst16 as texel offsets from the 16-byte boundary at or below it, and each row's phase shift from its image row
	uint8_t *const base = dev ? dst16 - (reinterpret_cast<uintptr_t>(dst16) & 15) : nullptr;
	size_t const lead = dev ? (size_t)(dst16 - base)/2 : 0;
	auto out_of = [&](tw_hmap_rect const &R, int y) {return lead + (size_t)y*(pitch/2) + (size_t)R.x;};
	auto shift_of = [&](tw_hmap_rect const &R, int y, size_t img) {return dev ? (unsigned)((out_of(R, y) - img) & 7) : 0u;};
	size_t group[8] = {0, 0, 0, 0, 0, 0, 0, 0}; // texels of each shift's rows in the staging
	for_hmap_rows(W, r->rects, nrects, [&](tw_hmap_rect const &R, int y, size_t img) {group[shift_of(R, y, img)] += (size_t)R.w + 7;});
	bool const shifted = dev && group[0] < texels, direct = dev && !shifted;
	size_t const ntab = shifted ? 2*nrows : nrows, stage = texels + 64; // each group starts on an 8-texel boundary
	twi_hmap_row *d_rows, *h_rows;
	uint8_t *d_s1 = nullptr, *d_s2 = nullptr, *h_data = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		d_rows = c.take<twi_hmap_row>(ntab);
		if (!direct) {d_s1 = c.take<uint8_t>(2*stage);}
		if (shifted) {d_s2 = c.take<uint8_t>(2*stage + 16);}
	}); if (rc) return rc;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {h_rows = c.take<twi_hmap_row>(ntab); if (!dev) {h_data = c.take<uint8_t>(2*stage);}}); if (rc) return rc;
	size_t g0[8], at[8]; // each group's first texel and next free texel in the staging
	for (size_t d = 0, o = 0; d < 8; o += (group[d] + 7) & ~(size_t)7, ++d) {g0[d] = at[d] = o;}
	size_t k = 0;
	for_hmap_rows(W, r->rects, nrects, [&](tw_hmap_rect const &R, int y, size_t img) {
		if (direct) {set_hmap_row(h_rows[k++], out_of(R, y), img, R.w); return;}
		unsigned const d = shift_of(R, y, img);
		size_t const packed = pack_hmap_row(at[d], img, (unsigned)R.w);
		set_hmap_row(h_rows[k], packed, img, R.w);
		if (shifted) {set_hmap_row(h_rows[nrows + k], out_of(R, y), packed + d, R.w);} // in the second staging, the row has its destination's phase
		++k;
	});
	twi_job pending;
	pending.reads_image = true; // no cancellation point
	pending.complete = [dev, h_rows, h_data, nrows, W, dst16, pitch](tw_ctx *) -> int {
		for (size_t i = 0; i < nrows && !dev; ++i) {
			twi_hmap_row const &R = h_rows[i];
			memcpy(dst16 + (R.src/W)*pitch + 2*(R.src % W), h_data + 2*R.dst, 2*(size_t)R.w);
		}
		return TW_OK;
	};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemcpyAsync(d_rows, h_rows, ntab*sizeof(twi_hmap_row), cudaMemcpyHostToDevice, ctx->stream));
		int g = twi_hmap_scatter(ctx, ctx->stream, d_rows, (uint32_t)nrows, ctx->d_hmap, direct ? base : d_s1); if (g) return g;
		TW_CUDA(ctx, cudaEventRecord(ctx->async.image_free, ctx->stream)); // a later edit waits for this kernel only
		ctx->async.image_free_set = true;
		if (shifted) {
			for (size_t d = 0; d < 8; ++d) {
				if (at[d] > g0[d]) {TW_CUDA(ctx, cudaMemcpyAsync(d_s2 + 2*(g0[d] + d), d_s1 + 2*g0[d], 2*(at[d] - g0[d]), cudaMemcpyDeviceToDevice, ctx->stream));}
			}
			g = twi_hmap_scatter(ctx, ctx->stream, d_rows + nrows, (uint32_t)nrows, d_s2, base); if (g) return g;
		}
		if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(h_data, d_s1, 2*at[0], cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
}

int tw_read_heightmap(tw_ctx *ctx, const tw_hmap_read *r) {
	int const rc = tw_read_heightmap_launch(ctx, r);
	return rc ? rc : poll_job(ctx, 1);
}

// The AO of heightmap tiles as one launch of tw_hmap_ao.cubin's kernel: one CTA per (tile, sub-square), each with the heights its rays reach in shared
// memory. Sub-squares have at most TWI_AO_MAX_SIDE cells a side; when the tiles would give fewer CTAs than the device has SMs (a frame's few new tiles), the
// tiles are cut finer so that every SM gets work. Slot 0: [origins | set slots | zvals (host zvals) | ao (host ao)]; pinned staging: [origins | set slots |
// zvals (host zvals) | ao (pageable ao)].
int tw_hmap_tile_ao_launch(tw_ctx *ctx, const tw_hmap_ao_job *job) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!job) return tw_set_error(ctx, TW_ERR_ARG, "null job");
	if (!job->hs) return tw_set_error(ctx, TW_ERR_ARG, "null heightmap sampler");
	if (job->hs->edge_mode < 0 || job->hs->edge_mode > 2) return tw_set_error(ctx, TW_ERR_ARG, "bad edge_mode %d", job->hs->edge_mode);
	if (job->zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "zvsize %u < 2", job->zvsize);
	if (!job->zvals == !job->set) return tw_set_error(ctx, TW_ERR_ARG, "exactly one of zvals and set is required");
	if (!job->ao) return tw_set_error(ctx, TW_ERR_ARG, "null ao");
	uint32_t const n = job->ntiles, zv = job->zvsize, stride = zv - 1;
	if (n && (!job->origins_xy || (job->set && !job->tile_xy))) return tw_set_error(ctx, TW_ERR_ARG, "null origins_xy, or a set without tile_xy, with ntiles > 0");
	if (n == 0) return TW_OK;
	rc = validate_hmap(ctx, job->hs, nullptr); if (rc) return rc;
	std::vector<int> slots;
	const float *slab = nullptr;
	cudaEvent_t set_ev = nullptr;
	if (job->set) {rc = twi_tile_set_tiles(ctx, job->set, job->tile_xy, n, zv, slots, &slab, &set_ev); if (rc) return rc;}
	unsigned nsub = (stride + TWI_AO_MAX_SIDE - 1)/TWI_AO_MAX_SIDE;
	while (nsub < stride && (size_t)n*nsub*nsub < ctx->num_sms) ++nsub;
	unsigned const side = (stride + nsub - 1)/nsub;
	nsub = (stride + side - 1)/side;
	if ((size_t)n*nsub*nsub > 0x7fffffffu) return tw_set_error(ctx, TW_ERR_ARG, "too many tiles in one job");
	size_t const ao_bytes = (size_t)n*stride*stride, smem = (size_t)(side + 2*TWI_AO_RAY_LEN)*(side + 2*TWI_AO_RAY_LEN)*sizeof(float);
	static const char *const names[] = {"tw_hmap_ao_kernel"};
	cudaKernel_t k;
	rc = twi_module_kernels(ctx, "tw_hmap_ao.cubin", names, 1, &k); if (rc) return rc;
	TW_CUDA(ctx, cudaKernelSetAttributeForDevice(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem, ctx->device));
	twi_user<const float> z(job->zvals, job->set ? 0 : (size_t)n*zv*zv);
	uint8_t *const ao = job->ao;
	bool const dev_out = tw_is_device_ptr(ao), locked_out = !dev_out && twi_is_page_locked(ao);
	int32_t *d_org, *h_org; int *d_slots = nullptr, *h_slots = nullptr;
	uint8_t *d_ao = ao, *h_ao = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		d_org = c.take<int32_t>(2*(size_t)n); if (job->set) {d_slots = c.take<int>(n);}
		z.take(c); if (!dev_out) {d_ao = c.take<uint8_t>(ao_bytes);}
	}); if (rc) return rc;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		h_org = c.take<int32_t>(2*(size_t)n); if (job->set) {h_slots = c.take<int>(n);}
		z.take_pinned(c); if (!dev_out && !locked_out) {h_ao = c.take<uint8_t>(ao_bytes);}
	}); if (rc) return rc;
	memcpy(h_org, job->origins_xy, 2*(size_t)n*sizeof(int32_t));
	if (job->set) {memcpy(h_slots, slots.data(), n*sizeof(int));}
	twi_hmap_ao_args A;
	A.img = ctx->d_hmap; A.origins = d_org; A.zvals = job->set ? slab : z.d; A.slots = d_slots; A.ao = d_ao; A.H = *job->hs;
	A.zvsize = zv; A.side = side; A.nsub = nsub; A.dz = (float)(0.5*job->half_dxy); // src/tiled_mesh.cpp:612
	twi_job pending;
	pending.reads_image = true; // one kernel: no cancellation point
	pending.complete = [h_ao, ao, ao_bytes](tw_ctx *) -> int {if (h_ao) {memcpy(ao, h_ao, ao_bytes);} return TW_OK;};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemcpyAsync(d_org, h_org, 2*(size_t)n*sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
		if (job->set) {TW_CUDA(ctx, cudaMemcpyAsync(d_slots, h_slots, n*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));}
		int r = z.in(ctx); if (r) return r;
		if (job->set) {TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, set_ev, 0));} // a frame on another context may still write the slab
		void *args[] = {&A};
		TW_CUDA(ctx, cudaLaunchKernel((const void *)k, dim3(n*nsub*nsub), dim3(TWI_AO_THREADS), args, smem, ctx->stream));
		ctx->launches++;
		TW_CUDA(ctx, cudaEventRecord(ctx->async.image_free, ctx->stream)); // a later edit waits for this kernel only
		ctx->async.image_free_set = true;
		if (job->set) {TW_CUDA(ctx, cudaEventRecord(set_ev, ctx->stream));}
		if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(locked_out ? ao : h_ao, d_ao, ao_bytes, cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
}

int tw_hmap_tile_ao(tw_ctx *ctx, const tw_hmap_ao_job *job) {
	int const rc = tw_hmap_tile_ao_launch(ctx, job);
	return rc ? rc : poll_job(ctx, 1);
}

int tw_create_tiles_launch_hmap(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                                float wpz_max, uint32_t size, const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_shadows *shadows)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate_hmap(ctx, hs, shading); if (rc) return rc;
	ctx->last_erosion_steps = 0;
	return tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, shadows, hs);
}

} // extern "C"

int twi_create_tiles_launch(tw_ctx *ctx, const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                            uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval, float wpz_max, uint32_t size,
                            const tw_tile_outputs *out, const tw_tile_shading *shading, twi_job_tail *tail)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	if (hs) {rc = validate_hmap(ctx, hs, shading); if (rc) return rc;}
	ctx->last_erosion_steps = 0;
	return tiles_launch(ctx, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, wpz_max, size, out, shading, nullptr, hs, tail);
}

extern "C" {

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
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!data16 || !hs || !origins_xy || !out || ntiles == 0 || zvsize == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (hs->width <= 0 || hs->height <= 0 || hs->edge_mode < 0 || hs->edge_mode > 2) return tw_set_error(ctx, TW_ERR_ARG, "bad heightmap sampler");
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	twi_user<const uint8_t> img(data16, (size_t)2*hs->width*hs->height);
	twi_user<float> o(out, (size_t)ntiles*zvsize*zvsize);
	int32_t *d_org;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {d_org = c.take<int32_t>((size_t)ntiles*2); img.take(c); o.take(c);}); if (rc) return rc;
	TW_CUDA(ctx, cudaMemcpyAsync(d_org, origins_xy, (size_t)ntiles*8, cudaMemcpyHostToDevice, ctx->stream));
	rc = img.in(ctx); if (rc) return rc;
	rc = twi_hmap_sample_tiles(ctx, img.d, hs, d_org, ntiles, zvsize, o.d); if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // origins_xy is the caller's buffer
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ per-tile normals and ambient occlusion (N1)
int tw_tile_normals_batch(tw_ctx *ctx, const float *zvals, uint32_t ntiles, uint32_t zvsize, float dx_val, float dy_val, uint8_t *rgba, float *min_normal_z) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!zvals || !rgba || ntiles == 0 || zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (ntiles > 65535) return tw_set_error(ctx, TW_ERR_ARG, "at most 65535 tiles per call");
	size_t const stride = zvsize - 1;
	twi_user<const float> z(zvals, (size_t)ntiles*zvsize*zvsize);
	twi_user<uint8_t> o(rgba, (size_t)ntiles*stride*stride*4);
	unsigned *d_mn;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {d_mn = c.take<unsigned>(ntiles); z.take(c); o.take(c);}); if (rc) return rc;
	rc = z.in(ctx); if (rc) return rc;
	{
		std::vector<unsigned> init(ntiles, tw_f2ord(1.0f)); // min_normal_z = 1.0, src/tiled_mesh.cpp:868
		TW_CUDA(ctx, cudaMemcpyAsync(d_mn, init.data(), ntiles*sizeof(unsigned), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	rc = twi_tile_normals(ctx, ctx->stream, z.d, ntiles, zvsize, dx_val, dy_val, o.d, d_mn); if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
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
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!zvals || !origins_xy || !p || !ao || ntiles == 0 || zvsize < 2) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	uint32_t const ray = 36, stride = zvsize - 1, csz = stride + 2*ray; // AO_RAY_LEN, context_sz (src/tiled_mesh.cpp:43,601)
	size_t const tile_elems = (size_t)zvsize*zvsize, ctx_elems = (size_t)csz*csz, ao_elems = (size_t)stride*stride;
	bool const dev_in = tw_is_device_ptr(zvals), dev_out = tw_is_device_ptr(ao);
	bool const ctx_inside = (p->gen_mode >= TW_MGEN_SIMPLEX_GPU); // use_ao_zvals: the rays test the un-eroded context inside the tile too (src/tiled_mesh.cpp:604)
	// chunk of tiles whose context grids fit in ~2 GB
	uint32_t chunk = (uint32_t)std::min<size_t>(ntiles, std::max<size_t>(1, ((size_t)2 << 30)/(ctx_elems*sizeof(float))));
	if (chunk > 65535) chunk = 65535;
	float *d_cz, *s_z = nullptr; unsigned char *s_ao = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		d_cz = c.take<float>((size_t)chunk*ctx_elems); if (!dev_in) {s_z = c.take<float>((size_t)chunk*tile_elems);}
		if (!dev_out) {s_ao = c.take<unsigned char>((size_t)chunk*ao_elems);}
	}); if (rc) return rc;
	std::vector<int32_t> org(2*(size_t)chunk);
	for (uint32_t t0 = 0; t0 < ntiles; t0 += chunk) {
		uint32_t const nt = (ntiles - t0 < chunk) ? ntiles - t0 : chunk;
		const float *d_z = zvals + (size_t)t0*tile_elems;
		if (!dev_in) {TW_CUDA(ctx, cudaMemcpyAsync(s_z, d_z, (size_t)nt*tile_elems*sizeof(float), cudaMemcpyHostToDevice, ctx->stream)); d_z = s_z;}
		unsigned char *d_ao = dev_out ? ao + (size_t)t0*ao_elems : s_ao;
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
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!xy || !p || !q || !out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (n == 0) return TW_OK;
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	twi_user<const float> pts(xy, 2*n);
	twi_user<float> o(out, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {pts.take(c); o.take(c);}); if (rc) return rc;
	rc = pts.in(ctx); if (rc) return rc;
	rc = twi_eval_points(ctx, pts.d, n, p, q, o.d);
	if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// tw_eval_points, or get_clamped_height of the context's image (TW_PQ_HMAP), as the context's asynchronous job: host xy is copied into the pinned staging
// during the launch and goes up from there; the results go to device or page-locked out directly, and to pageable out through the staging, which the
// completion copies. Device scratch slot 0: [xy (host xy) | out (host out)]; pinned staging: [xy (host xy) | out (pageable out)].
int tw_points_launch(tw_ctx *ctx, const tw_points_job *job) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!job) return tw_set_error(ctx, TW_ERR_ARG, "null job");
	size_t const n = job->n;
	if (n == 0) return TW_OK;
	if (!job->xy || !job->q || !job->out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	bool const hmap = (job->q->kind == TW_PQ_HMAP);
	if (hmap) {
		rc = validate_hmap(ctx, job->hs, nullptr); if (rc) return rc;
		if (n > (size_t)0x7fffffff*256) return tw_set_error(ctx, TW_ERR_ARG, "tw_points_launch: too many points");
	}
	else {
		if (!job->p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
		if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
		rc = twi_eval_points_check(ctx, n, job->p, job->q); if (rc) return rc;
	}
	twi_user<const float> pts(job->xy, 2*n);
	bool const dev_out = tw_is_device_ptr(job->out), locked_out = !dev_out && twi_is_page_locked(job->out);
	float *d_out = job->out, *h_out = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {pts.take(c); if (!dev_out) {d_out = c.take<float>(n);}}); if (rc) return rc;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {pts.take_pinned(c); if (!dev_out && !locked_out) {h_out = c.take<float>(n);}}); if (rc) return rc;
	float *const out = job->out;
	twi_job pending;
	pending.reads_image = hmap; // one kernel: not cancellable
	pending.complete = [h_out, out, n](tw_ctx *) -> int {if (h_out) {memcpy(out, h_out, n*sizeof(float));} return TW_OK;};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		rc = pts.in(ctx); if (rc) return rc;
		if (hmap) {
			int const r = twi_hmap_points(ctx, ctx->d_hmap, job->hs, pts.d, n, d_out); if (r) return r;
			TW_CUDA(ctx, cudaEventRecord(ctx->async.image_free, ctx->stream)); // a later edit waits for this kernel only
			ctx->async.image_free_set = true;
		}
		else {int const r = twi_eval_points(ctx, pts.d, n, job->p, job->q, d_out); if (r) return r;}
		if (!dev_out) {TW_CUDA(ctx, cudaMemcpyAsync(locked_out ? out : h_out, d_out, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
}

int tw_erode(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p) {
	return tw_erode_tiles(ctx, heightmap, 1, xsize, ysize, nullptr, min_zval, num_iters, p);
}

int tw_erode_parallel(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p, uint32_t num_threads) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!heightmap || !p) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	if (xsize <= 0 || ysize <= 0) return tw_set_error(ctx, TW_ERR_ARG, "empty heightmap");
	if (num_iters == 0 || p->erode_amount <= 0.0) {ctx->last_erosion_steps = 0; return TW_OK;} // src/erosion.cpp:16
	size_t const n = (size_t)xsize*ysize;
	twi_user<float> m(heightmap, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {m.take(c);}); if (rc) return rc;
	rc = m.in(ctx); if (rc) return rc;
	rc = twi_erode_parallel(ctx, m.d, xsize, ysize, min_zval, num_iters, p, num_threads);
	if (rc) return rc;
	rc = m.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// tw_erode / tw_erode_parallel of one map, or of the context's image between its unpack and its pack, as the context's asynchronous job: the work tw_erode
// (twi_erode's single-map paths) and tw_erode_parallel enqueue, with the step count, the no-progress flag and the pack's error flag staged in a
// twi_hmap_stage that the completing poll unpacks; the image's lower clamp is its minimum, computed into the stage's min_z on the device. The sweeps mode
// (tw_erode_launch_ex) enqueues tw_erode_sweeps' one-band work the same way (twi_erode_sweeps_enqueue).
int tw_erode_launch(tw_ctx *ctx, const tw_erosion_job *job) {return tw_erode_launch_ex(ctx, job, nullptr);}

int tw_erode_launch_ex(tw_ctx *ctx, const tw_erosion_job *job, const tw_sweep_params *sw) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!job || !job->ep) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	bool const image = (job->heightmap == nullptr);
	if (job->mode != TW_EROSION_SERIAL && job->mode != TW_EROSION_OPENMP && job->mode != TW_EROSION_SWEEPS) return tw_set_error(ctx, TW_ERR_ARG, "bad erosion mode %d", job->mode);
	if (job->mode != TW_EROSION_OPENMP && job->num_threads) return tw_set_error(ctx, TW_ERR_ARG, "num_threads is for TW_EROSION_OPENMP only");
	bool const sweeps = (job->mode == TW_EROSION_SWEEPS);
	if (sweeps != (sw != nullptr)) return tw_set_error(ctx, TW_ERR_ARG, sweeps ? "TW_EROSION_SWEEPS needs its tw_sweep_params" : "tw_sweep_params are for TW_EROSION_SWEEPS only");
	if (sweeps && (sw->sweep == 0 || sw->halo < twi_sweep_view() + 12)) return tw_set_error(ctx, TW_ERR_ARG, "sweep must be > 0 and halo >= %d (view + 12)", twi_sweep_view() + 12);
	if (image) {
		if (job->xsize || job->ysize) return tw_set_error(ctx, TW_ERR_ARG, "the image's size is the tw_set_heightmap image's: xsize and ysize must be 0");
		if (ctx->parent) return tw_set_error(ctx, TW_ERR_ARG, "tables are set on the parent context, not on a shared one");
		if (!ctx->hmap_w) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_heightmap() has not been called");
	}
	else {
		if (job->vals) return tw_set_error(ctx, TW_ERR_ARG, "vals is an output of the image's erosion only");
		if (job->xsize <= 0 || job->ysize <= 0) return tw_set_error(ctx, TW_ERR_ARG, "empty heightmap");
	}
	int const xsize = image ? ctx->hmap_w : job->xsize, ysize = image ? ctx->hmap_h : job->ysize;
	size_t const n = (size_t)xsize*ysize;
	bool const erode = (job->num_iters > 0 && job->ep->erode_amount > 0.0); // src/erosion.cpp:16
	if (erode && !ctx->d_dir_table) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	bool const openmp = (job->mode == TW_EROSION_OPENMP), spec = erode && !openmp && !sweeps && twi_erode_spec_eligible(1, xsize, ysize, job->num_iters);
	twi_user<float> u(image ? job->vals : job->heightmap, n); // the caller's floats: the map, or the image's optional eroded floats
	// slot 0: the floats (unless the caller's are on the device); slot 1: the erosion's scratch; slot 2: [fixed words (ordered min/max, droplet counter) | stage]
	if (erode) {rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {u.take(c);}); if (rc) return rc;}
	size_t const ebytes = !erode ? 0 : openmp ? twi_erode_parallel_scratch_bytes(xsize, ysize) : sweeps ? twi_erode_sweeps_scratch_bytes(xsize, ysize)
	                                 : spec ? twi_erode_spec_scratch_bytes(xsize, ysize) : twi_erode_scratch_bytes(ctx, 1, xsize, ysize);
	if (ebytes) {rc = tw_reserve(ctx, 1, ebytes); if (rc) return rc;}
	twi_slot2_words *words; twi_hmap_stage *d_st;
	rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {words = c.take<twi_slot2_words>(1); d_st = c.take<twi_hmap_stage>(1);}); if (rc) return rc;
	rc = tw_reserve_pinned(ctx, sizeof(twi_hmap_stage)); if (rc) return rc;
	twi_hmap_stage *const h_st = (twi_hmap_stage *)ctx->h_pinned;
	if (image) { // the shared contexts' jobs may read the image; the context has none until the completing poll
		rc = begin_table_change(ctx); if (rc) return rc;
		ctx->hmap_w = ctx->hmap_h = 0;
	}
	tw_erosion_params const ep = *job->ep;
	float *const d_vals = u.d;
	unsigned *const d_mm = words->mm;
	twi_job pending;
	pending.cancellable = true; pending.reads_image = image;
	pending.complete = hmap_completion(h_st, nullptr, image ? xsize : 0, image ? ysize : 0);
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(d_st, 0, sizeof(twi_hmap_stage), ctx->stream));
		if (erode) {
			const float *d_min = nullptr; // the float map's clamp is job->min_zval
			if (image) { // tw_heightmap_to_floats_u16, tw_minmax_f32 (run_erosion's min_zval, src/heightmap.cpp:155-156)
				int r = twi_to_floats_u16(ctx, ctx->d_hmap, n, job->val_mult, job->val_add, d_vals); if (r) return r;
				r = twi_init_minmax(ctx, d_mm, 1); if (r) return r;
				r = twi_minmax(ctx, d_vals, n, d_mm); if (r) return r;
				r = twi_ord_min(ctx, d_mm, &d_st->min_z); if (r) return r;
				d_min = &d_st->min_z;
			}
			else {int const r = u.in(ctx); if (r) return r;} // the image's floats are an output only
			int r;
			if (openmp) {r = twi_erode_parallel_enqueue(ctx, ctx->d_scratch[1], d_vals, xsize, ysize, d_min, job->min_zval, job->num_iters, &ep, job->num_threads, &d_st->steps, &words->next);}
			else if (sweeps) {r = twi_erode_sweeps_enqueue(ctx, ctx->d_scratch[1], d_vals, xsize, ysize, d_min, job->min_zval, job->num_iters, &ep, sw->sweep, sw->halo, &d_st->steps);}
			else if (spec) {r = twi_erode_spec_enqueue(ctx, ctx->d_scratch[1], d_vals, xsize, ysize, d_min, job->min_zval, job->num_iters, &ep, &d_st->steps, &d_st->fail, false);}
			else {r = twi_erode_enqueue(ctx, ctx->stream, 0, ctx->d_scratch[1], 1, d_vals, 1, xsize, ysize, d_min, job->min_zval, job->num_iters, &ep, &d_st->steps);}
			if (r) return r;
			if (image) {r = twi_from_floats_u16(ctx, d_vals, n, job->val_mult, job->val_add, ctx->d_hmap, &d_st->bad); if (r) return r;}
			r = u.out(ctx); if (r) return r;
		}
		TW_CUDA(ctx, cudaMemcpyAsync(h_st, d_st, sizeof(twi_hmap_stage), cudaMemcpyDeviceToHost, ctx->stream));
		return TW_OK;
	});
}

// ------------------------------------------------------------------------------------------------ voxels
int tw_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *out) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!vp || !out) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	size_t tab_bytes = 0;
	rc = twi_voxel_fill_check(ctx, vp, &tab_bytes); if (rc) return rc;
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	twi_user<float> o(out, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {o.take(c);}); if (rc) return rc;
	rc = twi_voxel_fill(ctx, vp, rdata420, o.d);
	if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ streaming passes
int tw_heightmap_from_floats_u16(tw_ctx *ctx, const float *vals, size_t n, float val_mult, float val_add, uint8_t *out2n) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!vals || !out2n || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	twi_user<const float> v(vals, n);
	twi_user<uint8_t> o(out2n, 2*n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {v.take(c); o.take(c);}); if (rc) return rc;
	rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words)); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	unsigned *d_bad = &twi_slot2(ctx)->bad;
	TW_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(unsigned), ctx->stream));
	rc = twi_from_floats_u16(ctx, v.d, n, val_mult, val_add, o.d, d_bad);
	if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
	unsigned bad = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (bad) return tw_set_error(ctx, TW_ERR_ARG, "from_floats: value outside [0,256) (the reference asserts, src/heightmap.cpp:211)");
	return TW_OK;
}

int tw_heightmap_to_floats_u16(tw_ctx *ctx, const uint8_t *data2n, size_t n, float val_mult, float val_add, float *vals) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!vals || !data2n || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	twi_user<const uint8_t> img(data2n, 2*n);
	twi_user<float> o(vals, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {o.take(c); img.take(c);}); if (rc) return rc;
	rc = img.in(ctx); if (rc) return rc;
	rc = twi_to_floats_u16(ctx, img.d, n, val_mult, val_add, o.d);
	if (rc) return rc;
	rc = o.out(ctx); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// heightmap_t::proc_gen as the context's asynchronous job: generation, erosion with the grid's minimum as a device value, the z range, the texture scalars
// (twi_hmap_scales) and the pack, all on ctx->stream; the scalars and the step count come back through the pinned stage the completing poll unpacks
int tw_proc_gen_heightmap_launch(tw_ctx *ctx, uint32_t width, uint32_t height, float dx_val, float dy_val, const tw_height_params *p,
                                 uint32_t erosion_iters, const tw_erosion_params *ep, const tw_heightmap_outputs *out)
{
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!p || !out || width == 0 || height == 0 || (!out->data16 && !out->set_image)) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	if (width > 0x7fffffffu || height > 0x7fffffffu) return tw_set_error(ctx, TW_ERR_ARG, "heightmap size %u x %u", width, height);
	if (out->set_image && ctx->parent) return tw_set_error(ctx, TW_ERR_ARG, "tables are set on the parent context, not on a shared one");
	tw_grid2d g; g.x0 = -0.5*width; g.y0 = -0.5*height; g.dx = dx_val; g.dy = dy_val; g.nx = width; g.ny = height; // src/heightmap.cpp:135
	rc = validate_gen(ctx, &g, p); if (rc) return rc;
	if (p->gen_mode == TW_MGEN_SINE && !ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called");
	size_t const n = (size_t)width*height;
	bool const erode = (erosion_iters > 0 && ep && ep->erode_amount > 0.0); // run_erosion (src/heightmap.cpp:153-156, src/erosion.cpp:16)
	bool const spec = erode && twi_erode_spec_eligible(1, (int)width, (int)height, erosion_iters);
	bool const vals_dev = (out->vals && tw_is_device_ptr(out->vals)), img_dev = (out->data16 && tw_is_device_ptr(out->data16));
	// slot 0: [vals (unless on the device)] [image (unless on the device or the context's)]; slot 1: the sine tables, then the erosion's scratch;
	// slot 2: [fixed words (ordered min/max) | stage]
	float *d_vals = out->vals; uint8_t *s_img = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {if (!vals_dev) {d_vals = c.take<float>(n);} if (!img_dev && !out->set_image) {s_img = c.take<uint8_t>(2*n);}}); if (rc) return rc;
	size_t const ebytes = !erode ? 0 : (spec ? twi_erode_spec_scratch_bytes((int)width, (int)height) : twi_erode_scratch_bytes(ctx, 1, (int)width, (int)height));
	size_t const s1 = std::max(ebytes, twi_heightgen_slot1_bytes(&g, p));
	if (s1) {rc = tw_reserve(ctx, 1, s1); if (rc) return rc;}
	twi_slot2_words *words; twi_hmap_stage *d_st;
	rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {words = c.take<twi_slot2_words>(1); d_st = c.take<twi_hmap_stage>(1);}); if (rc) return rc;
	unsigned *const d_mm = words->mm;
	rc = tw_reserve_pinned(ctx, sizeof(twi_hmap_stage)); if (rc) return rc;
	twi_hmap_stage *const h_st = (twi_hmap_stage *)ctx->h_pinned;
	if (out->set_image) { // the old image goes now; the context has none until the completing poll
		rc = begin_table_change(ctx); if (rc) return rc;
		rc = twi_image_settle(ctx); if (rc) return rc;
		size_t const bytes = 2*n, had = (size_t)2*ctx->hmap_w*ctx->hmap_h;
		if (ctx->d_hmap && bytes != had) {TW_CUDA(ctx, cudaFree(ctx->d_hmap)); ctx->d_hmap = nullptr;}
		ctx->hmap_w = ctx->hmap_h = 0;
		if (!ctx->d_hmap) {TW_CUDA(ctx, cudaMalloc(&ctx->d_hmap, bytes));}
	}
	uint8_t *const d_img = out->set_image ? ctx->d_hmap : (img_dev ? out->data16 : s_img);
	twi_job pending;
	pending.cancellable = true; pending.reads_image = (out->set_image != 0);
	pending.complete = hmap_completion(h_st, out->info, out->set_image ? (int)width : 0, out->set_image ? (int)height : 0);
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(d_st, 0, sizeof(twi_hmap_stage), ctx->stream));
		int r = twi_init_minmax(ctx, d_mm, 1); if (r) return r;
		r = twi_heightgen(ctx, &g, p, 1, 0, nullptr, 1, d_vals, d_mm); if (r) return r;
		r = twi_hmap_scales(ctx, d_mm, p->mesh_height_scale, p->mesh_scale_z_inv, d_st); if (r) return r; // min_z: run_erosion's min_zval (src/heightmap.cpp:155-156)
		if (erode) {
			if (spec) {r = twi_erode_spec_enqueue(ctx, ctx->d_scratch[1], d_vals, (int)width, (int)height, &d_st->min_z, 0.0f, erosion_iters, ep, &d_st->steps, &d_st->fail, false);}
			else {r = twi_erode_enqueue(ctx, ctx->stream, 0, ctx->d_scratch[1], 1, d_vals, 1, (int)width, (int)height, &d_st->min_z, 0.0f, erosion_iters, ep, &d_st->steps);}
			if (r) return r;
			r = twi_init_minmax(ctx, d_mm, 1); if (r) return r;
			r = twi_minmax(ctx, d_vals, n, d_mm); if (r) return r; // get_heightmap_z_range
			r = twi_hmap_scales(ctx, d_mm, p->mesh_height_scale, p->mesh_scale_z_inv, d_st); if (r) return r;
		}
		r = twi_from_floats_u16_dev(ctx, d_vals, n, d_st, d_img); if (r) return r;
		if (out->data16 && d_img != out->data16) {TW_CUDA(ctx, cudaMemcpyAsync(out->data16, d_img, 2*n, cudaMemcpyDefault, ctx->stream));}
		if (out->vals && !vals_dev) {TW_CUDA(ctx, cudaMemcpyAsync(out->vals, d_vals, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
		TW_CUDA(ctx, cudaMemcpyAsync(h_st, d_st, sizeof(twi_hmap_stage), cudaMemcpyDeviceToHost, ctx->stream));
		return TW_OK;
	});
}

int tw_proc_gen_heightmap(tw_ctx *ctx, uint32_t width, uint32_t height, float dx_val, float dy_val, const tw_height_params *p,
                          uint32_t erosion_iters, const tw_erosion_params *ep, uint8_t *data16, float *vals, tw_heightmap_info *info)
{
	if (!data16) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	tw_heightmap_outputs o;
	memset(&o, 0, sizeof(o));
	o.data16 = data16; o.vals = vals; o.info = info;
	int const rc = tw_proc_gen_heightmap_launch(ctx, width, height, dx_val, dy_val, p, erosion_iters, ep, &o);
	if (rc) return rc;
	return poll_job(ctx, 1);
}

// gen_mesh in ground mode as the context's asynchronous job: the mesh and the probe are generated, then one-thread kernels turn the data's min/max and the
// probe's max |z| into the record's z values (twi_gen_mesh_zvals), glaciation reads zmax_est from the record and writes zbottom / ztop back, and the erosion
// builds its parameters from the record (twi_erode_dev_enqueue); the record comes back through the pinned staging, which the completing poll unpacks.
// With lights, a mesh shadow pass (twi_mesh_pass) follows on the final mesh, its clip z range read from the record.
// Scratch slot 0: [mesh (unless on the device) | probe | the shadow pass's]; slot 1: the sine tables, then the erosion's scratch; slot 2: [fixed words |
// record]; pinned staging: [record | mesh (pageable mesh) | the shadow pass's].
int tw_gen_mesh_launch_shadows(tw_ctx *ctx, const tw_gen_mesh_job *job, uint32_t nlights, const tw_tile_light *lights) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!job || !job->p || !job->ep || !job->mesh) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	int const MX = job->mesh_x_size, MY = job->mesh_y_size;
	if (MX <= 0 || MY <= 0 || MY > 65535) return tw_set_error(ctx, TW_ERR_ARG, "mesh size %d x %d", MX, MY);
	if (nlights && !lights) return tw_set_error(ctx, TW_ERR_ARG, "nlights > 0 without lights");
	twi_mesh_pass pass;
	if (nlights) {rc = pass.make(ctx, MX, MY, nlights, lights); if (rc) return rc;}
	tw_height_params const p = *job->p;
	tw_erosion_params const ep = *job->ep;
	tw_grid2d const grid = {(float)(job->xoff2 - MX/2), (float)(job->yoff2 - MY/2), job->dx_val, job->dy_val, (uint32_t)MX, (uint32_t)MY}; // gen_mesh_sine_table, src/mesh_gen.cpp:201-210
	float const xy_scene_size(0.5f*(job->x_scene_size + job->y_scene_size));
	float const rm_scale(1000.0*xy_scene_size/p.mesh_scale);
	tw_grid2d const probe = {0.0f, 0.0f, rm_scale, rm_scale, 128, 128}; // estimate_zminmax's EST_RAND_PARAM grid, src/mesh_gen.cpp:468-472
	rc = validate_gen(ctx, &grid, &p); if (rc) return rc;
	if (p.gen_mode == TW_MGEN_SINE && !ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called");
	size_t const n = (size_t)MX*MY, nprobe = (size_t)probe.nx*probe.ny;
	uint32_t const iters = job->erosion_iters;
	bool const erode = (iters > 0 && ep.erode_amount > 0.0); // apply_erosion, src/erosion.cpp:16
	bool const dev = tw_is_device_ptr(job->mesh), locked = !dev && twi_is_page_locked(job->mesh);
	float *d_mesh = job->mesh, *d_probe;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {if (!dev) {d_mesh = c.take<float>(n);} d_probe = c.take<float>(nprobe); pass.carve_dev(c);}); if (rc) return rc;
	size_t const s1 = std::max(erode ? twi_erode_dev_scratch_bytes(ctx, MX, MY, iters) : 0, std::max(twi_heightgen_slot1_bytes(&grid, &p), twi_heightgen_slot1_bytes(&probe, &p)));
	if (s1) {rc = tw_reserve(ctx, 1, s1); if (rc) return rc;}
	twi_gen_mesh_rec *d_rec;
	rc = twi_reserve_carve(ctx, 2, [&](twi_carve &c) {c.take<twi_slot2_words>(1); d_rec = c.take<twi_gen_mesh_rec>(1);}); if (rc) return rc;
	twi_gen_mesh_rec *h_rec; float *h_mesh = nullptr;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {h_rec = c.take<twi_gen_mesh_rec>(1); if (!dev && !locked) {h_mesh = c.take<float>(n);} pass.carve_pin(c);});
	if (rc) return rc;
	float const wpz = twi_water_rel(p.glaciate, p.custom_glaciate_exp, job->water_h_off_rel);
	float *const mesh = job->mesh;
	tw_gen_mesh_info *const info = job->info;
	twi_job pending;
	pending.cancellable = true;
	pending.complete = [h_rec, h_mesh, mesh, n, info, pass](tw_ctx *c) -> int {
		twi_gen_mesh_rec const r = *h_rec;
		if (r.fail) {c->last_erosion_steps = 0; return tw_set_error(c, TW_ERR_STATE, "speculative erosion made no progress (%u rounds)", r.fail);}
		c->last_erosion_steps = r.steps;
		if (info) {
			info->zmin = r.zmin; info->zmax = r.zmax; info->zmax_est = r.zmax_est; info->zbottom = r.zbottom; info->ztop = r.ztop;
			info->water_plane_z = r.water_plane_z; info->erosion_moves = r.steps;
		}
		if (h_mesh) {memcpy(mesh, h_mesh, n*sizeof(float));}
		pass.complete();
		return TW_OK;
	};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(d_rec, 0, sizeof(twi_gen_mesh_rec), ctx->stream));
		int r = twi_init_minmax(ctx, d_rec->mm, 1); if (r) return r;
		r = twi_heightgen(ctx, &grid, &p, 0, 0, nullptr, 1, d_mesh, d_rec->mm); if (r) return r;     // the mesh and calc_zminmax
		r = twi_heightgen(ctx, &probe, &p, 0, 0, nullptr, 1, d_probe, nullptr); if (r) return r;
		r = twi_gen_mesh_zvals(ctx, d_rec, d_probe, nprobe, p.gen_mode == TW_MGEN_SINE, wpz, job->water_h_off, job->prev_zbottom, job->prev_ztop,
		                       job->prev_water_plane_z); if (r) return r;
		if (p.glaciate) { // gen_terrain_map -> glaciate(): zbottom / ztop of the glaciated mesh
			r = twi_glaciate_mesh_rec(ctx, d_mesh, MX, MY, job->xoff2, job->yoff2, MX, MY, &p, d_rec); if (r) return r;
			r = twi_gen_mesh_zbottom(ctx, d_rec); if (r) return r;
		}
		if (erode) {r = twi_erode_dev_enqueue(ctx, ctx->d_scratch[1], d_mesh, MX, MY, iters, &ep, d_rec); if (r) return r;}
		r = pass.enqueue(ctx, d_mesh, d_rec); if (r) return r; // calc_mesh_shadows per light on the final mesh, with the record's zmin / zmax
		if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(locked ? mesh : h_mesh, d_mesh, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
		TW_CUDA(ctx, cudaMemcpyAsync(h_rec, d_rec, sizeof(twi_gen_mesh_rec), cudaMemcpyDeviceToHost, ctx->stream));
		return TW_OK;
	});
}

int tw_gen_mesh_launch(tw_ctx *ctx, const tw_gen_mesh_job *job) {return tw_gen_mesh_launch_shadows(ctx, job, 0, nullptr);}

// calc_mesh_shadows over one whole mesh for every light of the job, as the context's pending job (twi_mesh_pass). Scratch slot 0: [mesh (unless on the device)
// | the pass's]; pinned staging: [host mesh | the pass's].
int tw_mesh_shadows_launch(tw_ctx *ctx, const tw_mesh_shadows_job *job) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!job || !job->mesh) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	twi_mesh_pass pass;
	rc = pass.make(ctx, job->xsize, job->ysize, job->nlights, job->lights); if (rc) return rc;
	twi_user<const float> z(job->mesh, (size_t)job->xsize*job->ysize);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {z.take(c); pass.carve_dev(c);}); if (rc) return rc;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {z.take_pinned(c); pass.carve_pin(c);}); if (rc) return rc;
	twi_job pending;
	pending.cancellable = true;
	pending.complete = [pass](tw_ctx *) -> int {pass.complete(); return TW_OK;};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		int r = z.in(ctx); if (r) return r;
		return pass.enqueue(ctx, z.d, nullptr);
	});
}

int tw_mesh_shadows(tw_ctx *ctx, const float *mesh, int xsize, int ysize, const tw_shadow_params *sp, const float *sh_in_x, const float *sh_in_y, uint8_t *smask,
                    float *sh_out_x, float *sh_out_y)
{
	if (!ctx) return TW_ERR_ARG;
	if (!sp) return tw_set_error(ctx, TW_ERR_ARG, "null argument");
	tw_tile_light L;
	L.sp = *sp; L.sh_in_x = sh_in_x; L.sh_in_y = sh_in_y; L.smask = smask; L.sh_out_x = sh_out_x; L.sh_out_y = sh_out_y;
	tw_mesh_shadows_job const job = {mesh, xsize, ysize, 1, &L};
	int const rc = tw_mesh_shadows_launch(ctx, &job);
	if (rc) return rc;
	return poll_job(ctx, 1);
}

int tw_minmax_f32(tw_ctx *ctx, const float *vals, size_t n, tw_minmax *mm) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!vals || !mm || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "null/empty argument");
	twi_user<const float> v(vals, n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {v.take(c);}); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words)); if (rc) return rc;
	unsigned *d_mm = twi_slot2(ctx)->mm;
	rc = twi_init_minmax(ctx, d_mm, 1); if (rc) return rc;
	rc = twi_minmax(ctx, v.d, n, d_mm); if (rc) return rc;
	return read_minmax(ctx, d_mm, mm, 1);
}

} // extern "C"
