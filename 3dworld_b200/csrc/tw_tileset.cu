// tw_tileset.cu - tile sets (include/tw3d.h, tw_tile_set_*): the live tiles' zvals kept in device memory the set owns, and per light slot the mesh shadows
// each tile was last computed with. A relight is the context's asynchronous job: it recomputes only the tiles whose result can have changed (the cache rules
// are in tw_tileset_rules.h) through the unchanged mesh-shadow plan and kernels of tw_shadows.cu, with the cached sh_out rows of valid neighbours as caller
// rows, so every output equals tw_tile_shadows_batch_ex on all resident tiles. The kernels here only move tiles: gather a batch's zvals and caller rows out
// of the slabs, scatter its results back, gather the requested outputs - one launch each per light, 16-byte accesses where the sizes and pointers allow.
// A frame launch (tw_tile_set_create_tiles_launch) appends the put and the relight to a tile job on any context of the set's family; the set's event orders
// the device work on its slabs across those contexts, while the host state is committed at launch, in launch order.
#include "tw_internal.h"
#include "tw_tileset_rules.h"
#include <algorithm>
#include <new>

struct tw_tile_set {
	struct slot_t {                                  // one light slot (its valid bits are st.valid[l])
		bool have = false;                           // sp holds the params the valid tiles were computed with
		tw_shadow_params sp;
		unsigned char *d_m = nullptr;                // capacity*zvsize^2 bytes: each tile's smask
		float *d_ox = nullptr, *d_oy = nullptr;      // capacity*zvsize floats each: each tile's sh_out_x / sh_out_y
	};
	tw_ctx *ctx = nullptr;
	uint32_t zvsize = 0, nlights = 0;
	twts::state st;                                  // resident tile -> slab slot, free slots, per light slot the valid bits
	uint32_t capacity = 0;                           // slots allocated
	float *d_z = nullptr;                            // capacity*zvsize^2 floats: the zvals slab (the set's own memory: tw_reserve may re-allocate scratch under a job)
	cudaEvent_t ev = nullptr;                        // recorded after the last device work that touched the slabs, on whichever context of the family enqueued it
	std::vector<slot_t> L;
};

namespace {

// tile i of dst (at slot dst_idx[i], or i) = tile src_idx[i] (or i) of src, or `fill` where src_idx[i] < 0
template <typename T>
__global__ void __launch_bounds__(256)
tiles_copy_kernel(T *__restrict__ dst, const int *__restrict__ dst_idx, const T *__restrict__ src, const int *__restrict__ src_idx, size_t words, uint32_t n, T fill) {
	for (uint32_t t = blockIdx.y; t < n; t += gridDim.y) {
		int const s = src_idx ? __ldg(src_idx + t) : (int)t, d = dst_idx ? __ldg(dst_idx + t) : (int)t;
		T *o = dst + (size_t)d*words;
		const T *in = (s >= 0) ? src + (size_t)s*words : nullptr;
		for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x*blockDim.x) {o[i] = in ? in[i] : fill;}
	}
}

// n tiles of tile_bytes each; fill = a 32-bit pattern (only used with a src_idx that holds negative entries, whose tiles are then whole 32-bit words)
int copy_tiles(tw_ctx *ctx, void *dst, const int *dst_idx, const void *src, const int *src_idx, size_t tile_bytes, uint32_t n, uint32_t fill = 0) {
	if (n == 0) return TW_OK;
	uintptr_t const a = (uintptr_t)dst | (uintptr_t)src | (uintptr_t)tile_bytes;
	unsigned const gy = std::min<uint32_t>(n, 65535);
	auto grid = [&](size_t words) {return dim3((unsigned)std::min<size_t>((words + 255)/256, 64), gy);};
	if (!(a & 15)) {
		size_t const w = tile_bytes/16;
		tiles_copy_kernel<uint4><<<grid(w), 256, 0, ctx->stream>>>((uint4 *)dst, dst_idx, (const uint4 *)src, src_idx, w, n, make_uint4(fill, fill, fill, fill));
	}
	else if (!(a & 3)) {
		size_t const w = tile_bytes/4;
		tiles_copy_kernel<unsigned><<<grid(w), 256, 0, ctx->stream>>>((unsigned *)dst, dst_idx, (const unsigned *)src, src_idx, w, n, fill);
	}
	else {tiles_copy_kernel<unsigned char><<<grid(tile_bytes), 256, 0, ctx->stream>>>((unsigned char *)dst, dst_idx, (const unsigned char *)src, src_idx, tile_bytes, n, (unsigned char)fill);}
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// unique keys of n (x, y) pairs, or false when one is named twice
bool read_keys(const int32_t *tile_xy, uint32_t n, std::vector<twts::key> &keys) {
	keys.resize(n);
	for (uint32_t i = 0; i < n; ++i) {keys[i] = twts::key(tile_xy[2*i], tile_xy[2*i+1]);}
	std::vector<twts::key> sorted(keys);
	std::sort(sorted.begin(), sorted.end());
	return std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end();
}

// slabs for at least `need` tiles: geometric growth, the old contents copied over on ctx's stream once the set's device work on any context is done (it holds
// the old slab pointers); nothing changes when an allocation fails
int grow(tw_tile_set *s, uint32_t need, tw_ctx *ctx) {
	if (need <= s->capacity) return TW_OK;
	TW_CUDA(ctx, cudaEventSynchronize(s->ev));
	uint32_t const cap = std::max(need, std::max<uint32_t>(16, 2*s->capacity));
	size_t const zt = (size_t)s->zvsize*s->zvsize, edge = (size_t)s->zvsize*sizeof(float);
	std::vector<void *> fresh; // zvals, then smask / sh_out_x / sh_out_y of every slot
	auto alloc = [&](size_t bytes) {void *p = nullptr; if (cudaMalloc(&p, bytes) != cudaSuccess) {cudaGetLastError(); return false;} fresh.push_back(p); return true;};
	bool ok = alloc(cap*zt*sizeof(float));
	for (uint32_t l = 0; ok && l < s->nlights; ++l) {ok = alloc(cap*zt + 4) && alloc(cap*edge) && alloc(cap*edge);}
	cudaError_t e = cudaSuccess;
	if (ok && s->capacity) {
		size_t const old = s->capacity;
		if (e == cudaSuccess) e = cudaMemcpyAsync(fresh[0], s->d_z, old*zt*sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream);
		for (uint32_t l = 0; l < s->nlights && e == cudaSuccess; ++l) {
			tw_tile_set::slot_t const &S = s->L[l];
			e = cudaMemcpyAsync(fresh[1 + 3*l], S.d_m, old*zt, cudaMemcpyDeviceToDevice, ctx->stream);
			if (e == cudaSuccess) e = cudaMemcpyAsync(fresh[2 + 3*l], S.d_ox, old*edge, cudaMemcpyDeviceToDevice, ctx->stream);
			if (e == cudaSuccess) e = cudaMemcpyAsync(fresh[3 + 3*l], S.d_oy, old*edge, cudaMemcpyDeviceToDevice, ctx->stream);
		}
		if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
	}
	if (!ok || e != cudaSuccess) {
		cudaStreamSynchronize(ctx->stream);
		for (void *p : fresh) cudaFree(p);
		if (!ok) return tw_set_error(ctx, TW_ERR_CUDA, "tile set: no device memory for %u tiles of %u^2", cap, s->zvsize);
		return tw_set_error(ctx, TW_ERR_CUDA, "tile set: growing the slabs: %s", cudaGetErrorString(e));
	}
	cudaFree(s->d_z); s->d_z = (float *)fresh[0];
	for (uint32_t l = 0; l < s->nlights; ++l) {
		tw_tile_set::slot_t &S = s->L[l];
		cudaFree(S.d_m); cudaFree(S.d_ox); cudaFree(S.d_oy);
		S.d_m = (unsigned char *)fresh[1 + 3*l]; S.d_ox = (float *)fresh[2 + 3*l]; S.d_oy = (float *)fresh[3 + 3*l];
		s->st.valid[l].resize(cap, 0);
	}
	s->capacity = cap;
	return TW_OK;
}

std::vector<twts::signs> slot_signs(const tw_tile_set *s) {
	std::vector<twts::signs> sg(s->nlights);
	for (uint32_t l = 0; l < s->nlights; ++l) {
		tw_tile_set::slot_t const &S = s->L[l];
		sg[l].sx = S.have ? twts::light_sign(S.sp.lpos[0]) : 1; sg[l].sy = S.have ? twts::light_sign(S.sp.lpos[1]) : 1;
	}
	return sg;
}

// per asked light: the slot's params differ from sps[l] (or it has none), so a relight recomputes all of it
std::vector<uint8_t> slot_resets(const tw_tile_set *s, const tw_shadow_params *sps, uint32_t nlights) {
	std::vector<uint8_t> reset(nlights);
	for (uint32_t l = 0; l < nlights; ++l) {reset[l] = !s->L[l].have || memcmp(&s->L[l].sp, &sps[l], sizeof(tw_shadow_params)) != 0;}
	return reset;
}

// the removes and puts of a frame (tw_tile_set_create_tiles_launch, tw_tile_set_stale_after): each list names a tile once, every removed tile is resident and
// no tile is both removed and put
int frame_keys(tw_ctx *ctx, const tw_tile_set *s, const int32_t *remove_xy, uint32_t nremove, const int32_t *put_xy, uint32_t nput,
               std::vector<twts::key> &rk, std::vector<twts::key> &pk) {
	if ((nremove && !remove_xy) || (nput && !put_xy)) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: null remove_xy or tile_xy with a count > 0");
	if (!read_keys(remove_xy, nremove, rk)) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: remove_xy names a tile twice");
	for (twts::key const &k : rk) {if (!s->st.where.count(k)) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: removed tile (%d, %d) is not resident", k.first, k.second);}
	if (!read_keys(put_xy, nput, pk)) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: tile_xy names a tile twice");
	std::vector<twts::key> sorted(rk);
	std::sort(sorted.begin(), sorted.end());
	for (twts::key const &k : pk) {
		if (std::binary_search(sorted.begin(), sorted.end(), k)) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: tile (%d, %d) is both removed and put", k.first, k.second);
	}
	return TW_OK;
}

// A relight planned on the host against a set state: per light the batch B (invalid requested tiles + their invalid upstream closure), its plan, and the
// slab slots it reads and writes. Its int region ([requested tiles' slots | per light: plan, B's slots, x and y caller-row sources]) is staged in pinned memory
// and goes up in one copy.
struct relight_t {
	struct batch_t {
		bool reset = false;                      // the slot's params differ: every tile of it is invalid
		std::vector<twts::key> B;
		twi_shadow_plan P;
		std::vector<int> ints;                   // [plan (3*nB) | B's slots | x caller-row sources | y caller-row sources]
		size_t off_ints = 0;                     // byte offset into the int region
	};
	uint32_t n = 0, nl = 0, zv = 0, maxB = 0;
	std::vector<tw_tile_set_light> lights;
	std::vector<int> req_slot;
	std::vector<char> dev_m, dev_x, dev_y;
	std::vector<batch_t> jobs;
	size_t ints_bytes = 0;
	// the device scratch: [B's zvals | mask | 64-bit keys | x edges (outputs, then caller rows) | y edges | per light: staging of the host-bound smask, sh_out_x
	// and sh_out_y (nullptr: none) | int region]
	struct dev_t {float *zB, *ox, *oy; unsigned char *mB; unsigned long long *keys; std::vector<unsigned char *> om; std::vector<float *> sx, sy; char *ints;};
	void dev_layout(twi_carve &c, dev_t &D) const {
		size_t const zt = (size_t)zv*zv, e2 = 2*(size_t)maxB*zv;
		D.zB = c.take<float>(maxB*zt); D.mB = c.take<unsigned char>(maxB*zt + 4); D.keys = c.take<unsigned long long>(e2); D.ox = c.take<float>(e2); D.oy = c.take<float>(e2);
		D.om.resize(nl); D.sx.resize(nl); D.sy.resize(nl);
		for (uint32_t l = 0; l < nl; ++l) {
			D.om[l] = dev_m[l] ? nullptr : c.take<unsigned char>(n*zt);
			D.sx[l] = (lights[l].sh_out_x && !dev_x[l]) ? c.take<float>((size_t)n*zv) : nullptr; D.sy[l] = (lights[l].sh_out_y && !dev_y[l]) ? c.take<float>((size_t)n*zv) : nullptr;
		}
		D.ints = c.take<char>(ints_bytes);
	}
	size_t dev_bytes() const {twi_carve c; dev_t D; dev_layout(c, D); return c.bytes;}
};

// validates req against st (TW_ERR_ARG on ctx; nothing changes) and plans it
int relight_plan(tw_ctx *ctx, const tw_tile_set *s, twts::state const &st, const tw_tile_set_request *req, relight_t &R) {
	if (!req || !req->tile_xy || req->n == 0 || !req->lights || req->nlights == 0 || req->nlights > s->nlights)
		return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: needs tile_xy, n >= 1 and 1 .. %u lights", s->nlights);
	uint32_t const n = req->n, nl = req->nlights;
	R.n = n; R.nl = nl; R.zv = s->zvsize;
	R.lights.assign(req->lights, req->lights + nl);
	std::vector<twts::key> keys;
	if (!read_keys(req->tile_xy, n, keys)) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: tile_xy names a tile twice");
	R.req_slot.resize(n);
	for (uint32_t i = 0; i < n; ++i) {
		auto const it = st.where.find(keys[i]);
		if (it == st.where.end()) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: tile (%d, %d) is not resident", keys[i].first, keys[i].second);
		R.req_slot[i] = (int)it->second;
	}
	R.dev_m.assign(nl, 0); R.dev_x.assign(nl, 0); R.dev_y.assign(nl, 0);
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_set_light const &Lr = R.lights[l];
		if (!Lr.smask) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: light %u has no smask", l);
		R.dev_m[l] = tw_is_device_ptr(Lr.smask);
		if (R.dev_m[l] && ((size_t)Lr.smask & 3)) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: light %u: a device smask must be 4-byte aligned", l);
		R.dev_x[l] = Lr.sh_out_x && tw_is_device_ptr(Lr.sh_out_x); R.dev_y[l] = Lr.sh_out_y && tw_is_device_ptr(Lr.sh_out_y);
	}
	R.jobs.resize(nl);
	twi_carve ints; ints.take<int>(n);                       // the int region's offsets: it starts with the requested tiles' slots
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_set::slot_t const &S = s->L[l];
		relight_t::batch_t &J = R.jobs[l];
		tw_shadow_params const &sp = R.lights[l].sp;
		J.reset = !S.have || memcmp(&S.sp, &sp, sizeof(sp)) != 0;
		int const sx = twts::light_sign(sp.lpos[0]), sy = twts::light_sign(sp.lpos[1]);
		std::vector<uint8_t> const none(J.reset ? st.valid[l].size() : 0, 0);
		std::vector<uint8_t> const &valid = J.reset ? none : st.valid[l];
		J.B = twts::recompute_batch(st.where, valid, keys, sx, sy);
		uint32_t const nB = (uint32_t)J.B.size();
		R.maxB = std::max(R.maxB, nB);
		if (nB) {
			std::vector<int32_t> bxy(2*(size_t)nB);
			for (uint32_t t = 0; t < nB; ++t) {bxy[2*t] = J.B[t].first; bxy[2*t+1] = J.B[t].second;}
			twi_shadow_plan_make(bxy.data(), nB, &sp, true, true, &J.P);
			J.ints.resize(twi_shadow_plan_ints(nB) + 3*(size_t)nB);
			twi_shadow_plan_pack(J.P, J.ints.data());
			int *bs = J.ints.data() + twi_shadow_plan_ints(nB), *rx = bs + nB, *ry = rx + nB;
			auto cached = [&](twts::key const &k) {auto const it = st.where.find(k); return (it != st.where.end() && valid[it->second]) ? (int)it->second : -1;};
			for (uint32_t t = 0; t < nB; ++t) {
				bs[t] = (int)st.where.find(J.B[t])->second;
				rx[t] = cached(twts::key(J.B[t].first, J.B[t].second + sy)); // sh_in_x row: the sh_out_x of (tx, ty + sy); not resident -> MESH_MIN_Z
				ry[t] = cached(twts::key(J.B[t].first + sx, J.B[t].second)); // sh_in_y row: the sh_out_y of (tx + sx, ty)
			}
		}
		J.off_ints = ints.bytes; ints.take<int>(J.ints.size());
	}
	R.ints_bytes = ints.bytes;
	return TW_OK;
}

// Enqueues R on ctx->stream into R.dev_bytes() of device scratch at d, its int region staged at h (R.ints_bytes of pinned memory that stays untouched until the
// work is done); records the set's event once the slabs are no longer read or written, then copies the host outputs. The caller has made the stream wait on the
// set's event.
int relight_enqueue(tw_ctx *ctx, tw_tile_set *s, relight_t const &R, char *d, char *h) {
	uint32_t const n = R.n, zv = s->zvsize;
	size_t const zt = (size_t)zv*zv, eb = (size_t)zv*sizeof(float);
	twi_carve c{d};
	relight_t::dev_t D; R.dev_layout(c, D);
	float *d_zB = D.zB, *d_ox = D.ox, *d_oy = D.oy; unsigned char *d_mB = D.mB; unsigned long long *d_keys = D.keys; char *d_ints = D.ints;
	memcpy(h, R.req_slot.data(), n*sizeof(int));
	for (relight_t::batch_t const &J : R.jobs) {memcpy(h + J.off_ints, J.ints.data(), J.ints.size()*sizeof(int));}
	uint32_t minz_bits; {float const m = TW_MESH_MIN_Z; memcpy(&minz_bits, &m, 4);}
	TW_CUDA(ctx, cudaMemcpyAsync(d_ints, h, R.ints_bytes, cudaMemcpyHostToDevice, ctx->stream));
	const int *d_req = (const int *)d_ints;
	for (uint32_t l = 0; l < R.nl; ++l) {
		tw_tile_set::slot_t &S = s->L[l];
		relight_t::batch_t const &J = R.jobs[l];
		uint32_t const nB = (uint32_t)J.B.size();
		tw_tile_set_light const &Lr = R.lights[l];
		if (nB) {
			const int *d_plan = (const int *)(d_ints + J.off_ints), *d_bs = d_plan + twi_shadow_plan_ints(nB), *d_rx = d_bs + nB, *d_ry = d_rx + nB;
			int r = copy_tiles(ctx, d_zB, nullptr, s->d_z, d_bs, zt*sizeof(float), nB); if (r) return r;            // B's zvals
			r = copy_tiles(ctx, d_ox + (size_t)nB*zv, nullptr, S.d_ox, d_rx, eb, nB, minz_bits); if (r) return r;  // caller rows: cached sh_out of valid neighbours
			r = copy_tiles(ctx, d_oy + (size_t)nB*zv, nullptr, S.d_oy, d_ry, eb, nB, minz_bits); if (r) return r;
			r = twi_shadow_enqueue(ctx, ctx->stream, J.P, d_zB, nB, zv, d_mB, d_keys, d_ox, d_oy, d_plan, true); if (r) return r;
			r = copy_tiles(ctx, S.d_m, d_bs, d_mB, nullptr, zt, nB); if (r) return r;                                 // results into the slot
			r = copy_tiles(ctx, S.d_ox, d_bs, d_ox, nullptr, eb, nB); if (r) return r;
			r = copy_tiles(ctx, S.d_oy, d_bs, d_oy, nullptr, eb, nB); if (r) return r;
		}
		// the requested tiles' outputs, in request order
		unsigned char *om = R.dev_m[l] ? Lr.smask : D.om[l];
		float *ox = !Lr.sh_out_x ? nullptr : (R.dev_x[l] ? Lr.sh_out_x : D.sx[l]);
		float *oy = !Lr.sh_out_y ? nullptr : (R.dev_y[l] ? Lr.sh_out_y : D.sy[l]);
		int r = copy_tiles(ctx, om, nullptr, S.d_m, d_req, zt, n); if (r) return r;
		if (ox) {r = copy_tiles(ctx, ox, nullptr, S.d_ox, d_req, eb, n); if (r) return r;}
		if (oy) {r = copy_tiles(ctx, oy, nullptr, S.d_oy, d_req, eb, n); if (r) return r;}
	}
	TW_CUDA(ctx, cudaEventRecord(s->ev, ctx->stream));
	for (uint32_t l = 0; l < R.nl; ++l) { // host outputs: one copy each, at the end
		tw_tile_set_light const &Lr = R.lights[l];
		if (D.om[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.smask, D.om[l], n*zt, cudaMemcpyDeviceToHost, ctx->stream));}
		if (D.sx[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.sh_out_x, D.sx[l], n*eb, cudaMemcpyDeviceToHost, ctx->stream));}
		if (D.sy[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.sh_out_y, D.sy[l], n*eb, cudaMemcpyDeviceToHost, ctx->stream));}
	}
	return TW_OK;
}

// after an enqueued relight: each slot holds the request's params, and B is valid in it
void relight_commit(tw_tile_set *s, relight_t const &R, uint8_t *recomputed) {
	std::vector<uint8_t> computed(s->capacity, 0);
	for (uint32_t l = 0; l < R.nl; ++l) {
		tw_tile_set::slot_t &S = s->L[l];
		relight_t::batch_t const &J = R.jobs[l];
		std::vector<uint8_t> &valid = s->st.valid[l];
		if (J.reset) {std::fill(valid.begin(), valid.end(), 0);}
		S.have = true; S.sp = R.lights[l].sp;
		for (twts::key const &k : J.B) {uint32_t const slot = s->st.where.find(k)->second; valid[slot] = 1; computed[slot] = 1;}
	}
	if (recomputed) {for (uint32_t i = 0; i < R.n; ++i) {recomputed[i] = computed[R.req_slot[i]];}}
}

void invalidate_all(tw_tile_set *s) { // what the slots hold is unknown: everything is recomputed next time
	for (uint32_t l = 0; l < s->nlights; ++l) {s->L[l].have = false; std::fill(s->st.valid[l].begin(), s->st.valid[l].end(), 0);}
}

// The set's part of a frame's tile job: prepare grows the slabs before the job enqueues anything; enqueue, after the chunk join, waits for the set's earlier
// device work, scatters the job's zvals into the put tiles' slots and runs the relight (or records the set's event itself).
struct frame_tail : twi_job_tail {
	tw_tile_set *s = nullptr;
	twts::state post;                // the set's host state after the frame's removes and puts
	std::vector<int> idx;            // the put tiles' slab slots, in tile_xy order
	uint32_t ntiles = 0;
	bool relight = false;
	relight_t R;
	// [put tiles' slots | the relight's memory] of the device scratch (d) and of the pinned staging (h)
	void layout(twi_carve &d, twi_carve &h, int *&d_idx, int *&h_idx, char *&d_rl, char *&h_rl) const {
		d_idx = d.take<int>(ntiles); h_idx = h.take<int>(ntiles);
		d_rl = relight ? d.take<char>(R.dev_bytes()) : nullptr; h_rl = relight ? h.take<char>(R.ints_bytes) : nullptr;
	}
	int prepare(tw_ctx *ctx) override {return grow(s, post.used, ctx);}
	// once this starts the slabs may be partly written, so every failure from here on is reported as TW_ERR_CUDA (the code that selects the error state)
	int enqueue(tw_ctx *ctx, const float *d_zvals, char *d, char *h) override {
		int const rc = enqueue_tail(ctx, d_zvals, d, h);
		return (rc && rc != TW_ERR_CUDA) ? TW_ERR_CUDA : rc;
	}
	int enqueue_tail(tw_ctx *ctx, const float *d_zvals, char *d, char *h) {
		twi_carve dc{d}, hc{h}; int *d_idx, *h_idx; char *d_rl, *h_rl;
		layout(dc, hc, d_idx, h_idx, d_rl, h_rl);
		memcpy(h_idx, idx.data(), ntiles*sizeof(int));
		TW_CUDA(ctx, cudaMemcpyAsync(d_idx, h_idx, ntiles*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
		TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, s->ev, 0));
		int rc = copy_tiles(ctx, s->d_z, d_idx, d_zvals, nullptr, (size_t)s->zvsize*s->zvsize*sizeof(float), ntiles); if (rc) return rc;
		if (relight) return relight_enqueue(ctx, s, R, d_rl, h_rl);
		TW_CUDA(ctx, cudaEventRecord(s->ev, ctx->stream));
		return TW_OK;
	}
};

} // namespace

extern "C" {

int tw_tile_set_create(tw_ctx *ctx, uint32_t zvsize, uint32_t nlights, tw_tile_set **out) {
	if (out) *out = nullptr;
	if (!ctx) return TW_ERR_ARG;
	if (!out || zvsize < 2 || nlights < 1) return tw_set_error(ctx, TW_ERR_ARG, "tile set: needs out, zvsize >= 2 and nlights >= 1 (zvsize %u, nlights %u)", zvsize, nlights);
	TW_CUDA(ctx, cudaSetDevice(ctx->device));
	tw_tile_set *s = new (std::nothrow) tw_tile_set();
	if (!s) return tw_set_error(ctx, TW_ERR_CUDA, "tile set: out of host memory");
	try {s->L.resize(nlights); s->st.valid.resize(nlights);} catch (...) {delete s; return tw_set_error(ctx, TW_ERR_CUDA, "tile set: out of host memory");}
	cudaError_t const e = cudaEventCreateWithFlags(&s->ev, cudaEventDisableTiming);
	if (e != cudaSuccess) {delete s; return tw_set_error(ctx, TW_ERR_CUDA, "tile set: event: %s", cudaGetErrorString(e));}
	try {ctx->sets.push_back(s);} catch (...) {cudaEventDestroy(s->ev); delete s; return tw_set_error(ctx, TW_ERR_CUDA, "tile set: out of host memory");}
	s->ctx = ctx; s->zvsize = zvsize; s->nlights = nlights;
	*out = s;
	return TW_OK;
}

void tw_tile_set_destroy(tw_tile_set *s) {
	if (!s) return;
	tw_ctx *ctx = s->ctx;
	cudaSetDevice(ctx->device);
	twi_finish_pending(ctx); // a relight may still read the slabs
	cudaEventSynchronize(s->ev); // and so may a frame's job on another context of the family
	cudaStreamSynchronize(ctx->stream);
	cudaEventDestroy(s->ev);
	cudaFree(s->d_z);
	for (tw_tile_set::slot_t &S : s->L) {cudaFree(S.d_m); cudaFree(S.d_ox); cudaFree(S.d_oy);}
	ctx->sets.erase(std::find(ctx->sets.begin(), ctx->sets.end(), s));
	delete s;
}

int tw_tile_set_put(tw_tile_set *s, const int32_t *tile_xy, uint32_t n, const float *zvals) {
	if (!s) return TW_ERR_ARG;
	tw_ctx *ctx = s->ctx;
	if (!tile_xy || !zvals || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tile set put: null or empty argument");
	std::vector<twts::key> keys;
	if (!read_keys(tile_xy, n, keys)) return tw_set_error(ctx, TW_ERR_ARG, "tile set put: tile_xy names a tile twice");
	int rc = twi_begin(ctx); if (rc) return rc;
	std::vector<uint32_t> free_left;
	std::vector<int> idx;
	uint32_t const next = twts::put_slots(s->st, keys, free_left, idx);
	rc = grow(s, next, ctx); if (rc) return rc;
	size_t const tb = (size_t)s->zvsize*s->zvsize*sizeof(float);
	bool const dev = tw_is_device_ptr(zvals);
	char *p = nullptr; int *d_idx;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {if (!dev) {p = c.take<char>(n*tb);} d_idx = c.take<int>(n);}); if (rc) return rc;
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(p, zvals, n*tb, cudaMemcpyHostToDevice, ctx->stream));}
	TW_CUDA(ctx, cudaMemcpyAsync(d_idx, idx.data(), n*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
	TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, s->ev, 0)); // a frame's job on another context may still read these slots
	rc = copy_tiles(ctx, s->d_z, d_idx, dev ? (const void *)zvals : (const void *)p, nullptr, tb, n); if (rc) return rc;
	TW_CUDA(ctx, cudaEventRecord(s->ev, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // zvals (and idx) have been read
	twts::put_tiles(s->st, keys, idx, free_left, next, slot_signs(s));
	return TW_OK;
}

int tw_tile_set_remove(tw_tile_set *s, const int32_t *tile_xy, uint32_t n) {
	if (!s) return TW_ERR_ARG;
	tw_ctx *ctx = s->ctx;
	if (!tile_xy || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: null or empty argument");
	std::vector<twts::key> keys;
	if (!read_keys(tile_xy, n, keys)) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: tile_xy names a tile twice");
	for (twts::key const &k : keys) {if (!s->st.where.count(k)) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: tile (%d, %d) is not resident", k.first, k.second);}
	int rc = twi_begin(ctx); if (rc) return rc;
	// host state only: the next writer of a freed slot waits on the set's event
	twts::remove_tiles(s->st, keys, slot_signs(s));
	return TW_OK;
}

int tw_tile_set_stale(tw_tile_set *s, const tw_shadow_params *sps, uint32_t nlights, int32_t *tile_xy_out, uint32_t capacity, uint32_t *nstale) {
	if (!s) return TW_ERR_ARG;
	if (!sps || !nstale || nlights == 0 || nlights > s->nlights || (capacity && !tile_xy_out))
		return tw_set_error(s->ctx, TW_ERR_ARG, "tile set stale: needs sps, nstale, 1 .. %u lights and tile_xy_out when capacity > 0", s->nlights);
	std::vector<twts::key> const stale = twts::stale_tiles(s->st, slot_resets(s, sps, nlights));
	for (size_t i = 0; i < stale.size() && i < capacity; ++i) {tile_xy_out[2*i] = stale[i].first; tile_xy_out[2*i+1] = stale[i].second;}
	*nstale = (uint32_t)stale.size();
	return TW_OK;
}

int tw_tile_set_stale_after(tw_tile_set *s, const tw_shadow_params *sps, uint32_t nlights, const int32_t *remove_xy, uint32_t nremove, const int32_t *put_xy,
                            uint32_t nput, int32_t *tile_xy_out, uint32_t capacity, uint32_t *nstale) {
	if (!s) return TW_ERR_ARG;
	if (!sps || !nstale || nlights == 0 || nlights > s->nlights || (capacity && !tile_xy_out))
		return tw_set_error(s->ctx, TW_ERR_ARG, "tile set stale_after: needs sps, nstale, 1 .. %u lights and tile_xy_out when capacity > 0", s->nlights);
	std::vector<twts::key> rk, pk;
	int const rc = frame_keys(s->ctx, s, remove_xy, nremove, put_xy, nput, rk, pk); if (rc) return rc;
	std::vector<twts::key> const stale = twts::stale_after(s->st, rk, pk, slot_signs(s), slot_resets(s, sps, nlights));
	for (size_t i = 0; i < stale.size() && i < capacity; ++i) {tile_xy_out[2*i] = stale[i].first; tile_xy_out[2*i+1] = stale[i].second;}
	*nstale = (uint32_t)stale.size();
	return TW_OK;
}

int tw_tile_set_shadows_launch(tw_tile_set *s, const tw_tile_set_request *req) {
	if (!s) return TW_ERR_ARG;
	tw_ctx *ctx = s->ctx;
	TW_CUDA(ctx, cudaSetDevice(ctx->device));
	relight_t R;
	int rc = relight_plan(ctx, s, s->st, req, R); if (rc) return rc;
	rc = twi_finish_pending(ctx); if (rc) return rc;
	// everything is reserved before anything is enqueued (tw_reserve synchronises the stream and may re-allocate)
	rc = tw_reserve(ctx, 0, R.dev_bytes()); if (rc) return rc;
	rc = tw_reserve_pinned(ctx, R.ints_bytes); if (rc) return rc;
	twi_job pending;
	pending.complete = [](tw_ctx *) {return TW_OK;}; // a relight stages nothing for the poll
	rc = twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, s->ev, 0)); // a frame's job on another context may still use the slabs
		return relight_enqueue(ctx, s, R, (char *)ctx->d_scratch[0], (char *)ctx->h_pinned);
	});
	if (rc) {invalidate_all(s); return rc;} // what the slots hold is unknown now, so they are recomputed next time
	relight_commit(s, R, req->recomputed);
	return TW_OK;
}

int tw_tile_set_create_tiles_launch(tw_ctx *ctx, tw_tile_set *s, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                    const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval, float wpz_max, uint32_t size,
                                    const tw_tile_outputs *out, const tw_tile_shading *shading, const tw_tile_set_frame *frame) {
	if (!ctx || !s) return TW_ERR_ARG;
	tw_ctx const *root = ctx->parent ? ctx->parent : ctx, *set_root = s->ctx->parent ? s->ctx->parent : s->ctx;
	if (root != set_root || ctx->device != s->ctx->device) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: ctx is neither the set's context, its parent nor a shared context of that parent");
	if (!frame || !frame->tile_xy) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: needs frame and frame->tile_xy");
	if (frame->hs && shading && shading->ao) return tw_set_error(ctx, TW_ERR_ARG, "tile set frame: the AO map is not available for heightmap tiles");
	frame_tail T;
	T.s = s;
	std::vector<twts::key> rk, pk;
	int rc = frame_keys(ctx, s, frame->remove_xy, frame->nremove, frame->tile_xy, ntiles, rk, pk); if (rc) return rc;
	// the state the sequential calls would leave: remove, then put (the job's zvals), then the relight planned against that
	std::vector<twts::signs> const sg = slot_signs(s);
	T.post = s->st;
	if (!rk.empty()) twts::remove_tiles(T.post, rk, sg);
	if (!pk.empty()) {
		std::vector<uint32_t> free_left;
		uint32_t const used = twts::put_slots(T.post, pk, free_left, T.idx);
		twts::put_tiles(T.post, pk, T.idx, free_left, used, sg);
	}
	if (frame->relight) {rc = relight_plan(ctx, s, T.post, frame->relight, T.R); if (rc) return rc; T.relight = true;}
	T.ntiles = ntiles;
	{twi_carve dc, hc; int *d_idx, *h_idx; char *d_rl, *h_rl; T.layout(dc, hc, d_idx, h_idx, d_rl, h_rl); T.dev_bytes = dc.bytes; T.pin_bytes = hc.bytes;}
	tw_tile_outputs const none = {nullptr, nullptr, nullptr, nullptr, nullptr};
	rc = twi_create_tiles_launch(ctx, frame->hs, origins_xy, ntiles, mesh_x_size, mesh_y_size, dx, dy, s->zvsize, p, erosion_iters, ep, min_zval, wpz_max, size,
	                             out ? out : &none, shading, &T);
	if (rc) {
		if (rc == TW_ERR_CUDA) { // what reached the slabs is unknown: the removes have happened, no put tile is resident, every slot is invalid
			if (!rk.empty()) twts::remove_tiles(s->st, rk, sg);
			std::vector<twts::key> dropped;
			for (twts::key const &k : pk) {if (s->st.where.count(k)) dropped.push_back(k);}
			if (!dropped.empty()) twts::remove_tiles(s->st, dropped, sg);
			invalidate_all(s);
		}
		return rc;
	}
	// commit at launch: later launches plan against this state, and the set's event orders their device work after this job's
	s->st = std::move(T.post);
	for (uint32_t l = 0; l < s->nlights; ++l) {if (s->st.valid[l].size() < s->capacity) s->st.valid[l].resize(s->capacity, 0);}
	if (T.relight) relight_commit(s, T.R, frame->relight->recomputed);
	return TW_OK;
}

} // extern "C"
