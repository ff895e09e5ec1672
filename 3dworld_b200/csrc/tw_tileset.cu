// tw_tileset.cu - tile sets (include/tw3d.h, tw_tile_set_*): the live tiles' zvals kept in device memory the set owns, and per light slot the mesh shadows
// each tile was last computed with. A relight is the context's asynchronous job: it recomputes only the tiles whose result can have changed (the cache rules
// are in tw_tileset_rules.h) through the unchanged mesh-shadow plan and kernels of tw_shadows.cu, with the cached sh_out rows of valid neighbours as caller
// rows, so every output equals tw_tile_shadows_batch_ex on all resident tiles. The kernels here only move tiles: gather a batch's zvals and caller rows out
// of the slabs, scatter its results back, gather the requested outputs - one launch each per light, 16-byte accesses where the sizes and pointers allow.
#include "tw_internal.h"
#include "tw_tileset_rules.h"
#include <algorithm>
#include <new>

struct tw_tile_set {
	struct slot_t {                                  // one light slot
		bool have = false;                           // sp holds the params the valid tiles were computed with
		tw_shadow_params sp;
		std::vector<uint8_t> valid;                  // per slab slot
		unsigned char *d_m = nullptr;                // capacity*zvsize^2 bytes: each tile's smask
		float *d_ox = nullptr, *d_oy = nullptr;      // capacity*zvsize floats each: each tile's sh_out_x / sh_out_y
	};
	tw_ctx *ctx = nullptr;
	uint32_t zvsize = 0, nlights = 0;
	twts::index_map where;                           // resident tile -> slab slot
	std::vector<uint32_t> free_slots;                // slots of removed tiles, reused first
	uint32_t used = 0, capacity = 0;                 // slots handed out so far, slots allocated
	float *d_z = nullptr;                            // capacity*zvsize^2 floats: the zvals slab (the set's own memory: tw_reserve may re-allocate scratch under a job)
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

size_t al(size_t b) {return (b + 255) & ~(size_t)255;}

int begin_call(tw_tile_set *s) { // the context's device, its tables, and its pending job completed
	TW_CUDA(s->ctx, cudaSetDevice(s->ctx->device));
	return twi_finish_pending(s->ctx);
}

// unique keys of n (x, y) pairs, or false when one is named twice
bool read_keys(const int32_t *tile_xy, uint32_t n, std::vector<twts::key> &keys) {
	keys.resize(n);
	for (uint32_t i = 0; i < n; ++i) {keys[i] = twts::key(tile_xy[2*i], tile_xy[2*i+1]);}
	std::vector<twts::key> sorted(keys);
	std::sort(sorted.begin(), sorted.end());
	return std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end();
}

// slabs for at least `need` tiles: geometric growth, the old contents copied over on the context's stream (nothing of the set's is in flight: put has completed
// the pending job); nothing changes when an allocation fails
int grow(tw_tile_set *s, uint32_t need) {
	if (need <= s->capacity) return TW_OK;
	tw_ctx *ctx = s->ctx;
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
		S.valid.resize(cap, 0);
	}
	s->capacity = cap;
	return TW_OK;
}

void slot_signs(tw_tile_set::slot_t const &S, int &sx, int &sy) {
	sx = S.have ? twts::light_sign(S.sp.lpos[0]) : 1; sy = S.have ? twts::light_sign(S.sp.lpos[1]) : 1;
}

} // namespace

extern "C" {

int tw_tile_set_create(tw_ctx *ctx, uint32_t zvsize, uint32_t nlights, tw_tile_set **out) {
	if (out) *out = nullptr;
	if (!ctx) return TW_ERR_ARG;
	if (!out || zvsize < 2 || nlights < 1) return tw_set_error(ctx, TW_ERR_ARG, "tile set: needs out, zvsize >= 2 and nlights >= 1 (zvsize %u, nlights %u)", zvsize, nlights);
	TW_CUDA(ctx, cudaSetDevice(ctx->device));
	tw_tile_set *s = new (std::nothrow) tw_tile_set();
	if (!s) return tw_set_error(ctx, TW_ERR_CUDA, "tile set: out of host memory");
	try {s->L.resize(nlights); ctx->sets.push_back(s);} catch (...) {delete s; return tw_set_error(ctx, TW_ERR_CUDA, "tile set: out of host memory");}
	s->ctx = ctx; s->zvsize = zvsize; s->nlights = nlights;
	*out = s;
	return TW_OK;
}

void tw_tile_set_destroy(tw_tile_set *s) {
	if (!s) return;
	tw_ctx *ctx = s->ctx;
	cudaSetDevice(ctx->device);
	twi_finish_pending(ctx); // a relight may still read the slabs
	cudaStreamSynchronize(ctx->stream);
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
	int rc = begin_call(s); if (rc) return rc;
	// slots: a resident tile keeps its own, new tiles take freed slots first, then fresh ones
	std::vector<uint32_t> free_left(s->free_slots);
	uint32_t next = s->used;
	std::vector<int> idx(n);
	for (uint32_t i = 0; i < n; ++i) {
		auto const it = s->where.find(keys[i]);
		if (it != s->where.end()) {idx[i] = (int)it->second;}
		else if (!free_left.empty()) {idx[i] = (int)free_left.back(); free_left.pop_back();}
		else {idx[i] = (int)next++;}
	}
	rc = grow(s, next); if (rc) return rc;
	size_t const tb = (size_t)s->zvsize*s->zvsize*sizeof(float);
	bool const dev = tw_is_device_ptr(zvals);
	size_t const zb = dev ? 0 : al(n*tb);
	rc = tw_reserve(ctx, 0, zb + al(n*sizeof(int))); if (rc) return rc;
	char *p = (char *)ctx->d_scratch[0];
	if (!dev) {TW_CUDA(ctx, cudaMemcpyAsync(p, zvals, n*tb, cudaMemcpyHostToDevice, ctx->stream));}
	int *d_idx = (int *)(p + zb);
	TW_CUDA(ctx, cudaMemcpyAsync(d_idx, idx.data(), n*sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
	rc = copy_tiles(ctx, s->d_z, d_idx, dev ? (const void *)zvals : (const void *)p, nullptr, tb, n); if (rc) return rc;
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // zvals (and idx) have been read
	// commit: the new tiles are resident; each put tile and its downstream closure are invalid in every slot
	for (uint32_t i = 0; i < n; ++i) {s->where.emplace(keys[i], (uint32_t)idx[i]);}
	s->free_slots.swap(free_left); s->used = next;
	for (tw_tile_set::slot_t &S : s->L) {
		int sx, sy; slot_signs(S, sx, sy);
		twts::invalidate_downstream(s->where, keys, sx, sy, S.valid);
	}
	return TW_OK;
}

int tw_tile_set_remove(tw_tile_set *s, const int32_t *tile_xy, uint32_t n) {
	if (!s) return TW_ERR_ARG;
	tw_ctx *ctx = s->ctx;
	if (!tile_xy || n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: null or empty argument");
	std::vector<twts::key> keys;
	if (!read_keys(tile_xy, n, keys)) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: tile_xy names a tile twice");
	for (twts::key const &k : keys) {if (!s->where.count(k)) return tw_set_error(ctx, TW_ERR_ARG, "tile set remove: tile (%d, %d) is not resident", k.first, k.second);}
	int rc = begin_call(s); if (rc) return rc;
	for (twts::key const &k : keys) {
		uint32_t const slot = s->where[k];
		s->where.erase(k);
		s->free_slots.push_back(slot);
		for (tw_tile_set::slot_t &S : s->L) {S.valid[slot] = 0;}
	}
	for (tw_tile_set::slot_t &S : s->L) { // the removed tiles' downstream neighbours lose an incoming row
		int sx, sy; slot_signs(S, sx, sy);
		std::vector<twts::key> seeds;
		for (twts::key const &k : keys) {seeds.push_back(twts::key(k.first - sx, k.second)); seeds.push_back(twts::key(k.first, k.second - sy));}
		twts::invalidate_downstream(s->where, seeds, sx, sy, S.valid);
	}
	return TW_OK;
}

int tw_tile_set_stale(tw_tile_set *s, const tw_shadow_params *sps, uint32_t nlights, int32_t *tile_xy_out, uint32_t capacity, uint32_t *nstale) {
	if (!s) return TW_ERR_ARG;
	if (!sps || !nstale || nlights == 0 || nlights > s->nlights || (capacity && !tile_xy_out))
		return tw_set_error(s->ctx, TW_ERR_ARG, "tile set stale: needs sps, nstale, 1 .. %u lights and tile_xy_out when capacity > 0", s->nlights);
	uint32_t count = 0;
	for (auto const &kv : s->where) { // a relight of every resident tile recomputes exactly the invalid ones (their upstream closure is invalid too)
		bool stale = false;
		for (uint32_t l = 0; l < nlights && !stale; ++l) {
			tw_tile_set::slot_t const &S = s->L[l];
			stale = !S.have || memcmp(&S.sp, &sps[l], sizeof(tw_shadow_params)) != 0 || !S.valid[kv.second];
		}
		if (!stale) continue;
		if (count < capacity) {tile_xy_out[2*count] = kv.first.first; tile_xy_out[2*count+1] = kv.first.second;}
		++count;
	}
	*nstale = count;
	return TW_OK;
}

int tw_tile_set_shadows_launch(tw_tile_set *s, const tw_tile_set_request *req) {
	if (!s) return TW_ERR_ARG;
	tw_ctx *ctx = s->ctx;
	if (!req || !req->tile_xy || req->n == 0 || !req->lights || req->nlights == 0 || req->nlights > s->nlights)
		return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: needs tile_xy, n >= 1 and 1 .. %u lights", s->nlights);
	TW_CUDA(ctx, cudaSetDevice(ctx->device));
	uint32_t const n = req->n, nl = req->nlights, zv = s->zvsize;
	size_t const zt = (size_t)zv*zv, eb = (size_t)zv*sizeof(float);
	std::vector<tw_tile_set_light> const lights(req->lights, req->lights + nl);
	std::vector<twts::key> keys;
	if (!read_keys(req->tile_xy, n, keys)) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: tile_xy names a tile twice");
	std::vector<int> req_slot(n);
	for (uint32_t i = 0; i < n; ++i) {
		auto const it = s->where.find(keys[i]);
		if (it == s->where.end()) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: tile (%d, %d) is not resident", keys[i].first, keys[i].second);
		req_slot[i] = (int)it->second;
	}
	std::vector<char> dev_m(nl), dev_x(nl), dev_y(nl);
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_set_light const &Lr = lights[l];
		if (!Lr.smask) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: light %u has no smask", l);
		dev_m[l] = tw_is_device_ptr(Lr.smask);
		if (dev_m[l] && ((size_t)Lr.smask & 3)) return tw_set_error(ctx, TW_ERR_ARG, "tile set relight: light %u: a device smask must be 4-byte aligned", l);
		dev_x[l] = Lr.sh_out_x && tw_is_device_ptr(Lr.sh_out_x); dev_y[l] = Lr.sh_out_y && tw_is_device_ptr(Lr.sh_out_y);
	}
	int rc = twi_finish_pending(ctx); if (rc) return rc;
	// per light: the batch B (invalid requested tiles + their invalid upstream closure), its plan, and the slab slots it reads and writes
	struct batch_t {
		bool reset = false;                      // the slot's params differ: every tile of it is invalid
		std::vector<twts::key> B;
		twi_shadow_plan P;
		std::vector<int> ints;                   // [plan (3*nB) | B's slots | x caller-row sources | y caller-row sources]
		size_t off_ints = 0, off_out = 0;        // byte offsets into the int region / the output staging
	};
	std::vector<batch_t> jobs(nl);
	uint32_t maxB = 0;
	size_t ints_bytes = al(n*sizeof(int)), out_bytes = 0;    // the int region starts with the requested tiles' slots
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_set::slot_t const &S = s->L[l];
		batch_t &J = jobs[l];
		tw_shadow_params const &sp = lights[l].sp;
		J.reset = !S.have || memcmp(&S.sp, &sp, sizeof(sp)) != 0;
		int const sx = twts::light_sign(sp.lpos[0]), sy = twts::light_sign(sp.lpos[1]);
		std::vector<uint8_t> const none(J.reset ? s->capacity : 0, 0);
		std::vector<uint8_t> const &valid = J.reset ? none : S.valid;
		J.B = twts::recompute_batch(s->where, valid, keys, sx, sy);
		uint32_t const nB = (uint32_t)J.B.size();
		maxB = std::max(maxB, nB);
		if (nB) {
			std::vector<int32_t> bxy(2*(size_t)nB);
			for (uint32_t t = 0; t < nB; ++t) {bxy[2*t] = J.B[t].first; bxy[2*t+1] = J.B[t].second;}
			twi_shadow_plan_make(bxy.data(), nB, &sp, true, true, &J.P);
			J.ints.resize(twi_shadow_plan_ints(nB) + 3*(size_t)nB);
			twi_shadow_plan_pack(J.P, J.ints.data());
			int *bs = J.ints.data() + twi_shadow_plan_ints(nB), *rx = bs + nB, *ry = rx + nB;
			auto cached = [&](twts::key const &k) {auto const it = s->where.find(k); return (it != s->where.end() && valid[it->second]) ? (int)it->second : -1;};
			for (uint32_t t = 0; t < nB; ++t) {
				bs[t] = (int)s->where.find(J.B[t])->second;
				rx[t] = cached(twts::key(J.B[t].first, J.B[t].second + sy)); // sh_in_x row: the sh_out_x of (tx, ty + sy); not resident -> MESH_MIN_Z
				ry[t] = cached(twts::key(J.B[t].first + sx, J.B[t].second)); // sh_in_y row: the sh_out_y of (tx + sx, ty)
			}
		}
		J.off_ints = ints_bytes; ints_bytes += al(J.ints.size()*sizeof(int));
		J.off_out = out_bytes;
		out_bytes += (dev_m[l] ? 0 : al(n*zt)) + ((lights[l].sh_out_x && !dev_x[l]) ? al(n*eb) : 0) + ((lights[l].sh_out_y && !dev_y[l]) ? al(n*eb) : 0);
	}
	// everything is reserved before anything is enqueued (tw_reserve synchronises the stream and may re-allocate): slot 0 = [B's zvals | mask | 64-bit keys |
	// x edges (outputs, then caller rows) | y edges | host-bound output staging | int region], the int region staged in pinned memory
	size_t const zb = al((size_t)maxB*zt*sizeof(float)), mb = al((size_t)maxB*zt + 4), kb = al(2*(size_t)maxB*eb*2), fb = al(2*(size_t)maxB*eb);
	size_t const off_out = zb + mb + kb + 2*fb, off_ints = off_out + out_bytes;
	rc = tw_reserve(ctx, 0, off_ints + ints_bytes); if (rc) return rc;
	rc = tw_reserve_pinned(ctx, ints_bytes); if (rc) return rc;
	char *const s0 = (char *)ctx->d_scratch[0], *const h = (char *)ctx->h_pinned;
	float *d_zB = (float *)s0;
	unsigned char *d_mB = (unsigned char *)(s0 + zb);
	unsigned long long *d_keys = (unsigned long long *)(s0 + zb + mb);
	float *d_ox = (float *)(s0 + zb + mb + kb), *d_oy = (float *)(s0 + zb + mb + kb + fb);
	char *d_ints = s0 + off_ints;
	memcpy(h, req_slot.data(), n*sizeof(int));
	for (batch_t const &J : jobs) {memcpy(h + J.off_ints, J.ints.data(), J.ints.size()*sizeof(int));}
	uint32_t minz_bits; {float const m = TW_MESH_MIN_Z; memcpy(&minz_bits, &m, 4);}
	auto enqueue = [&]() -> int {
		TW_CUDA(ctx, cudaMemcpyAsync(d_ints, h, ints_bytes, cudaMemcpyHostToDevice, ctx->stream));
		const int *d_req = (const int *)d_ints;
		for (uint32_t l = 0; l < nl; ++l) {
			tw_tile_set::slot_t &S = s->L[l];
			batch_t const &J = jobs[l];
			uint32_t const nB = (uint32_t)J.B.size();
			tw_tile_set_light const &Lr = lights[l];
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
			char *st = s0 + off_out + J.off_out; // the requested tiles' outputs, in request order
			unsigned char *om = dev_m[l] ? Lr.smask : (unsigned char *)st; st += dev_m[l] ? 0 : al(n*zt);
			float *ox = !Lr.sh_out_x ? nullptr : (dev_x[l] ? Lr.sh_out_x : (float *)st); st += (Lr.sh_out_x && !dev_x[l]) ? al(n*eb) : 0;
			float *oy = !Lr.sh_out_y ? nullptr : (dev_y[l] ? Lr.sh_out_y : (float *)st);
			int r = copy_tiles(ctx, om, nullptr, S.d_m, d_req, zt, n); if (r) return r;
			if (ox) {r = copy_tiles(ctx, ox, nullptr, S.d_ox, d_req, eb, n); if (r) return r;}
			if (oy) {r = copy_tiles(ctx, oy, nullptr, S.d_oy, d_req, eb, n); if (r) return r;}
		}
		for (uint32_t l = 0; l < nl; ++l) { // host outputs: one copy each, at the end
			tw_tile_set_light const &Lr = lights[l];
			char *st = s0 + off_out + jobs[l].off_out;
			if (!dev_m[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.smask, st, n*zt, cudaMemcpyDeviceToHost, ctx->stream)); st += al(n*zt);}
			if (Lr.sh_out_x && !dev_x[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.sh_out_x, st, n*eb, cudaMemcpyDeviceToHost, ctx->stream)); st += al(n*eb);}
			if (Lr.sh_out_y && !dev_y[l]) {TW_CUDA(ctx, cudaMemcpyAsync(Lr.sh_out_y, st, n*eb, cudaMemcpyDeviceToHost, ctx->stream));}
		}
		TW_CUDA(ctx, cudaEventRecord(ctx->async.done, ctx->stream));
		return TW_OK;
	};
	rc = enqueue();
	if (rc) { // nothing may still run on the scratch; what the slots hold is unknown now, so they are recomputed next time
		cudaStreamSynchronize(ctx->stream);
		for (tw_tile_set::slot_t &S : s->L) {S.have = false; std::fill(S.valid.begin(), S.valid.end(), 0);}
		return rc;
	}
	// commit: each slot holds this request's params, and B is valid in it
	std::vector<uint8_t> computed(s->capacity, 0);
	for (uint32_t l = 0; l < nl; ++l) {
		tw_tile_set::slot_t &S = s->L[l];
		batch_t const &J = jobs[l];
		if (J.reset) {std::fill(S.valid.begin(), S.valid.end(), 0);}
		S.have = true; S.sp = lights[l].sp;
		for (twts::key const &k : J.B) {uint32_t const slot = s->where.find(k)->second; S.valid[slot] = 1; computed[slot] = 1;}
	}
	if (req->recomputed) {for (uint32_t i = 0; i < n; ++i) {req->recomputed[i] = computed[req_slot[i]];}}
	tw_async_state &a = ctx->async;
	a.pending = true; a.tiles = true; a.steps = false; a.n_mm = 0;
	a.host_mm = nullptr; a.host_bounds = nullptr; a.host_min_nz = nullptr; a.host_flags = nullptr;
	return TW_OK;
}

} // extern "C"
