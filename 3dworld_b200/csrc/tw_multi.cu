// tw_multi.cu - multi-GPU host layer (include/tw3d.h "Multi-GPU"): one tw_ctx per device driven by one host worker thread each, the row-band /
// tile-band partition, NUMA-local pinned host buffers, and the only collective of the path - the 2-float z-range reduction
// (get_heightmap_z_range, src/map_view.cpp:399-407) - as an ncclAllReduce over NVLink inside the library.
// NCCL is loaded at run time (dlopen "libnccl.so.2"): a process that already has one loaded (e.g. torch's bundled copy) gets the same handle,
// and the single-GPU library keeps no link-time dependency on it.
#include "tw_internal.h"
#include <nccl.h>       // types and prototypes only; every call goes through the function table below
#include <dlfcn.h>
#include <sched.h>
#include <stdarg.h>
#include <stdlib.h>
#include <ctype.h>
#include <string>
#include <thread>
#include <vector>

namespace {

struct NcclApi {
	void *lib = nullptr;
	ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*GroupStart)() = nullptr;
	ncclResult_t (*GroupEnd)() = nullptr;
	const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi *nccl_api(std::string &err) {
	static NcclApi api;
	static bool tried = false;
	if (!tried) {
		tried = true;
		const char *names[] = {getenv("TW_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
		for (const char *n : names) {if (n && (api.lib = dlopen(n, RTLD_NOW | RTLD_LOCAL))) break;}
		if (api.lib) {
#define TW_SYM(field, name) *(void **)(&api.field) = dlsym(api.lib, name)
			TW_SYM(GetUniqueId, "ncclGetUniqueId"); TW_SYM(CommInitRank, "ncclCommInitRank"); TW_SYM(CommInitAll, "ncclCommInitAll"); TW_SYM(CommDestroy, "ncclCommDestroy");
			TW_SYM(AllReduce, "ncclAllReduce"); TW_SYM(Send, "ncclSend"); TW_SYM(Recv, "ncclRecv"); TW_SYM(GroupStart, "ncclGroupStart"); TW_SYM(GroupEnd, "ncclGroupEnd");
			TW_SYM(GetErrorString, "ncclGetErrorString");
#undef TW_SYM
			if (!api.GetUniqueId || !api.CommInitRank || !api.CommInitAll || !api.CommDestroy || !api.AllReduce || !api.Send || !api.Recv || !api.GroupStart || !api.GroupEnd) {dlclose(api.lib); api.lib = nullptr;}
		}
	}
	if (!api.lib) {err = "libnccl.so.2 could not be loaded (set TW_NCCL_LIB)"; return nullptr;}
	return &api;
}

bool parse_cpulist(const char *s, cpu_set_t &set) { // "0-31,64-95"
	CPU_ZERO(&set);
	int n = 0;
	while (*s) {
		while (*s && !isdigit((unsigned char)*s)) ++s;
		if (!*s) break;
		char *e; long a = strtol(s, &e, 10), b = a;
		if (*e == '-') {b = strtol(e + 1, &e, 10);}
		for (long c = a; c <= b && c < CPU_SETSIZE; ++c) {CPU_SET((int)c, &set); ++n;}
		s = e;
	}
	return n > 0;
}

} // namespace

extern "C" int tw_bind_thread_to_device(int device) {
	char bus[32] = {0};
	if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {cudaGetLastError(); return TW_ERR_ARG;}
	for (char *c = bus; *c; ++c) {*c = (char)tolower((unsigned char)*c);}
	std::string const path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
	FILE *f = fopen(path.c_str(), "r");
	if (!f) return TW_ERR_ARG;
	char line[4096] = {0};
	bool const got = (fgets(line, sizeof(line), f) != nullptr);
	fclose(f);
	cpu_set_t want, have, both;
	if (!got || !parse_cpulist(line, want)) return TW_ERR_ARG;
	if (sched_getaffinity(0, sizeof(have), &have) != 0) return TW_ERR_ARG;
	CPU_AND(&both, &want, &have);                 // never widen beyond what the process is allowed (cgroup / taskset)
	if (CPU_COUNT(&both) == 0) return TW_ERR_ARG;
	return (sched_setaffinity(0, sizeof(both), &both) == 0) ? TW_OK : TW_ERR_ARG;
}

// ------------------------------------------------------------------------------------------------ one process per GPU
struct tw_dist_state {ncclComm_t comm = nullptr; int nranks = 0, rank = 0; float *d_buf = nullptr;};

extern "C" int tw_dist_unique_id(char id128[128]) {
	std::string err;
	NcclApi *N = nccl_api(err);
	if (!N || !id128) return TW_ERR_STATE;
	static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
	ncclUniqueId id;
	if (N->GetUniqueId(&id) != ncclSuccess) return TW_ERR_CUDA;
	memcpy(id128, &id, 128);
	return TW_OK;
}

extern "C" int tw_dist_init(tw_ctx *ctx, int nranks, int rank, const char id128[128]) {
	if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return TW_ERR_ARG;
	std::string err;
	NcclApi *N = nccl_api(err);
	if (!N) return tw_set_error(ctx, TW_ERR_STATE, "%s", err.c_str());
	if (ctx->dist) return tw_set_error(ctx, TW_ERR_STATE, "tw_dist_init: already initialised");
	TW_CUDA(ctx, cudaSetDevice(ctx->device));
	tw_dist_state *d = new tw_dist_state();
	ncclUniqueId id;
	memcpy(&id, id128, 128);
	ncclResult_t const r = N->CommInitRank(&d->comm, nranks, id, rank);
	if (r != ncclSuccess) {delete d; return tw_set_error(ctx, TW_ERR_CUDA, "ncclCommInitRank: %s", N->GetErrorString ? N->GetErrorString(r) : "error");}
	d->nranks = nranks; d->rank = rank;
	if (cudaMalloc(&d->d_buf, 2*sizeof(float)) != cudaSuccess) {N->CommDestroy(d->comm); delete d; return tw_set_error(ctx, TW_ERR_CUDA, "cudaMalloc");}
	ctx->dist = d;
	return TW_OK;
}

extern "C" int tw_dist_allreduce_minmax(tw_ctx *ctx, tw_minmax *inout) {
	if (!ctx || !inout) return TW_ERR_ARG;
	tw_dist_state *d = (tw_dist_state *)ctx->dist;
	if (!d) return tw_set_error(ctx, TW_ERR_STATE, "tw_dist_init() has not been called");
	std::string err;
	NcclApi *N = nccl_api(err);
	int const rc = twi_begin(ctx); if (rc) return rc;
	float h[2] = {-inout->zmin, inout->zmax}; // one MAX reduction gives both ends of the range
	TW_CUDA(ctx, cudaMemcpyAsync(d->d_buf, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
	ncclResult_t const r = N->AllReduce(d->d_buf, d->d_buf, 2, ncclFloat, ncclMax, d->comm, ctx->stream);
	if (r != ncclSuccess) return tw_set_error(ctx, TW_ERR_CUDA, "ncclAllReduce: %s", N->GetErrorString ? N->GetErrorString(r) : "error");
	TW_CUDA(ctx, cudaMemcpyAsync(h, d->d_buf, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	inout->zmin = -h[0]; inout->zmax = h[1];
	return TW_OK;
}

extern "C" void tw_dist_finalize(tw_ctx *ctx) {
	if (!ctx || !ctx->dist) return;
	tw_dist_state *d = (tw_dist_state *)ctx->dist;
	std::string err;
	NcclApi *N = nccl_api(err);
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	if (d->d_buf) cudaFree(d->d_buf);
	if (N && d->comm) N->CommDestroy(d->comm);
	delete d;
	ctx->dist = nullptr;
}

// ------------------------------------------------------------------------------------------------ one process, all GPUs
struct tw_multi {
	int n = 0;
	std::vector<int> dev;
	std::vector<tw_ctx *> ctx;
	std::vector<ncclComm_t> comm;
	std::vector<float *> d_range; // 2 floats per device: {-zmin, zmax}
	char err[512] = {0};
};

static int multi_error(tw_multi *m, int status, const char *fmt, ...) {
	if (m) {va_list ap; va_start(ap, fmt); vsnprintf(m->err, sizeof(m->err), fmt, ap); va_end(ap);}
	return status;
}

extern "C" void tw_multi_range(uint32_t n, int ndev, int i, uint32_t *begin, uint32_t *end) {
	if (begin) *begin = (uint32_t)((uint64_t)n*(uint64_t)i/(uint64_t)ndev);
	if (end)   *end   = (uint32_t)((uint64_t)n*(uint64_t)(i + 1)/(uint64_t)ndev);
}

extern "C" void tw_multi_destroy(tw_multi *m) {
	if (!m) return;
	std::string err;
	NcclApi *N = m->comm.empty() ? nullptr : nccl_api(err);
	for (int i = 0; i < m->n; ++i) {
		if (i < (int)m->d_range.size() && m->d_range[i]) {cudaSetDevice(m->dev[i]); cudaFree(m->d_range[i]);}
		if (N && i < (int)m->comm.size() && m->comm[i]) N->CommDestroy(m->comm[i]);
		if (i < (int)m->ctx.size() && m->ctx[i]) tw_destroy(m->ctx[i]);
	}
	delete m;
}

extern "C" int tw_multi_create(const int *devices, int ndev, tw_multi **out) {
	if (!out || ndev < 1) return TW_ERR_ARG;
	*out = nullptr;
	int have = 0;
	if (cudaGetDeviceCount(&have) != cudaSuccess || have == 0) {cudaGetLastError(); return TW_ERR_NO_DEVICE;}
	tw_multi *m = new tw_multi();
	m->n = ndev;
	m->dev.resize(ndev); m->ctx.assign(ndev, nullptr); m->d_range.assign(ndev, nullptr);
	for (int i = 0; i < ndev; ++i) {
		m->dev[i] = devices ? devices[i] : i;
		if (m->dev[i] < 0 || m->dev[i] >= have) {tw_multi_destroy(m); return TW_ERR_ARG;}
	}
	for (int i = 0; i < ndev; ++i) {
		int rc = tw_create(m->dev[i], &m->ctx[i]);
		if (rc == TW_OK) rc = tw_set_sin_table(m->ctx[i], nullptr);
		if (rc == TW_OK && cudaMalloc(&m->d_range[i], 2*sizeof(float)) != cudaSuccess) rc = TW_ERR_CUDA;
		if (rc) {tw_multi_destroy(m); return rc;}
	}
	if (ndev > 1) { // the communicator of the z-range reduction
		std::string err;
		NcclApi *N = nccl_api(err);
		if (!N) {tw_multi_destroy(m); return TW_ERR_STATE;}
		m->comm.assign(ndev, nullptr);
		if (N->CommInitAll(m->comm.data(), ndev, m->dev.data()) != ncclSuccess) {m->comm.clear(); tw_multi_destroy(m); return TW_ERR_CUDA;}
	}
	*out = m;
	return TW_OK;
}

extern "C" int tw_multi_size(const tw_multi *m) {return m ? m->n : 0;}
extern "C" tw_ctx *tw_multi_ctx(tw_multi *m, int i) {return (m && i >= 0 && i < m->n) ? m->ctx[i] : nullptr;}
extern "C" const char *tw_multi_last_error(const tw_multi *m) {return m ? m->err : "null tw_multi";}

extern "C" int tw_multi_set_sine_params(tw_multi *m, const float *sp) {
	if (!m || !sp) return TW_ERR_ARG;
	for (int i = 0; i < m->n; ++i) {int const rc = tw_set_sine_params(m->ctx[i], sp); if (rc) return multi_error(m, rc, "device %d: %s", m->dev[i], tw_last_error(m->ctx[i]));}
	return TW_OK;
}

extern "C" int tw_multi_alloc_host(tw_multi *m, int i, size_t bytes, void **ptr) {
	if (!m || !ptr || i < 0 || i >= m->n || bytes == 0) return TW_ERR_ARG;
	*ptr = nullptr;
	cudaError_t e = cudaSuccess;
	std::thread t([&] { // a short-lived thread bound to the GPU's local CPUs: the pages are first touched (and therefore placed) on that NUMA node
		tw_bind_thread_to_device(m->dev[i]);
		cudaSetDevice(m->dev[i]);
		e = cudaHostAlloc(ptr, bytes, cudaHostAllocPortable);
		if (e == cudaSuccess) {memset(*ptr, 0, bytes);}
	});
	t.join();
	if (e != cudaSuccess) {cudaGetLastError(); return multi_error(m, TW_ERR_CUDA, "cudaHostAlloc(%zu): %s", bytes, cudaGetErrorString(e));}
	return TW_OK;
}
extern "C" void tw_multi_free_host(tw_multi *, void *ptr) {if (ptr) cudaFreeHost(ptr);}

// runs fn(i) on one host thread per device (bound to the device's local CPUs), then reduces the per-device ranges with one grouped ncclAllReduce
template<typename F>
static int run_sharded(tw_multi *m, F fn, std::vector<tw_minmax> &local, tw_minmax *zrange) {
	std::vector<int> rc(m->n, TW_OK);
	std::vector<std::thread> th;
	for (int i = 0; i < m->n; ++i) {
		th.emplace_back([&, i] {
			tw_bind_thread_to_device(m->dev[i]);
			rc[i] = fn(i);
		});
	}
	for (auto &t : th) t.join();
	for (int i = 0; i < m->n; ++i) {if (rc[i]) return multi_error(m, rc[i], "device %d: %s", m->dev[i], tw_last_error(m->ctx[i]));}
	if (!zrange) return TW_OK;
	if (m->n == 1) {*zrange = local[0]; return TW_OK;}
	std::string err;
	NcclApi *N = nccl_api(err);
	if (!N) return multi_error(m, TW_ERR_STATE, "%s", err.c_str());
	for (int i = 0; i < m->n; ++i) {
		float const h[2] = {-local[i].zmin, local[i].zmax};
		if (cudaSetDevice(m->dev[i]) != cudaSuccess || cudaMemcpy(m->d_range[i], h, sizeof(h), cudaMemcpyHostToDevice) != cudaSuccess) return multi_error(m, TW_ERR_CUDA, "z-range upload");
	}
	N->GroupStart();
	for (int i = 0; i < m->n; ++i) {N->AllReduce(m->d_range[i], m->d_range[i], 2, ncclFloat, ncclMax, m->comm[i], (cudaStream_t)tw_stream(m->ctx[i]));}
	if (N->GroupEnd() != ncclSuccess) return multi_error(m, TW_ERR_CUDA, "ncclAllReduce(z range) failed");
	float h[2] = {0, 0};
	for (int i = 0; i < m->n; ++i) { // every device holds the global range; read it back from each (also the synchronisation point of its stream)
		if (cudaSetDevice(m->dev[i]) != cudaSuccess || cudaStreamSynchronize((cudaStream_t)tw_stream(m->ctx[i])) != cudaSuccess ||
		    cudaMemcpy(h, m->d_range[i], sizeof(h), cudaMemcpyDeviceToHost) != cudaSuccess) return multi_error(m, TW_ERR_CUDA, "z-range read-back");
		if (i == 0) {zrange->zmin = -h[0]; zrange->zmax = h[1];}
		else if (zrange->zmin != -h[0] || zrange->zmax != h[1]) return multi_error(m, TW_ERR_CUDA, "z range differs between devices after the all-reduce");
	}
	return TW_OK;
}

extern "C" int tw_create_zvals_sharded(tw_multi *m, const int32_t *origins_xy, uint32_t ntiles, int mesh_x_size, int mesh_y_size, float dx, float dy,
                                       uint32_t zvsize, const tw_height_params *p, uint32_t erosion_iters, const tw_erosion_params *ep, float min_zval,
                                       float *const *out_bands, tw_minmax *mm, tw_minmax *zrange)
{
	if (!m || !origins_xy || !p || !out_bands || ntiles < (uint32_t)m->n) return multi_error(m, TW_ERR_ARG, "null argument or fewer tiles than devices");
	std::vector<tw_minmax> local(m->n);
	std::vector<std::vector<tw_minmax>> band_mm(m->n);
	return run_sharded(m, [&](int i) -> int {
		uint32_t t0, t1;
		tw_multi_range(ntiles, m->n, i, &t0, &t1);
		tw_minmax *bm = mm ? mm + t0 : nullptr;
		if (!bm && zrange) {band_mm[i].resize(t1 - t0); bm = band_mm[i].data();}
		int const rc = tw_create_zvals_batch(m->ctx[i], origins_xy + 2*(size_t)t0, t1 - t0, mesh_x_size, mesh_y_size, dx, dy, zvsize, p, erosion_iters, ep, min_zval, out_bands[i], bm);
		if (rc) return rc;
		if (bm) {
			tw_minmax r = bm[0];
			for (uint32_t t = 1; t < t1 - t0; ++t) {r.zmin = (bm[t].zmin < r.zmin) ? bm[t].zmin : r.zmin; r.zmax = (r.zmax < bm[t].zmax) ? bm[t].zmax : r.zmax;}
			local[i] = r;
		}
		return TW_OK;
	}, local, zrange);
}

extern "C" int tw_heightgen_2d_sharded(tw_multi *m, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, float *const *out_bands, tw_minmax *zrange) {
	if (!m || !g || !p || !out_bands || g->ny < (uint32_t)m->n) return multi_error(m, TW_ERR_ARG, "null argument or fewer rows than devices");
	std::vector<tw_minmax> local(m->n);
	return run_sharded(m, [&](int i) -> int {
		uint32_t r0, r1;
		tw_multi_range(g->ny, m->n, i, &r0, &r1);
		tw_grid2d b = *g;
		b.y0 = g->y0 + (float)r0;   // build_arrays(x0, y0 + r0, ...): my0 = dy*(y0 + r0); exact while |y0| + ny < 2^24 (grid coordinates are integers)
		b.ny = r1 - r0;
		return tw_heightgen_2d(m->ctx[i], &b, p, enable_glaciate, 0, out_bands[i], &local[i]);
	}, local, zrange);
}

// ------------------------------------------------------------------------------------------------ coherent erosion of ONE map sharded over the devices
// tw_erode_sweeps / tw_erode_sweeps_sharded (include/tw3d.h): the batched droplet algorithm of droplet_kernel<M_FROZEN> on row bands, with ONE grouped
// NCCL exchange per sweep: after the droplets of a sweep have been walked, neighbours swap the fixed-point deltas of the 2*halo rows around their
// common border (each side's own rows next to the border + its halo copy of the other side's rows), add what they receive (integer sums: exact), and
// apply the deltas to their band +- halo - after which every device's halo is current again without a second exchange.
namespace {
struct SweepBand {
	int y0 = 0, y1 = 0;       // owned un-padded rows
	int R0 = 0, R1 = 0;       // owned padded rows
	int E0 = 0, E1 = 0;       // stored padded rows (band +- halo)
	int u0 = 0, u1 = 0;       // un-padded rows needed to build them
	float *U = nullptr, *P = nullptr;
	long long *D = nullptr, *Rlo = nullptr, *Rhi = nullptr;
	unsigned long long *d_steps = nullptr;
	float *d_out = nullptr;   // staging of the result when the caller's band is host memory
};
int clampi_h(int v, int hi) {return v < 0 ? 0 : (v > hi ? hi : v);}
}

static int erode_sweeps_core(int n, tw_ctx **ctxs, ncclComm_t *comms, float *const *bands, int xsize, int ysize, float min_zval, uint32_t num_iters,
                             const tw_erosion_params *ep, uint32_t sweep, int halo, uint64_t *moves, char *err, size_t errlen)
{
#define SW_FAIL(status, ...) do {snprintf(err, errlen, __VA_ARGS__); rc = (status); goto done;} while (0)
#define SW_CUDA(call) do {cudaError_t e_ = (call); if (e_ != cudaSuccess) SW_FAIL(TW_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_));} while (0)
	int rc = TW_OK;
	bool local = false;
	int const PADR = 4, NX = xsize + 2*PADR, NY = ysize + 2*PADR;
	std::vector<SweepBand> B(n);
	std::string nerr;
	NcclApi *N = (n > 1 && comms) ? nccl_api(nerr) : nullptr;
	if (moves) *moves = 0;
	if (num_iters == 0 || ep->erode_amount <= 0.0) return TW_OK; // src/erosion.cpp:16
	int const view = twi_sweep_view();
	if (sweep == 0 || halo < view + 12 || xsize <= 0 || ysize <= 0) {snprintf(err, errlen, "sweep must be > 0 and halo >= %d (view + 12)", view + 12); return TW_ERR_ARG;}
	if (n > 1 && comms && !N) {snprintf(err, errlen, "%s", nerr.c_str()); return TW_ERR_STATE;}
	for (int i = 0; i < n; ++i) {
		uint32_t a, b;
		tw_multi_range((uint32_t)ysize, n, i, &a, &b);
		SweepBand &s = B[i];
		s.y0 = (int)a; s.y1 = (int)b;
		if (n > 1 && s.y1 - s.y0 < 2*halo + 2*PADR) {snprintf(err, errlen, "bands of %d rows are too thin for a halo of %d rows", s.y1 - s.y0, halo); return TW_ERR_ARG;}
		s.R0 = (i == 0) ? 0 : s.y0 + PADR; s.R1 = (i == n - 1) ? NY : s.y1 + PADR;
		s.E0 = std::max(0, s.R0 - halo); s.E1 = std::min(NY, s.R1 + halo);
		s.u0 = clampi_h(s.E0 - PADR, ysize - 1); s.u1 = clampi_h(s.E1 - 1 - PADR, ysize - 1) + 1;
	}
	for (int i = 0; i < n; ++i) { // buffers + the caller's band into the un-padded staging rows
		SweepBand &s = B[i];
		size_t const band = (size_t)(s.E1 - s.E0)*NX;
		SW_CUDA(cudaSetDevice(ctxs[i]->device));
		SW_CUDA(cudaMalloc(&s.U, (size_t)(s.u1 - s.u0)*xsize*sizeof(float)));
		SW_CUDA(cudaMalloc(&s.P, band*sizeof(float)));
		SW_CUDA(cudaMalloc(&s.D, band*sizeof(long long)));
		SW_CUDA(cudaMalloc(&s.d_steps, sizeof(unsigned long long)));
		if (n > 1) {SW_CUDA(cudaMalloc(&s.Rlo, (size_t)2*halo*NX*sizeof(long long))); SW_CUDA(cudaMalloc(&s.Rhi, (size_t)2*halo*NX*sizeof(long long)));}
		SW_CUDA(cudaMemsetAsync(s.D, 0, band*sizeof(long long), ctxs[i]->stream));
		SW_CUDA(cudaMemsetAsync(s.d_steps, 0, sizeof(unsigned long long), ctxs[i]->stream));
		SW_CUDA(cudaMemcpyAsync(s.U + (size_t)(s.y0 - s.u0)*xsize, bands[i], (size_t)(s.y1 - s.y0)*xsize*sizeof(float), cudaMemcpyDefault, ctxs[i]->stream));
	}
	local = (n > 1 && comms == nullptr); // all bands on ONE device (tw_erode_sweeps_banded): neighbours exchange with device-to-device copies on the one stream
	if (local) {
		for (int i = 0; i < n; ++i) {
			SweepBand &s = B[i];
			if (i > 0)     SW_CUDA(cudaMemcpyAsync(s.U, B[i-1].U + (size_t)(s.u0 - B[i-1].u0)*xsize, (size_t)(s.y0 - s.u0)*xsize*sizeof(float), cudaMemcpyDeviceToDevice, ctxs[i]->stream));
			if (i < n - 1) SW_CUDA(cudaMemcpyAsync(s.U + (size_t)(s.y1 - s.u0)*xsize, B[i+1].U + (size_t)(s.y1 - B[i+1].u0)*xsize, (size_t)(s.u1 - s.y1)*xsize*sizeof(float), cudaMemcpyDeviceToDevice, ctxs[i]->stream));
		}
	}
	else if (n > 1) { // initial halo of HEIGHTS: rows [u0, y0) come from the lower neighbour, [y1, u1) from the upper one
		N->GroupStart();
		for (int i = 0; i < n; ++i) {
			SweepBand &s = B[i];
			cudaStream_t const st = ctxs[i]->stream;
			if (i > 0) {
				N->Send(s.U + (size_t)(s.y0 - s.u0)*xsize, (size_t)(B[i-1].u1 - s.y0)*xsize, ncclFloat, i - 1, comms[i], st);
				N->Recv(s.U, (size_t)(s.y0 - s.u0)*xsize, ncclFloat, i - 1, comms[i], st);
			}
			if (i < n - 1) {
				N->Send(s.U + (size_t)(B[i+1].u0 - s.u0)*xsize, (size_t)(s.y1 - B[i+1].u0)*xsize, ncclFloat, i + 1, comms[i], st);
				N->Recv(s.U + (size_t)(s.y1 - s.u0)*xsize, (size_t)(s.u1 - s.y1)*xsize, ncclFloat, i + 1, comms[i], st);
			}
		}
		if (N->GroupEnd() != ncclSuccess) SW_FAIL(TW_ERR_CUDA, "NCCL halo exchange (heights) failed");
	}
	for (int i = 0; i < n; ++i) {
		SW_CUDA(cudaSetDevice(ctxs[i]->device));
		rc = twi_sweep_pad(ctxs[i], B[i].U, B[i].u0, xsize, ysize, B[i].E0, B[i].E1 - B[i].E0, B[i].P);
		if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));
	}
	for (uint32_t it0 = 0; it0 < num_iters; it0 += sweep) {
		uint32_t const it1 = (num_iters - it0 < sweep) ? num_iters : it0 + sweep;
		for (int i = 0; i < n; ++i) { // every device walks the droplets of this sweep that start in its own rows, on its frozen band
			SW_CUDA(cudaSetDevice(ctxs[i]->device));
			rc = twi_sweep_walk(ctxs[i], B[i].P, B[i].D, xsize, ysize, B[i].E0, B[i].R0, B[i].R1, halo - view - PADR, it0, it1, ep, B[i].d_steps);
			if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));
		}
		if (n > 1) { // THE halo exchange of the sweep: 2*halo rows of deltas around every internal border, both directions, one NCCL group
			size_t const cnt = (size_t)2*halo*NX;
			if (local) { // every copy reads the senders' un-summed deltas: all copies are enqueued before the first add below (one stream)
				for (int i = 0; i < n; ++i) {
					SweepBand &s = B[i];
					if (i < n - 1) SW_CUDA(cudaMemcpyAsync(s.Rhi, B[i+1].D + (size_t)(B[i+1].R0 - halo - B[i+1].E0)*NX, cnt*sizeof(long long), cudaMemcpyDeviceToDevice, ctxs[i]->stream));
					if (i > 0)     SW_CUDA(cudaMemcpyAsync(s.Rlo, B[i-1].D + (size_t)(B[i-1].R1 - halo - B[i-1].E0)*NX, cnt*sizeof(long long), cudaMemcpyDeviceToDevice, ctxs[i]->stream));
				}
			}
			else {
			N->GroupStart();
			for (int i = 0; i < n; ++i) {
				SweepBand &s = B[i];
				cudaStream_t const st = ctxs[i]->stream;
				if (i < n - 1) {N->Send(s.D + (size_t)(s.R1 - halo - s.E0)*NX, cnt, ncclInt64, i + 1, comms[i], st); N->Recv(s.Rhi, cnt, ncclInt64, i + 1, comms[i], st);}
				if (i > 0)     {N->Send(s.D + (size_t)(s.R0 - halo - s.E0)*NX, cnt, ncclInt64, i - 1, comms[i], st); N->Recv(s.Rlo, cnt, ncclInt64, i - 1, comms[i], st);}
			}
			if (N->GroupEnd() != ncclSuccess) SW_FAIL(TW_ERR_CUDA, "NCCL halo exchange (deltas) failed");
			}
			for (int i = 0; i < n; ++i) {
				SweepBand &s = B[i];
				SW_CUDA(cudaSetDevice(ctxs[i]->device));
				if (i < n - 1) {rc = twi_sweep_add(ctxs[i], s.D + (size_t)(s.R1 - halo - s.E0)*NX, s.Rhi, cnt); if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));}
				if (i > 0)     {rc = twi_sweep_add(ctxs[i], s.D + (size_t)(s.R0 - halo - s.E0)*NX, s.Rlo, cnt); if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));}
			}
		}
		for (int i = 0; i < n; ++i) {
			SW_CUDA(cudaSetDevice(ctxs[i]->device));
			rc = twi_sweep_apply(ctxs[i], B[i].P, B[i].D, (size_t)(B[i].E1 - B[i].E0)*NX);
			if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));
		}
	}
	for (int i = 0; i < n; ++i) { // remove the padding, clamp, hand the band back
		SweepBand &s = B[i];
		SW_CUDA(cudaSetDevice(ctxs[i]->device));
		bool const dev = tw_is_device_ptr(bands[i]);
		float *out = bands[i];
		size_t const bytes = (size_t)(s.y1 - s.y0)*xsize*sizeof(float);
		if (!dev) {SW_CUDA(cudaMalloc(&s.d_out, bytes)); out = s.d_out;}
		rc = twi_sweep_unpad(ctxs[i], s.P, s.E0, xsize, s.y0, s.y1, min_zval, out);
		if (rc) SW_FAIL(rc, "%s", tw_last_error(ctxs[i]));
		if (!dev) {SW_CUDA(cudaMemcpyAsync(bands[i], s.d_out, bytes, cudaMemcpyDeviceToHost, ctxs[i]->stream));}
	}
	for (int i = 0; i < n; ++i) {
		unsigned long long h = 0;
		SW_CUDA(cudaSetDevice(ctxs[i]->device));
		SW_CUDA(cudaMemcpyAsync(&h, B[i].d_steps, sizeof(h), cudaMemcpyDeviceToHost, ctxs[i]->stream));
		SW_CUDA(cudaStreamSynchronize(ctxs[i]->stream));
		if (moves) *moves += h;
	}
done:
	for (int i = 0; i < n; ++i) {
		SweepBand &s = B[i];
		cudaSetDevice(ctxs[i]->device);
		cudaStreamSynchronize(ctxs[i]->stream);
		if (s.U) cudaFree(s.U); if (s.P) cudaFree(s.P); if (s.D) cudaFree(s.D); if (s.Rlo) cudaFree(s.Rlo); if (s.Rhi) cudaFree(s.Rhi);
		if (s.d_steps) cudaFree(s.d_steps); if (s.d_out) cudaFree(s.d_out);
	}
	return rc;
#undef SW_FAIL
#undef SW_CUDA
}

extern "C" int tw_erode_sweeps(tw_ctx *ctx, float *heightmap, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                               uint32_t sweep, int halo, uint64_t *moves)
{
	if (!ctx || !heightmap || !p) return TW_ERR_ARG;
	int const rc = twi_begin(ctx); if (rc) return rc;
	float *bands[1] = {heightmap};
	tw_ctx *ctxs[1] = {ctx};
	return erode_sweeps_core(1, ctxs, nullptr, bands, xsize, ysize, min_zval, num_iters, p, sweep, halo, moves, ctx->err, sizeof(ctx->err));
}

extern "C" int tw_erode_sweeps_banded(tw_ctx *ctx, float *const *bands, int nbands, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                                      uint32_t sweep, int halo, uint64_t *moves)
{
	if (!ctx || !bands || !p || nbands < 1 || nbands > 1024) return TW_ERR_ARG;
	int const rc = twi_begin(ctx); if (rc) return rc;
	std::vector<tw_ctx *> ctxs((size_t)nbands, ctx);
	return erode_sweeps_core(nbands, ctxs.data(), nullptr, bands, xsize, ysize, min_zval, num_iters, p, sweep, halo, moves, ctx->err, sizeof(ctx->err));
}

extern "C" int tw_erode_sweeps_sharded(tw_multi *m, float *const *bands, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p,
                                       uint32_t sweep, int halo, uint64_t *moves)
{
	if (!m || !bands || !p) return TW_ERR_ARG;
	return erode_sweeps_core(m->n, m->ctx.data(), m->comm.empty() ? nullptr : m->comm.data(), bands, xsize, ysize, min_zval, num_iters, p, sweep, halo, moves, m->err, sizeof(m->err));
}
