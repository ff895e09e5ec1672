// Drives tiles_job::cancel() the way an engine drops work it no longer wants: a pool slot whose tiles went out of range, an erosion of a map that is being
// replaced. Checks that
//   - a cancelled long tile job on a tile_job_pool slot is ready soon, reports cancelled(), and the slot then runs a new job whose outputs equal
//     tw3d::create_zvals_batch byte for byte;
//   - a cancelled pool job that the pool's next launch completes still reports cancelled();
//   - a tiles_job destroyed right after cancel() waits only briefly;
//   - cancel() on a job that is already complete changes nothing (not cancelled, outputs exact).
// Prints "identical" when every check holds. usage: test_cancel <long droplets per tile>
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cuda_runtime_api.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>

namespace {
double seconds_since(std::chrono::steady_clock::time_point t0) {return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();}
}

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_cancel <long droplets per tile>\n"); return 1;}
	unsigned const long_iters = (unsigned)atoi(argv[1]);
	try {
		tw3d::scene_globals g;
		g.mesh_seed = 1; g.mesh_gen_mode = TW_MGEN_DWARP_GPU; g.zmin = -2.0f; g.zmax = 2.0f; g.water_plane_z = -0.5f;
		tw3d::set_globals(g);
		float const dx = 1.0f/g.DX_VAL_INV, dy = 1.0f/g.DY_VAL_INV;
		unsigned const S = 32, zv = S + 1, nt = 16, iters = 200;
		std::vector<int32_t> origins;
		for (unsigned t = 0; t < nt; ++t) {origins.push_back((int32_t)(t % 4)*(int32_t)S*8 - 400); origins.push_back((int32_t)(t / 4)*(int32_t)S*8 + 300);}
		size_t const cells = (size_t)nt*zv*zv;
		std::vector<float> ref(cells), z(cells);
		float *zl = nullptr; // the long jobs' output: pinned, so that their launches do not wait for the job (a pageable copy would)
		if (cudaMallocHost((void **)&zl, cells*sizeof(float)) != cudaSuccess) {fprintf(stderr, "cudaMallocHost failed\n"); return 3;}
		tw3d::create_zvals_batch(origins.data(), nt, zv, dx, dy, iters, ref.data(), nullptr);
		tw_tile_outputs o;
		bool ok = true;
		tw3d::tile_job_pool pool(1);
		// a long job on the pool's one slot, cancelled at once
		memset(&o, 0, sizeof(o)); o.zvals = zl;
		auto t0 = std::chrono::steady_clock::now();
		{
			tw3d::tiles_job job = pool.create_tiles_async(origins.data(), nt, zv, dx, dy, long_iters, 0.0f, S, o);
			job.cancel();
			job.wait();
			double const dt = seconds_since(t0);
			printf("cancelled pool job ready after %.3f s, cancelled() = %d\n", dt, (int)job.cancelled());
			if (!job.cancelled() || dt > 2.0) {fprintf(stderr, "the cancelled job was not cut short\n"); ok = false;}
		}
		// the same, but the pool's next launch completes the cancelled job (its slot scan, then the relaunch): the old handle still reports cancelled()
		memset(&o, 0, sizeof(o)); o.zvals = zl;
		{
			tw3d::tiles_job old_job = pool.create_tiles_async(origins.data(), nt, zv, dx, dy, long_iters, 0.0f, S, o);
			old_job.cancel();
			std::vector<float> z2(cells);
			tw_tile_outputs o2;
			memset(&o2, 0, sizeof(o2)); o2.zvals = z2.data();
			tw3d::tiles_job job = pool.create_tiles_async(origins.data(), nt, zv, dx, dy, iters, 0.0f, S, o2);
			job.wait();
			if (!old_job.ready() || !old_job.cancelled()) {fprintf(stderr, "a cancelled job completed by the pool's next launch is not reported cancelled\n"); ok = false;}
			if (job.cancelled() || memcmp(z2.data(), ref.data(), cells*sizeof(float))) {fprintf(stderr, "the pool's job after a cancelled one differs\n"); ok = false;}
		}
		// the slot is free again: the next job on it is exact
		memset(&o, 0, sizeof(o)); o.zvals = z.data();
		{
			tw3d::tiles_job job = pool.create_tiles_async(origins.data(), nt, zv, dx, dy, iters, 0.0f, S, o);
			job.wait();
			job.cancel(); // complete: changes nothing
			if (job.cancelled() || memcmp(z.data(), ref.data(), cells*sizeof(float))) {fprintf(stderr, "the job after the cancelled one differs\n"); ok = false;}
		}
		// a cancelled job's handle destroyed at once: its destructor's wait is short
		memset(&o, 0, sizeof(o)); o.zvals = zl;
		t0 = std::chrono::steady_clock::now();
		{
			tw3d::tiles_job job = tw3d::create_tiles_async(origins.data(), nt, zv, dx, dy, long_iters, 0.0f, S, o);
			job.cancel();
		}
		double const dd = seconds_since(t0);
		printf("destructor after cancel returned after %.3f s\n", dd);
		if (dd > 2.0) {fprintf(stderr, "the destructor waited too long\n"); ok = false;}
		memset(&o, 0, sizeof(o)); o.zvals = z.data();
		std::fill(z.begin(), z.end(), 0.0f);
		tw3d::create_tiles_async(origins.data(), nt, zv, dx, dy, iters, 0.0f, S, o).wait();
		if (memcmp(z.data(), ref.data(), cells*sizeof(float))) {fprintf(stderr, "the context's next job differs\n"); ok = false;}
		cudaFreeHost(zl);
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
