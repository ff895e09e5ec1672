// Drives tw3d::tile_set::create_tiles_async: a camera's frames (a far row evicted, a row of new tiles on the sun's side, the stale tiles relit with the sun
// and the moon) launched in one job each - on the thread's context, then on the slots of a tw3d::tile_job_pool with several frames in flight - against the
// same frames as separate calls on a second set (create_tiles_async, put, relight_async), made after all the launches. Prints "identical" when every byte of every output agrees.
// usage: test_tile_set_frame <mode> <pool slots>        (mode = mesh_gen_mode 0..4; 0 slots = the thread's context)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cuda_runtime_api.h>
#include <cstdio>
#include <cstdlib>
#include <deque>

namespace {
unsigned const SIZE = 64, ZV = SIZE + 2, COLS = 4;
size_t const ZT = (size_t)ZV*ZV;

struct frame_out { // pinned, so that a launch never blocks
	unsigned n = 0, nr = 0;
	float *z = nullptr; unsigned char *m[2] = {nullptr, nullptr}; float *ox[2] = {nullptr, nullptr};
	std::vector<uint8_t> rec;
	void alloc(unsigned n_, unsigned nr_) {
		n = n_; nr = nr_; rec.assign(nr, 0);
		if (cudaMallocHost((void **)&z, n*ZT*sizeof(float)) != cudaSuccess) {fprintf(stderr, "cudaMallocHost failed\n"); exit(3);}
		for (int l = 0; l < 2; ++l) {
			if (cudaMallocHost((void **)&m[l], nr*ZT) != cudaSuccess || cudaMallocHost((void **)&ox[l], nr*ZV*sizeof(float)) != cudaSuccess) {fprintf(stderr, "cudaMallocHost failed\n"); exit(3);}
		}
	}
	void release() {cudaFreeHost(z); for (int l = 0; l < 2; ++l) {cudaFreeHost(m[l]); cudaFreeHost(ox[l]);}}
	bool same(frame_out const &o) const {
		bool s = n == o.n && nr == o.nr && rec == o.rec && !memcmp(z, o.z, n*ZT*sizeof(float));
		for (int l = 0; l < 2 && s; ++l) {s = !memcmp(m[l], o.m[l], nr*ZT) && !memcmp(ox[l], o.ox[l], nr*ZV*sizeof(float));}
		return s;
	}
};
}

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_tile_set_frame <mode> <pool slots>\n"); return 1;}
	int const mode = atoi(argv[1]);
	unsigned const slots = (unsigned)atoi(argv[2]);
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = mode; g.mesh_seed = 1; g.start_eval_sin = tw_compute_scale(1.0f, 1); g.zmax_est = 2.3f;
		g.hmap_params.sine_mag = 5.0f; g.hmap_params.sine_freq = 0.001f; g.hmap_params.sine_bias = -4.0f;
		g.MESH_X_SIZE = g.MESH_Y_SIZE = 64;
		g.zmin = -2.3f; g.zmax = 2.3f; g.water_plane_z = -0.5f; g.clip_hd1 = 0.5f;
		g.X_SCENE_SIZE = g.Y_SCENE_SIZE = 2.0f;
		std::vector<float> sinTable(450);
		tw_rng rng = {1, 1};
		tw_gen_sine_params(&rng, g.MESH_HEIGHT*g.mesh_height_scale, 128, 128, 4.0f, 4.0f, g.mesh_seed, g.mesh_rgen_index, mode, 0.02f, 240.0f, 2.0f, 0.5f, sinTable.data());
		tw3d::set_globals(g, nullptr, sinTable.data());
		float const DX = 0.0625f, DY = 0.0625f;
		float const sun[3] = {3.0f, 2.0f, 0.3f}, moon[3] = {-2.0f, -3.0f, 0.4f};
		tw_shadow_params const sps[2] = {tw3d::shadow_params(sun, DX, DY), tw3d::shadow_params(moon, DX, DY)};
		tw3d::tile_set set(ZV, 2), ref(ZV, 2);
		std::unique_ptr<tw3d::tile_job_pool> pool(slots ? new tw3d::tile_job_pool(slots) : nullptr);
		tw_tile_shading const no_shading = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		int const FRAMES = 6;
		std::deque<frame_out> outs, refs;
		std::vector<tw3d::tiles_job> jobs;
		bool same = true;
		size_t recomputed = 0, shadowed = 0;
		// the frame launches on set, all of them first: with a pool, no launch waits for another frame, and the frames alternate heavy and light erosion, so a
		// light frame's set tail has to wait for the heavy frame launched before it
		struct frame_rec {std::vector<int32_t> origins, txy, rem, req; unsigned iters;};
		std::vector<frame_rec> plan(FRAMES);
		for (int f = 0; f < FRAMES; ++f) {
			// frame 0: a 4x3 block; then a row of COLS tiles at y = 2 + f on the sun's side (+y), the row at y = f - 3 evicted from frame 3 on
			frame_rec &F = plan[f];
			unsigned const rows = f ? 1 : 3, nt = rows*COLS, y0 = f ? 2 + f : 0;
			F.iters = (f % 2) ? 20 : 2000;
			for (unsigned t = 0; t < nt; ++t) {
				F.origins.push_back((int32_t)(t % COLS)*(int32_t)SIZE); F.origins.push_back((int32_t)(y0 + t/COLS)*(int32_t)SIZE + 300);
				F.txy.push_back((int32_t)(t % COLS)); F.txy.push_back((int32_t)(y0 + t/COLS));
			}
			if (f >= 3) {for (unsigned x = 0; x < COLS; ++x) {F.rem.push_back((int32_t)x); F.rem.push_back(f - 3);}}
			unsigned const nrem = (unsigned)F.rem.size()/2;
			F.req = set.stale_after(sps, 2, F.rem.data(), nrem, F.txy.data(), nt); // the host state of the frames launched so far is committed
			unsigned const nr = (unsigned)F.req.size()/2;
			outs.emplace_back(); frame_out &o = outs.back(); o.alloc(nt, nr);
			tw_tile_set_light const lights[2] = {{sps[0], o.m[0], o.ox[0], nullptr}, {sps[1], o.m[1], o.ox[1], nullptr}};
			tw_tile_set_request const rq = {F.req.data(), nr, 2, lights, o.rec.data()}; // read during the launch
			tw_tile_set_frame const frame = {nrem ? F.rem.data() : nullptr, nrem, F.txy.data(), nullptr, &rq};
			tw_tile_outputs const out = {o.z, nullptr, nullptr, nullptr, nullptr};
			jobs.push_back(set.create_tiles_async(F.origins.data(), nt, DX, DY, F.iters, 0.0f, SIZE, out, no_shading, frame, pool.get()));
			if (!pool) jobs.back().wait(); // one context: a frame at a time, as the thread's other calls would complete it anyway
		}
		// then the separate calls on ref, one after the other, with the same relight requests
		for (int f = 0; f < FRAMES; ++f) {
			frame_rec const &F = plan[f];
			unsigned const nt = (unsigned)F.txy.size()/2, nrem = (unsigned)F.rem.size()/2, nr = (unsigned)F.req.size()/2;
			if (F.req != ref.stale_after(sps, 2, F.rem.data(), nrem, F.txy.data(), nt)) {printf("stale_after differs\n"); same = false;}
			refs.emplace_back(); frame_out &r = refs.back(); r.alloc(nt, nr);
			if (nrem) ref.remove(F.rem.data(), nrem);
			{
				tw_tile_outputs const out = {r.z, nullptr, nullptr, nullptr, nullptr};
				tw3d::tiles_job job = tw3d::create_tiles_async(F.origins.data(), nt, ZV, DX, DY, F.iters, 0.0f, SIZE, out);
				job.wait();
			}
			ref.put(F.txy.data(), nt, r.z);
			{
				tw_tile_set_light const lights[2] = {{sps[0], r.m[0], r.ox[0], nullptr}, {sps[1], r.m[1], r.ox[1], nullptr}};
				tw3d::tiles_job job = ref.relight_async(F.req.data(), nr, lights, 2, r.rec.data());
				job.wait();
			}
		}
		for (tw3d::tiles_job &j : jobs) {j.wait();}
		for (int f = 0; f < FRAMES; ++f) {
			if (!outs[f].same(refs[f])) {printf("frame %d differs\n", f); same = false;}
			for (uint8_t v : outs[f].rec) {recomputed += v;}
			for (size_t i = 0; i < (size_t)outs[f].nr*ZT; ++i) {shadowed += (outs[f].m[0][i] != 0) + (outs[f].m[1][i] != 0);}
		}
		// both sets agree on what a relight with the sun moved would recompute
		float const sun2[3] = {2.0f, 3.5f, 0.25f};
		tw_shadow_params const sps2[2] = {tw3d::shadow_params(sun2, DX, DY), sps[1]};
		if (set.stale(sps2, 2) != ref.stale(sps2, 2) || set.stale(sps, 2) != ref.stale(sps, 2)) {printf("stale differs\n"); same = false;}
		for (frame_out &o : outs) o.release();
		for (frame_out &o : refs) o.release();
		printf("%zu shadowed cells, %zu recomputed\n", shadowed, recomputed);
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
