// Drives tw3d::tile_set: a frame's new tiles from create_tiles_async into device memory, put() into the set straight from there, relit with the sun and the
// moon through relight_async() (polled with ready() as tile_draw_t::update would); then a second row of tiles on the sun's side is put and only the stale
// tiles are relit. Every relight is compared with the adapter's calc_mesh_shadows over all resident tiles; prints "identical" when every byte agrees.
// usage: test_tile_set <mode>        (mode = mesh_gen_mode 0..4)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cuda_runtime_api.h>
#include <cstdio>
#include <cstdlib>

namespace {
bool same_as_full(std::vector<float> const &zvals, std::vector<int32_t> const &all_xy, std::vector<int32_t> const &req_xy, unsigned zvsize, float dx, float dy,
                  const float lpos[3], std::vector<unsigned char> const &m, std::vector<float> const &ox, std::vector<float> const &oy) {
	unsigned const nt = (unsigned)all_xy.size()/2, n = (unsigned)req_xy.size()/2;
	size_t const zt = (size_t)zvsize*zvsize;
	std::vector<unsigned char> em(nt*zt);
	std::vector<float> ex((size_t)nt*zvsize), ey((size_t)nt*zvsize);
	tw3d::calc_mesh_shadows(lpos, zvals.data(), all_xy.data(), nt, zvsize, dx, dy, nullptr, nullptr, em.data(), ex.data(), ey.data());
	for (unsigned i = 0; i < n; ++i) {
		unsigned t = 0;
		while (all_xy[2*t] != req_xy[2*i] || all_xy[2*t+1] != req_xy[2*i+1]) {++t;}
		if (memcmp(&m[i*zt], &em[t*zt], zt) || memcmp(&ox[(size_t)i*zvsize], &ex[(size_t)t*zvsize], zvsize*sizeof(float)) ||
		    memcmp(&oy[(size_t)i*zvsize], &ey[(size_t)t*zvsize], zvsize*sizeof(float))) return false;
	}
	return true;
}
}

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_tile_set <mode>\n"); return 1;}
	int const mode = atoi(argv[1]);
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
		unsigned const size = 64, zvsize = size + 2, cols = 4;
		size_t const zt = (size_t)zvsize*zvsize;
		float const DX = 0.0625f, DY = 0.0625f;
		float const sun[3] = {3.0f, 2.0f, 0.3f}, moon[3] = {-2.0f, -3.0f, 0.4f};
		tw3d::tile_set set(zvsize, 2);
		std::vector<int32_t> all_xy;
		std::vector<float> all_z;
		float *d_z = nullptr;
		if (cudaMalloc((void **)&d_z, 3*cols*zt*sizeof(float)) != cudaSuccess) {fprintf(stderr, "cudaMalloc failed\n"); return 3;}
		bool same = true;
		size_t shadowed = 0, recomputed_total = 0;
		for (int step = 0; step < 2; ++step) {
			// step 0: a 4x3 block; step 1: a row of 4 new tiles on the sun's side (+y) of it
			unsigned const rows = step ? 1 : 3, nt = rows*cols, y0 = step ? 3 : 0;
			std::vector<int32_t> origins, txy;
			for (unsigned t = 0; t < nt; ++t) {
				origins.push_back((int32_t)(t % cols)*(int32_t)size); origins.push_back((int32_t)(y0 + t/cols)*(int32_t)size + 300);
				txy.push_back((int32_t)(t % cols)); txy.push_back((int32_t)(y0 + t/cols) + 5);
			}
			tw_tile_outputs out = {d_z, nullptr, nullptr, nullptr, nullptr};
			{
				tw3d::tiles_job job = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, 0.0f, size, out);
				while (!job.ready()) {}
			}
			set.put(txy.data(), nt, d_z);
			std::vector<float> z(nt*zt);
			if (cudaMemcpy(z.data(), d_z, nt*zt*sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {fprintf(stderr, "cudaMemcpy failed\n"); return 3;}
			all_xy.insert(all_xy.end(), txy.begin(), txy.end());
			all_z.insert(all_z.end(), z.begin(), z.end());
			tw_shadow_params const sps[2] = {tw3d::shadow_params(sun, DX, DY), tw3d::shadow_params(moon, DX, DY)};
			std::vector<int32_t> req = step ? set.stale(sps, 2) : all_xy; // after the new row: only what its arrival changed
			unsigned const n = (unsigned)req.size()/2;
			std::vector<unsigned char> m_sun(n*zt), m_moon(n*zt), rec(n);
			std::vector<float> ox_sun((size_t)n*zvsize), oy_sun((size_t)n*zvsize), ox_moon((size_t)n*zvsize), oy_moon((size_t)n*zvsize);
			tw_tile_set_light const lights[2] = {{sps[0], m_sun.data(), ox_sun.data(), oy_sun.data()}, {sps[1], m_moon.data(), ox_moon.data(), oy_moon.data()}};
			{
				tw3d::tiles_job job = set.relight_async(req.data(), n, lights, 2, rec.data());
				while (!job.ready()) {}
			}
			for (unsigned i = 0; i < n; ++i) {recomputed_total += rec[i];}
			for (size_t i = 0; i < m_sun.size(); ++i) {shadowed += (m_sun[i] != 0) + (m_moon[i] != 0);}
			printf("step %d: %u tiles relit\n", step, n);
			same = same && same_as_full(all_z, all_xy, req, zvsize, DX, DY, sun, m_sun, ox_sun, oy_sun) && same_as_full(all_z, all_xy, req, zvsize, DX, DY, moon, m_moon, ox_moon, oy_moon);
		}
		cudaFree(d_z);
		printf("%zu shadowed cells, %zu recomputed\n", shadowed, recomputed_total);
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
