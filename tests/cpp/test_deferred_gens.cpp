// Drives tw3d::set_deferred_gens(8) and tw3d::tile_job_pool the way tile_draw_t::update drives the reference (src/tiled_mesh.cpp:2367-2417): eight tiles'
// mesh_xy_grid_cache_t::build_arrays(..., no_wait=1) + enable_glaciate() launched before any of them is collected, then every grid read through eval_index;
// and two frames' create_tiles_async on a tile_job_pool(2) in flight together. Compares with the blocking forms (build_arrays without no_wait, the synchronous
// create_zvals_batch + tile_bounds + tile_normals) and prints "identical" when every value agrees.
// usage: test_deferred_gens <mode>      (mode = mesh_gen_mode 3 or 4: the GPU modes whose build_arrays(no_wait) launches asynchronously)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_deferred_gens <mode>\n"); return 1;}
	int const mode = atoi(argv[1]);
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = mode; g.mesh_seed = 1; g.start_eval_sin = tw_compute_scale(1.0f, 1); g.zmax_est = 2.3f;
		g.hmap_params.sine_mag = 5.0f; g.hmap_params.sine_freq = 0.001f; g.hmap_params.sine_bias = -4.0f;
		g.MESH_X_SIZE = g.MESH_Y_SIZE = 64;
		g.zmin = -2.3f; g.zmax = 2.3f; g.water_plane_z = -0.5f; g.clip_hd1 = 0.5f;
		tw3d::set_globals(g);
		float const DX = 0.0625f, DY = 0.0625f;
		// 1. eight deferred height generations (setup_height_gen_async per tile), then the frames that collect them
		unsigned const N = 8, nx = 258, ny = 197;
		tw3d::set_deferred_gens(N);
		std::vector<tw3d::mesh_xy_grid_cache_t> gens(N), blocking(N);
		auto x0 = [&](unsigned i) {return DX*(float)((int)(i % 4)*300 - 700);};
		auto y0 = [&](unsigned i) {return DY*(float)((int)(i / 4)*260 + 150);};
		unsigned launched_zero = 0, pending_zero = 0;
		for (unsigned i = 0; i < N; ++i) {
			launched_zero += !gens[i].build_arrays(x0(i), y0(i), DX, DY, nx, ny, 0, 0, 1);
			gens[i].enable_glaciate();
		}
		for (unsigned i = 0; i < N; ++i) {pending_zero += !gens[i].build_arrays(x0(i), y0(i), DX, DY, nx, ny, 0, 0, 1);} // the next frame asks again
		printf("build_arrays(no_wait) returned 0 for %u of %u tiles at launch, %u on the next frame\n", launched_zero, N, pending_zero);
		unsigned const contexts = (unsigned)tw3d::detail::tls().gens.size();
		bool same = (launched_zero == N && contexts == N);
		for (unsigned i = 0; i < N; ++i) {
			gens[i].enable_glaciate();
			blocking[i].build_arrays(x0(i), y0(i), DX, DY, nx, ny);
			blocking[i].enable_glaciate();
			for (unsigned y = 0; y < ny; ++y) {
				for (unsigned x = 0; x < nx; ++x) {
					float const a = gens[i].eval_index(x, y), b = blocking[i].eval_index(x, y);
					if (memcmp(&a, &b, sizeof(a))) {if (same) {fprintf(stderr, "tile %u cell (%u, %u): %.9g != %.9g\n", i, x, y, a, b);} same = false;}
				}
			}
		}
		// 2. two frames' tile jobs on a pool of two shared contexts, the second launched while the first may still run
		unsigned const size = 64, zvsize = size + 2, nt = 12, stride = zvsize - 1;
		float const wpz_max = g.water_plane_z;
		std::vector<int32_t> org[2];
		for (unsigned f = 0; f < 2; ++f) {
			for (unsigned t = 0; t < nt; ++t) {org[f].push_back((int32_t)(t % 4)*(int32_t)size*7 - 900 + (int32_t)(f*size*40)); org[f].push_back((int32_t)(t/4)*(int32_t)size*5 + 300);}
		}
		std::vector<float> zv[2], mnz[2];
		std::vector<unsigned char> nrm[2];
		std::vector<tw_minmax> mm[2];
		std::vector<tw_tile_bounds> bd[2];
		{
			tw3d::tile_job_pool pool(2);
			tw3d::tiles_job jobs[2];
			for (unsigned f = 0; f < 2; ++f) {
				zv[f].resize((size_t)nt*zvsize*zvsize); mnz[f].resize(nt); nrm[f].resize((size_t)nt*stride*stride*4); mm[f].resize(nt); bd[f].resize(nt);
				tw_tile_outputs const out = {zv[f].data(), mm[f].data(), bd[f].data(), nrm[f].data(), mnz[f].data()};
				jobs[f] = pool.create_tiles_async(org[f].data(), nt, zvsize, DX, DY, 300, wpz_max, size, out);
			}
			int frames = 0;
			while (!(jobs[0].ready() & jobs[1].ready())) {++frames;}
			printf("two frames' tiles ready after %d frame(s)\n", frames);
		}
		for (unsigned f = 0; f < 2; ++f) {
			std::vector<float> ez(zv[f].size()), emnz(nt);
			std::vector<unsigned char> en(nrm[f].size());
			std::vector<tw_minmax> emm(nt);
			std::vector<tw_tile_bounds> eb(nt);
			tw3d::create_zvals_batch(org[f].data(), nt, zvsize, DX, DY, 300, ez.data(), emm.data());
			tw3d::tile_bounds(ez.data(), nt, zvsize, wpz_max, DX, DY, size, eb.data());
			tw3d::tile_normals(ez.data(), nt, zvsize, DX, DY, en.data(), emnz.data());
			bool const ok = !memcmp(zv[f].data(), ez.data(), ez.size()*sizeof(float)) && !memcmp(mm[f].data(), emm.data(), nt*sizeof(tw_minmax)) &&
			                !memcmp(bd[f].data(), eb.data(), nt*sizeof(tw_tile_bounds)) && !memcmp(nrm[f].data(), en.data(), en.size()) &&
			                !memcmp(mnz[f].data(), emnz.data(), nt*sizeof(float));
			if (!ok) {fprintf(stderr, "frame %u: pooled tile job differs from the synchronous calls\n", f);}
			same = same && ok;
		}
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
