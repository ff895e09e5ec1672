// Drives the shading overload of tw3d::create_tiles_async: one launch for a frame's new tiles with heights, erosion, the AO map and the terrain
// weights texture, polled with ready() as tile_draw_t::update would. Compares them with the adapter's synchronous calls on the same tiles
// (create_zvals_batch - in the GPU gen modes tw_heightgen_tiles of the AO contexts cut to their interior and tw_erode_tiles -, tile_ao_lighting,
// create_texture_weights)
// and prints "identical" when every byte agrees.
// usage: test_tiles_shading <mode>        (mode = mesh_gen_mode 0..4)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_tiles_shading <mode>\n"); return 1;}
	int const mode = atoi(argv[1]);
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = mode; g.mesh_seed = 1; g.start_eval_sin = tw_compute_scale(1.0f, 1); g.zmax_est = 2.3f;
		g.hmap_params.sine_mag = 5.0f; g.hmap_params.sine_freq = 0.001f; g.hmap_params.sine_bias = -4.0f;
		g.MESH_X_SIZE = g.MESH_Y_SIZE = 64;
		g.zmin = -2.3f; g.zmax = 2.3f; g.water_plane_z = -0.5f; g.clip_hd1 = 0.5f;
		std::vector<float> sinTable(450);
		tw_rng rng = {1, 1};
		tw_gen_sine_params(&rng, g.MESH_HEIGHT*g.mesh_height_scale, 128, 128, 4.0f, 4.0f, g.mesh_seed, g.mesh_rgen_index, mode, 0.02f, 240.0f, 2.0f, 0.5f, sinTable.data());
		tw3d::set_globals(g, nullptr, sinTable.data());
		unsigned const size = 64, zvsize = size + 2, nt = 12, stride = zvsize - 1;
		float const DX = 0.0625f, DY = 0.0625f;
		std::vector<int32_t> origins;
		for (unsigned t = 0; t < nt; ++t) {origins.push_back((int32_t)(t % 4)*(int32_t)size*7 - 900); origins.push_back((int32_t)(t/4)*(int32_t)size*5 + 300);}
		tw3d::weight_tables wt = {{-0.5f, -0.2f, 0.3f, 0.7f, 1.0f}, {TW_TEX_SAND, TW_TEX_DIRT, TW_TEX_GROUND, TW_TEX_ROCK, TW_TEX_SNOW}, {{0.6f, 0.8f}, {0.4f, 0.6f}}, -0.5f, 1.0f, false, 0, 1.0f};
		tw_weight_params const W = tw3d::weight_params(wt, zvsize, DX, DY);
		std::vector<float> tile_params((size_t)nt*8);
		for (size_t i = 0; i < tile_params.size(); ++i) {tile_params[i] = 0.125f*(float)(i % 9);}
		std::vector<float> zvals((size_t)nt*zvsize*zvsize);
		std::vector<unsigned char> ao((size_t)nt*stride*stride), weights((size_t)nt*stride*stride*4), grass(nt);
		tw_tile_outputs out = {zvals.data(), nullptr, nullptr, nullptr, nullptr};
		tw_tile_shading sh = {g.HALF_DXY, &W, tile_params.data(), ao.data(), weights.data(), grass.data()};
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, 0.0f, size, out, sh);
			while (!job.ready()) {++frames;}
		}
		printf("tiles ready after %d frame(s)\n", frames);
		std::vector<float> ezvals(zvals.size());
		std::vector<unsigned char> eao(ao.size()), eweights(weights.size()), egrass(nt);
		if (mode >= TW_MGEN_SIMPLEX_GPU) { // the context grids (origin x1 - 36, y1 - 36) cut to their interior, then eroded: what the job does, by separate calls
			unsigned const csz = stride + 72;
			std::vector<int32_t> corg(origins);
			for (int32_t &v : corg) {v -= 36;}
			std::vector<float> cz((size_t)nt*csz*csz);
			tw_height_params const p = tw3d::height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
			tw_erosion_params const e = tw3d::erosion_params_from_globals();
			if (tw_heightgen_tiles(tw3d::ctx(), corg.data(), nt, g.MESH_X_SIZE, g.MESH_Y_SIZE, DX, DY, csz, &p, cz.data(), nullptr) != TW_OK) {fprintf(stderr, "heightgen_tiles\n"); return 2;}
			for (unsigned t = 0; t < nt; ++t) {
				for (unsigned y = 0; y < zvsize; ++y) {memcpy(&ezvals[((size_t)t*zvsize + y)*zvsize], &cz[((size_t)t*csz + y + 36)*csz + 36], zvsize*sizeof(float));}
			}
			if (tw_erode_tiles(tw3d::ctx(), ezvals.data(), nt, (int)zvsize, (int)zvsize, nullptr, g.zmin, 300, &e) != TW_OK) {fprintf(stderr, "erode_tiles\n"); return 2;}
		}
		else {tw3d::create_zvals_batch(origins.data(), nt, zvsize, DX, DY, 300, ezvals.data());}
		tw3d::tile_ao_lighting(ezvals.data(), origins.data(), nt, zvsize, DX, DY, eao.data());
		tw3d::create_texture_weights(ezvals.data(), origins.data(), nt, zvsize, DX, DY, wt, tile_params.data(), eweights.data(), egrass.data());
		bool const same = !memcmp(zvals.data(), ezvals.data(), zvals.size()*sizeof(float)) && ao == eao && weights == eweights && grass == egrass;
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
