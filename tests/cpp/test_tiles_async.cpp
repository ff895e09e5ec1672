// Drives tw3d::create_tiles_async the way tile_draw_t::update would (src/tiled_mesh.cpp:2367-2417): launch a frame's new tiles, keep drawing frames
// while ready() says no, then use heights, z ranges, bounds and normal maps. Compares them with the synchronous adapter calls (create_zvals_batch,
// tile_bounds, tile_normals) on the same tiles and prints "identical" when every byte agrees.
// usage: test_tiles_async <mode>        (mode = mesh_gen_mode 0..4);  "test_tiles_async probe" only checks that the library loads
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main(int argc, char **argv) {
	if (argc >= 2 && std::string(argv[1]) == "probe") {printf("abi %d\n", tw_abi_version()); return 0;}
	if (argc < 2) {fprintf(stderr, "usage: test_tiles_async <mode>\n"); return 1;}
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
		float const DX = 0.0625f, DY = 0.0625f, wpz_max = g.water_plane_z;
		std::vector<int32_t> origins;
		for (unsigned t = 0; t < nt; ++t) {origins.push_back((int32_t)(t % 4)*(int32_t)size*7 - 900); origins.push_back((int32_t)(t/4)*(int32_t)size*5 + 300);}
		std::vector<float> zvals((size_t)nt*zvsize*zvsize), min_nz(nt);
		std::vector<unsigned char> normals((size_t)nt*stride*stride*4);
		std::vector<tw_minmax> mm(nt);
		std::vector<tw_tile_bounds> bounds(nt);
		tw_tile_outputs out = {zvals.data(), mm.data(), bounds.data(), normals.data(), min_nz.data()};
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, wpz_max, size, out);
			while (!job.ready()) {++frames;} // the frames drawn while the tiles are created
		}
		printf("tiles ready after %d frame(s)\n", frames);
		// the synchronous calls on the same tiles
		std::vector<float> ezvals(zvals.size()), emin_nz(nt);
		std::vector<unsigned char> enormals(normals.size());
		std::vector<tw_minmax> emm(nt);
		std::vector<tw_tile_bounds> ebounds(nt);
		tw3d::create_zvals_batch(origins.data(), nt, zvsize, DX, DY, 300, ezvals.data(), emm.data());
		tw3d::tile_bounds(ezvals.data(), nt, zvsize, wpz_max, DX, DY, size, ebounds.data());
		tw3d::tile_normals(ezvals.data(), nt, zvsize, DX, DY, enormals.data(), emin_nz.data());
		bool const same = !memcmp(zvals.data(), ezvals.data(), zvals.size()*sizeof(float)) && !memcmp(mm.data(), emm.data(), nt*sizeof(tw_minmax)) &&
		                  !memcmp(bounds.data(), ebounds.data(), nt*sizeof(tw_tile_bounds)) && !memcmp(normals.data(), enormals.data(), normals.size()) &&
		                  !memcmp(min_nz.data(), emin_nz.data(), nt*sizeof(float));
		// a handle that is dropped while its job runs waits for it; a second launch completes the first one
		{
			std::vector<float> z2(zvals.size());
			tw_tile_outputs o2 = {z2.data(), nullptr, nullptr, nullptr, nullptr};
			tw3d::tiles_job a = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, wpz_max, size, o2);
			tw3d::tiles_job b = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, wpz_max, size, out);
			if (!a.ready()) {fprintf(stderr, "first job not complete after the second launch\n"); return 3;}
			b.wait();
			if (memcmp(z2.data(), ezvals.data(), z2.size()*sizeof(float)) || memcmp(zvals.data(), ezvals.data(), zvals.size()*sizeof(float))) {fprintf(stderr, "chained jobs differ\n"); return 3;}
		}
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
