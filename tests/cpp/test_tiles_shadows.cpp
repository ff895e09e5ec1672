// Drives the shadows overload of tw3d::create_tiles_async: one launch for a frame's new tiles with heights, erosion and the mesh shadows of two lights (the
// sun, and the moon with incoming heights from tiles outside the batch), polled with ready() as tile_draw_t::update would. Compares the shadows with the
// adapter's calc_mesh_shadows overloads on the job's own zvals and prints "identical" when every byte agrees.
// usage: test_tiles_shadows <mode>        (mode = mesh_gen_mode 0..4)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_tiles_shadows <mode>\n"); return 1;}
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
		unsigned const size = 64, zvsize = size + 2, nt = 12;
		float const DX = 0.0625f, DY = 0.0625f;
		std::vector<int32_t> origins, tile_xy;
		for (unsigned t = 0; t < nt; ++t) {
			origins.push_back((int32_t)(t % 4)*(int32_t)size); origins.push_back((int32_t)(t/4)*(int32_t)size + 300);
			tile_xy.push_back((int32_t)(t % 4)); tile_xy.push_back((int32_t)(t/4) + 5);
		}
		size_t const cells = (size_t)nt*zvsize*zvsize, edge = (size_t)nt*zvsize;
		float const sun[3] = {3.0f, 2.0f, 0.3f}, moon[3] = {-2.0f, -3.0f, 0.4f};
		std::vector<float> in_x(edge), in_y(edge); // the moon's incoming heights from existing tiles: a ramp, every third entry "none"
		for (size_t i = 0; i < edge; ++i) {in_x[i] = (i % 3) ? -1.5f + 0.002f*(float)(i % 997) : TW_MESH_MIN_Z; in_y[i] = (i % 3 == 1) ? TW_MESH_MIN_Z : -1.0f + 0.003f*(float)(i % 701);}
		std::vector<float> zvals(cells);
		std::vector<unsigned char> m_sun(cells), m_moon(cells);
		std::vector<float> ox_sun(edge), oy_sun(edge), ox_moon(edge), oy_moon(edge);
		tw_tile_outputs out = {zvals.data(), nullptr, nullptr, nullptr, nullptr};
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		tw_tile_light const lights[2] = {
			{tw3d::shadow_params(sun, DX, DY), nullptr, nullptr, m_sun.data(), ox_sun.data(), oy_sun.data()},
			{tw3d::shadow_params(moon, DX, DY), in_x.data(), in_y.data(), m_moon.data(), ox_moon.data(), oy_moon.data()}};
		tw_tile_shadows const shadows = {tile_xy.data(), 2, lights};
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::create_tiles_async(origins.data(), nt, zvsize, DX, DY, 300, 0.0f, size, out, none, shadows);
			while (!job.ready()) {++frames;}
		}
		printf("tiles ready after %d frame(s)\n", frames);
		std::vector<unsigned char> e_sun(cells), e_moon(cells);
		std::vector<float> ex_sun(edge), ey_sun(edge), ex_moon(edge), ey_moon(edge);
		tw3d::calc_mesh_shadows(sun, zvals.data(), tile_xy.data(), nt, zvsize, DX, DY, e_sun.data(), ex_sun.data(), ey_sun.data());
		tw3d::calc_mesh_shadows(moon, zvals.data(), tile_xy.data(), nt, zvsize, DX, DY, in_x.data(), in_y.data(), e_moon.data(), ex_moon.data(), ey_moon.data());
		size_t shadowed = 0;
		for (size_t i = 0; i < cells; ++i) {shadowed += (m_sun[i] != 0) + (m_moon[i] != 0);}
		printf("%zu shadowed cells\n", shadowed);
		bool const same = m_sun == e_sun && m_moon == e_moon && !memcmp(ox_sun.data(), ex_sun.data(), edge*sizeof(float)) && !memcmp(oy_sun.data(), ey_sun.data(), edge*sizeof(float)) &&
		                  !memcmp(ox_moon.data(), ex_moon.data(), edge*sizeof(float)) && !memcmp(oy_moon.data(), ey_moon.data(), edge*sizeof(float));
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
