// Drives tw3d::hmap_tile_ao_async: a heightmap tile frame goes into a tile set on a tile_job_pool slot with no CPU copy of the zvals, and the tiles' AO maps
// are launched at once on another slot (tile_set::hmap_ao_async), with no wait in between. Compares them with the blocking tw3d::hmap_tile_ao on the zvals of
// the synchronous chain (create_zvals_from_heightmap, apply_erosion per tile) and with tile_job_pool::hmap_tile_ao_async on the same zvals, and prints
// "identical" when every byte agrees.
// usage: test_hmap_ao
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main() {
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = 1; g.MESH_X_SIZE = g.MESH_Y_SIZE = 64;
		g.mesh_file_scale = 25.0f; g.mesh_file_tz = -2.5f;
		g.zmin = -2.3f; g.zmax = 2.3f; g.water_plane_z = -0.5f; g.clip_hd1 = 0.5f;
		g.X_SCENE_SIZE = g.Y_SCENE_SIZE = 2.0f;
		tw3d::set_globals(g);
		int const W = 700, H = 500;
		std::vector<uint8_t> img((size_t)2*W*H);
		for (int y = 0; y < H; ++y) {
			for (int x = 0; x < W; ++x) { // hills and valleys steep enough to shade each other: value = hi + lo/256
				float const v = 128.0f + 100.0f*sinf(0.05f*(float)x)*cosf(0.04f*(float)y);
				img[2*((size_t)y*W + x)] = (uint8_t)(256.0f*(v - floorf(v))); img[2*((size_t)y*W + x) + 1] = (uint8_t)v;
			}
		}
		unsigned const size = 64, zvsize = size + 2, stride = zvsize - 1, nt = 12, iters = 300;
		float const DX = 0.0625f, DY = 0.0625f;
		std::vector<int32_t> origins, tile_xy;
		for (unsigned t = 0; t < nt; ++t) { // the block overhangs the image's left edge (mirrored)
			origins.push_back((int32_t)(t % 4)*(int32_t)size - 400); origins.push_back((int32_t)(t/4)*(int32_t)size - 100);
			tile_xy.push_back((int32_t)(t % 4)); tile_xy.push_back((int32_t)(t/4));
		}
		size_t const cells = (size_t)nt*zvsize*zvsize, texels = (size_t)nt*stride*stride;
		tw3d::set_heightmap(img.data(), W, H);
		std::vector<unsigned char> ao(texels), ao_pool(texels), ao_ref(texels);
		tw_hmap_sampler const hs = tw3d::hmap_sampler(W, H, TW_HMAP_EDGE_MIRROR);
		int frames = 0;
		{
			tw3d::tile_job_pool pool(2);
			tw3d::tile_set set(zvsize, 1);
			tw_tile_outputs const out = {nullptr, nullptr, nullptr, nullptr, nullptr};
			tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
			tw_tile_set_frame const frame = {nullptr, 0, tile_xy.data(), &hs, nullptr};
			tw3d::tiles_job fj = set.create_tiles_async(origins.data(), nt, DX, DY, iters, g.water_plane_z, size, out, none, frame, &pool);
			tw3d::tiles_job aj = set.hmap_ao_async(tile_xy.data(), origins.data(), nt, zvsize, ao.data(), &pool);
			while (!aj.ready()) {++frames;}
			fj.wait();
		}
		printf("AO ready after %d frame(s)\n", frames);
		std::vector<float> ez(cells);
		tw3d::create_zvals_from_heightmap(img.data(), W, H, origins.data(), nt, zvsize, ez.data());
		for (unsigned t = 0; t < nt; ++t) {tw3d::apply_erosion(ez.data() + (size_t)t*zvsize*zvsize, zvsize, zvsize, g.zmin, iters);} // tile_t::create_zvals
		tw3d::hmap_tile_ao(origins.data(), nt, zvsize, ez.data(), ao_ref.data());
		{
			tw3d::tile_job_pool pool(2);
			pool.hmap_tile_ao_async(origins.data(), nt, zvsize, ez.data(), ao_pool.data()).wait();
		}
		size_t shaded = 0;
		for (size_t i = 0; i < texels; ++i) {shaded += (ao_ref[i] != 255);}
		tw_hmap_rect const brush = {10, 10, 20, 20};
		std::vector<uint8_t> touched(nt);
		tw3d::hmap_ao_tiles_touched(origins.data(), nt, zvsize, &brush, 1, touched.data());
		unsigned nt_touched = 0;
		for (unsigned t = 0; t < nt; ++t) {nt_touched += touched[t];}
		printf("%zu occluded texels, %u of %u tiles re-shaded by the brush\n", shaded, nt_touched, nt);
		bool const same = ao == ao_ref && ao_pool == ao_ref && shaded > 0;
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
