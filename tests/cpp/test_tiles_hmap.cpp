// Drives tw3d::create_tiles_async_from_heightmap: the heightmap image is set once with tw3d::set_heightmap, then one launch for a frame's new tiles with
// heights from the image, erosion, the normal map and the mesh shadows of the sun, polled with ready() as tile_draw_t::update would. Compares every output
// with create_zvals_from_heightmap followed by the synchronous tail (apply_erosion per tile, tile_normals, calc_mesh_shadows) and prints "identical" when
// every byte agrees.
// usage: test_tiles_hmap
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main() {
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = 1; g.MESH_X_SIZE = g.MESH_Y_SIZE = 64;
		g.mesh_file_scale = 25.0f; g.mesh_file_tz = -2.5f; // texel value v -> (0.0008*25*v - 2.5): about -1.9 .. 2.1 over the image below
		g.zmin = -2.3f; g.zmax = 2.3f; g.water_plane_z = -0.5f; g.clip_hd1 = 0.5f;
		g.X_SCENE_SIZE = g.Y_SCENE_SIZE = 2.0f;
		tw3d::set_globals(g);
		int const W = 700, H = 500;
		std::vector<uint8_t> img((size_t)2*W*H);
		for (int y = 0; y < H; ++y) {
			for (int x = 0; x < W; ++x) { // smooth hills and valleys: value = hi + lo/256
				float const v = 128.0f + 100.0f*sinf(0.021f*(float)x)*cosf(0.017f*(float)y);
				img[2*((size_t)y*W + x)] = (uint8_t)(256.0f*(v - floorf(v))); img[2*((size_t)y*W + x) + 1] = (uint8_t)v;
			}
		}
		unsigned const size = 64, zvsize = size + 2, nt = 12, iters = 300;
		float const DX = 0.0625f, DY = 0.0625f;
		std::vector<int32_t> origins, tile_xy;
		for (unsigned t = 0; t < nt; ++t) { // the block overhangs the image's left edge (mirrored)
			origins.push_back((int32_t)(t % 4)*(int32_t)size - 400); origins.push_back((int32_t)(t/4)*(int32_t)size - 100);
			tile_xy.push_back((int32_t)(t % 4)); tile_xy.push_back((int32_t)(t/4));
		}
		size_t const cells = (size_t)nt*zvsize*zvsize, edge = (size_t)nt*zvsize, texels = (size_t)nt*(zvsize - 1)*(zvsize - 1);
		float const sun[3] = {3.0f, 2.0f, 0.3f};
		std::vector<float> zvals(cells), ox(edge), oy(edge);
		std::vector<unsigned char> nrm(texels*4), mask(cells);
		tw_tile_outputs out = {zvals.data(), nullptr, nullptr, nrm.data(), nullptr};
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		tw_tile_light const light = {tw3d::shadow_params(sun, DX, DY), nullptr, nullptr, mask.data(), ox.data(), oy.data()};
		tw_tile_shadows const shadows = {tile_xy.data(), 1, &light};
		tw3d::set_heightmap(img.data(), W, H);
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::create_tiles_async_from_heightmap(origins.data(), nt, zvsize, DX, DY, iters, g.water_plane_z, size, out, none, shadows);
			while (!job.ready()) {++frames;}
		}
		printf("tiles ready after %d frame(s)\n", frames);
		std::vector<float> ez(cells), eox(edge), eoy(edge);
		std::vector<unsigned char> en(texels*4), em(cells);
		tw3d::create_zvals_from_heightmap(img.data(), W, H, origins.data(), nt, zvsize, ez.data());
		size_t moved = 0;
		std::vector<float> raw(ez);
		for (unsigned t = 0; t < nt; ++t) {tw3d::apply_erosion(ez.data() + (size_t)t*zvsize*zvsize, zvsize, zvsize, g.zmin, iters);} // tile_t::create_zvals
		for (size_t i = 0; i < cells; ++i) {moved += (raw[i] != ez[i]);}
		tw3d::tile_normals(ez.data(), nt, zvsize, DX, DY, en.data());
		tw3d::calc_mesh_shadows(sun, ez.data(), tile_xy.data(), nt, zvsize, DX, DY, em.data(), eox.data(), eoy.data());
		size_t shadowed = 0;
		for (size_t i = 0; i < cells; ++i) {shadowed += (mask[i] != 0);}
		printf("%zu eroded cells, %zu shadowed cells\n", moved, shadowed);
		bool const same = !memcmp(zvals.data(), ez.data(), cells*sizeof(float)) && nrm == en && mask == em && !memcmp(ox.data(), eox.data(), edge*sizeof(float)) &&
		                  !memcmp(oy.data(), eoy.data(), edge*sizeof(float));
		printf(same ? "identical\n" : "DIFFERENT\n");
		return same ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
