// Drives tw3d::proc_gen_heightmap_async the way an engine would build its heightmap without stalling its frames: launch it, keep drawing while ready() says
// no, then use the image, the heights and the info. Compares them with the synchronous tw3d::proc_gen_heightmap on the same grid and prints "identical" when
// every byte agrees; a second job with set_image and no data16 must give heightmap tiles (create_tiles_async_from_heightmap) equal to the set_heightmap route.
// usage: test_heightmap_job <gen_mode> <size> <erosion droplets>
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main(int argc, char **argv) {
	if (argc < 4) {fprintf(stderr, "usage: test_heightmap_job <gen_mode> <size> <erosion droplets>\n"); return 1;}
	int const mode = atoi(argv[1]);
	unsigned const n = (unsigned)atoi(argv[2]), iters = (unsigned)atoi(argv[3]);
	try {
		tw3d::scene_globals g;
		g.mesh_seed = 1; g.mesh_gen_mode = mode; g.zmin = -2.0f; g.zmax = 2.0f; g.water_plane_z = -0.5f;
		tw3d::set_globals(g);
		float const dx = 1.0f/g.DX_VAL_INV, dy = 1.0f/g.DY_VAL_INV;
		size_t const cells = (size_t)n*n;
		std::vector<uint8_t> img_sync(2*cells), img_async(2*cells, 0xEE);
		std::vector<float> vals_sync(cells), vals_async(cells);
		tw_heightmap_info info_sync, info_async;
		memset(&info_async, 0, sizeof(info_async));
		tw3d::proc_gen_heightmap(n, n, dx, dy, iters, img_sync.data(), vals_sync.data(), &info_sync);
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::proc_gen_heightmap_async(n, n, dx, dy, iters, img_async.data(), vals_async.data(), &info_async);
			while (!job.ready()) {++frames;}
		}
		printf("heightmap ready after %d frame(s), %llu droplet moves\n", frames, (unsigned long long)info_async.erosion_moves);
		bool const same = !memcmp(img_async.data(), img_sync.data(), 2*cells) && !memcmp(vals_async.data(), vals_sync.data(), cells*sizeof(float)) &&
		                  !memcmp(&info_async, &info_sync, sizeof(info_sync));
		// the image for heightmap tiles: set_heightmap(data16) against set_image
		tw3d::scene_globals g2 = g;
		g2.mesh_file_scale = info_sync.mesh_file_scale; g2.mesh_file_tz = info_sync.mesh_file_tz;
		tw3d::set_globals(g2);
		unsigned const S = 64, zv = S + 1, nt = 4;
		int32_t const origins[2*nt] = {-100, -100, 0, 0, 64, -64, 30, 90};
		std::vector<float> z_ref((size_t)nt*zv*zv), z_img((size_t)nt*zv*zv);
		tw_tile_outputs o;
		memset(&o, 0, sizeof(o));
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		tw_tile_shadows const no_lights = {nullptr, 0, nullptr};
		tw3d::set_heightmap(img_sync.data(), (int)n, (int)n);
		o.zvals = z_ref.data();
		tw3d::create_tiles_async_from_heightmap(origins, nt, zv, dx, dy, 0, 0.0f, 0, o, none, no_lights).wait();
		tw_heightmap_info info_img;
		tw3d::tiles_job job = tw3d::proc_gen_heightmap_async(n, n, dx, dy, iters, nullptr, nullptr, &info_img, true);
		o.zvals = z_img.data();
		tw3d::create_tiles_async_from_heightmap(origins, nt, zv, dx, dy, 0, 0.0f, 0, o, none, no_lights).wait(); // completes the heightmap job first
		bool const tiles = !memcmp(z_img.data(), z_ref.data(), z_ref.size()*sizeof(float)) && !memcmp(&info_img, &info_sync, sizeof(info_sync));
		if (!tiles) {fprintf(stderr, "heightmap tiles from set_image differ\n");}
		printf(same && tiles ? "identical\n" : "DIFFERENT\n");
		return (same && tiles) ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
