// Drives the adapter's object placement without stalling the frame: tw3d::get_exact_zvals_async and tw3d::heightmap_heights_async, on the thread's context
// and on a tile_job_pool slot while a heightmap frame runs on another slot. Checks that
//   - get_exact_zvals_async gives get_exact_zvals' heights, byte for byte (domain-warp terrain, scrolled, with the hmap sine and glaciation);
//   - heightmap_heights_async at integer cells gives the heights create_zvals_from_heightmap gives for tiles containing them, and the pool's frame is
//     unchanged by the placement beside it;
//   - cancel() on a placement job throws tw3d::error with TW_ERR_STATE.
// Prints "identical" when every check holds.
// usage: test_points_job
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main() {
	try {
		tw3d::scene_globals g;
		g.mesh_gen_mode = TW_MGEN_DWARP_GPU; g.zmax_est = 2.3f; g.xoff2 = -37; g.yoff2 = 12;
		g.hmap_params.sine_mag = 5.0f; g.hmap_params.sine_freq = 0.001f; g.hmap_params.sine_bias = -4.0f;
		g.mesh_file_scale = 25.0f; g.mesh_file_tz = -2.5f;
		tw3d::set_globals(g);
		size_t const n = 100000;
		std::vector<float> xy(2*n);
		for (size_t i = 0; i < 2*n; ++i) {xy[i] = -3.0f + 6.0f*(float)((i*2654435761u) % 100003u)/100003.0f;}
		std::vector<float> want(n), got(n, -1.0f);
		tw3d::get_exact_zvals(xy.data(), n, want.data());
		{
			tw3d::tiles_job job = tw3d::get_exact_zvals_async(xy.data(), n, got.data());
			while (!job.ready()) {}
		}
		bool ok = (memcmp(got.data(), want.data(), n*sizeof(float)) == 0);
		if (!ok) printf("get_exact_zvals_async differs from get_exact_zvals\n");

		int const W = 301, H = 203;
		std::vector<uint8_t> img((size_t)2*W*H);
		for (size_t i = 0; i < img.size(); ++i) {img[i] = (uint8_t)((i*2654435761u) >> 13);}
		tw3d::set_heightmap(img.data(), W, H);
		unsigned const zvsize = 34, nt = 6;
		std::vector<int32_t> origins;
		for (unsigned t = 0; t < nt; ++t) {origins.push_back((int32_t)(t % 3)*150 - 260); origins.push_back((int32_t)(t/3)*120 - 150);} // across the edges
		size_t const cells = (size_t)nt*zvsize*zvsize;
		std::vector<float> tiles(cells), pts(2*cells), heights(cells, -1.0f), pool_heights(cells, -1.0f), frame(cells), frame_alone(cells);
		tw3d::create_zvals_from_heightmap(img.data(), W, H, origins.data(), nt, zvsize, tiles.data());
		for (unsigned t = 0; t < nt; ++t) {
			for (unsigned j = 0; j < zvsize; ++j) {
				for (unsigned i = 0; i < zvsize; ++i) {
					size_t const c = ((size_t)t*zvsize + j)*zvsize + i;
					pts[2*c] = (float)(origins[2*t] + (int)i); pts[2*c + 1] = (float)(origins[2*t + 1] + (int)j);
				}
			}
		}
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		tw_tile_shadows const no_shadows = {nullptr, 0, nullptr};
		{
			tw3d::tiles_job job = tw3d::heightmap_heights_async(pts.data(), cells, heights.data());
			job.wait();
			tw3d::tile_job_pool pool(2);
			tw_tile_outputs alone = {frame_alone.data(), nullptr, nullptr, nullptr, nullptr};
			pool.create_tiles_async_from_heightmap(origins.data(), nt, zvsize, 1.0f, 1.0f, 0, 0.0f, zvsize - 2, alone, none, no_shadows).wait();
			tw_tile_outputs out = {frame.data(), nullptr, nullptr, nullptr, nullptr};
			tw3d::tiles_job f = pool.create_tiles_async_from_heightmap(origins.data(), nt, zvsize, 1.0f, 1.0f, 0, 0.0f, zvsize - 2, out, none, no_shadows);
			tw3d::tiles_job p = pool.heightmap_heights_async(pts.data(), cells, pool_heights.data());
			int refused = 0;
			try {p.cancel();} catch (tw3d::error const &e) {refused = (e.status == TW_ERR_STATE);}
			if (!refused) {printf("cancel() of a placement job did not throw TW_ERR_STATE\n"); ok = false;}
			tw3d::tiles_job z = pool.get_exact_zvals_async(xy.data(), n, got.data()); // every slot busy: completes the frame's slot first
			p.wait(); f.wait(); z.wait();
			if (memcmp(got.data(), want.data(), n*sizeof(float)) != 0) {printf("the pool's get_exact_zvals_async differs\n"); ok = false;}
		}
		if (memcmp(heights.data(), tiles.data(), cells*sizeof(float)) != 0) {printf("heightmap_heights_async differs from the tiles\n"); ok = false;}
		if (memcmp(pool_heights.data(), tiles.data(), cells*sizeof(float)) != 0) {printf("the pool's heightmap_heights_async differs from the tiles\n"); ok = false;}
		if (memcmp(frame.data(), frame_alone.data(), cells*sizeof(float)) != 0 || memcmp(frame.data(), tiles.data(), cells*sizeof(float)) != 0) {
			printf("the frame beside the placement differs\n"); ok = false;
		}
		if (ok) printf("identical\n");
		return ok ? 0 : 2;
	}
	catch (std::exception const &e) {fprintf(stderr, "error: %s\n", e.what()); return 3;}
}
