// Drives tw3d::update_heightmap and tw3d::hmap_tiles_touched the way an engine applies a brush stroke: set_heightmap once, change the CPU image inside the
// brush's rect, update_heightmap with that rect, hmap_tiles_touched over the live tiles. Checks that
//   - a frame launched after the edit (create_tiles_async_from_heightmap) gives the zvals create_zvals_from_heightmap gives on the edited image;
//   - the tiles hmap_tiles_touched leaves out have the same zvals on the old and the edited image, and it flags at least one tile;
//   - an edit of a rect outside the image, and one with an image size other than set_heightmap's, throw tw3d::error with TW_ERR_ARG.
// Prints "identical" when every check holds.
// usage: test_hmap_edit
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

int main() {
	try {
		tw3d::scene_globals g;
		g.mesh_file_scale = 25.0f; g.mesh_file_tz = -2.5f;
		tw3d::set_globals(g);
		int const W = 700, H = 500;
		std::vector<uint8_t> img((size_t)2*W*H);
		for (size_t i = 0; i < img.size(); ++i) {img[i] = (uint8_t)((i*2654435761u) >> 13);}
		std::vector<uint8_t> const old(img);
		unsigned const size = 64, zvsize = size + 2, nt = 24;
		std::vector<int32_t> origins;
		for (unsigned t = 0; t < nt; ++t) {origins.push_back((int32_t)(t % 6)*(int32_t)size - 400); origins.push_back((int32_t)(t/6)*(int32_t)size - 200);}
		size_t const cells = (size_t)nt*zvsize*zvsize;
		tw3d::set_heightmap(img.data(), W, H);
		tw_hmap_rect const brush = {100, 90, 37, 21};
		for (int y = brush.y; y < brush.y + brush.h; ++y) {
			for (int x = brush.x; x < brush.x + brush.w; ++x) {img[2*((size_t)y*W + x) + 1] ^= 0x5a;}
		}
		tw3d::update_heightmap(img.data(), W, H, &brush, 1);
		std::vector<uint8_t> touched(nt);
		tw3d::hmap_tiles_touched(origins.data(), nt, zvsize, &brush, 1, touched.data());
		std::vector<float> z(cells), want(cells), before(cells);
		tw_tile_outputs out = {z.data(), nullptr, nullptr, nullptr, nullptr};
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		tw_tile_shadows const no_shadows = {nullptr, 0, nullptr};
		{
			tw3d::tiles_job job = tw3d::create_tiles_async_from_heightmap(origins.data(), nt, zvsize, 1.0f, 1.0f, 0, 0.0f, size, out, none, no_shadows);
			job.wait();
		}
		tw3d::create_zvals_from_heightmap(img.data(), W, H, origins.data(), nt, zvsize, want.data());
		tw3d::create_zvals_from_heightmap(old.data(), W, H, origins.data(), nt, zvsize, before.data());
		bool ok = (memcmp(z.data(), want.data(), cells*sizeof(float)) == 0);
		if (!ok) printf("the frame after the edit differs from the edited image's tiles\n");
		unsigned nflag = 0;
		for (unsigned t = 0; t < nt; ++t) {
			size_t const o = (size_t)t*zvsize*zvsize;
			bool const same = (memcmp(before.data() + o, want.data() + o, zvsize*zvsize*sizeof(float)) == 0);
			nflag += touched[t];
			if (!touched[t] && !same) {printf("tile %u changed but is not flagged\n", t); ok = false;}
		}
		if (nflag == 0) {printf("no tile flagged\n"); ok = false;}
		printf("%u of %u tiles touched\n", nflag, nt);
		int refused = 0;
		tw_hmap_rect const outside = {W - 3, 0, 4, 1};
		try {tw3d::update_heightmap(img.data(), W, H, &outside, 1);} catch (tw3d::error const &e) {refused += (e.status == TW_ERR_ARG);}
		try {tw3d::update_heightmap(img.data(), W + 1, H, &brush, 1);} catch (tw3d::error const &e) {refused += (e.status == TW_ERR_ARG);}
		if (refused != 2) {printf("refusals: %d of 2\n", refused); ok = false;}
		if (ok) printf("identical\n");
		return ok ? 0 : 2;
	}
	catch (std::exception const &e) {fprintf(stderr, "error: %s\n", e.what()); return 3;}
}
