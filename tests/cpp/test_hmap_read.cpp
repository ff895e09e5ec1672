// Drives tw3d::read_heightmap / read_heightmap_async the way an engine keeps its CPU heightmap in line with the device's image. On a generated n x n map:
//   - set_heightmap, then read_heightmap of the whole image: equals the uploaded image;
//   - read_heightmap_async of three rects into device memory, and on a tile_job_pool slot into host memory: the rects' texels, the rest left alone;
//   - erode_heightmap_async, then read_heightmap_async once it is ready: equals the chain to_floats -> minmax -> apply_erosion -> from_floats;
//   - the brush workflow: a brush stroke on that CPU copy, update_heightmap with the brush's rect, read_heightmap: equals the CPU copy, which is the
//     eroded map outside the rect;
//   - a read with an image size other than set_heightmap's, and one of a rect outside the image, throw tw3d::error with TW_ERR_ARG.
// Prints "identical" when every check holds.
// usage: test_hmap_read <size> <erosion droplets>
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>

namespace {
void check(int rc, const char *what) {if (rc != TW_OK) {throw tw3d::error(rc, std::string(what) + ": " + tw_last_error(tw3d::ctx()));}}

// img's texels inside rects over a buffer of `fill` bytes
std::vector<uint8_t> rects_of(std::vector<uint8_t> const &img, int n, const tw_hmap_rect *rects, unsigned nr, uint8_t fill) {
	std::vector<uint8_t> out(img.size(), fill);
	for (unsigned r = 0; r < nr; ++r) {
		for (int y = rects[r].y; y < rects[r].y + rects[r].h; ++y) {
			size_t const o = 2*((size_t)y*n + rects[r].x);
			memcpy(&out[o], &img[o], 2*(size_t)rects[r].w);
		}
	}
	return out;
}
}

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_hmap_read <size> <erosion droplets>\n"); return 1;}
	int const n = atoi(argv[1]);
	unsigned const iters = (unsigned)atoi(argv[2]);
	try {
		tw3d::scene_globals g;
		g.mesh_seed = 1; g.mesh_gen_mode = TW_MGEN_DWARP_GPU; g.zmin = -2.0f; g.zmax = 2.0f; g.water_plane_z = -0.5f;
		tw3d::set_globals(g);
		float const dx = 1.0f/g.DX_VAL_INV, dy = 1.0f/g.DY_VAL_INV;
		size_t const cells = (size_t)n*n, bytes = 2*cells;
		std::vector<uint8_t> img(bytes);
		tw_heightmap_info info;
		tw3d::proc_gen_heightmap((unsigned)n, (unsigned)n, dx, dy, 0, img.data(), nullptr, &info);
		bool ok = true;
		// the whole image, blocking
		tw3d::set_heightmap(img.data(), n, n);
		std::vector<uint8_t> back(bytes, 0);
		tw3d::read_heightmap(back.data(), n, n);
		if (back != img) {fprintf(stderr, "read_heightmap differs from the uploaded image\n"); ok = false;}
		// rects into device memory, and on a pool slot into host memory
		tw_hmap_rect const rects[3] = {{3, 5, 17, 9}, {n - 40, n - 3, 40, 3}, {0, n/2, n, 1}};
		std::vector<uint8_t> const want = rects_of(img, n, rects, 3, 0x77);
		uint8_t *d_buf = nullptr;
		if (cudaMalloc(&d_buf, bytes) != cudaSuccess || cudaMemset(d_buf, 0x77, bytes) != cudaSuccess) {fprintf(stderr, "cudaMalloc failed\n"); return 3;}
		tw3d::read_heightmap_async(d_buf, n, n, rects, 3).wait();
		std::vector<uint8_t> got(bytes);
		if (cudaMemcpy(got.data(), d_buf, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) {fprintf(stderr, "cudaMemcpy failed\n"); return 3;}
		cudaFree(d_buf);
		if (got != want) {fprintf(stderr, "read_heightmap_async into device memory differs\n"); ok = false;}
		{
			std::vector<uint8_t> pooled(bytes, 0x77);
			tw3d::tile_job_pool pool(2);
			tw3d::tiles_job job = pool.read_heightmap_async(pooled.data(), n, n, rects, 3);
			job.wait();
			if (pooled != want) {fprintf(stderr, "tile_job_pool::read_heightmap_async differs\n"); ok = false;}
		}
		// an erosion of the image on the device, then the read
		tw_ctx *c = tw3d::ctx();
		std::vector<float> chain(cells);
		std::vector<uint8_t> chain_img(bytes);
		tw_minmax mm;
		check(tw_heightmap_to_floats_u16(c, img.data(), cells, info.val_mult, info.val_add, chain.data()), "to_floats");
		check(tw_minmax_f32(c, chain.data(), cells, &mm), "minmax");
		tw3d::apply_erosion(chain.data(), n, n, mm.zmin, iters);
		check(tw_heightmap_from_floats_u16(c, chain.data(), cells, info.val_mult, info.val_add, chain_img.data()), "from_floats");
		if (chain_img == img) {fprintf(stderr, "the erosion changed nothing\n"); ok = false;}
		tw3d::tiles_job erosion = tw3d::erode_heightmap_async(info.val_mult, info.val_add, iters);
		int frames = 0;
		while (!erosion.ready()) {++frames;}
		std::vector<uint8_t> cpu(bytes, 0);
		tw3d::tiles_job read = tw3d::read_heightmap_async(cpu.data(), n, n);
		read.wait();
		printf("erosion ready after %d frame(s)\n", frames);
		if (cpu != chain_img) {fprintf(stderr, "the read after erode_heightmap_async differs from the chain's image\n"); ok = false;}
		// a brush stroke on the CPU copy, then update_heightmap: the device's image is the CPU copy, eroded outside the brush
		tw_hmap_rect const brush = {n/3, n/4, 29, 13};
		for (int y = brush.y; y < brush.y + brush.h; ++y) {
			for (int x = brush.x; x < brush.x + brush.w; ++x) {cpu[2*((size_t)y*n + x) + 1] ^= 0x21;}
		}
		tw3d::update_heightmap(cpu.data(), n, n, &brush, 1);
		std::vector<uint8_t> after(bytes, 0);
		tw3d::read_heightmap(after.data(), n, n);
		if (after != cpu) {fprintf(stderr, "the image after the brush differs from the CPU copy\n"); ok = false;}
		int refused = 0;
		try {tw3d::read_heightmap(after.data(), n + 1, n);} catch (tw3d::error const &e) {refused += (e.status == TW_ERR_ARG);}
		tw_hmap_rect const outside = {n - 3, 0, 4, 1};
		try {tw3d::read_heightmap(after.data(), n, n, &outside, 1);} catch (tw3d::error const &e) {refused += (e.status == TW_ERR_ARG);}
		if (refused != 2) {fprintf(stderr, "refusals: %d of 2\n", refused); ok = false;}
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
