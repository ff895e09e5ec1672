// Drives the adapter's sweeps erosion jobs the way an engine would erode the island without stalling its frames: launch, keep drawing while ready() says
// no, then use the map. On a generated size x size terrain, compares
//   apply_erosion_sweeps_async        with apply_erosion_sweeps (the map and the moves),
//   erode_heightmap_sweeps_async      with to_floats -> minmax -> apply_erosion_sweeps -> from_floats (the eroded floats, and heightmap tiles over the whole
//                                     image against those of set_heightmap(the chain's image)),
// then cancels a long job (cancelled() is true, the next job is exact again) and a job that has finished (cancelled() is false, its output exact),
// and prints "identical" when every check passes.
// usage: test_erosion_sweeps_job <size> <erosion droplets> <sweep> <halo>
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

namespace {
bool same(std::vector<float> const &a, std::vector<float> const &b) {return a.size() == b.size() && !memcmp(a.data(), b.data(), a.size()*sizeof(float));}

void check(int rc, const char *what) {if (rc != TW_OK) {throw tw3d::error(rc, std::string(what) + ": " + tw_last_error(tw3d::ctx()));}}

int frames_until_ready(tw3d::tiles_job job) {int frames = 0; while (!job.ready()) {++frames;} return frames;}

// heightmap tiles of this thread's set_heightmap image covering all of it (texel (0,0) is the image centre)
std::vector<float> image_tiles(int n, float dx, float dy) {
	unsigned const S = 64, zv = S + 1;
	std::vector<int32_t> origins;
	for (int y = -n/2; y < n/2; y += (int)S) {for (int x = -n/2; x < n/2; x += (int)S) {origins.push_back(x); origins.push_back(y);}}
	unsigned const nt = (unsigned)origins.size()/2;
	std::vector<float> z((size_t)nt*zv*zv);
	tw_tile_outputs o;
	memset(&o, 0, sizeof(o));
	o.zvals = z.data();
	tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
	tw_tile_shadows const no_lights = {nullptr, 0, nullptr};
	tw3d::create_tiles_async_from_heightmap(origins.data(), nt, zv, dx, dy, 0, 0.0f, 0, o, none, no_lights).wait();
	return z;
}
}

int main(int argc, char **argv) {
	if (argc < 5) {fprintf(stderr, "usage: test_erosion_sweeps_job <size> <erosion droplets> <sweep> <halo>\n"); return 1;}
	int const n = atoi(argv[1]);
	unsigned const iters = (unsigned)atoi(argv[2]), sweep = (unsigned)atoi(argv[3]);
	int const halo = atoi(argv[4]);
	try {
		tw3d::scene_globals g;
		g.mesh_seed = 1; g.mesh_gen_mode = TW_MGEN_DWARP_GPU; g.zmin = -2.0f; g.zmax = 2.0f; g.water_plane_z = -0.5f;
		tw3d::set_globals(g);
		float const dx = 1.0f/g.DX_VAL_INV, dy = 1.0f/g.DY_VAL_INV;
		size_t const cells = (size_t)n*n;
		std::vector<uint8_t> img(2*cells);
		std::vector<float> terrain(cells);
		tw_heightmap_info info;
		tw3d::proc_gen_heightmap((unsigned)n, (unsigned)n, dx, dy, 0, img.data(), terrain.data(), &info);
		float const zmin = info.min_z;
		tw_ctx *c = tw3d::ctx();
		bool ok = true;
		// the float map
		std::vector<float> ref = terrain, map = terrain;
		uint64_t const moves = tw3d::apply_erosion_sweeps(ref.data(), n, n, zmin, iters, sweep, halo);
		int const frames = frames_until_ready(tw3d::apply_erosion_sweeps_async(map.data(), n, n, zmin, iters, sweep, halo));
		printf("apply_erosion_sweeps_async ready after %d frame(s), %llu droplet moves\n", frames, (unsigned long long)moves);
		if (moves == 0 || same(ref, terrain) || !same(map, ref) || tw_last_erosion_steps(c) != moves) {fprintf(stderr, "apply_erosion_sweeps_async differs\n"); ok = false;}
		// the image: the synchronous chain
		std::vector<float> chain(cells);
		std::vector<uint8_t> chain_img(2*cells);
		tw_minmax mm;
		check(tw_heightmap_to_floats_u16(c, img.data(), cells, info.val_mult, info.val_add, chain.data()), "to_floats");
		check(tw_minmax_f32(c, chain.data(), cells, &mm), "minmax");
		uint64_t const chain_moves = tw3d::apply_erosion_sweeps(chain.data(), n, n, mm.zmin, iters, sweep, halo);
		check(tw_heightmap_from_floats_u16(c, chain.data(), cells, info.val_mult, info.val_add, chain_img.data()), "from_floats");
		tw3d::scene_globals g2 = g;
		g2.mesh_file_scale = info.mesh_file_scale; g2.mesh_file_tz = info.mesh_file_tz;
		tw3d::set_globals(g2);
		tw3d::set_heightmap(chain_img.data(), n, n);
		std::vector<float> const z_ref = image_tiles(n, dx, dy);
		// ... and the job on the original image
		std::vector<float> vals(cells);
		tw3d::set_heightmap(img.data(), n, n);
		tw3d::tiles_job job = tw3d::erode_heightmap_sweeps_async(info.val_mult, info.val_add, iters, sweep, halo, vals.data());
		job.wait();
		if (job.cancelled() || tw_last_erosion_steps(c) != chain_moves || !same(vals, chain) || !same(image_tiles(n, dx, dy), z_ref)) {fprintf(stderr, "erode_heightmap_sweeps_async differs\n"); ok = false;}
		// a long job cancelled at once: cancelled(), and the next job is exact. It erodes the image without vals: a job with a pageable host map or vals
		// would hold the launch until its copies, i.e. the whole job, are done
		{
			tw3d::set_heightmap(img.data(), n, n);
			tw3d::tiles_job long_job = tw3d::erode_heightmap_sweeps_async(info.val_mult, info.val_add, 4000000u, 1000u, halo);
			long_job.cancel();
			long_job.wait();
			if (!long_job.cancelled() || tw_last_erosion_steps(c) != 0) {fprintf(stderr, "the cancelled job was not reported as cancelled\n"); ok = false;}
			std::vector<float> again = terrain;
			tw3d::apply_erosion_sweeps_async(again.data(), n, n, zmin, iters, sweep, halo).wait();
			if (!same(again, ref) || tw_last_erosion_steps(c) != moves) {fprintf(stderr, "the job after a cancelled one differs\n"); ok = false;}
		}
		// a cancel after the job has finished changes nothing
		{
			std::vector<float> m2 = terrain;
			tw3d::tiles_job j2 = tw3d::apply_erosion_sweeps_async(m2.data(), n, n, zmin, iters, sweep, halo);
			check(tw_sync(c), "tw_sync");
			j2.cancel();
			j2.wait();
			if (j2.cancelled() || !same(m2, ref) || tw_last_erosion_steps(c) != moves) {fprintf(stderr, "a cancel after the job ended changed it\n"); ok = false;}
		}
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
