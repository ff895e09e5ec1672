// Drives the adapter's ground-mode mesh without stalling the frame: tw3d::gen_mesh_async against tw3d::gen_mesh, on the thread's context and on a
// tile_job_pool slot. Checks that
//   - the mesh, the returned z values and tw_last_erosion_steps() equal gen_mesh's, byte for byte (sine mode with glaciation and 1500 droplets, a scrolled
//     domain-warp mesh, and a flat mesh whose previous zbottom / ztop / water_plane_z must survive);
//   - the scene_globals gen_mesh_async leaves once the job is ready equal the ones gen_mesh leaves, and stay untouched until then;
//   - the sine-table generator state advances as gen_mesh advances it.
// Prints "identical" when every check holds.
// usage: test_gen_mesh_job
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>

static bool same_globals(tw3d::scene_globals const &a, tw3d::scene_globals const &b) {
	return !memcmp(&a.zmax_est, &b.zmax_est, 4) && !memcmp(&a.zmin, &b.zmin, 4) && !memcmp(&a.zmax, &b.zmax, 4) && !memcmp(&a.water_plane_z, &b.water_plane_z, 4)
	    && !memcmp(&a.zbottom, &b.zbottom, 4) && !memcmp(&a.ztop, &b.ztop, 4);
}

int main() {
	try {
		bool ok = true;
		struct Case {int mode, shape, xoff2, yoff2; unsigned iters; bool flat; bool pool;};
		Case const cases[] = {{TW_MGEN_SINE, 0, 0, 0, 1500, false, false}, {TW_MGEN_DWARP_GPU, 1, -37, 512, 800, false, true}, {TW_MGEN_SIMPLEX, 2, 5, 9, 300, false, false},
		                      {TW_MGEN_SINE, 0, 3, -4, 400, true, false}};
		for (Case const &k : cases) {
			tw3d::scene_globals g;
			g.mesh_gen_mode = k.mode; g.mesh_gen_shape = k.shape; g.mesh_seed = 6; g.relh_adj_tex = 0.02f; g.clip_hd1 = 0.45f;
			g.zbottom = 0.25f; g.ztop = 0.75f; g.water_plane_z = -0.125f;
			if (k.flat) {g.MESH_START_MAG = 0.0f; g.GLACIATE = 0;} // every sine magnitude 0; without glaciation zbottom / ztop stay the previous ones
			tw3d::set_globals(g);
			size_t const n = (size_t)g.MESH_X_SIZE*g.MESH_Y_SIZE;
			std::vector<float> want(n), got(n, -1.0f);
			tw_rng r1 = {1, 1}, r2 = {1, 1};
			tw3d::gen_mesh_result const rw = tw3d::gen_mesh(want.data(), r1, 4.0f, 4.0f, k.iters, k.xoff2, k.yoff2, 0.0f, 0.0f, 0.05f, -0.03f);
			uint64_t const steps_w = tw_last_erosion_steps(tw3d::ctx());
			tw3d::scene_globals const gw = tw3d::globals();
			tw3d::set_globals(g);
			tw3d::gen_mesh_result rg;
			memset(&rg, 0xee, sizeof(rg));
			uint64_t steps = 0;
			if (k.pool) {
				tw3d::tile_job_pool pool(2);
				tw3d::tiles_job job = pool.gen_mesh_async(got.data(), r2, 4.0f, 4.0f, k.iters, k.xoff2, k.yoff2, 0.0f, 0.0f, 0.05f, -0.03f, &rg);
				if (!same_globals(tw3d::globals(), g)) {printf("globals changed before the job was ready\n"); ok = false;}
				job.wait();
				// the pool's slot context ran the job; its step count is that context's (the pool is about to go)
			}
			else {
				tw3d::tiles_job job = tw3d::gen_mesh_async(got.data(), r2, 4.0f, 4.0f, k.iters, k.xoff2, k.yoff2, 0.0f, 0.0f, 0.05f, -0.03f, &rg);
				if (!same_globals(tw3d::globals(), g)) {printf("globals changed before the job was ready\n"); ok = false;}
				while (!job.ready()) {}
				steps = tw_last_erosion_steps(tw3d::ctx());
				if (steps != steps_w) {printf("case %d: steps %llu vs %llu\n", k.mode, (unsigned long long)steps, (unsigned long long)steps_w); ok = false;}
			}
			if (memcmp(got.data(), want.data(), n*sizeof(float))) {printf("case %d/%d: the mesh differs\n", k.mode, k.shape); ok = false;}
			if (memcmp(&rg, &rw, sizeof(rw))) {printf("case %d/%d: the z values differ\n", k.mode, k.shape); ok = false;}
			if (!same_globals(tw3d::globals(), gw)) {printf("case %d/%d: the globals differ\n", k.mode, k.shape); ok = false;}
			if (r1.rseed1 != r2.rseed1 || r1.rseed2 != r2.rseed2) {printf("case %d/%d: the sine generator state differs\n", k.mode, k.shape); ok = false;}
			if (k.flat && (rw.zbottom != 0.25f || rw.ztop != 0.75f || rw.water_plane_z != -0.125f)) {printf("the flat mesh did not keep its values\n"); ok = false;}
		}
		if (ok) printf("identical\n");
		return ok ? 0 : 2;
	}
	catch (std::exception const &e) {fprintf(stderr, "error: %s\n", e.what()); return 3;}
}
