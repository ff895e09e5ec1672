// Drives the adapter's mesh shadows of the ground-mode mesh: the blocking tw3d::calc_mesh_shadows(lpos, mh, smask, xsize, ysize, ...), tw3d::mesh_shadows_async
// (thread context and tile_job_pool slot) and tw3d::gen_mesh_async with lights. Checks that
//   - on the mesh the Python side wrote (dir/mesh.f32, xsize x ysize, globals from dir/params.f32), the blocking overload and both async forms give the masks
//     and edges the oracle gave (dir/oracle_<l>.bin: smask bytes, sh_out_x, sh_out_y), byte for byte;
//   - gen_mesh_async with lights equals gen_mesh followed by calc_mesh_shadows with the zmin / zmax gen_mesh left in scene_globals.
// Prints "identical" when every check holds.
// usage: test_mesh_shadows <dir>
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>
#include <string>

static std::vector<char> slurp(std::string const &path) {
	FILE *f = fopen(path.c_str(), "rb");
	if (!f) {fprintf(stderr, "cannot open %s\n", path.c_str()); exit(4);}
	std::vector<char> b;
	char buf[65536];
	size_t n;
	while ((n = fread(buf, 1, sizeof(buf), f)) > 0) {b.insert(b.end(), buf, buf + n);}
	fclose(f);
	return b;
}

struct result {std::vector<unsigned char> m; std::vector<float> ox, oy;};
static result make(int xs, int ys) {return result{std::vector<unsigned char>((size_t)xs*ys), std::vector<float>(xs), std::vector<float>(ys)};}
static bool same(result const &a, result const &b) {
	return a.m == b.m && !memcmp(a.ox.data(), b.ox.data(), a.ox.size()*4) && !memcmp(a.oy.data(), b.oy.data(), a.oy.size()*4);
}
static tw_tile_light light(const float lpos[3], result &r) {
	tw_tile_light L;
	L.sp = tw3d::mesh_shadow_params(lpos); L.sh_in_x = nullptr; L.sh_in_y = nullptr; L.smask = r.m.data(); L.sh_out_x = r.ox.data(); L.sh_out_y = r.oy.data();
	return L;
}

int main(int argc, char **argv) {
	if (argc < 2) {fprintf(stderr, "usage: test_mesh_shadows <dir>\n"); return 1;}
	try {
		std::string const dir = argv[1];
		bool ok = true;
		std::vector<char> const pb = slurp(dir + "/params.f32");
		float const *P = (const float *)pb.data(); // xsize, ysize, x_scene, y_scene, zmin, zmax, nlights, then lpos per light
		int const xs = (int)P[0], ys = (int)P[1], nl = (int)P[6];
		tw3d::scene_globals g;
		g.MESH_X_SIZE = xs; g.MESH_Y_SIZE = ys; g.X_SCENE_SIZE = P[2]; g.Y_SCENE_SIZE = P[3]; g.zmin = P[4]; g.zmax = P[5];
		g.DX_VAL_INV = 1.0f/(2.0f*g.X_SCENE_SIZE/xs); g.DY_VAL_INV = 1.0f/(2.0f*g.Y_SCENE_SIZE/ys);
		tw3d::set_globals(g);
		std::vector<char> const mb = slurp(dir + "/mesh.f32");
		const float *mh = (const float *)mb.data();
		std::vector<tw_tile_light> lights;
		std::vector<result> blocking, async1, async2;
		for (int l = 0; l < nl; ++l) {blocking.push_back(make(xs, ys)); async1.push_back(make(xs, ys)); async2.push_back(make(xs, ys));}
		for (int l = 0; l < nl; ++l) {
			const float *lp = P + 7 + 3*l;
			tw3d::calc_mesh_shadows(lp, mh, blocking[l].m.data(), xs, ys, nullptr, nullptr, blocking[l].ox.data(), blocking[l].oy.data());
			std::vector<char> const ob = slurp(dir + "/oracle_" + std::to_string(l) + ".bin");
			result want = make(xs, ys);
			memcpy(want.m.data(), ob.data(), want.m.size());
			memcpy(want.ox.data(), ob.data() + want.m.size(), xs*4);
			memcpy(want.oy.data(), ob.data() + want.m.size() + xs*4, ys*4);
			if (!same(blocking[l], want)) {printf("light %d: calc_mesh_shadows differs from the oracle\n", l); ok = false;}
			lights.push_back(light(lp, async1[l]));
		}
		tw3d::mesh_shadows_async(mh, xs, ys, lights).wait();
		{
			tw3d::tile_job_pool pool(2);
			std::vector<tw_tile_light> l2;
			for (int l = 0; l < nl; ++l) {l2.push_back(light(P + 7 + 3*l, async2[l]));}
			pool.mesh_shadows_async(mh, xs, ys, l2).wait();
		}
		for (int l = 0; l < nl; ++l) {
			if (!same(async1[l], blocking[l])) {printf("light %d: mesh_shadows_async differs\n", l); ok = false;}
			if (!same(async2[l], blocking[l])) {printf("light %d: tile_job_pool::mesh_shadows_async differs\n", l); ok = false;}
		}
		// the ground-mode mesh: gen_mesh then calc_mesh_shadows with the globals it leaves, against one gen_mesh_async with lights
		for (bool pool : {false, true}) {
			tw3d::scene_globals h;
			h.mesh_gen_mode = TW_MGEN_SINE; h.mesh_seed = 6;
			tw3d::set_globals(h);
			size_t const n = (size_t)h.MESH_X_SIZE*h.MESH_Y_SIZE;
			std::vector<float> want(n), got(n);
			tw_rng r1 = {1, 1}, r2 = {1, 1};
			tw3d::gen_mesh(want.data(), r1, 4.0f, 4.0f, 1500);
			std::vector<result> w, r;
			std::vector<tw_tile_light> gl;
			for (int l = 0; l < nl; ++l) {w.push_back(make(h.MESH_X_SIZE, h.MESH_Y_SIZE)); r.push_back(make(h.MESH_X_SIZE, h.MESH_Y_SIZE));}
			for (int l = 0; l < nl; ++l) {
				tw3d::calc_mesh_shadows(P + 7 + 3*l, want.data(), w[l].m.data(), h.MESH_X_SIZE, h.MESH_Y_SIZE, nullptr, nullptr, w[l].ox.data(), w[l].oy.data());
				gl.push_back(light(P + 7 + 3*l, r[l]));
			}
			tw3d::set_globals(h);
			if (pool) {tw3d::tile_job_pool p(2); p.gen_mesh_async(got.data(), r2, 4.0f, 4.0f, 1500, gl).wait();}
			else {tw3d::gen_mesh_async(got.data(), r2, 4.0f, 4.0f, 1500, gl).wait();}
			if (memcmp(got.data(), want.data(), n*4)) {printf("gen_mesh_async with lights: the mesh differs\n"); ok = false;}
			for (int l = 0; l < nl; ++l) {if (!same(r[l], w[l])) {printf("gen_mesh_async with lights: light %d differs\n", l); ok = false;}}
		}
		if (ok) printf("identical\n");
		return ok ? 0 : 2;
	}
	catch (std::exception const &e) {fprintf(stderr, "error: %s\n", e.what()); return 3;}
}
