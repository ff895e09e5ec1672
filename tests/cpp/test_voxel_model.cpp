// Drives tw3d::voxel_model the way an engine keeps a brush-edited voxel model: a GLM simplex grid built once per block, then brush boxes re-meshing only
// the blocks they change, outputs in page-locked memory. Checks, and prints "identical" when all hold:
// - a one-block model's mesh equals tw3d::voxel_mesh on the field and flags of create_procedural + voxel_build, byte for byte;
// - the blocked model's field and flags equal that chain's;
// - after each edit the raw field equals the caller's edited copy, and every re-meshed block equals the same block of a model built from that copy.
// usage: test_voxel_model <tables dir> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>

template<typename T> static std::vector<T> load(std::string const &path, size_t n) {
	std::vector<T> v(n);
	std::ifstream f(path, std::ios::binary);
	f.read((char *)v.data(), n*sizeof(T));
	if (!f) {fprintf(stderr, "cannot read %s\n", path.c_str()); exit(1);}
	return v;
}

struct blocks_out { // page-locked outputs and the host table of one job
	float *verts; uint32_t *indices; size_t vcap, tcap;
	std::vector<tw_voxel_block_mesh> table;
	uint32_t nblocks = 0; uint64_t nverts = 0, ntris = 0;
	tw_voxel_blocks_out out() {return {verts, vcap, indices, tcap, table.data(), &nblocks, &nverts, &ntris, nullptr};}
	// block -> its vertex bytes followed by its index bytes
	std::map<uint32_t, std::string> meshes() const {
		std::map<uint32_t, std::string> r;
		for (uint32_t k = 0; k < nblocks; ++k) {
			tw_voxel_block_mesh const &b = table[k];
			r[b.block] = std::string((const char *)(verts + 3*b.voff), 12*b.nverts) + std::string((const char *)(indices + 3*b.toff), 12*b.ntris);
		}
		return r;
	}
};

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_voxel_model <tables dir> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	unsigned const rm = (unsigned)atoi(argv[2]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = 1;
		tw3d::set_globals(g);
		unsigned const nx = 97, ny = 79, nz = 71, B = 16;
		std::vector<float> f_sync;
		tw3d::voxel_grid_view vs = {nx, ny, nz, {16.0f/96, 16.0f/78, 4.0f/71}, {-8.0f, -8.0f, -1.0f}, &f_sync};
		float const offset[3] = {0.5f, -0.25f, 0.0f}, zscale = -2.0f/(float)(nz - 1);
		tw3d::create_procedural(vs, 1.0f, 1.0f, offset, true, 123, 456, 1, zscale, 2);
		std::vector<float> raw = f_sync;
		std::vector<unsigned char> o_sync;
		tw3d::voxel_build(vs, o_sync, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data());
		tw3d::voxel_mesh_t const whole = tw3d::voxel_mesh(vs, o_sync, -1.0f, false, true, false, et.data(), tt.data(), e2v.data());
		size_t const cap = 2*whole.indices.size()/3 + 4096;
		tw3d::multi_gpu mg(1);
		void *pv[2] = {nullptr, nullptr}, *pi[2] = {nullptr, nullptr};
		for (int k = 0; k < 2; ++k) {
			if (tw_multi_alloc_host(mg.handle(), 0, cap*12, &pv[k]) != TW_OK || tw_multi_alloc_host(mg.handle(), 0, cap*12, &pi[k]) != TW_OK) {fprintf(stderr, "no pinned memory\n"); return 2;}
		}
		auto outs = [&](int k, size_t nblocks) {blocks_out o; o.verts = (float *)pv[k]; o.indices = (uint32_t *)pi[k]; o.vcap = o.tcap = cap; o.table.resize(nblocks); return o;};
		bool ok = true;
		{ // one block
			tw3d::voxel_model one(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), nx, ny);
			blocks_out o = outs(0, 1);
			tw_voxel_blocks_out const d = o.out();
			one.build_async(nullptr, raw.data(), d).wait();
			ok = ok && o.nblocks == 1 && o.nverts*3 == whole.verts.size() && o.ntris*3 == whole.indices.size() &&
			     !memcmp(o.verts, whole.verts.data(), whole.verts.size()*4) && !memcmp(o.indices, whole.indices.data(), whole.indices.size()*4);
			if (!ok) fprintf(stderr, "one block differs from voxel_mesh\n");
		}
		unsigned const nb = ((nx - 1 + B - 1)/B)*((ny - 1 + B - 1)/B);
		tw3d::voxel_model model(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), B, B);
		blocks_out o = outs(0, nb);
		tw_voxel_blocks_out d = o.out();
		tw_voxel_params const fp = tw3d::procedural_params(vs, 1.0f, 1.0f, offset, true, 123, 456, 1, zscale, 2);
		int frames = 0;
		{
			tw3d::tiles_job job = model.build_async(&fp, nullptr, d);
			while (!job.ready()) {++frames;}
		}
		std::vector<float> r, v;
		std::vector<unsigned char> fl;
		model.read(&r, &v, &fl);
		ok = ok && o.nblocks == nb && r == raw && !memcmp(v.data(), f_sync.data(), v.size()*4) && fl == o_sync;
		printf("build ready after %d poll(s): %u blocks, %llu vertices, %llu triangles\n", frames, o.nblocks, (unsigned long long)o.nverts, (unsigned long long)o.ntris);
		for (int e = 0; e < 6 && ok; ++e) { // brush boxes of 7^3, alternately inside and outside, some on block faces
			unsigned const x0 = std::min((e % 2) ? B*(1 + e) - 3 : 11*e + 5, nx - 7), y0 = (e % 3) ? B*2 - 4 : 7*e + 3, z0 = 20 + 3*e;
			std::vector<tw_voxel_box> const boxes = {{x0, y0, z0, 7, 7, 7}};
			std::vector<float> vals(343, (e % 2) ? 2.0f : -3.0f);
			for (unsigned y = 0; y < 7; ++y) for (unsigned x = 0; x < 7; ++x) for (unsigned z = 0; z < 7; ++z) raw[(z0 + z) + ((size_t)(x0 + x) + (size_t)(y0 + y)*nx)*nz] = vals[0];
			blocks_out eo = outs(0, nb);
			tw_voxel_blocks_out const ed = eo.out();
			model.edit_async(boxes, vals.data(), ed).wait();
			model.read(&r, nullptr, nullptr);
			tw3d::voxel_model fresh(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), B, B);
			blocks_out fo = outs(1, nb);
			tw_voxel_blocks_out const fd = fo.out();
			fresh.build_async(nullptr, raw.data(), fd).wait();
			std::map<uint32_t, std::string> const got = eo.meshes(), want = fo.meshes();
			bool same = (r == raw) && eo.nblocks > 0;
			for (auto const &kv : got) same = same && want.count(kv.first) && want.at(kv.first) == kv.second;
			printf("edit %d: %u block(s) re-meshed, %s\n", e, eo.nblocks, same ? "equal" : "DIFFERENT");
			ok = ok && same;
		}
		for (int k = 0; k < 2; ++k) {tw_multi_free_host(mg.handle(), pv[k]); tw_multi_free_host(mg.handle(), pi[k]);}
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
