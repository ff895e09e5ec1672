// Drives tw3d::voxel_model::edit_async with a change list the way an engine keeps its voxel_manager field and outside flags in step with the device: one
// read after the build, then per brush edit only the listed voxels, patched into the engine's copies once the job is ready. Checks, and prints "identical"
// when all hold:
// - after each edit, the patched copies equal voxel_model::read byte for byte, and the list is ascending;
// - an edit whose list does not fit its capacity reports its full count, writes no more than the capacity and makes apply_changes return false.
// usage: test_voxel_changes <tables dir> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>

template<typename T> static std::vector<T> load(std::string const &path, size_t n) {
	std::vector<T> v(n);
	std::ifstream f(path, std::ios::binary);
	f.read((char *)v.data(), n*sizeof(T));
	if (!f) {fprintf(stderr, "cannot read %s\n", path.c_str()); exit(1);}
	return v;
}

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_voxel_changes <tables dir> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	unsigned const rm = (unsigned)atoi(argv[2]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = 1;
		tw3d::set_globals(g);
		unsigned const nx = 97, ny = 79, nz = 71, B = 16;
		std::vector<float> field;
		tw3d::voxel_grid_view vs = {nx, ny, nz, {16.0f/96, 16.0f/78, 4.0f/71}, {-8.0f, -8.0f, -1.0f}, &field};
		float const offset[3] = {0.5f, -0.25f, 0.0f}, zscale = -2.0f/(float)(nz - 1);
		tw_voxel_params const fp = tw3d::procedural_params(vs, 1.0f, 1.0f, offset, true, 123, 456, 1, zscale, 2);
		tw3d::voxel_model model(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), B, B);
		unsigned const nb = ((nx - 1 + B - 1)/B)*((ny - 1 + B - 1)/B);
		std::vector<tw_voxel_block_mesh> table(nb);
		uint32_t nblocks = 0; uint64_t nverts = 0, ntris = 0;
		tw_voxel_blocks_out const out = {nullptr, 0, nullptr, 0, table.data(), &nblocks, &nverts, &ntris, nullptr};
		model.build_async(&fp, nullptr, out).wait();
		std::vector<float> vals, v;
		std::vector<unsigned char> outside, o;
		model.read(nullptr, &vals, &outside); // the engine's copies, read once
		size_t const cap = (size_t)nx*ny*nz;
		tw3d::multi_gpu mg(1);
		void *pi = nullptr, *pv = nullptr, *po = nullptr;
		if (tw_multi_alloc_host(mg.handle(), 0, cap*4, &pi) != TW_OK || tw_multi_alloc_host(mg.handle(), 0, cap*4, &pv) != TW_OK ||
		    tw_multi_alloc_host(mg.handle(), 0, cap, &po) != TW_OK) {fprintf(stderr, "no pinned memory\n"); return 2;}
		uint64_t nchanged = 0;
		tw_voxel_changes ch = {(uint32_t *)pi, (float *)pv, (uint8_t *)po, cap, &nchanged};
		bool ok = true;
		for (int e = 0; e < 6 && ok; ++e) { // brush boxes of 7^3, alternately inside and outside, some on block faces
			unsigned const x0 = std::min((e % 2) ? B*(1 + e) - 3 : 11*e + 5, nx - 7), y0 = (e % 3) ? B*2 - 4 : 7*e + 3, z0 = 20 + 3*e;
			std::vector<tw_voxel_box> const boxes = {{x0, y0, z0, 7, 7, 7}};
			std::vector<float> const box(343, (e % 2) ? 2.0f : -3.0f);
			model.edit_async(boxes, box.data(), out, ch).wait();
			bool const fits = tw3d::voxel_model::apply_changes(ch, &vals, &outside);
			model.read(nullptr, &v, &o);
			bool const asc = std::is_sorted(ch.index, ch.index + nchanged) && std::adjacent_find(ch.index, ch.index + nchanged) == ch.index + nchanged;
			bool const same = fits && asc && nchanged > 0 && !memcmp(v.data(), vals.data(), cap*4) && o == outside;
			printf("edit %d: %llu voxel(s) changed, %u block(s) re-meshed, %s\n", e, (unsigned long long)nchanged, nblocks, same ? "equal" : "DIFFERENT");
			ok = ok && same;
		}
		{ // a list that overflows: the count is complete, nothing past the capacity is written, and apply_changes refuses it
			std::vector<tw_voxel_box> const boxes = {{40, 30, 10, 9, 9, 30}};
			std::vector<float> const box(9*9*30, 3.0f);
			uint32_t *const idx = (uint32_t *)pi;
			std::fill(idx, idx + 16, 0xdeadbeefu);
			tw_voxel_changes const small = {idx, nullptr, nullptr, 8, &nchanged};
			model.edit_async(boxes, box.data(), out, small).wait();
			bool const over = nchanged > 8 && idx[8] == 0xdeadbeefu && idx[7] != 0xdeadbeefu && !tw3d::voxel_model::apply_changes(small, &vals, &outside);
			printf("overflowing list: %llu voxel(s) changed, capacity 8, %s\n", (unsigned long long)nchanged, over ? "refused" : "WRONG");
			ok = ok && over;
		}
		tw_multi_free_host(mg.handle(), pi); tw_multi_free_host(mg.handle(), pv); tw_multi_free_host(mg.handle(), po);
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
