// Drives tw3d::voxel_model_build_batch_async / voxel_model_edit_batch_async the way an engine loads and hits its rock models: six small GLM rocks of
// different sizes built in one job, then four frames of brush strokes (one model left out of each frame) edited in one job, on the thread's context and on
// a tile_job_pool slot. Each model has a twin driven by voxel_model::build_async / edit_async. Checks, and prints "identical" when all hold: every job's
// block table, counts and change list count, and the final reads, are the same for each model and its twin, and each build lists all its blocks.
// usage: test_voxel_model_batch <tables dir> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <deque>
#include <memory>

template<typename T> static std::vector<T> load(std::string const &path, size_t n) {
	std::vector<T> v(n);
	std::ifstream f(path, std::ios::binary);
	f.read((char *)v.data(), n*sizeof(T));
	if (!f) {fprintf(stderr, "cannot read %s\n", path.c_str()); exit(1);}
	return v;
}

struct job_out { // one job's host results; o and ch point at its own members, so it is neither copied nor moved (held in a std::deque)
	std::vector<tw_voxel_block_mesh> table;
	uint32_t nblocks = 0; uint64_t nverts = 0, ntris = 0, changed = 0, nchanged = 0;
	tw_voxel_blocks_out o;
	tw_voxel_changes ch;
	explicit job_out(unsigned nb) : table(nb) {o = {nullptr, 0, nullptr, 0, table.data(), &nblocks, &nverts, &ntris, &changed}; ch = {nullptr, nullptr, nullptr, 0, &nchanged};}
	job_out(job_out const &) = delete;
	job_out &operator=(job_out const &) = delete;
	bool operator==(job_out const &b) const {
		return nblocks == b.nblocks && nverts == b.nverts && ntris == b.ntris && changed == b.changed && nchanged == b.nchanged &&
		       !memcmp(table.data(), b.table.data(), nblocks*sizeof(tw_voxel_block_mesh));
	}
};

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_voxel_model_batch <tables dir> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	unsigned const rm = (unsigned)atoi(argv[2]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = 1;
		tw3d::set_globals(g);
		unsigned const M = 6, F = 4;
		std::vector<std::vector<float>> field(M);
		std::vector<tw3d::voxel_grid_view> views;
		std::vector<tw_voxel_params> fills;
		std::vector<std::unique_ptr<tw3d::voxel_model>> A, B;
		std::vector<unsigned> nb;
		for (unsigned i = 0; i < M; ++i) {
			unsigned const nx = 20 + 7*i, ny = 18 + 5*i, nz = 24 + 3*i, bx = 3 + i, by = 5;
			views.push_back({nx, ny, nz, {2.0f/(nx - 1), 2.0f/(ny - 1), 2.0f/(nz - 1)}, {-1.0f, -1.0f, -1.0f}, &field[i]});
			float const offset[3] = {0.5f*i, -0.25f, 0.0f};
			fills.push_back(tw3d::procedural_params(views[i], 1.0f, 1.0f, offset, true, 123 + i, 456, 1, 0.0f, 3));
			for (int k = 0; k < 2; ++k) {
				(k ? B : A).emplace_back(new tw3d::voxel_model(views[i], 0.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), bx, by));
			}
			nb.push_back(((nx - 2 + bx)/bx)*((ny - 2 + by)/by));
		}
		tw3d::tile_job_pool pool(2);
		bool ok = true;
		auto compare = [&](const char *what, unsigned f, std::deque<job_out> const &a, std::deque<job_out> const &b) {
			for (unsigned i = 0; i < M; ++i) {
				bool const same = a[i] == b[i];
				if (!same) {printf("%s %u, model %u: DIFFERENT\n", what, f, i);}
				ok = ok && same;
			}
			printf("%s %u: %llu verts over %u models\n", what, f, (unsigned long long)[&] {uint64_t s = 0; for (auto const &j : a) {s += j.nverts;} return s;}(), M);
		};
		std::deque<job_out> ra, rb;
		for (unsigned i = 0; i < M; ++i) {ra.emplace_back(nb[i]); rb.emplace_back(nb[i]);}
		std::vector<tw3d::voxel_model_build_args> builds;
		for (unsigned i = 0; i < M; ++i) {builds.push_back({A[i].get(), &fills[i], nullptr, &ra[i].o});}
		tw3d::voxel_model_build_batch_async(builds).wait();
		for (unsigned i = 0; i < M; ++i) {B[i]->build_async(&fills[i], nullptr, rb[i].o).wait();}
		compare("build", 0, ra, rb);
		for (unsigned i = 0; i < M; ++i) { // a build lists every block: the comparison above covered each model's whole table
			if (ra[i].nblocks != nb[i]) {printf("build, model %u: %u of %u blocks listed\n", i, ra[i].nblocks, nb[i]); ok = false;}
		}
		for (unsigned f = 0; f < F; ++f) {
			std::deque<job_out> ea, eb;
			for (unsigned i = 0; i < M; ++i) {ea.emplace_back(nb[i]); eb.emplace_back(nb[i]);}
			std::vector<tw3d::voxel_model_edit_args> edits;
			std::vector<std::vector<float>> vals(M);
			for (unsigned i = 0; i < M; ++i) {
				std::vector<tw_voxel_box> boxes;
				if (i != f) { // model f is not hit this frame
					unsigned const w = 5, x = (3*f + 2*i) % (views[i].nx - w), y = (5*f + i) % (views[i].ny - w), z = (7*f + 3*i) % (views[i].nz - w);
					boxes.push_back({x, y, z, w, w, w});
					vals[i].assign(w*w*w, (f % 2) ? 2.0f : -3.0f);
				}
				edits.push_back({A[i].get(), boxes, vals[i].data(), &ea[i].o, &ea[i].ch});
			}
			tw3d::voxel_model_edit_batch_async(edits, (f % 2) ? &pool : nullptr).wait();
			for (unsigned i = 0; i < M; ++i) {B[i]->edit_async(edits[i].boxes, vals[i].data(), eb[i].o, eb[i].ch).wait();}
			compare("edit frame", f, ea, eb);
		}
		for (unsigned i = 0; i < M; ++i) {
			size_t const n = (size_t)views[i].nx*views[i].ny*views[i].nz;
			std::vector<float> ar(n), av(n), br(n), bv(n); std::vector<unsigned char> ao(n), bo(n);
			A[i]->read(&ar, &av, &ao); B[i]->read(&br, &bv, &bo);
			bool const same = !memcmp(ar.data(), br.data(), n*4) && !memcmp(av.data(), bv.data(), n*4) && ao == bo;
			if (!same) {printf("final read of model %u: DIFFERENT\n", i);}
			ok = ok && same;
		}
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
