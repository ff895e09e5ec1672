// Drives tw3d::voxel_model's jobs on the slots of a tile_job_pool the way an engine issues brush strokes, one per frame, without waiting for the last one:
// the same build, brush edits and reads run on a model through the thread's context alone (every job waited for at once) and on a second model through a
// pool of 4 slots (every stroke launched before any is waited for, then the jobs waited for newest first). Checks, and prints "identical" when all hold:
// - each edit's block table and counts, and each read, are the same both ways;
// - a read_async launched between two strokes sees the first and not the second;
// - a read_async of boxes into pageable memory equals the boxes cut from a whole-grid read.
// usage: test_voxel_model_family <tables dir> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <memory>

template<typename T> static std::vector<T> load(std::string const &path, size_t n) {
	std::vector<T> v(n);
	std::ifstream f(path, std::ios::binary);
	f.read((char *)v.data(), n*sizeof(T));
	if (!f) {fprintf(stderr, "cannot read %s\n", path.c_str()); exit(1);}
	return v;
}

struct job_out { // one job's host results
	std::vector<tw_voxel_block_mesh> table;
	uint32_t nblocks = 0; uint64_t nverts = 0, ntris = 0, changed = 0;
	explicit job_out(unsigned nb) : table(nb) {}
	tw_voxel_blocks_out out() {return {nullptr, 0, nullptr, 0, table.data(), &nblocks, &nverts, &ntris, &changed};}
	bool operator==(job_out const &o) const {
		return nblocks == o.nblocks && nverts == o.nverts && ntris == o.ntris && changed == o.changed && !memcmp(table.data(), o.table.data(), nblocks*sizeof(tw_voxel_block_mesh));
	}
};

int main(int argc, char **argv) {
	if (argc < 3) {fprintf(stderr, "usage: test_voxel_model_family <tables dir> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	unsigned const rm = (unsigned)atoi(argv[2]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = 1;
		tw3d::set_globals(g);
		unsigned const nx = 97, ny = 79, nz = 71, B = 16, E = 6;
		size_t const n = (size_t)nx*ny*nz;
		std::vector<float> field;
		tw3d::voxel_grid_view vs = {nx, ny, nz, {16.0f/96, 16.0f/78, 4.0f/71}, {-8.0f, -8.0f, -1.0f}, &field};
		float const offset[3] = {0.5f, -0.25f, 0.0f}, zscale = -2.0f/(float)(nz - 1);
		tw_voxel_params const fp = tw3d::procedural_params(vs, 1.0f, 1.0f, offset, true, 123, 456, 1, zscale, 2);
		unsigned const nb = ((nx - 1 + B - 1)/B)*((ny - 1 + B - 1)/B);
		auto brush = [&](unsigned e, std::vector<tw_voxel_box> &boxes, std::vector<float> &vals) { // 7^3 boxes, alternately inside and outside
			unsigned const x0 = std::min((e % 2) ? B*(1 + e) - 3 : 11*e + 5, nx - 7), y0 = (e % 3) ? B*2 - 4 : 7*e + 3, z0 = 20 + 3*e;
			boxes = {{x0, y0, z0, 7, 7, 7}};
			vals.assign(343, (e % 2) ? 2.0f : -3.0f);
		};
		std::vector<tw_voxel_box> const rboxes = {{3, 5, 7, 11, 6, 9}, {40, 30, 0, 5, 13, nz}};
		size_t const rn = 11*6*9 + 5*13*(size_t)nz;
		// the thread's context alone
		tw3d::voxel_model a(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), B, B);
		std::vector<job_out> ra(E + 1, job_out(nb));
		std::vector<float> ra_mid(n), ra_end(n), rb_box(rn);
		a.build_async(&fp, nullptr, ra[0].out()).wait();
		std::vector<tw_voxel_box> boxes; std::vector<float> vals;
		for (unsigned e = 0; e < E; ++e) {
			brush(e, boxes, vals);
			a.edit_async(boxes, vals.data(), ra[e + 1].out()).wait();
			if (e == 2) {a.read_async({}, nullptr, ra_mid.data(), nullptr).wait();}
		}
		std::vector<float> a_raw(n), a_vals(n); std::vector<unsigned char> a_out(n);
		a.read(&a_raw, &a_vals, &a_out);
		// the same on pool slots, nothing waited for until every job is launched
		tw3d::tile_job_pool pool(4);
		tw3d::voxel_model b(vs, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), B, B);
		std::vector<job_out> rb(E + 1, job_out(nb));
		std::vector<std::unique_ptr<tw3d::tiles_job>> jobs;
		std::vector<std::vector<float>> held(E); // the values stay alive until the launch returns; kept to the end anyway
		jobs.emplace_back(new tw3d::tiles_job(b.build_async(&fp, nullptr, rb[0].out(), &pool)));
		std::vector<float> rb_mid(n), rb_raw(n), rb_vals(n); std::vector<unsigned char> rb_out(n);
		for (unsigned e = 0; e < E; ++e) {
			brush(e, boxes, held[e]);
			jobs.emplace_back(new tw3d::tiles_job(b.edit_async(boxes, held[e].data(), rb[e + 1].out(), &pool)));
			if (e == 2) {jobs.emplace_back(new tw3d::tiles_job(b.read_async({}, nullptr, rb_mid.data(), nullptr, &pool)));}
		}
		jobs.emplace_back(new tw3d::tiles_job(b.read_async({}, rb_raw.data(), rb_vals.data(), rb_out.data(), &pool)));
		jobs.emplace_back(new tw3d::tiles_job(b.read_async(rboxes, nullptr, rb_box.data(), nullptr, &pool)));
		for (size_t k = jobs.size(); k-- > 0;) {jobs[k]->wait();}
		bool ok = true;
		for (unsigned e = 0; e <= E; ++e) {
			bool const same = ra[e] == rb[e];
			printf("%s %u: %u block(s), %llu verts, %llu tris, %s\n", e ? "edit" : "build", e, rb[e].nblocks, (unsigned long long)rb[e].nverts,
			       (unsigned long long)rb[e].ntris, same ? "equal" : "DIFFERENT");
			ok = ok && same;
		}
		bool const mid = !memcmp(ra_mid.data(), rb_mid.data(), n*4) && memcmp(rb_mid.data(), rb_vals.data(), n*4) != 0;
		bool const end = !memcmp(a_raw.data(), rb_raw.data(), n*4) && !memcmp(a_vals.data(), rb_vals.data(), n*4) && a_out == rb_out;
		size_t k = 0; bool box = true;
		for (tw_voxel_box const &q : rboxes) {
			for (unsigned y = q.y; y < q.y + q.h; ++y) {
				for (unsigned x = q.x; x < q.x + q.w; ++x) {
					for (unsigned z = q.z; z < q.z + q.d; ++z, ++k) {box = box && !memcmp(&rb_box[k], &a_vals[z + ((size_t)x + (size_t)y*nx)*nz], 4);}
				}
			}
		}
		printf("read between strokes 3 and 4: %s; final reads: %s; box read: %s\n", mid ? "equal" : "DIFFERENT", end ? "equal" : "DIFFERENT", box ? "equal" : "DIFFERENT");
		ok = ok && mid && end && box;
		printf(ok ? "identical\n" : "DIFFERENT\n");
		return ok ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
