// Drives tw3d::voxel_build_async the way an engine would build a voxel model without stalling its frames: launch the fill + build, keep drawing while
// ready() says no, then use the field, the flags and the triangles. Compares them with the synchronous adapter calls (create_procedural + voxel_build) on
// the same grid and prints "identical" when every byte agrees; a second job with no field output and a capacity of 7 must give the first 7 triangles
// and the full count, and leave the rest of its buffer alone.
// usage: test_voxel_build <tables dir> <gen_mode> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
#define TW3D_NO_ABORT
#include "tw3d_adapter.h"
#include <cmath>
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
	if (argc < 4) {fprintf(stderr, "usage: test_voxel_build <tables dir> <gen_mode> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	int const mode = atoi(argv[2]);
	unsigned const rm = (unsigned)atoi(argv[3]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = mode;
		tw3d::set_globals(g);
		unsigned const nx = 97, ny = 79, nz = 71; // n % 4 == 1: the job's padded flags
		std::vector<float> f_sync, f_async;
		tw3d::voxel_grid_view vs = {nx, ny, nz, {16.0f/96, 16.0f/78, 4.0f/71}, {-8.0f, -8.0f, -1.0f}, &f_sync};
		tw3d::voxel_grid_view va = vs;
		va.data = &f_async;
		float const offset[3] = {0.5f, -0.25f, 0.0f}, zscale = -2.0f/(float)(nz - 1);
		// the synchronous chain
		tw3d::create_procedural(vs, 1.0f, 1.0f, offset, true, 123, 456, mode, zscale, 2);
		std::vector<unsigned char> o_sync;
		std::vector<float> const t_sync = tw3d::voxel_build(vs, o_sync, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data());
		size_t const n = (size_t)nx*ny*nz, nt = t_sync.size()/9;
		if (nt < 100) {fprintf(stderr, "only %zu triangles\n", nt); return 3;}
		// the job: page-locked flags and triangles (with room for sentinels past the capacity)
		tw3d::multi_gpu m(1);
		void *po = nullptr, *pt = nullptr;
		if (tw_multi_alloc_host(m.handle(), 0, n, &po) != TW_OK || tw_multi_alloc_host(m.handle(), 0, (nt + 16)*9*sizeof(float), &pt) != TW_OK) {fprintf(stderr, "no pinned memory\n"); return 2;}
		unsigned char *o_async = (unsigned char *)po;
		float *t_async = (float *)pt;
		for (size_t i = 0; i < (nt + 16)*9; ++i) t_async[i] = NAN;
		tw_voxel_params const fp = tw3d::procedural_params(va, 1.0f, 1.0f, offset, true, 123, 456, mode, zscale, 2);
		uint64_t ntris = 0;
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::voxel_build_async(va, &fp, o_async, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), t_async, nt + 16, ntris);
			while (!job.ready()) {++frames;}
		}
		printf("build ready after %d frame(s), %llu triangles\n", frames, (unsigned long long)ntris);
		bool same = ntris == nt && f_async.size() == n && !memcmp(f_async.data(), f_sync.data(), n*sizeof(float)) && !memcmp(o_async, o_sync.data(), n) &&
		            !memcmp(t_async, t_sync.data(), nt*9*sizeof(float));
		for (size_t i = nt*9; i < (nt + 16)*9; ++i) same = same && std::isnan(t_async[i]);
		// triangles only, capacity 7
		for (size_t i = 0; i < (nt + 16)*9; ++i) t_async[i] = NAN;
		tw3d::voxel_grid_view vn = va;
		vn.data = nullptr;
		uint64_t n7 = 0;
		tw3d::voxel_build_async(vn, &fp, nullptr, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(), t_async, 7, n7).wait();
		bool cut = n7 == nt && !memcmp(t_async, t_sync.data(), 7*9*sizeof(float));
		for (size_t i = 7*9; i < (nt + 16)*9; ++i) cut = cut && std::isnan(t_async[i]);
		if (!cut) {fprintf(stderr, "capacity 7: count %llu, or bytes differ\n", (unsigned long long)n7);}
		tw_multi_free_host(m.handle(), po); tw_multi_free_host(m.handle(), pt);
		printf(same && cut ? "identical\n" : "DIFFERENT\n");
		return (same && cut) ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
