// Drives tw3d::voxel_mesh and the voxel_build_async overload with mesh outputs the way an engine builds a voxel model's indexed mesh: the synchronous
// chain (create_procedural + voxel_build + voxel_mesh) against one job that fills the grid and returns the soup and the welded mesh in page-locked memory.
// Prints "identical" when the field, the soup and the mesh agree byte for byte, the counts agree, the mesh indices are below the vertex count and the
// sentinels past the capacities are untouched; a second job with the mesh only (no soup) must give the same mesh.
// usage: test_voxel_mesh <tables dir> <gen_mode> <remove_unconnected>   (the dir holds edge_table.bin, tri_table.bin, edge_to_vals.bin)
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
	if (argc < 4) {fprintf(stderr, "usage: test_voxel_mesh <tables dir> <gen_mode> <remove_unconnected>\n"); return 1;}
	std::string const dir = argv[1];
	int const mode = atoi(argv[2]);
	unsigned const rm = (unsigned)atoi(argv[3]);
	try {
		std::vector<unsigned> const et = load<unsigned>(dir + "/edge_table.bin", 256), e2v = load<unsigned>(dir + "/edge_to_vals.bin", 24);
		std::vector<int> const tt = load<int>(dir + "/tri_table.bin", 256*16);
		tw3d::scene_globals g;
		g.mesh_seed = 3; g.mesh_gen_mode = mode;
		tw3d::set_globals(g);
		unsigned const nx = 97, ny = 79, nz = 71;
		std::vector<float> f_sync, f_async;
		tw3d::voxel_grid_view vs = {nx, ny, nz, {16.0f/96, 16.0f/78, 4.0f/71}, {-8.0f, -8.0f, -1.0f}, &f_sync};
		tw3d::voxel_grid_view va = vs;
		va.data = &f_async;
		float const offset[3] = {0.5f, -0.25f, 0.0f}, zscale = -2.0f/(float)(nz - 1);
		tw3d::create_procedural(vs, 1.0f, 1.0f, offset, true, 123, 456, mode, zscale, 2);
		std::vector<unsigned char> o_sync;
		std::vector<float> const t_sync = tw3d::voxel_build(vs, o_sync, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data());
		tw3d::voxel_mesh_t const m_sync = tw3d::voxel_mesh(vs, o_sync, -1.0f, false, true, false, et.data(), tt.data(), e2v.data());
		size_t const nt = t_sync.size()/9, mv = m_sync.verts.size()/3, mt = m_sync.indices.size()/3;
		if (nt < 100 || mv < 50) {fprintf(stderr, "only %zu triangles, %zu vertices\n", nt, mv); return 3;}
		bool in_range = true;
		for (uint32_t i : m_sync.indices) in_range = in_range && i < mv;
		tw3d::multi_gpu m(1);
		void *pt = nullptr, *pv = nullptr, *pi = nullptr;
		if (tw_multi_alloc_host(m.handle(), 0, (nt + 16)*9*sizeof(float), &pt) != TW_OK || tw_multi_alloc_host(m.handle(), 0, (mv + 16)*3*sizeof(float), &pv) != TW_OK ||
		    tw_multi_alloc_host(m.handle(), 0, (mt + 16)*3*sizeof(uint32_t), &pi) != TW_OK) {fprintf(stderr, "no pinned memory\n"); return 2;}
		float *t_async = (float *)pt, *v_async = (float *)pv;
		uint32_t *i_async = (uint32_t *)pi;
		auto reset = [&]() {
			for (size_t i = 0; i < (nt + 16)*9; ++i) t_async[i] = NAN;
			for (size_t i = 0; i < (mv + 16)*3; ++i) v_async[i] = NAN;
			for (size_t i = 0; i < (mt + 16)*3; ++i) i_async[i] = 0xdeadbeefu;
		};
		auto mesh_same = [&](uint64_t nv, uint64_t nm) {
			bool s = nv == mv && nm == mt && !memcmp(v_async, m_sync.verts.data(), mv*3*sizeof(float)) && !memcmp(i_async, m_sync.indices.data(), mt*3*sizeof(uint32_t));
			for (size_t i = mv*3; i < (mv + 16)*3; ++i) s = s && std::isnan(v_async[i]);
			for (size_t i = mt*3; i < (mt + 16)*3; ++i) s = s && i_async[i] == 0xdeadbeefu;
			return s;
		};
		tw_voxel_params const fp = tw3d::procedural_params(va, 1.0f, 1.0f, offset, true, 123, 456, mode, zscale, 2);
		reset();
		uint64_t ntris = 0, nverts = 0, nmesh = 0;
		int frames = 0;
		{
			tw3d::tiles_job job = tw3d::voxel_build_async(va, &fp, nullptr, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(),
			                                              t_async, nt + 16, &ntris, v_async, mv + 16, i_async, mt + 16, nverts, nmesh);
			while (!job.ready()) {++frames;}
		}
		printf("build ready after %d frame(s): %llu triangles, mesh %llu vertices / %llu triangles\n", frames, (unsigned long long)ntris,
		       (unsigned long long)nverts, (unsigned long long)nmesh);
		bool same = in_range && ntris == nt && f_async.size() == f_sync.size() && !memcmp(f_async.data(), f_sync.data(), f_sync.size()*sizeof(float)) &&
		            !memcmp(t_async, t_sync.data(), nt*9*sizeof(float)) && mesh_same(nverts, nmesh);
		// the mesh only
		reset();
		tw3d::voxel_grid_view vn = va;
		vn.data = nullptr;
		nverts = nmesh = 0;
		tw3d::voxel_build_async(vn, &fp, nullptr, -1.0f, false, true, rm, false, true, false, nullptr, et.data(), tt.data(), e2v.data(),
		                        nullptr, 0, nullptr, v_async, mv + 16, i_async, mt + 16, nverts, nmesh).wait();
		bool const only = mesh_same(nverts, nmesh) && std::isnan(t_async[0]);
		if (!only) {fprintf(stderr, "mesh-only job differs: %llu / %llu\n", (unsigned long long)nverts, (unsigned long long)nmesh);}
		tw_multi_free_host(m.handle(), pt); tw_multi_free_host(m.handle(), pv); tw_multi_free_host(m.handle(), pi);
		printf(same && only ? "identical\n" : "DIFFERENT\n");
		return (same && only) ? 0 : 4;
	}
	catch (tw3d::error const &e) {fprintf(stderr, "tw3d error %d: %s\n", e.status, e.what()); return 2;}
}
