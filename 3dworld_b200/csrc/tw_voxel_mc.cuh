// tw_voxel_mc.cuh - the voxel pipeline's device code shared by tw_voxel_post.cu (the library) and tw_voxel_batch.cu (the batch module, which tw_voxel_post.cu
// loads at run time): the outside flag of a voxel, and the welded marching-cubes mesh - its owner rule, its per-cube work and one MC_BLOCK-cube block of its
// count and emit passes. Included at file scope; everything here has internal linkage, so each translation unit keeps its own copy and its own kernels' names.
#pragma once
#include "../../include/tw3d.h"
#include "tw_voxel_math.cuh"

namespace {

constexpr float VOX_TOLERANCE = 1.0E-12f; // TOLERANCE, src/3DWorld.h:50


// a voxel's value for outside_flag: read from the field (read-only in the kernel), or already in a register
__device__ __forceinline__ float vox_val(const float *__restrict__ vals, size_t i) {return __ldg(vals + i);}
__device__ __forceinline__ float vox_val(float val, size_t) {return val;}
// determine_voxels_outside + calc_outside_val + val_is_outside (src/voxels.cpp:571-604) of voxel i = (x, y, z)
template<typename V>
__device__ __forceinline__ unsigned char outside_flag(V vals, size_t i, unsigned x, unsigned y, unsigned z, tw_voxel_post_params P, const unsigned *__restrict__ zix_xy) {
	bool const on_edge = (P.make_closed_surface && ((x == 0 || x == P.nx-1) || (y == 0 || y == P.ny-1) || (z == 0 || z == P.nz-1)));
	float const val = vox_val(vals, i);
	unsigned char ival = on_edge ? (unsigned char)TW_VOX_ON_EDGE : (unsigned char)((val == P.isolevel) ? 1 : (((val < P.isolevel) != (P.invert != 0)) ? 1 : 0)); // val_is_outside
	if (zix_xy && z < __ldg(zix_xy + (size_t)y*P.nx + x)) {ival |= TW_VOX_UNDER_MESH;}
	return ival;
}

struct McTables {const unsigned *edge_table; const int *tri_table; const unsigned *edge_to_vals;};
constexpr int MC_BLOCK = 1024;
__device__ __forceinline__ void interpolate_pt(float isolevel, const float *pt1, const float *pt2, float val1, float val2, float *pt) { // src/voxels.cpp:485-493
	if (fabsf(isolevel - val1) < VOX_TOLERANCE) {pt[0] = pt1[0]; pt[1] = pt1[1]; pt[2] = pt1[2]; return;}
	if (fabsf(isolevel - val2) < VOX_TOLERANCE) {pt[0] = pt2[0]; pt[1] = pt2[1]; pt[2] = pt2[2]; return;}
	if (fabsf(val1     - val2) < VOX_TOLERANCE) {pt[0] = pt1[0]; pt[1] = pt1[1]; pt[2] = pt1[2]; return;}
	float const mu = smax(0.0f, smin(1.0f, __fdiv_rn(isolevel - val1, val2 - val1))); // CLIP_TO_01
#pragma unroll
	for (int i = 0; i < 3; ++i) {pt[i] = pt1[i] + mu*(pt2[i] - pt1[i]);}
}


// The cube's 12 edges as grid edges, from edge_to_vals: s_edge[i] = axis | ox << 2 | oy << 3 | oz << 4 (axis 0 x, 1 y, 2 z; o = the edge's low corner in
// the cube); s_look[4*axis + 2*o1 + o2] = the local edge along axis whose low corner is at o1, o2 on the axis' other two (perp() order).
// edge_to_vals must name each edge of the cube once (Bourke's table does).
__device__ __forceinline__ void perp(unsigned a, unsigned &p1, unsigned &p2) {p1 = (a == 1) ? 0u : 1u; p2 = (a == 2) ? 0u : 2u;} // y > x > z in index weight
__device__ void mesh_edge_tables(const unsigned *__restrict__ etv, unsigned char *s_edge, unsigned char *s_look) {
	unsigned const t = threadIdx.x;
	if (t < 12) {
		unsigned c[2][3];
		for (unsigned d = 0; d < 2; ++d) {
			unsigned const e = __ldg(etv + 2*t + d), yhi = (e & 2) >> 1;
			c[d][0] = yhi ^ (e & 1); c[d][1] = yhi; c[d][2] = (e >> 2) & 1;
		}
		unsigned const a = (c[0][0] != c[1][0]) ? 0u : ((c[0][1] != c[1][1]) ? 1u : 2u);
		s_edge[t] = (unsigned char)(a | (min(c[0][0], c[1][0]) << 2) | (min(c[0][1], c[1][1]) << 3) | (min(c[0][2], c[1][2]) << 4));
	}
	__syncthreads();
	if (t < 12) {
		unsigned char look = 0;
		for (unsigned i = 0; i < 12; ++i) {
			unsigned const e = s_edge[i], a = e & 3;
			unsigned p1, p2; perp(a, p1, p2);
			if (4*a + 2*((e >> (2 + p1)) & 1) + ((e >> (2 + p2)) & 1) == t) {look = (unsigned char)i;}
		}
		s_look[t] = look;
	}
	__syncthreads();
}

// A block of a voxel model (tw_voxel_model): the cubes x in [x0, x1), y in [y0, y1), every z. A cube's index within it is ((y - y0)*(x1 - x0) + x - x0)*nz + z.
struct CubeRange {unsigned x0, x1, y0, y1;};

// cube (c[0], c[1], c[2]) makes triangles: inside the grid (with BLK: inside R), not in the last layer of an axis, and not skip_under_mesh with its 4 low
// corners under the mesh
template<bool BLK = false>
__device__ __forceinline__ bool cube_valid(const unsigned char *__restrict__ outside, const tw_voxel_post_params &P, const int *c, const CubeRange &R = CubeRange()) {
	if (c[0] < 0 || c[1] < 0 || c[2] < 0 || (unsigned)c[0] + 1 >= P.nx || (unsigned)c[1] + 1 >= P.ny || (unsigned)c[2] + 1 >= P.nz) return false;
	if (BLK && ((unsigned)c[0] < R.x0 || (unsigned)c[0] >= R.x1 || (unsigned)c[1] < R.y0 || (unsigned)c[1] >= R.y1)) return false;
	if (!P.skip_under_mesh) return true;
	for (unsigned k = 0; k < 4; ++k) {
		size_t const ix = (unsigned)c[2] + ((size_t)(c[0] + (k & 1)) + (size_t)(c[1] + (k >> 1))*P.nx)*P.nz;
		if (!(__ldg(outside + ix) & TW_VOX_UNDER_MESH)) return true;
	}
	return false;
}

// One cube of the welded mesh: the welded position of each of its crossing edges (vlist), each edge's owner (linear index) and local edge there (own, oj),
// the edges it owns (mask) and the triangles whose welded positions have a nonzero normal (kept, bit k = the k-th triangle of tri_table). Returns the
// number of kept triangles. With BLK the cube is one of block R's, only R's cubes can own an edge, and own / ci are indices within R.
struct MeshCube {float vlist[12][3]; unsigned own[12]; unsigned char oj[12], tri[5][3]; unsigned mask, kept;};
template<bool EMIT, bool BLK = false>
__device__ unsigned cube_mesh(const float *__restrict__ vals, const unsigned char *__restrict__ outside, const tw_voxel_post_params &P, const McTables &T,
	const unsigned char *s_edge, const unsigned char *s_look, unsigned x, unsigned y, unsigned z, unsigned ci, MeshCube &m, const CubeRange &R = CubeRange())
{
	m.mask = 0; m.kept = 0;
	unsigned const nx = P.nx, ny = P.ny, nz = P.nz;
	if (x + 1 >= nx || y + 1 >= ny || z + 1 >= nz) return 0; // last layer of an axis
	unsigned cix = 0;
	bool all_under_mesh = (P.skip_under_mesh != 0);
#pragma unroll
	for (unsigned yhi = 0; yhi < 2; ++yhi) {
#pragma unroll
		for (unsigned xhi = 0; xhi < 2; ++xhi) {
			size_t const ix = z + ((size_t)(x + xhi) + (size_t)(y + yhi)*nx)*nz;
			if (all_under_mesh) {all_under_mesh = ((__ldg(outside + ix) & TW_VOX_UNDER_MESH) != 0);}
#pragma unroll
			for (unsigned zhi = 0; zhi < 2; ++zhi) {if (__ldg(outside + ix + zhi) & 7) {cix |= 1u << ((xhi ^ yhi) + 2*yhi + 4*zhi);}}
		}
	}
	if (all_under_mesh) return 0;
	unsigned const edge_val = __ldg(T.edge_table + cix);
	if (edge_val == 0) return 0;
	for (unsigned i = 0; i < 12; ++i) {
		if (EMIT) {m.own[i] = ci; m.oj[i] = (unsigned char)i;}
		if (!(edge_val & (1u << i))) continue;
		unsigned const e = s_edge[i], a = e & 3;
		unsigned p1, p2; perp(a, p1, p2);
		int const g[3] = {(int)(x + ((e >> 2) & 1)), (int)(y + ((e >> 3) & 1)), (int)(z + ((e >> 4) & 1))};
		int o[3] = {(int)x, (int)y, (int)z};
		unsigned j = i;
		for (unsigned k = 0; k < 4; ++k) { // the edge's cubes in increasing index: (d1, d2) = (1, 1), (1, 0), (0, 1), (0, 0) below its low corner
			unsigned const d1 = (k < 2), d2 = !(k & 1);
			int c[3] = {g[0], g[1], g[2]};
			c[p1] -= (int)d1; c[p2] -= (int)d2;
			if (c[0] == (int)x && c[1] == (int)y && c[2] == (int)z) {m.mask |= 1u << i; break;} // no earlier cube makes triangles: this one owns it
			if (cube_valid<BLK>(outside, P, c, R)) {o[0] = c[0]; o[1] = c[1]; o[2] = c[2]; j = s_look[4*a + 2*d1 + d2]; break;}
		}
		if (EMIT) {
			m.own[i] = (m.mask & (1u << i)) ? ci : BLK ? (((unsigned)o[1] - R.y0)*(R.x1 - R.x0) + (unsigned)o[0] - R.x0)*nz + (unsigned)o[2]
			                                            : (unsigned)o[2] + ((unsigned)o[0] + (unsigned)o[1]*nx)*nz;
			m.oj[i] = (unsigned char)j;
		}
		float v2[2], pts[2][3];
#pragma unroll
		for (unsigned d = 0; d < 2; ++d) { // the owner's interpolation: its corners, in its order
			unsigned const ev = __ldg(T.edge_to_vals + 2*j + d), yhi = (ev & 2) >> 1, xhi = yhi ^ (ev & 1), zhi = (ev >> 2) & 1;
			unsigned const cx = (unsigned)o[0] + xhi, cy = (unsigned)o[1] + yhi, cz = (unsigned)o[2] + zhi;
			size_t const ix = cz + ((size_t)cx + (size_t)cy*nx)*nz;
			v2[d] = ((__ldg(outside + ix) & 7) == TW_VOX_ON_EDGE) ? P.isolevel : __ldg(vals + ix);
			pts[d][0] = (float)cx*P.vsz[0] + P.lo_pos[0]; pts[d][1] = (float)cy*P.vsz[1] + P.lo_pos[1]; pts[d][2] = (float)cz*P.vsz[2] + P.lo_pos[2];
		}
		interpolate_pt(P.isolevel, pts[0], pts[1], v2[0], v2[1], m.vlist[i]);
	}
	const int *t = T.tri_table + 16*cix;
	unsigned count = 0;
	for (unsigned i = 0, k = 0; i < 15; i += 3, ++k) {
		int const t0 = __ldg(t + i);
		if (t0 < 0) break;
		int const t1 = __ldg(t + i + 1), t2 = __ldg(t + i + 2);
		const float *p0 = m.vlist[t0], *p1 = m.vlist[t1], *p2 = m.vlist[t2];
		float const a0 = p1[0] - p0[0], a1 = p1[1] - p0[1], a2 = p1[2] - p0[2], b0 = p2[0] - p1[0], b1 = p2[1] - p1[1], b2 = p2[2] - p1[2]; // get_normal
		float const cx = a1*b2 - a2*b1, cy = a2*b0 - a0*b2, cz = a0*b1 - a1*b0;
		if (cx == 0.0f && cy == 0.0f && cz == 0.0f) continue; // degenerate in the welded positions: the reference tests the cached points
		if (EMIT) {m.tri[count][0] = (unsigned char)t0; m.tri[count][1] = (unsigned char)t1; m.tri[count][2] = (unsigned char)t2;}
		++count;
	}
	return count;
}

} // namespace
