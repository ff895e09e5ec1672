// tw_voxel_post.cu - voxel post-processing on the device (SURVEY.md 8f row N3): the steps of voxel_model::build after the density fill
// (src/voxels.cpp:1496-1530): determine_voxels_outside (:571-604), remove_unconnected_outside / remove_interior_holes (:606-610, :729-868) and the marching
// cubes of add_triangles_for_voxel (:485-566) for the whole grid in create_block order (:1077-1108). Layout: index z + (x + y*nx)*nz (src/voxels.h:141-144).
//   outside_kernel      one thread per voxel, streaming (4 B read + 1 B written per voxel)
//   flood fills         breadth-first frontier expansion: a voxel is claimed by whoever first sets its ANCHORED bit (atomicOr on the 32-bit word that holds
//                       its flag byte), so it enters the next frontier exactly once; the SET of reached voxels is what the reference's depth-first stack
//                       reaches, the visiting order is irrelevant. One cooperative launch per fill runs every generation with one grid barrier each and
//                       ends on the device when a frontier is empty (flood_fill_kernel): the host never reads a count, and no kernel is launched per generation.
//   mc_kernel<EMIT>     1024 consecutive voxels per block = 1024 cubes in the reference's (y, x, z) order; every thread builds its cube's <= 5 triangles,
//                       a block scan of the per-cube counts plus the scanned block totals give every triangle its slot, i.e. the output is in the
//                       reference's emission order without atomics (pass 1: counts only; pass 2: write).
// All fp32 arithmetic is the reference's (separate multiply and add: the TU is compiled with -fmad=false), std::min/max argument order kept.
#include "tw_internal.h"
#include <vector>

namespace {

constexpr float VOX_TOLERANCE = 1.0E-12f; // TOLERANCE, src/3DWorld.h:50

__device__ __forceinline__ float smin(float a, float b) {return (b < a) ? b : a;} // std::min
__device__ __forceinline__ float smax(float a, float b) {return (a < b) ? b : a;} // std::max

__global__ void outside_kernel(const float *__restrict__ vals, tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, unsigned char *__restrict__ outside, size_t n) {
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		unsigned const z = (unsigned)(i % P.nz);
		size_t const xy = i / P.nz;
		unsigned const x = (unsigned)(xy % P.nx), y = (unsigned)(xy / P.nx);
		bool const on_edge = (P.make_closed_surface && ((x == 0 || x == P.nx-1) || (y == 0 || y == P.ny-1) || (z == 0 || z == P.nz-1)));
		float const val = __ldg(vals + i);
		unsigned char ival = on_edge ? (unsigned char)TW_VOX_ON_EDGE : (unsigned char)((val == P.isolevel) ? 1 : (((val < P.isolevel) != (P.invert != 0)) ? 1 : 0)); // val_is_outside
		if (zix_xy && z < __ldg(zix_xy + (size_t)y*P.nx + x)) {ival |= TW_VOX_UNDER_MESH;}
		outside[i] = ival;
	}
}

// ---- flood fill ----
__device__ __forceinline__ bool claim(unsigned char *outside, size_t ix, unsigned char fill_val, unsigned char bit) { // outside[ix] == fill_val -> |= bit, true for exactly one caller
	if (*(volatile unsigned char *)(outside + ix) != fill_val) return false;
	unsigned *word = (unsigned *)(outside + (ix & ~(size_t)3));
	unsigned const shift = (unsigned)(ix & 3)*8u;
	unsigned const old = atomicOr(word, (unsigned)bit << shift);
	return (((old >> shift) & 0xffu) == fill_val);
}
// seeds of remove_unconnected_outside_range (src/voxels.cpp:768-805); mode 0: voxels under the mesh (outside == UNDER_MESH), 1: scene-edge columns (outside != 1),
// 2: top plane of remove_interior_holes (outside != 0, :835-842)
__global__ void seed_kernel(unsigned char *outside, tw_voxel_post_params P, int mode, unsigned *frontier, unsigned *count, size_t n) {
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		unsigned char const o = outside[i];
		bool seed = false;
		if (mode == 0) {seed = (o == TW_VOX_UNDER_MESH);}
		else {
			unsigned const z = (unsigned)(i % P.nz);
			size_t const xy = i / P.nz;
			unsigned const x = (unsigned)(xy % P.nx), y = (unsigned)(xy / P.nx);
			if (mode == 1) {seed = ((x == 0 || x + 1 == P.nx || y == 0 || y + 1 == P.ny) && o != 1 && !(o & TW_VOX_ANCHORED));}
			else           {seed = (z == P.nz - 1 && o != 0);}
		}
		if (seed) { // flag bytes of one word may be seeded by different threads: set the bit atomically
			unsigned *word = (unsigned *)(outside + (i & ~(size_t)3));
			atomicOr(word, (unsigned)TW_VOX_ANCHORED << ((unsigned)(i & 3)*8u));
			frontier[atomicAdd(count, 1u)] = (unsigned)i;
		}
	}
}
__global__ void seed_centre_kernel(unsigned char *outside, tw_voxel_post_params P, unsigned *frontier, unsigned *count) { // :769-776
	size_t const ix = (P.nz/2) + ((size_t)(P.nx/2) + (size_t)(P.ny/2)*P.nx)*P.nz;
	outside[ix] |= TW_VOX_ANCHORED;
	frontier[atomicAdd(count, 1u)] = (unsigned)ix;
}
// The flood's grid barrier. It is only correct in a cooperative launch (cudaLaunchCooperativeKernel guarantees that every block is resident; in a plain
// launch a waiting block could hold the SM a missing block needs). It is cooperative_groups' grid.sync() protocol - arrive with one atomic per block, the
// last block to arrive releases the others by advancing a generation word - except that the waiting blocks poll with __nanosleep between reads: with
// grid.sync()'s tight polling loop, 528 blocks hammering one L2 line made the wide 512^3 fills about 4x slower than one launch per generation. On one H100
// 80GB HBM3 at 400 W (tools/bench_voxel_build.py --remove-only, 512^3 sine / GLM / 20000-generation column): grid.sync() 135 / 138 / 84 ms, 64 ns sleeps
// 36.8 / 33.0 / 90.5 ms, 128 ns 35.6 / 32.4 / 91.8 ms, 256 ns 35.5 / 32.4 / 91.8 ms, the former launch per generation 35.3 / 32.5 / 157 ms.
// bar[0]: arrivals, bar[1]: generation; both 0 before the launch.
// tw_cancel: only the last block to arrive acts on the job words, before it releases the others: in a cancelled job it zeroes the next frontier's count
// (*next, final once every block has arrived), which every thread reads after the barrier - so all blocks leave in the same generation. (Every block
// loads the words beside its arrival, so the load adds no latency to the barrier; the others drop the value.)
#ifndef TW_FLOOD_SLEEP_NS
#define TW_FLOOD_SLEEP_NS 128
#endif
__device__ __forceinline__ void grid_barrier(unsigned *bar, unsigned *next, twi_job_words *jw) {
	__syncthreads();
	if (threadIdx.x == 0) {
		volatile unsigned *gen = bar + 1;
		unsigned const g0 = *gen; // cannot advance before this block arrives
		__threadfence();          // this block's frontier, counts and flags before the arrival
		unsigned long long const words = twi_job_words_load(jw);
		if (atomicAdd(bar, 1u) == gridDim.x - 1) {
			bar[0] = 0;
			if (twi_job_words_hit(words) && *(volatile unsigned *)next != 0u) {*next = 0u; twi_mark_stopped(jw);}
			__threadfence(); atomicAdd(bar + 1, 1u);
		}
		else {while (*gen == g0) {__nanosleep(TW_FLOOD_SLEEP_NS);}}
		__threadfence();
	}
	__syncthreads();
}
// flood_fill_range + FLOOD_FILL_INNER (src/voxels.cpp:729-757): the whole fill in one cooperative launch. The seeds are in f0, their count in cnt[0], and
// cnt[1], cnt[4], cnt[5] are 0. Generation g expands frontier f[g & 1] of cnt[g % 3] voxels into f[(g + 1) & 1], counting in cnt[(g + 1) % 3], while thread 0
// zeroes cnt[(g + 2) % 3] for the next generation: nothing writes the count a generation reads, so after the one grid barrier per generation (cnt[4..5]) every
// thread reads the same next count and all leave together when it is 0. cnt[3] = the seed count (the pass-1 finish reads it). Counts and frontiers written
// by other blocks are read past L1 (__ldcg); flag bytes are read volatile by claim().
constexpr int FLOOD_THREADS = 256;
__global__ void __launch_bounds__(FLOOD_THREADS)
flood_fill_kernel(unsigned char *outside, unsigned nx, unsigned ny, unsigned nz, unsigned *f0, unsigned *f1, unsigned *cnt, unsigned char fill_val, unsigned char bit,
                  twi_job_words *jw)
{
	unsigned const nxnz = nx*nz, tid = blockIdx.x*blockDim.x + threadIdx.x, stride = gridDim.x*blockDim.x;
	if (tid == 0) {cnt[3] = __ldcg(cnt);}
	for (unsigned g = 0;; ++g) {
		unsigned const n = __ldcg(cnt + g%3);
		if (n == 0) return;
		if (tid == 0) {cnt[(g + 2)%3] = 0;}
		const unsigned *fin = (g & 1) ? f1 : f0;
		unsigned *fout = (g & 1) ? f0 : f1, *n_out = cnt + (g + 1)%3;
		for (unsigned i = tid; i < n; i += stride) {
			unsigned const cur = __ldcg(fin + i);
			unsigned const y = cur/nxnz, cur_xz = cur - y*nxnz, x = cur_xz/nz, z = cur_xz - x*nz;
#define TW_FF(pos, max_range, step) \
			if (pos >= 1)            {unsigned const ix = cur - step; if (claim(outside, ix, fill_val, bit)) {fout[atomicAdd(n_out, 1u)] = ix;}} \
			if (pos + 1 < max_range) {unsigned const ix = cur + step; if (claim(outside, ix, fill_val, bit)) {fout[atomicAdd(n_out, 1u)] = ix;}}
			TW_FF(x, nx, nz)
			TW_FF(y, ny, nxnz)
			TW_FF(z, nz, 1u)
#undef TW_FF
		}
		grid_barrier(cnt + 4, n_out, jw);
	}
}
// :808-826 (pass 0) and :847-857 (pass 1); gate (optional): does nothing when *gate == 0 (remove_interior_holes bails out without a seed, :844)
__global__ void flood_finish_kernel(float *__restrict__ vals, unsigned char *__restrict__ outside, float isolevel, int invert, int pass, unsigned long long *changed, size_t n,
	const unsigned *gate)
{
	if (gate && *gate == 0) return;
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	unsigned long long c = 0;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		unsigned char const o = outside[i];
		if (pass == 0) {
			if (o > 1) {outside[i] = o & (unsigned char)~TW_VOX_ANCHORED;}
			else if (o != 1) {outside[i] = 1; vals[i] = isolevel - (invert ? -VOX_TOLERANCE : VOX_TOLERANCE); ++c;} // make_voxel_outside, :861-864
		}
		else {
			if (o & TW_VOX_ANCHORED) {outside[i] = o & (unsigned char)~TW_VOX_ANCHORED;}
			else if (o == 1) {outside[i] = 0; vals[i] = isolevel + (invert ? -VOX_TOLERANCE : VOX_TOLERANCE); ++c;} // make_voxel_inside, :865-868
		}
	}
	for (int o = 16; o > 0; o >>= 1) {c += __shfl_xor_sync(0xffffffffu, c, o);}
	if ((threadIdx.x & 31) == 0 && c) {atomicAdd(changed, c);}
}

// ---- marching cubes ----
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

// add_triangles_for_voxel(x, y, z) at lod 0 (src/voxels.cpp:495-566): returns the number of valid triangles, written to tri[k][9] when EMIT
template<bool EMIT>
__device__ unsigned cube_triangles(const float *__restrict__ vals, const unsigned char *__restrict__ outside, const tw_voxel_post_params &P, const McTables &T,
	unsigned x, unsigned y, unsigned z, float (*tri)[9])
{
	unsigned const nx = P.nx, ny = P.ny, nz = P.nz;
	unsigned const x2 = min(x + 1, nx - 1), y2 = min(y + 1, ny - 1), z2 = min(z + 1, nz - 1);
	if (x2 <= x || y2 <= y || z2 <= z) return 0; // invalid (empty) range
	unsigned const xv[2] = {x, x2}, yv[2] = {y, y2}, zv[2] = {z, z2};
	unsigned cix = 0;
	bool all_under_mesh = (P.skip_under_mesh != 0);
#pragma unroll
	for (unsigned yhi = 0; yhi < 2; ++yhi) {
#pragma unroll
		for (unsigned xhi = 0; xhi < 2; ++xhi) {
			size_t const ix = z + ((size_t)xv[xhi] + (size_t)yv[yhi]*nx)*nz;
			if (all_under_mesh) {all_under_mesh = ((__ldg(outside + ix) & TW_VOX_UNDER_MESH) != 0);}
#pragma unroll
			for (unsigned zhi = 0; zhi < 2; ++zhi) {if (__ldg(outside + ix + zv[zhi] - z) & 7) {cix |= 1u << ((xhi ^ yhi) + 2*yhi + 4*zhi);}} // outside or on edge
		}
	}
	if (all_under_mesh) return 0;
	unsigned const edge_val = __ldg(T.edge_table + cix);
	if (edge_val == 0) return 0; // no polygons
	const int *t = T.tri_table + 16*cix;
	float const cube[3][2] = {{(float)x*P.vsz[0] + P.lo_pos[0], (float)x2*P.vsz[0] + P.lo_pos[0]}, {(float)y*P.vsz[1] + P.lo_pos[1], (float)y2*P.vsz[1] + P.lo_pos[1]},
	                          {(float)z*P.vsz[2] + P.lo_pos[2], (float)z2*P.vsz[2] + P.lo_pos[2]}}; // get_xv / get_yv / get_zv
	float vlist[12][3];
	for (unsigned i = 0; i < 12; ++i) {
		if (!(edge_val & (1u << i))) continue;
		float v2[2], pts[2][3];
#pragma unroll
		for (unsigned d = 0; d < 2; ++d) {
			unsigned const e = __ldg(T.edge_to_vals + 2*i + d), yhi = (e & 2) >> 1, xhi = yhi ^ (e & 1), zhi = e >> 2;
			size_t const ix = zv[zhi] + ((size_t)xv[xhi] + (size_t)yv[yhi]*nx)*nz;
			v2[d] = ((__ldg(outside + ix) & 7) == TW_VOX_ON_EDGE) ? P.isolevel : __ldg(vals + ix);
			pts[d][0] = cube[0][xhi]; pts[d][1] = cube[1][yhi]; pts[d][2] = cube[2][zhi];
		}
		interpolate_pt(P.isolevel, pts[0], pts[1], v2[0], v2[1], vlist[i]);
	}
	unsigned count = 0;
	for (unsigned i = 0; i < 15; i += 3) {
		int const t0 = __ldg(t + i);
		if (t0 < 0) break;
		const float *p0 = vlist[t0], *p1 = vlist[__ldg(t + i + 1)], *p2 = vlist[__ldg(t + i + 2)];
		float const a0 = p1[0] - p0[0], a1 = p1[1] - p0[1], a2 = p1[2] - p0[2], b0 = p2[0] - p1[0], b1 = p2[1] - p1[1], b2 = p2[2] - p1[2]; // get_normal: cross(v2 - v1, v3 - v2)
		float const cx = a1*b2 - a2*b1, cy = a2*b0 - a0*b2, cz = a0*b1 - a1*b0;
		if (cx == 0.0f && cy == 0.0f && cz == 0.0f) continue; // normal == zero_vector: invalid triangle (:550)
		if (EMIT) {
#pragma unroll
			for (int k = 0; k < 3; ++k) {tri[count][k] = p0[k]; tri[count][3 + k] = p1[k]; tri[count][6 + k] = p2[k];}
		}
		++count;
	}
	return count;
}

template<bool EMIT>
__global__ void __launch_bounds__(MC_BLOCK)
mc_kernel(const float *__restrict__ vals, const unsigned char *__restrict__ outside, tw_voxel_post_params P, McTables T, size_t n, unsigned *__restrict__ block_sums,
	const unsigned long long *__restrict__ block_offsets, float *__restrict__ tris, unsigned long long capacity)
{
	__shared__ unsigned warp_sums[MC_BLOCK/32];
	size_t const i = (size_t)blockIdx.x*MC_BLOCK + threadIdx.x;
	float tri[5][9];
	unsigned cnt = 0;
	if (i < n) {
		unsigned const z = (unsigned)(i % P.nz);
		size_t const xy = i / P.nz;
		cnt = cube_triangles<EMIT>(vals, outside, P, T, (unsigned)(xy % P.nx), (unsigned)(xy / P.nx), z, tri);
	}
	// exclusive scan of cnt over the block (cube order == thread order)
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += v;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned w = warp_sums[lane], wi = w;
		for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
		warp_sums[lane] = wi - w; // exclusive
		if (!EMIT && lane == 31) {block_sums[blockIdx.x] = wi;}
	}
	__syncthreads();
	if (EMIT && cnt) {
		unsigned long long const base = block_offsets[blockIdx.x] + warp_sums[warp] + (incl - cnt);
		for (unsigned k = 0; k < cnt; ++k) {
			unsigned long long const slot = base + k;
			if (slot < capacity) {float *o = tris + 9*slot; for (int c = 0; c < 9; ++c) {o[c] = tri[k][c];}}
		}
	}
}
// exclusive scan of the block totals into 64-bit offsets (one block; nblocks is ~1e5 for a 512^3 grid); total[0] = grand total
__global__ void __launch_bounds__(1024)
scan_blocks_kernel(const unsigned *__restrict__ sums, unsigned nblocks, unsigned long long *__restrict__ offsets, unsigned long long *__restrict__ total) {
	__shared__ unsigned long long warp_sums[32];
	__shared__ unsigned long long carry;
	if (threadIdx.x == 0) {carry = 0;}
	__syncthreads();
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (unsigned base = 0; base < nblocks; base += 1024) {
		unsigned const i = base + threadIdx.x;
		unsigned long long const v = (i < nblocks) ? sums[i] : 0ull;
		unsigned long long incl = v;
		for (int o = 1; o < 32; o <<= 1) {unsigned long long const u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += u;}
		if (lane == 31) {warp_sums[warp] = incl;}
		__syncthreads();
		if (warp == 0) {
			unsigned long long w = warp_sums[lane], wi = w;
			for (int o = 1; o < 32; o <<= 1) {unsigned long long const u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += u;}
			warp_sums[lane] = wi - w;
		}
		__syncthreads();
		unsigned long long const excl = carry + warp_sums[warp] + (incl - v);
		if (i < nblocks) {offsets[i] = excl;}
		__syncthreads();
		if (threadIdx.x == 1023) {carry = excl + v;}
		__syncthreads();
	}
	if (threadIdx.x == 0) {*total = carry;}
}

// ---- the welded mesh (create_block's shared vertex cache, src/voxels.cpp:1077-1108 + :495-566) ----
// A grid edge's vertex belongs to its OWNER, the first cube containing it in (y, x, z) order - i.e. the lowest linear index - that is not skipped; the
// owner's interpolate_pt along its local edge, in its edge_to_vals corner order, is the position every cube on the edge uses. The eager cache of the
// reference creates vertices in owner order and, per owner, in local edge order, so a vertex's index is the owned-vertex prefix of its owner plus its rank
// among the owner's owned edges. mesh_kernel<false> counts per cube and stores word[c] = (block-exclusive owned-vertex prefix << 16) | owned-edge mask;
// mesh_kernel<true> reads the words of the owners it references. Per block <= 12*1024 vertices and 5*1024 triangles: both prefixes fit 16 bits.

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

template<bool EMIT>
__global__ void __launch_bounds__(MC_BLOCK)
mesh_kernel(const float *__restrict__ vals, const unsigned char *__restrict__ outside, tw_voxel_post_params P, McTables T, size_t n, unsigned *__restrict__ words,
	unsigned *__restrict__ vsums, unsigned *__restrict__ tsums, const unsigned long long *__restrict__ voff, const unsigned long long *__restrict__ toff,
	float *__restrict__ verts, unsigned long long vcap, uint32_t *__restrict__ indices, unsigned long long tcap)
{
	__shared__ unsigned warp_sums[MC_BLOCK/32];
	__shared__ unsigned char s_edge[12], s_look[12];
	mesh_edge_tables(T.edge_to_vals, s_edge, s_look);
	size_t const i = (size_t)blockIdx.x*MC_BLOCK + threadIdx.x;
	MeshCube m;
	m.mask = 0;
	unsigned cnt = 0; // owned vertices << 16 | kept triangles
	if (i < n) {
		unsigned const z = (unsigned)(i % P.nz);
		size_t const xy = i / P.nz;
		unsigned const nt = cube_mesh<EMIT>(vals, outside, P, T, s_edge, s_look, (unsigned)(xy % P.nx), (unsigned)(xy / P.nx), z, (unsigned)i, m);
		cnt = ((unsigned)__popc(m.mask) << 16) | nt;
	}
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += v;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned w = warp_sums[lane], wi = w;
		for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
		warp_sums[lane] = wi - w;
		if (!EMIT && lane == 31) {vsums[blockIdx.x] = wi >> 16; tsums[blockIdx.x] = wi & 0xffffu;}
	}
	__syncthreads();
	unsigned const excl = warp_sums[warp] + (incl - cnt);
	if (!EMIT) {
		if (i < n) {words[i] = (excl & 0xffff0000u) | m.mask;}
		return;
	}
	if (i >= n) return;
	unsigned long long const vbase = voff[blockIdx.x] + (excl >> 16);
	for (unsigned mk = m.mask; mk; mk &= mk - 1) {
		unsigned const e = __ffs(mk) - 1;
		unsigned long long const slot = vbase + __popc(m.mask & ((1u << e) - 1));
		if (slot < vcap) {float *o = verts + 3*slot; o[0] = m.vlist[e][0]; o[1] = m.vlist[e][1]; o[2] = m.vlist[e][2];}
	}
	unsigned long long const tbase = toff[blockIdx.x] + (excl & 0xffffu);
	for (unsigned k = 0; k < (cnt & 0xffffu); ++k) {
		unsigned long long const slot = tbase + k;
		if (slot >= tcap) break;
		for (unsigned v = 0; v < 3; ++v) {
			unsigned const e = m.tri[k][v], owner = m.own[e], w = __ldg(words + owner);
			indices[3*slot + v] = (uint32_t)(voff[owner / MC_BLOCK] + (w >> 16) + __popc(w & 0xfffu & ((1u << m.oj[e]) - 1)));
		}
	}
}

// both passes of the welded mesh after the flags are final: count -> two block scans -> emit (when a capacity is > 0). Scratch: words n, vsums / tsums
// nblocks, voff / toff nblocks, totals[2] = vertices, triangles.
struct MeshScratch {unsigned *words, *vsums, *tsums; unsigned long long *voff, *toff, *totals;};
int enqueue_mesh(tw_ctx *ctx, const float *d_v, const unsigned char *d_o, const tw_voxel_post_params &P, const McTables &T, const MeshScratch &S, float *verts,
                 unsigned long long vcap, uint32_t *indices, unsigned long long tcap)
{
	size_t const n = (size_t)P.nx*P.ny*P.nz;
	unsigned const nblocks = (unsigned)((n + MC_BLOCK - 1)/MC_BLOCK);
	mesh_kernel<false><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, P, T, n, S.words, S.vsums, S.tsums, nullptr, nullptr, nullptr, 0, nullptr, 0);
	TW_LAUNCH_CHECK(ctx);
	scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(S.vsums, nblocks, S.voff, S.totals);
	TW_LAUNCH_CHECK(ctx);
	scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(S.tsums, nblocks, S.toff, S.totals + 1);
	TW_LAUNCH_CHECK(ctx);
	if (vcap || tcap) {
		mesh_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, P, T, n, S.words, nullptr, nullptr, S.voff, S.toff, verts, vcap, indices, tcap);
		TW_LAUNCH_CHECK(ctx);
	}
	return TW_OK;
}
MeshScratch mesh_scratch(twi_carve &c, size_t n, unsigned nblocks) {
	MeshScratch S;
	S.words = c.take<unsigned>(n);
	S.vsums = c.take<unsigned>(nblocks);
	S.tsums = c.take<unsigned>(nblocks);
	S.voff = c.take<unsigned long long>(nblocks);
	S.toff = c.take<unsigned long long>(nblocks);
	S.totals = c.take<unsigned long long>(2);
	return S;
}

int validate(tw_ctx *ctx, const tw_voxel_post_params *vp) {
	if (!vp || vp->nx == 0 || vp->ny == 0 || vp->nz == 0) return tw_set_error(ctx, TW_ERR_ARG, "empty voxel grid");
	if ((unsigned long long)vp->nx*vp->ny*vp->nz >= 0xffffffffull) return tw_set_error(ctx, TW_ERR_ARG, "voxel grids are indexed with 32 bits, as in the reference (src/voxels.h:141)");
	return TW_OK;
}
unsigned stream_grid(const tw_ctx *ctx, size_t n) {size_t const b = (n + 255)/256; return (unsigned)(b < ctx->num_sms*16u ? (b ? b : 1) : ctx->num_sms*16u);}

// the flood's grid: 4 blocks per SM, fewer if fewer fit at once (a cooperative launch needs every block resident)
int flood_blocks(tw_ctx *ctx, unsigned *blocks) {
	int coop = 0, per_sm = 0;
	TW_CUDA(ctx, cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device));
	if (!coop) return tw_set_error(ctx, TW_ERR_CUDA, "device %d has no cooperative launch (the voxel flood fills run as one)", ctx->device);
	TW_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, flood_fill_kernel, FLOOD_THREADS, 0));
	unsigned const cap = (unsigned)per_sm*ctx->num_sms;
	if (cap == 0) return tw_set_error(ctx, TW_ERR_CUDA, "flood_fill_kernel: no block fits on an SM");
	*blocks = (ctx->num_sms*4 < cap) ? ctx->num_sms*4 : cap;
	return TW_OK;
}

int launch_flood(tw_ctx *ctx, unsigned blocks, unsigned char *d_o, const tw_voxel_post_params *vp, unsigned *f0, unsigned *f1, unsigned *cnt, unsigned char fill_val) {
	unsigned nx = vp->nx, ny = vp->ny, nz = vp->nz;
	unsigned char bit = TW_VOX_ANCHORED;
	twi_job_words *jw = ctx->d_job_words;
	void *args[] = {&d_o, &nx, &ny, &nz, &f0, &f1, &cnt, &fill_val, &bit, &jw};
	TW_CUDA(ctx, cudaLaunchCooperativeKernel((const void *)flood_fill_kernel, dim3(blocks), dim3(FLOOD_THREADS), args, 0, ctx->stream));
	ctx->launches++;
	return TW_OK;
}

// remove_unconnected_outside_range(keep_at_edge, 0, 0, nx, ny) (+ remove_interior_holes) on ctx->stream for remove_unconnected > 0: d_o 4-byte aligned with
// room for the word of its last byte; f0, f1: n + 16 entries each; cnt: 4 counters; d_changed accumulates the flipped voxels (the caller zeroes it)
int enqueue_remove_unconnected(tw_ctx *ctx, unsigned blocks, float *d_v, unsigned char *d_o, const tw_voxel_post_params *vp, unsigned *f0, unsigned *f1, unsigned *cnt,
                               unsigned long long *d_changed)
{
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	// anchors, fill of the inside voxels, verdict
	TW_CUDA(ctx, cudaMemsetAsync(cnt, 0, 8*sizeof(unsigned), ctx->stream));
	if (vp->centre_seed) {seed_centre_kernel<<<1, 1, 0, ctx->stream>>>(d_o, *vp, f0, cnt);}
	else {seed_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_o, *vp, 0, f0, cnt, n);}
	TW_LAUNCH_CHECK(ctx);
	if (vp->keep_at_edge) {seed_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_o, *vp, 1, f0, cnt, n); TW_LAUNCH_CHECK(ctx);}
	int rc = launch_flood(ctx, blocks, d_o, vp, f0, f1, cnt, 0); if (rc) return rc;
	flood_finish_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_v, d_o, vp->isolevel, vp->invert, 0, d_changed, n, nullptr);
	TW_LAUNCH_CHECK(ctx);
	if (vp->remove_unconnected > 2) { // remove_interior_holes: seeds on the top plane; without one the finish does nothing
		TW_CUDA(ctx, cudaMemsetAsync(cnt, 0, 8*sizeof(unsigned), ctx->stream));
		seed_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_o, *vp, 2, f0, cnt, n);
		TW_LAUNCH_CHECK(ctx);
		rc = launch_flood(ctx, blocks, d_o, vp, f0, f1, cnt, 1); if (rc) return rc;
		flood_finish_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_v, d_o, vp->isolevel, vp->invert, 1, d_changed, n, cnt + 3);
		TW_LAUNCH_CHECK(ctx);
	}
	return TW_OK;
}

} // namespace

extern "C" int tw_voxel_outside(tw_ctx *ctx, const float *vals, const tw_voxel_post_params *vp, const uint32_t *zix_xy, uint8_t *outside) {
	if (!ctx || !vals || !outside) return TW_ERR_ARG;
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate(ctx, vp); if (rc) return rc;
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz, nxy = (size_t)vp->nx*vp->ny;
	bool const dev_v = tw_is_device_ptr(vals), dev_o = tw_is_device_ptr(outside), dev_z = (zix_xy && tw_is_device_ptr(zix_xy));
	float *s_v = nullptr; uint8_t *d_o = outside; unsigned *s_z = nullptr;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		if (!dev_v) {s_v = c.take<float>(n);} if (!dev_o) {d_o = c.take<uint8_t>(n);} if (zix_xy && !dev_z) {s_z = c.take<unsigned>(nxy);}
	}); if (rc) return rc;
	const float *d_v = dev_v ? vals : s_v; const unsigned *d_z = s_z ? s_z : zix_xy;
	if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(s_v, vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
	if (s_z) {TW_CUDA(ctx, cudaMemcpyAsync(s_z, zix_xy, nxy*sizeof(unsigned), cudaMemcpyHostToDevice, ctx->stream));}
	outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_v, *vp, d_z, d_o, n);
	TW_LAUNCH_CHECK(ctx);
	if (!dev_o) {TW_CUDA(ctx, cudaMemcpyAsync(outside, d_o, n, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

extern "C" int tw_voxel_remove_unconnected(tw_ctx *ctx, float *vals, uint8_t *outside, const tw_voxel_post_params *vp, uint64_t *changed) {
	if (!ctx || !vals || !outside) return TW_ERR_ARG;
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate(ctx, vp); if (rc) return rc;
	if (changed) *changed = 0;
	if (vp->remove_unconnected <= 0) return TW_OK;
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	bool const dev_v = tw_is_device_ptr(vals), dev_o = tw_is_device_ptr(outside);
	if (dev_o && ((size_t)outside & 3)) return tw_set_error(ctx, TW_ERR_ARG, "outside must be 4-byte aligned (flag bytes are claimed with 32-bit atomics)");
	// the 32-bit word that holds the last flag byte reaches up to 3 bytes past a buffer of n % 4 != 0 bytes: such a device buffer is staged like a host one
	bool const stage_o = !dev_o || (n & 3);
	unsigned blocks = 0;
	rc = flood_blocks(ctx, &blocks); if (rc) return rc;
	float *d_v = vals; unsigned char *d_o = outside; unsigned *f0, *f1, *cnt; unsigned long long *d_changed;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		if (!dev_v) {d_v = c.take<float>(n);} if (stage_o) {d_o = c.take<unsigned char>(n + 4);} f0 = c.take<unsigned>(n + 16); f1 = c.take<unsigned>(n + 16);
		cnt = c.take<unsigned>(8); d_changed = c.take<unsigned long long>(1);
	}); if (rc) return rc;
	if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(d_v, vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
	if (stage_o) {TW_CUDA(ctx, cudaMemcpyAsync(d_o, outside, n, dev_o ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));}
	TW_CUDA(ctx, cudaMemsetAsync(d_changed, 0, sizeof(unsigned long long), ctx->stream));
	rc = enqueue_remove_unconnected(ctx, blocks, d_v, d_o, vp, f0, f1, cnt, d_changed);
	if (rc) {cudaStreamSynchronize(ctx->stream); return rc;}
	unsigned long long hc = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&hc, d_changed, sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
	if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(vals, d_v, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	if (stage_o) {TW_CUDA(ctx, cudaMemcpyAsync(outside, d_o, n, dev_o ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (changed) *changed = hc;
	return TW_OK;
}

extern "C" int tw_voxel_triangles(tw_ctx *ctx, const float *vals, const uint8_t *outside, const tw_voxel_post_params *vp, const uint32_t *edge_table256,
                                  const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, float *tris, uint64_t capacity, uint64_t *ntris)
{
	if (!ctx || !vals || !outside || !edge_table256 || !tri_table256x16 || !edge_to_vals12x2 || !ntris || (capacity && !tris)) return TW_ERR_ARG;
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate(ctx, vp); if (rc) return rc;
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	unsigned const nblocks = (unsigned)((n + MC_BLOCK - 1)/MC_BLOCK);
	bool const dev_v = tw_is_device_ptr(vals), dev_o = tw_is_device_ptr(outside), dev_t = (tris && tw_is_device_ptr(tris));
	float *s_v = nullptr; unsigned char *s_o = nullptr, *sp; unsigned *d_sums; unsigned long long *d_offsets, *d_total;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		if (!dev_v) {s_v = c.take<float>(n);} if (!dev_o) {s_o = c.take<unsigned char>(n);} sp = c.take<unsigned char>(1024 + 16384 + 96);
		d_sums = c.take<unsigned>(nblocks); d_offsets = c.take<unsigned long long>(nblocks); d_total = c.take<unsigned long long>(1);
	}); if (rc) return rc;
	const float *d_v = dev_v ? vals : s_v; const unsigned char *d_o = dev_o ? outside : s_o;
	if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(s_v, vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
	if (!dev_o) {TW_CUDA(ctx, cudaMemcpyAsync(s_o, outside, n, cudaMemcpyHostToDevice, ctx->stream));}
	McTables T;
	T.edge_table = (const unsigned *)sp; T.tri_table = (const int *)(sp + 1024); T.edge_to_vals = (const unsigned *)(sp + 1024 + 16384);
	TW_CUDA(ctx, cudaMemcpyAsync(sp, edge_table256, 1024, cudaMemcpyDefault, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(sp + 1024, tri_table256x16, 16384, cudaMemcpyDefault, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(sp + 1024 + 16384, edge_to_vals12x2, 96, cudaMemcpyDefault, ctx->stream));
	mc_kernel<false><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, *vp, T, n, d_sums, nullptr, nullptr, 0);
	TW_LAUNCH_CHECK(ctx);
	scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(d_sums, nblocks, d_offsets, d_total);
	TW_LAUNCH_CHECK(ctx);
	unsigned long long total = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*ntris = total;
	if (capacity == 0 || total == 0) return TW_OK;
	uint64_t const nw = (total < capacity) ? total : capacity;
	float *d_t = tris;
	if (!dev_t) {rc = tw_reserve(ctx, 1, (size_t)nw*9*sizeof(float)); if (rc) return rc; d_t = (float *)ctx->d_scratch[1];}
	mc_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, *vp, T, n, nullptr, d_offsets, d_t, nw);
	TW_LAUNCH_CHECK(ctx);
	if (!dev_t) {TW_CUDA(ctx, cudaMemcpyAsync(tris, d_t, (size_t)nw*9*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

namespace {
int validate_mesh(tw_ctx *ctx, const tw_voxel_post_params *vp, const tw_voxel_mesh *m) {
	if (!m->nverts || !m->ntris) return tw_set_error(ctx, TW_ERR_ARG, "the welded mesh needs nverts and ntris");
	if ((m->vcapacity && !m->verts) || (m->tcapacity && !m->indices)) return tw_set_error(ctx, TW_ERR_ARG, "a mesh capacity without its buffer");
	if (3ull*vp->nx*vp->ny*vp->nz >= 0x100000000ull) return tw_set_error(ctx, TW_ERR_ARG, "the welded mesh's indices are 32-bit: 3*nx*ny*nz must be below 2^32");
	return TW_OK;
}
// device or page-locked host memory as the device addresses it (the emit passes of the job write their outputs directly); nullptr for anything else
void *device_view(void *p) {
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {cudaGetLastError(); return nullptr;}
	if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return p;
	if (a.type == cudaMemoryTypeHost && a.devicePointer) return a.devicePointer;
	return nullptr;
}
} // namespace

extern "C" int tw_voxel_mesh_welded(tw_ctx *ctx, const float *vals, const uint8_t *outside, const tw_voxel_post_params *vp, const uint32_t *edge_table256,
                                    const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, const tw_voxel_mesh *out)
{
	if (!ctx || !vals || !outside || !edge_table256 || !tri_table256x16 || !edge_to_vals12x2 || !out) return TW_ERR_ARG;
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate(ctx, vp); if (rc) return rc;
	tw_voxel_mesh const M = *out;
	rc = validate_mesh(ctx, vp, &M); if (rc) return rc;
	size_t const n = (size_t)vp->nx*vp->ny*vp->nz;
	unsigned const nblocks = (unsigned)((n + MC_BLOCK - 1)/MC_BLOCK);
	bool const dev_v = tw_is_device_ptr(vals), dev_o = tw_is_device_ptr(outside);
	float *s_v = nullptr; unsigned char *s_o = nullptr, *sp; MeshScratch S;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		if (!dev_v) {s_v = c.take<float>(n);} if (!dev_o) {s_o = c.take<unsigned char>(n);} sp = c.take<unsigned char>(1024 + 16384 + 96); S = mesh_scratch(c, n, nblocks);
	}); if (rc) return rc;
	const float *d_v = dev_v ? vals : s_v; const unsigned char *d_o = dev_o ? outside : s_o;
	if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(s_v, vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
	if (!dev_o) {TW_CUDA(ctx, cudaMemcpyAsync(s_o, outside, n, cudaMemcpyHostToDevice, ctx->stream));}
	McTables T;
	T.edge_table = (const unsigned *)sp; T.tri_table = (const int *)(sp + 1024); T.edge_to_vals = (const unsigned *)(sp + 1024 + 16384);
	TW_CUDA(ctx, cudaMemcpyAsync(sp, edge_table256, 1024, cudaMemcpyDefault, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(sp + 1024, tri_table256x16, 16384, cudaMemcpyDefault, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(sp + 1024 + 16384, edge_to_vals12x2, 96, cudaMemcpyDefault, ctx->stream));
	// count and scan first: the emit pass writes at most min(count, capacity) of each, so host outputs are staged at that size
	rc = enqueue_mesh(ctx, d_v, d_o, *vp, T, S, nullptr, 0, nullptr, 0); if (rc) return rc;
	unsigned long long tot[2] = {0, 0};
	TW_CUDA(ctx, cudaMemcpyAsync(tot, S.totals, sizeof(tot), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*M.nverts = tot[0]; *M.ntris = tot[1];
	uint64_t const nv = (tot[0] < M.vcapacity) ? tot[0] : M.vcapacity, nt = (tot[1] < M.tcapacity) ? tot[1] : M.tcapacity;
	if (nv == 0 && nt == 0) return TW_OK;
	bool const dev_vt = nv && tw_is_device_ptr(M.verts), dev_ix = nt && tw_is_device_ptr(M.indices);
	float *d_vt = M.verts; uint32_t *d_ix = M.indices;
	rc = twi_reserve_carve(ctx, 1, [&](twi_carve &c) {
		if (!dev_vt) {d_vt = c.take<float>((size_t)nv*3);} if (!dev_ix) {d_ix = c.take<uint32_t>((size_t)nt*3);}
	}); if (rc) return rc;
	mesh_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, *vp, T, n, S.words, nullptr, nullptr, S.voff, S.toff, d_vt, nv, d_ix, nt);
	TW_LAUNCH_CHECK(ctx);
	if (nv && !dev_vt) {TW_CUDA(ctx, cudaMemcpyAsync(M.verts, d_vt, (size_t)nv*12, cudaMemcpyDeviceToHost, ctx->stream));}
	if (nt && !dev_ix) {TW_CUDA(ctx, cudaMemcpyAsync(M.indices, d_ix, (size_t)nt*12, cudaMemcpyDeviceToHost, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ the whole build as one asynchronous job
// The counts the build stages; nverts, mesh_ntris: the welded mesh (tw_voxel_build_launch_ex)
struct twi_voxel_stage {unsigned long long ntris, changed, nverts, mesh_ntris;};

// fill (optional) -> outside -> remove_unconnected -> marching cubes (count, block scan, emit with the caller's capacity) on ctx->stream; nothing is read back
// before the end: the triangle count and the flipped voxels go to pinned staging that the completing poll unpacks. Every buffer is reserved before anything is
// enqueued, so no re-allocation synchronises in the middle.
//   device slot 0: [counters | field (unless vals is device memory) | padded flags | 2 frontiers (remove_unconnected > 0) | tables | block sums | block
//                  offsets | zix_xy (host input)]
//   pinned:        [twi_voxel_stage | sine coefficients | tables | zix_xy (host input)]
//   with a welded mesh, device slot 0 ends with the mesh's scratch (mesh_scratch)
extern "C" int tw_voxel_build_launch(tw_ctx *ctx, const tw_voxel_build *b) {return tw_voxel_build_launch_ex(ctx, b, nullptr);}

extern "C" int tw_voxel_build_launch_ex(tw_ctx *ctx, const tw_voxel_build *b, const tw_voxel_mesh *mesh) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!b || !b->post) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_build_launch: null argument");
	tw_voxel_post_params const P = *b->post;
	rc = validate(ctx, &P); if (rc) return rc;
	bool const fill = (b->fill != nullptr);
	tw_voxel_params F;
	size_t tab_bytes = 0;
	if (fill) {
		F = *b->fill;
		if (F.nx != P.nx || F.ny != P.ny || F.nz != P.nz) return tw_set_error(ctx, TW_ERR_ARG, "the fill's grid %ux%ux%u differs from post's %ux%ux%u", F.nx, F.ny, F.nz, P.nx, P.ny, P.nz);
		rc = twi_voxel_fill_check(ctx, &F, &tab_bytes); if (rc) return rc;
	}
	else if (!b->vals) return tw_set_error(ctx, TW_ERR_ARG, "vals is the input field when there is no fill");
	int const ntab = (b->edge_table256 != nullptr) + (b->tri_table256x16 != nullptr) + (b->edge_to_vals12x2 != nullptr);
	if (ntab != 0 && ntab != 3) return tw_set_error(ctx, TW_ERR_ARG, "pass all three marching-cubes tables or none");
	bool const wm = (mesh != nullptr);
	if (wm && ntab != 3) return tw_set_error(ctx, TW_ERR_ARG, "the welded mesh needs the three marching-cubes tables");
	bool const mc = (ntab == 3) && (b->ntris || !wm); // the soup: without a mesh, the tables ask for it
	if (mc && !b->ntris) return tw_set_error(ctx, TW_ERR_ARG, "the tables need ntris");
	if (b->capacity && !b->tris) return tw_set_error(ctx, TW_ERR_ARG, "capacity > 0 without tris");
	if (wm && !mc && b->tris) return tw_set_error(ctx, TW_ERR_ARG, "tris without ntris");
	float *d_t = nullptr;
	if (b->tris) { // the emit pass writes tris directly: device memory, or page-locked host memory through its mapping
		d_t = (float *)device_view(b->tris);
		if (!d_t) return tw_set_error(ctx, TW_ERR_ARG, "tris must be device or page-locked host memory (the emit pass writes it directly)");
	}
	tw_voxel_mesh M;
	memset(&M, 0, sizeof(M));
	float *d_mv = nullptr;
	uint32_t *d_mi = nullptr;
	if (wm) {
		M = *mesh;
		rc = validate_mesh(ctx, &P, &M); if (rc) return rc;
		if (M.verts && !(d_mv = (float *)device_view(M.verts))) return tw_set_error(ctx, TW_ERR_ARG, "mesh verts must be device or page-locked host memory");
		if (M.indices && !(d_mi = (uint32_t *)device_view(M.indices))) return tw_set_error(ctx, TW_ERR_ARG, "mesh indices must be device or page-locked host memory");
	}
	bool const rm = (P.remove_unconnected > 0);
	unsigned blocks = 0;
	if (rm) {rc = flood_blocks(ctx, &blocks); if (rc) return rc;}
	size_t const n = (size_t)P.nx*P.ny*P.nz, nxy = (size_t)P.nx*P.ny;
	unsigned const nblocks = (unsigned)((n + MC_BLOCK - 1)/MC_BLOCK);
	bool const dev_v = b->vals && tw_is_device_ptr(b->vals), dev_z = b->zix_xy && tw_is_device_ptr(b->zix_xy);
	size_t const TAB = 1024 + 16384 + 96;
	bool const tabs = (ntab == 3), stage_z = (b->zix_xy && !dev_z);
	unsigned *cnt, *f0 = nullptr, *f1 = nullptr, *d_sums = nullptr, *s_z = nullptr;
	float *d_v = b->vals;
	unsigned char *d_o, *tab = nullptr;
	unsigned long long *d_offsets = nullptr;
	MeshScratch S;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		cnt = c.take<unsigned>(64); // [flood counters | changed at byte 64 | triangle total at byte 128], zeroed together
		if (!dev_v) {d_v = c.take<float>(n);}
		d_o = c.take<unsigned char>(n + 4);
		if (rm) {f0 = c.take<unsigned>(n + 16); f1 = c.take<unsigned>(n + 16);}
		if (tabs) {tab = c.take<unsigned char>(TAB);}
		if (mc) {d_sums = c.take<unsigned>(nblocks); d_offsets = c.take<unsigned long long>(nblocks);}
		if (stage_z) {s_z = c.take<unsigned>(nxy);}
		if (wm) S = mesh_scratch(c, n, nblocks);
	}); if (rc) return rc;
	if (tab_bytes) {rc = tw_reserve(ctx, 1, tab_bytes); if (rc) return rc;}
	twi_voxel_stage *st; float *h_rdata; unsigned char *h_tab = nullptr; unsigned *h_z = nullptr;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		st = c.take<twi_voxel_stage>(1); h_rdata = c.take<float>(TW_N3D_RDATA); if (tabs) {h_tab = c.take<unsigned char>(TAB);} if (stage_z) {h_z = c.take<unsigned>(nxy);}
	}); if (rc) return rc;
	if (fill && F.gen_mode != TW_MGEN_SINE) {rc = twi_ensure_glm3_lut(ctx); if (rc) return rc;}
	unsigned long long *d_changed = (unsigned long long *)(cnt + 16), *d_total = (unsigned long long *)(cnt + 32);
	McTables T = {};
	if (tabs) {T.edge_table = (const unsigned *)tab; T.tri_table = (const int *)(tab + 1024); T.edge_to_vals = (const unsigned *)(tab + 1024 + 16384);}
	const unsigned *d_z = dev_z ? b->zix_xy : s_z;
	twi_job pending;
	pending.cancellable = true;
	pending.complete = [st, ntris = mc ? b->ntris : nullptr, changed = b->changed, nverts = M.nverts, mesh_ntris = M.ntris](tw_ctx *) -> int {
		if (ntris) {*ntris = st->ntris;}
		if (changed) {*changed = st->changed;}
		if (nverts) {*nverts = st->nverts; *mesh_ntris = st->mesh_ntris;}
		return TW_OK;
	};
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(cnt, 0, 256, ctx->stream));
		if (fill) {int const r = twi_voxel_fill(ctx, &F, b->rdata420, d_v, h_rdata); if (r) return r;}
		else if (!dev_v) {TW_CUDA(ctx, cudaMemcpyAsync(d_v, b->vals, n*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
		if (stage_z) {memcpy(h_z, b->zix_xy, nxy*sizeof(unsigned)); TW_CUDA(ctx, cudaMemcpyAsync(s_z, h_z, nxy*sizeof(unsigned), cudaMemcpyHostToDevice, ctx->stream));}
		if (tabs) {
			const void *src[3] = {b->edge_table256, b->tri_table256x16, b->edge_to_vals12x2};
			size_t const off[3] = {0, 1024, 1024 + 16384}, len[3] = {1024, 16384, 96};
			for (int k = 0; k < 3; ++k) {
				// host tables are copied during the launch; device tables are read by the job
				if (tw_is_device_ptr(src[k])) {TW_CUDA(ctx, cudaMemcpyAsync(tab + off[k], src[k], len[k], cudaMemcpyDeviceToDevice, ctx->stream)); continue;}
				memcpy(h_tab + off[k], src[k], len[k]);
				TW_CUDA(ctx, cudaMemcpyAsync(tab + off[k], h_tab + off[k], len[k], cudaMemcpyHostToDevice, ctx->stream));
			}
		}
		outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_v, P, d_z, d_o, n);
		TW_LAUNCH_CHECK(ctx);
		if (rm) {int const r = enqueue_remove_unconnected(ctx, blocks, d_v, d_o, &P, f0, f1, cnt, d_changed); if (r) return r;}
		if (mc) {
			mc_kernel<false><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, P, T, n, d_sums, nullptr, nullptr, 0);
			TW_LAUNCH_CHECK(ctx);
			scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(d_sums, nblocks, d_offsets, d_total);
			TW_LAUNCH_CHECK(ctx);
			if (b->capacity) { // slots at or past the capacity are not written; the device total bounds the rest
				mc_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(d_v, d_o, P, T, n, nullptr, d_offsets, d_t, b->capacity);
				TW_LAUNCH_CHECK(ctx);
			}
		}
		if (wm) {int const r = enqueue_mesh(ctx, d_v, d_o, P, T, S, d_mv, M.vcapacity, d_mi, M.tcapacity); if (r) return r;}
		if (b->vals && !dev_v && (fill || rm)) {TW_CUDA(ctx, cudaMemcpyAsync(b->vals, d_v, n*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));}
		if (b->outside) {TW_CUDA(ctx, cudaMemcpyAsync(b->outside, d_o, n, cudaMemcpyDefault, ctx->stream));}
		TW_CUDA(ctx, cudaMemcpyAsync(&st->ntris, d_total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
		TW_CUDA(ctx, cudaMemcpyAsync(&st->changed, d_changed, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
		if (wm) {TW_CUDA(ctx, cudaMemcpyAsync(&st->nverts, S.totals, 2*sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));}
		return TW_OK;
	});
}

// ------------------------------------------------------------------------------------------------ resident voxel models (tw_voxel_model_*)
// The model's device state (one allocation): raw field and flags, the field and flags after remove_unconnected (post), a working copy of those (work),
// zix_xy, the tables, one mark byte per block, and two block lists {count, blocks...}: every block in order (build) and the marked ones (edit).
// A job meshes the blocks of a list with block_mesh_kernel: launch block k handles chunk k % chunks of the block in list slot k / chunks (chunks = MC_BLOCK-cube
// chunks of the largest block), so the grid is sized for every block listed and the slots past the device-side count exit at once. Count, the two scans of
// mesh_kernel (over slots x chunks, so a block's vertices and triangles are contiguous and in list order), emit, then the table of the listed blocks.
struct tw_voxel_model {
	tw_ctx *ctx = nullptr;
	tw_voxel_post_params P;
	unsigned bx = 1, by = 1, nbx = 0, nblocks = 0, chunks = 0;
	bool built = false, have_zix = false;
	char *mem = nullptr;
	float *raw = nullptr, *post = nullptr, *work = nullptr;
	unsigned char *raw_o = nullptr, *post_o = nullptr, *work_o = nullptr, *mark = nullptr;
	unsigned *zix = nullptr, *all = nullptr, *marked = nullptr;
	void *tables = nullptr;
};

namespace {

struct BlockGrid {unsigned bx, by, nbx, chunks;};

__device__ __forceinline__ CubeRange block_range(const tw_voxel_post_params &P, const BlockGrid &G, unsigned b) {
	CubeRange R;
	R.x0 = (b % G.nbx)*G.bx; R.y0 = (b / G.nbx)*G.by;
	R.x1 = min(R.x0 + G.bx, P.nx - 1); R.y1 = min(R.y0 + G.by, P.ny - 1);
	return R;
}

// the welded mesh of the blocks list[1 .. 1 + list[0]) (see above); words: slots x chunks x MC_BLOCK, the per-cube words of mesh_kernel at the block's local
// cube index; vsums / tsums / voff / toff: one entry per launch block
template<bool EMIT>
__global__ void __launch_bounds__(MC_BLOCK)
block_mesh_kernel(const float *__restrict__ vals, const unsigned char *__restrict__ outside, tw_voxel_post_params P, McTables T, BlockGrid G,
	const unsigned *__restrict__ list, unsigned *__restrict__ words, unsigned *__restrict__ vsums, unsigned *__restrict__ tsums,
	const unsigned long long *__restrict__ voff, const unsigned long long *__restrict__ toff, float *__restrict__ verts, unsigned long long vcap,
	uint32_t *__restrict__ indices, unsigned long long tcap)
{
	unsigned const slot = blockIdx.x / G.chunks;
	if (slot >= __ldg(list)) { // not listed: nothing to count (the scans read zeros), nothing to emit
		if (!EMIT && threadIdx.x == 0) {vsums[blockIdx.x] = 0; tsums[blockIdx.x] = 0;}
		return;
	}
	__shared__ unsigned warp_sums[MC_BLOCK/32];
	__shared__ unsigned char s_edge[12], s_look[12];
	mesh_edge_tables(T.edge_to_vals, s_edge, s_look);
	CubeRange const R = block_range(P, G, __ldg(list + 1 + slot));
	unsigned const w = R.x1 - R.x0, ncubes = (R.y1 - R.y0)*w*P.nz;
	unsigned const l = (blockIdx.x - slot*G.chunks)*MC_BLOCK + threadIdx.x;
	MeshCube m;
	m.mask = 0;
	unsigned cnt = 0;
	if (l < ncubes) {
		unsigned const xy = l / P.nz;
		unsigned const nt = cube_mesh<EMIT, true>(vals, outside, P, T, s_edge, s_look, R.x0 + xy % w, R.y0 + xy / w, l - xy*P.nz, l, m, R);
		cnt = ((unsigned)__popc(m.mask) << 16) | nt;
	}
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += v;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned w = warp_sums[lane], wi = w;
		for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
		warp_sums[lane] = wi - w;
		if (!EMIT && lane == 31) {vsums[blockIdx.x] = wi >> 16; tsums[blockIdx.x] = wi & 0xffffu;}
	}
	__syncthreads();
	unsigned const excl = warp_sums[warp] + (incl - cnt);
	unsigned *const bw = words + (size_t)slot*G.chunks*MC_BLOCK;
	if (!EMIT) {
		if (l < ncubes) {bw[l] = (excl & 0xffff0000u) | m.mask;}
		return;
	}
	if (l >= ncubes) return;
	const unsigned long long *const bvoff = voff + (size_t)slot*G.chunks;
	unsigned long long const vbase = voff[blockIdx.x] + (excl >> 16);
	for (unsigned mk = m.mask; mk; mk &= mk - 1) {
		unsigned const e = __ffs(mk) - 1;
		unsigned long long const s = vbase + __popc(m.mask & ((1u << e) - 1));
		if (s < vcap) {float *o = verts + 3*s; o[0] = m.vlist[e][0]; o[1] = m.vlist[e][1]; o[2] = m.vlist[e][2];}
	}
	unsigned long long const tbase = toff[blockIdx.x] + (excl & 0xffffu);
	for (unsigned k = 0; k < (cnt & 0xffffu); ++k) {
		unsigned long long const s = tbase + k;
		if (s >= tcap) break;
		for (unsigned v = 0; v < 3; ++v) {
			unsigned const e = m.tri[k][v], owner = m.own[e], ow = bw[owner];
			indices[3*s + v] = (uint32_t)(bvoff[owner / MC_BLOCK] - bvoff[0] + (ow >> 16) + __popc(ow & 0xfffu & ((1u << m.oj[e]) - 1)));
		}
	}
}

// the listed blocks' ranges: entry s of slot s < list[0] (nslots: the grid's slots; offsets past the last are the totals)
__global__ void block_table_kernel(const unsigned *__restrict__ list, unsigned chunks, unsigned nslots, const unsigned long long *__restrict__ voff,
	const unsigned long long *__restrict__ toff, const unsigned long long *__restrict__ totals, tw_voxel_block_mesh *__restrict__ table)
{
	unsigned const s = blockIdx.x*blockDim.x + threadIdx.x;
	if (s >= list[0]) return;
	size_t const a = (size_t)s*chunks, b = a + chunks;
	unsigned long long const v1 = (s + 1 < nslots) ? voff[b] : totals[0], t1 = (s + 1 < nslots) ? toff[b] : totals[1];
	tw_voxel_block_mesh e;
	e.block = list[1 + s]; e.pad = 0; e.voff = voff[a]; e.nverts = v1 - voff[a]; e.toff = toff[a]; e.ntris = t1 - toff[a];
	table[s] = e;
}

// list = {count, the marked blocks in ascending order}; clears the marks (one block)
__global__ void __launch_bounds__(1024) list_marked_kernel(unsigned char *__restrict__ mark, unsigned nblocks, unsigned *__restrict__ list) {
	__shared__ unsigned warp_sums[32];
	__shared__ unsigned carry;
	if (threadIdx.x == 0) {carry = 0;}
	__syncthreads();
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (unsigned base = 0; base < nblocks; base += 1024) {
		unsigned const i = base + threadIdx.x;
		bool const f = (i < nblocks) && mark[i];
		if (f) {mark[i] = 0;}
		unsigned const bal = __ballot_sync(0xffffffffu, f);
		if (lane == 0) {warp_sums[warp] = __popc(bal);}
		__syncthreads();
		if (warp == 0) {
			unsigned w = warp_sums[lane], wi = w;
			for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
			warp_sums[lane] = wi - w;
		}
		__syncthreads();
		if (f) {list[1 + carry + warp_sums[warp] + __popc(bal & ((1u << lane) - 1))] = i;}
		__syncthreads();
		if (threadIdx.x == 1023) {carry += warp_sums[31] + __popc(bal);}
		__syncthreads();
	}
	if (threadIdx.x == 0) {list[0] = carry;}
}

// every block whose cubes read voxel column (x, y): the cubes x-1, x and y-1, y that exist
__device__ __forceinline__ void mark_readers(unsigned char *mark, const tw_voxel_post_params &P, const BlockGrid &G, unsigned x, unsigned y) {
	for (unsigned cy = (y ? y - 1 : 0); cy <= y && cy + 1 < P.ny; ++cy) {
		for (unsigned cx = (x ? x - 1 : 0); cx <= x && cx + 1 < P.nx; ++cx) {mark[(cy / G.by)*G.nbx + cx / G.bx] = 1;}
	}
}

// an edit's box and the index of its first value among the packed values; later: a later box overlaps it
struct twi_box {unsigned x, y, z, w, h, d; unsigned long long off; unsigned later, pad;};

// the edit's values into the raw field, with the raw flags of outside_kernel; post (rm == 0, where the post field is the raw one): also compared with the
// model's field and flags, which take the new values, marking the blocks that read a changed voxel
__global__ void box_scatter_kernel(const twi_box *__restrict__ boxes, unsigned nboxes, const float *__restrict__ values, unsigned long long total,
	tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, BlockGrid G, float *__restrict__ raw, unsigned char *__restrict__ raw_o, float *post,
	unsigned char *post_o, unsigned char *mark)
{
	unsigned long long const stride = (unsigned long long)gridDim.x*blockDim.x;
	for (unsigned long long t = (unsigned long long)blockIdx.x*blockDim.x + threadIdx.x; t < total; t += stride) {
		unsigned lo = 0, hi = nboxes - 1;
		while (lo < hi) {unsigned const mid = (lo + hi + 1) >> 1; if (boxes[mid].off <= t) lo = mid; else hi = mid - 1;}
		twi_box const B = boxes[lo];
		unsigned long long const r = t - B.off, xy = r / B.d;
		unsigned const z = B.z + (unsigned)(r - xy*B.d), x = B.x + (unsigned)(xy % B.w), y = B.y + (unsigned)(xy / B.w);
		bool overwritten = false;
		for (unsigned k = lo + 1; B.later && k < nboxes && !overwritten; ++k) {
			twi_box const &C = boxes[k];
			overwritten = (x - C.x < C.w && y - C.y < C.h && z - C.z < C.d);
		}
		if (overwritten) continue;
		size_t const i = z + ((size_t)x + (size_t)y*P.nx)*P.nz;
		float const val = values[t];
		bool const on_edge = (P.make_closed_surface && ((x == 0 || x == P.nx-1) || (y == 0 || y == P.ny-1) || (z == 0 || z == P.nz-1)));
		unsigned char o = on_edge ? (unsigned char)TW_VOX_ON_EDGE : (unsigned char)((val == P.isolevel) ? 1 : (((val < P.isolevel) != (P.invert != 0)) ? 1 : 0));
		if (zix_xy && z < __ldg(zix_xy + (size_t)y*P.nx + x)) {o |= TW_VOX_UNDER_MESH;}
		raw[i] = val; raw_o[i] = o;
		if (post && (__float_as_uint(post[i]) != __float_as_uint(val) || post_o[i] != o)) {post[i] = val; post_o[i] = o; mark_readers(mark, P, G, x, y);}
	}
}

// the model's field and flags (ov, oo) take the new ones (nv, no) where they differ, marking the blocks that read a changed voxel
__global__ void diff_kernel(const float *__restrict__ nv, const unsigned char *__restrict__ no, float *__restrict__ ov, unsigned char *__restrict__ oo,
	tw_voxel_post_params P, BlockGrid G, unsigned char *__restrict__ mark, size_t n)
{
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		float const v = nv[i];
		unsigned char const o = no[i];
		if (__float_as_uint(v) == __float_as_uint(ov[i]) && o == oo[i]) continue;
		ov[i] = v; oo[i] = o;
		size_t const xy = i / P.nz;
		mark_readers(mark, P, G, (unsigned)(xy % P.nx), (unsigned)(xy / P.nx));
	}
}

BlockGrid block_grid(const tw_voxel_model *m) {BlockGrid G; G.bx = m->bx; G.by = m->by; G.nbx = m->nbx; G.chunks = m->chunks; return G;}
McTables model_tables(const tw_voxel_model *m) {
	McTables T;
	T.edge_table = (const unsigned *)m->tables; T.tri_table = (const int *)((const char *)m->tables + 1024);
	T.edge_to_vals = (const unsigned *)((const char *)m->tables + 1024 + 16384);
	return T;
}

// A model job's counts in its pinned staging
struct twi_vmodel_stage {unsigned long long nblocks, nverts, ntris, changed;};

// A model job's slot-0 scratch: [counters (changed at byte 64), zeroed together | frontiers (remove_unconnected > 0) | mesh scratch | table | boxes | values]
// and pinned staging: [twi_vmodel_stage (64 B), then the table | boxes | values | fill coefficients]
struct ModelScratch {
	unsigned *cnt, *f0, *f1; unsigned long long *changed; MeshScratch S; tw_voxel_block_mesh *table; twi_box *boxes; float *values;
	twi_vmodel_stage *h_stage; tw_voxel_block_mesh *h_table; char *h_boxes, *h_values, *h_rdata;
};
int model_scratch(tw_voxel_model *m, size_t nboxes, size_t nvalues, ModelScratch *X) {
	tw_ctx *ctx = m->ctx;
	size_t const n = (size_t)m->P.nx*m->P.ny*m->P.nz, ng = (size_t)m->nblocks*m->chunks;
	X->f0 = X->f1 = nullptr;
	int rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		X->cnt = c.take<unsigned>(64); if (m->P.remove_unconnected > 0) {X->f0 = c.take<unsigned>(n + 16); X->f1 = c.take<unsigned>(n + 16);}
		X->S = mesh_scratch(c, ng*MC_BLOCK, (unsigned)ng); X->table = c.take<tw_voxel_block_mesh>(m->nblocks); X->boxes = c.take<twi_box>(nboxes);
		X->values = c.take<float>(nvalues);
	}); if (rc) return rc;
	char *h_head;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		h_head = c.take<char>(64 + (size_t)m->nblocks*sizeof(tw_voxel_block_mesh)); X->h_boxes = c.take<char>(nboxes*sizeof(twi_box));
		X->h_values = c.take<char>(nvalues*sizeof(float)); X->h_rdata = c.take<char>(TW_N3D_RDATA*sizeof(float));
	}); if (rc) return rc;
	X->h_stage = (twi_vmodel_stage *)h_head; X->h_table = (tw_voxel_block_mesh *)(h_head + 64);
	X->changed = (unsigned long long *)(X->cnt + 16);
	return TW_OK;
}

int validate_blocks_out(tw_ctx *ctx, const tw_voxel_blocks_out *o, float **d_vt, uint32_t **d_ix) {
	if (!o || !o->blocks || !o->nblocks || !o->nverts || !o->ntris) return tw_set_error(ctx, TW_ERR_ARG, "the block meshes need blocks, nblocks, nverts and ntris");
	if ((o->vcapacity && !o->verts) || (o->tcapacity && !o->indices)) return tw_set_error(ctx, TW_ERR_ARG, "a mesh capacity without its buffer");
	*d_vt = nullptr; *d_ix = nullptr;
	if (o->verts && !(*d_vt = (float *)device_view(o->verts))) return tw_set_error(ctx, TW_ERR_ARG, "verts must be device or page-locked host memory");
	if (o->indices && !(*d_ix = (uint32_t *)device_view(o->indices))) return tw_set_error(ctx, TW_ERR_ARG, "indices must be device or page-locked host memory");
	return TW_OK;
}

// the meshes of the blocks in d_list, their table and the job's counts into the pinned stage
int enqueue_block_meshes(tw_voxel_model *m, const unsigned *d_list, const ModelScratch &X, float *d_vt, uint64_t vcap, uint32_t *d_ix, uint64_t tcap) {
	tw_ctx *ctx = m->ctx;
	twi_vmodel_stage *const st = X.h_stage;
	if (m->nblocks) {
		unsigned const ng = m->nblocks*m->chunks;
		McTables const T = model_tables(m);
		BlockGrid const G = block_grid(m);
		MeshScratch const &S = X.S;
		block_mesh_kernel<false><<<ng, MC_BLOCK, 0, ctx->stream>>>(m->post, m->post_o, m->P, T, G, d_list, S.words, S.vsums, S.tsums, nullptr, nullptr, nullptr, 0, nullptr, 0);
		TW_LAUNCH_CHECK(ctx);
		scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(S.vsums, ng, S.voff, S.totals);
		TW_LAUNCH_CHECK(ctx);
		scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(S.tsums, ng, S.toff, S.totals + 1);
		TW_LAUNCH_CHECK(ctx);
		if (vcap || tcap) {
			block_mesh_kernel<true><<<ng, MC_BLOCK, 0, ctx->stream>>>(m->post, m->post_o, m->P, T, G, d_list, S.words, nullptr, nullptr, S.voff, S.toff, d_vt, vcap, d_ix, tcap);
			TW_LAUNCH_CHECK(ctx);
		}
		block_table_kernel<<<(m->nblocks + 255)/256, 256, 0, ctx->stream>>>(d_list, m->chunks, m->nblocks, S.voff, S.toff, S.totals, X.table);
		TW_LAUNCH_CHECK(ctx);
		TW_CUDA(ctx, cudaMemcpyAsync(&st->nblocks, d_list, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream)); // the low word (little-endian)
		TW_CUDA(ctx, cudaMemcpyAsync(&st->nverts, S.totals, 2*sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
		TW_CUDA(ctx, cudaMemcpyAsync(X.h_table, X.table, (size_t)m->nblocks*sizeof(tw_voxel_block_mesh), cudaMemcpyDeviceToHost, ctx->stream));
	}
	TW_CUDA(ctx, cudaMemcpyAsync(&st->changed, X.changed, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
	return TW_OK;
}

// a model job (not cancellable: it commits the model's state) whose completion unpacks X's stage and table into o
twi_job model_job(const ModelScratch &X, const tw_voxel_blocks_out &o) {
	twi_job j;
	j.complete = [st = X.h_stage, table = X.h_table, o](tw_ctx *) -> int {
		*o.nblocks = (uint32_t)st->nblocks; *o.nverts = st->nverts; *o.ntris = st->ntris;
		if (o.changed) {*o.changed = st->changed;}
		memcpy(o.blocks, table, (size_t)st->nblocks*sizeof(tw_voxel_block_mesh));
		return TW_OK;
	};
	return j;
}

int model_begin(tw_voxel_model *m) {return m ? twi_begin(m->ctx) : TW_ERR_ARG;}

} // namespace

extern "C" int tw_voxel_model_create(tw_ctx *ctx, const tw_voxel_post_params *vp, const uint32_t *edge_table256, const int32_t *tri_table256x16,
                                     const uint32_t *edge_to_vals12x2, const uint32_t *zix_xy, uint32_t bx, uint32_t by, tw_voxel_model **out)
{
	if (!ctx) return TW_ERR_ARG;
	if (!out || !edge_table256 || !tri_table256x16 || !edge_to_vals12x2) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_create: null argument");
	*out = nullptr;
	int rc = twi_begin(ctx); if (rc) return rc;
	rc = validate(ctx, vp); if (rc) return rc;
	if (bx == 0 || by == 0) return tw_set_error(ctx, TW_ERR_ARG, "block sizes must be >= 1");
	tw_voxel_post_params const P = *vp;
	unsigned const ncx = P.nx - 1, ncy = P.ny - 1, bw = (bx < ncx) ? bx : ncx, bh = (by < ncy) ? by : ncy;
	if (3ull*(bw + 1)*(bh + 1)*P.nz >= 0x100000000ull) return tw_set_error(ctx, TW_ERR_ARG, "a block's indices are 32-bit: 3*(bx+1)*(by+1)*nz must be below 2^32");
	size_t const n = (size_t)P.nx*P.ny*P.nz, nxy = (size_t)P.nx*P.ny;
	unsigned const nbx = (ncx + bx - 1)/bx, nby = (ncy + by - 1)/by, nblocks = nbx*nby;
	tw_voxel_model *m = new (std::nothrow) tw_voxel_model();
	if (!m) return tw_set_error(ctx, TW_ERR_CUDA, "tw_voxel_model_create: out of host memory");
	try {ctx->models.push_back(m);} catch (...) {delete m; return tw_set_error(ctx, TW_ERR_CUDA, "tw_voxel_model_create: out of host memory");}
	m->ctx = ctx; m->P = P; m->bx = bx; m->by = by; m->nbx = nbx; m->nblocks = nblocks; m->chunks = (unsigned)(((size_t)bw*bh*P.nz + MC_BLOCK - 1)/MC_BLOCK);
	m->have_zix = (zix_xy != nullptr);
	auto layout = [&](twi_carve &c) {
		m->raw = c.take<float>(n); m->post = c.take<float>(n); m->work = c.take<float>(n);
		m->raw_o = c.take<unsigned char>(n + 4); m->post_o = c.take<unsigned char>(n + 4); m->work_o = c.take<unsigned char>(n + 4);
		m->zix = zix_xy ? c.take<unsigned>(nxy) : nullptr; m->tables = c.take<char>(1024 + 16384 + 96); m->mark = c.take<unsigned char>((size_t)nblocks + 1);
		m->all = c.take<unsigned>((size_t)nblocks + 1); m->marked = c.take<unsigned>((size_t)nblocks + 1);
	};
	twi_carve c;
	layout(c);
	if (cudaMalloc(&m->mem, c.bytes) != cudaSuccess) {
		cudaGetLastError(); m->mem = nullptr; tw_voxel_model_destroy(m);
		return tw_set_error(ctx, TW_ERR_CUDA, "tw_voxel_model_create: no device memory for %zu voxels", n);
	}
	c = twi_carve{m->mem};
	layout(c);
	std::vector<unsigned> all((size_t)nblocks + 1);
	all[0] = nblocks;
	for (unsigned b = 0; b < nblocks; ++b) {all[1 + b] = b;}
	rc = TW_OK;
	auto up = [&](void *dst, const void *src, size_t len) {if (rc == TW_OK && cudaMemcpyAsync(dst, src, len, cudaMemcpyDefault, ctx->stream) != cudaSuccess) rc = TW_ERR_CUDA;};
	up(m->tables, edge_table256, 1024); up((char *)m->tables + 1024, tri_table256x16, 16384); up((char *)m->tables + 1024 + 16384, edge_to_vals12x2, 96);
	if (zix_xy) {up(m->zix, zix_xy, nxy*sizeof(unsigned));}
	up(m->all, all.data(), all.size()*sizeof(unsigned));
	if (rc == TW_OK && cudaMemsetAsync(m->mark, 0, nblocks + 1, ctx->stream) != cudaSuccess) rc = TW_ERR_CUDA;
	if (rc == TW_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = TW_ERR_CUDA;
	if (rc != TW_OK) {
		cudaStreamSynchronize(ctx->stream);
		char msg[256]; snprintf(msg, sizeof(msg), "tw_voxel_model_create: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
		tw_voxel_model_destroy(m);
		return tw_set_error(ctx, TW_ERR_CUDA, "%s", msg);
	}
	*out = m;
	return TW_OK;
}

extern "C" void tw_voxel_model_destroy(tw_voxel_model *m) {
	if (!m) return;
	tw_ctx *ctx = m->ctx;
	cudaSetDevice(ctx->device);
	twi_finish_pending(ctx); // the job may still read or write the model
	if (m->mem) cudaFree(m->mem);
	for (size_t i = 0; i < ctx->models.size(); ++i) {if (ctx->models[i] == m) {ctx->models.erase(ctx->models.begin() + i); break;}}
	delete m;
}

extern "C" int tw_voxel_model_build_launch(tw_voxel_model *m, const tw_voxel_params *fill, const float *rdata420, const float *vals, const tw_voxel_blocks_out *out) {
	int rc = model_begin(m); if (rc) return rc;
	tw_ctx *ctx = m->ctx;
	if ((fill != nullptr) == (vals != nullptr)) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_build_launch: give either fill or vals");
	float *d_vt; uint32_t *d_ix;
	rc = validate_blocks_out(ctx, out, &d_vt, &d_ix); if (rc) return rc;
	tw_voxel_blocks_out const O = *out;
	tw_voxel_post_params const &P = m->P;
	size_t tab_bytes = 0;
	tw_voxel_params F;
	if (fill) {
		F = *fill;
		if (F.nx != P.nx || F.ny != P.ny || F.nz != P.nz) return tw_set_error(ctx, TW_ERR_ARG, "the fill's grid %ux%ux%u differs from the model's %ux%ux%u", F.nx, F.ny, F.nz, P.nx, P.ny, P.nz);
		rc = twi_voxel_fill_check(ctx, &F, &tab_bytes); if (rc) return rc;
		if (tab_bytes) {rc = tw_reserve(ctx, 1, tab_bytes); if (rc) return rc;}
		if (F.gen_mode != TW_MGEN_SINE) {rc = twi_ensure_glm3_lut(ctx); if (rc) return rc;}
	}
	bool const rm = (P.remove_unconnected > 0);
	unsigned blocks = 0;
	if (rm) {rc = flood_blocks(ctx, &blocks); if (rc) return rc;}
	ModelScratch X;
	rc = model_scratch(m, 0, 0, &X); if (rc) return rc;
	size_t const n = (size_t)P.nx*P.ny*P.nz;
	memset(X.h_stage, 0, sizeof(twi_vmodel_stage));
	m->built = true; // the job commits the model's state
	return twi_launch_job(ctx, model_job(X, O), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(X.cnt, 0, 256, ctx->stream));
		if (fill) {int const r = twi_voxel_fill(ctx, &F, rdata420, m->raw, X.h_rdata); if (r) return r;}
		else {TW_CUDA(ctx, cudaMemcpyAsync(m->raw, vals, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(m->raw, P, m->zix, m->raw_o, n);
		TW_LAUNCH_CHECK(ctx);
		TW_CUDA(ctx, cudaMemcpyAsync(m->post, m->raw, n*sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
		TW_CUDA(ctx, cudaMemcpyAsync(m->post_o, m->raw_o, n, cudaMemcpyDeviceToDevice, ctx->stream));
		if (rm) {int const r = enqueue_remove_unconnected(ctx, blocks, m->post, m->post_o, &P, X.f0, X.f1, X.cnt, X.changed); if (r) return r;}
		return enqueue_block_meshes(m, m->all, X, d_vt, O.vcapacity, d_ix, O.tcapacity);
	});
}

extern "C" int tw_voxel_model_edit_launch(tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values, const tw_voxel_blocks_out *out) {
	int rc = model_begin(m); if (rc) return rc;
	tw_ctx *ctx = m->ctx;
	if (nboxes && (!boxes || !values)) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_edit_launch: null boxes or values");
	float *d_vt; uint32_t *d_ix;
	rc = validate_blocks_out(ctx, out, &d_vt, &d_ix); if (rc) return rc;
	tw_voxel_blocks_out const O = *out;
	tw_voxel_post_params const &P = m->P;
	unsigned long long total = 0;
	std::vector<twi_box> B(nboxes);
	for (uint32_t k = 0; k < nboxes; ++k) {
		tw_voxel_box const &b = boxes[k];
		if (b.w == 0 || b.h == 0 || b.d == 0) return tw_set_error(ctx, TW_ERR_ARG, "box %u is empty", k);
		if (b.x >= P.nx || b.w > P.nx - b.x || b.y >= P.ny || b.h > P.ny - b.y || b.z >= P.nz || b.d > P.nz - b.z)
			return tw_set_error(ctx, TW_ERR_ARG, "box %u reaches outside the %ux%ux%u grid", k, P.nx, P.ny, P.nz);
		twi_box &t = B[k];
		t.x = b.x; t.y = b.y; t.z = b.z; t.w = b.w; t.h = b.h; t.d = b.d; t.off = total; t.later = 0; t.pad = 0;
		total += (unsigned long long)b.w*b.h*b.d;
	}
	for (uint32_t k = 0; k < nboxes; ++k) { // overlaps: the later box's value wins
		for (uint32_t j = k + 1; j < nboxes && !B[k].later; ++j) {
			const twi_box &a = B[k], &b = B[j];
			B[k].later = (a.x < b.x + b.w && b.x < a.x + a.w && a.y < b.y + b.h && b.y < a.y + a.h && a.z < b.z + b.d && b.z < a.z + a.d);
		}
	}
	if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "the voxel model has no field yet (tw_voxel_model_build_launch)");
	bool const rm = (P.remove_unconnected > 0);
	unsigned blocks = 0;
	if (rm && total) {rc = flood_blocks(ctx, &blocks); if (rc) return rc;}
	ModelScratch X;
	rc = model_scratch(m, nboxes, total, &X); if (rc) return rc;
	size_t const n = (size_t)P.nx*P.ny*P.nz;
	memset(X.h_stage, 0, sizeof(twi_vmodel_stage));
	if (nboxes) {memcpy(X.h_boxes, B.data(), nboxes*sizeof(twi_box)); memcpy(X.h_values, values, total*sizeof(float));}
	return twi_launch_job(ctx, model_job(X, O), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(X.cnt, 0, 256, ctx->stream));
		if (total) {
			TW_CUDA(ctx, cudaMemcpyAsync(X.boxes, X.h_boxes, nboxes*sizeof(twi_box), cudaMemcpyHostToDevice, ctx->stream));
			TW_CUDA(ctx, cudaMemcpyAsync(X.values, X.h_values, total*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
			box_scatter_kernel<<<stream_grid(ctx, total), 256, 0, ctx->stream>>>(X.boxes, nboxes, X.values, total, P, m->zix, block_grid(m), m->raw, m->raw_o,
			                                                                     rm ? nullptr : m->post, rm ? nullptr : m->post_o, m->mark);
			TW_LAUNCH_CHECK(ctx);
			if (rm) {
				TW_CUDA(ctx, cudaMemcpyAsync(m->work, m->raw, n*sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
				TW_CUDA(ctx, cudaMemcpyAsync(m->work_o, m->raw_o, n, cudaMemcpyDeviceToDevice, ctx->stream));
				int const r = enqueue_remove_unconnected(ctx, blocks, m->work, m->work_o, &P, X.f0, X.f1, X.cnt, X.changed); if (r) return r;
				diff_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(m->work, m->work_o, m->post, m->post_o, P, block_grid(m), m->mark, n);
				TW_LAUNCH_CHECK(ctx);
			}
		}
		if (m->nblocks) {list_marked_kernel<<<1, 1024, 0, ctx->stream>>>(m->mark, m->nblocks, m->marked); TW_LAUNCH_CHECK(ctx);}
		return enqueue_block_meshes(m, m->marked, X, d_vt, O.vcapacity, d_ix, O.tcapacity);
	});
}

extern "C" int tw_voxel_model_read(tw_voxel_model *m, float *raw, float *vals, uint8_t *outside) {
	int rc = model_begin(m); if (rc) return rc;
	tw_ctx *ctx = m->ctx;
	if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "the voxel model has no field yet (tw_voxel_model_build_launch)");
	size_t const n = (size_t)m->P.nx*m->P.ny*m->P.nz;
	if (raw) {TW_CUDA(ctx, cudaMemcpyAsync(raw, m->raw, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
	if (vals) {TW_CUDA(ctx, cudaMemcpyAsync(vals, m->post, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
	if (outside) {TW_CUDA(ctx, cudaMemcpyAsync(outside, m->post_o, n, cudaMemcpyDefault, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}
