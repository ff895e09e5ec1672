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
#include "tw_voxel_edit.cuh"
#include "tw_voxel_mc.cuh"
#include "tw_voxel_batch.h"
#include "tw_voxel_model_batch.h"
#include <dlfcn.h>
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

namespace {

__global__ void outside_kernel(const float *__restrict__ vals, tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, unsigned char *__restrict__ outside, size_t n) {
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		unsigned const z = (unsigned)(i % P.nz);
		size_t const xy = i / P.nz;
		unsigned const x = (unsigned)(xy % P.nx), y = (unsigned)(xy / P.nx);
		outside[i] = outside_flag(vals, i, x, y, z, P, zix_xy);
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
// The three tables in one device region of MC_TAB_BYTES: [edge_table 1024 B | tri_table 16384 B | edge_to_vals 96 B]
constexpr size_t MC_TAB_OFF[3] = {0, 1024, 1024 + 16384}, MC_TAB_LEN[3] = {1024, 16384, 96}, MC_TAB_BYTES = MC_TAB_OFF[2] + MC_TAB_LEN[2];
McTables mc_tables(const void *tab) {
	const char *t = (const char *)tab;
	return McTables{(const unsigned *)t, (const int *)(t + MC_TAB_OFF[1]), (const unsigned *)(t + MC_TAB_OFF[2])};
}
// Copies the caller's tables into the region `tab` on ctx->stream. h_bounce (optional): MC_TAB_BYTES of pinned staging that host tables are copied into
// first, so the caller may reuse them once this returns (device tables are read when the copy runs).
int mc_tables_upload(tw_ctx *ctx, void *tab, const uint32_t *edge_table256, const int32_t *tri_table256x16, const uint32_t *edge_to_vals12x2, char *h_bounce = nullptr) {
	const void *src[3] = {edge_table256, tri_table256x16, edge_to_vals12x2};
	for (int k = 0; k < 3; ++k) {
		if (h_bounce && !tw_is_device_ptr(src[k])) {memcpy(h_bounce + MC_TAB_OFF[k], src[k], MC_TAB_LEN[k]); src[k] = h_bounce + MC_TAB_OFF[k];}
		TW_CUDA(ctx, cudaMemcpyAsync((char *)tab + MC_TAB_OFF[k], src[k], MC_TAB_LEN[k], cudaMemcpyDefault, ctx->stream));
	}
	return TW_OK;
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
	twi_user<const float> v(vals, n);
	twi_user<uint8_t> o(outside, n);
	twi_user<const uint32_t> z(zix_xy, nxy);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {v.take(c); o.take(c); if (zix_xy) {z.take(c);}}); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	rc = z.in(ctx); if (rc) return rc;
	outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(v.d, *vp, z.d, o.d, n);
	TW_LAUNCH_CHECK(ctx);
	rc = o.out(ctx); if (rc) return rc;
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
	twi_user<float> v(vals, n);
	bool const dev_o = tw_is_device_ptr(outside);
	if (dev_o && ((size_t)outside & 3)) return tw_set_error(ctx, TW_ERR_ARG, "outside must be 4-byte aligned (flag bytes are claimed with 32-bit atomics)");
	// the 32-bit word that holds the last flag byte reaches up to 3 bytes past a buffer of n % 4 != 0 bytes: such a device buffer is staged like a host one
	bool const stage_o = !dev_o || (n & 3);
	unsigned blocks = 0;
	rc = flood_blocks(ctx, &blocks); if (rc) return rc;
	unsigned char *d_o = outside; unsigned *f0, *f1, *cnt; unsigned long long *d_changed;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		v.take(c); if (stage_o) {d_o = c.take<unsigned char>(n + 4);} f0 = c.take<unsigned>(n + 16); f1 = c.take<unsigned>(n + 16);
		cnt = c.take<unsigned>(8); d_changed = c.take<unsigned long long>(1);
	}); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	if (stage_o) {TW_CUDA(ctx, cudaMemcpyAsync(d_o, outside, n, dev_o ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));}
	TW_CUDA(ctx, cudaMemsetAsync(d_changed, 0, sizeof(unsigned long long), ctx->stream));
	rc = enqueue_remove_unconnected(ctx, blocks, v.d, d_o, vp, f0, f1, cnt, d_changed);
	if (rc) {cudaStreamSynchronize(ctx->stream); return rc;}
	unsigned long long hc = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&hc, d_changed, sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
	rc = v.out(ctx); if (rc) return rc;
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
	twi_user<const float> v(vals, n);
	twi_user<const uint8_t> o(outside, n);
	char *tab; unsigned *d_sums; unsigned long long *d_offsets, *d_total;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		v.take(c); o.take(c); tab = c.take<char>(MC_TAB_BYTES);
		d_sums = c.take<unsigned>(nblocks); d_offsets = c.take<unsigned long long>(nblocks); d_total = c.take<unsigned long long>(1);
	}); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	rc = o.in(ctx); if (rc) return rc;
	rc = mc_tables_upload(ctx, tab, edge_table256, tri_table256x16, edge_to_vals12x2); if (rc) return rc;
	McTables const T = mc_tables(tab);
	mc_kernel<false><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(v.d, o.d, *vp, T, n, d_sums, nullptr, nullptr, 0);
	TW_LAUNCH_CHECK(ctx);
	scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(d_sums, nblocks, d_offsets, d_total);
	TW_LAUNCH_CHECK(ctx);
	unsigned long long total = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*ntris = total;
	if (capacity == 0 || total == 0) return TW_OK;
	uint64_t const nw = (total < capacity) ? total : capacity;
	twi_user<float> t(tris, (size_t)nw*9);
	rc = twi_reserve_carve(ctx, 1, [&](twi_carve &c) {t.take(c);}); if (rc) return rc;
	mc_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(v.d, o.d, *vp, T, n, nullptr, d_offsets, t.d, nw);
	TW_LAUNCH_CHECK(ctx);
	rc = t.out(ctx); if (rc) return rc;
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
	twi_user<const float> v(vals, n);
	twi_user<const uint8_t> o(outside, n);
	char *tab; MeshScratch S;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {v.take(c); o.take(c); tab = c.take<char>(MC_TAB_BYTES); S = mesh_scratch(c, n, nblocks);}); if (rc) return rc;
	rc = v.in(ctx); if (rc) return rc;
	rc = o.in(ctx); if (rc) return rc;
	rc = mc_tables_upload(ctx, tab, edge_table256, tri_table256x16, edge_to_vals12x2); if (rc) return rc;
	McTables const T = mc_tables(tab);
	// count and scan first: the emit pass writes at most min(count, capacity) of each, so host outputs are staged at that size
	rc = enqueue_mesh(ctx, v.d, o.d, *vp, T, S, nullptr, 0, nullptr, 0); if (rc) return rc;
	unsigned long long tot[2] = {0, 0};
	TW_CUDA(ctx, cudaMemcpyAsync(tot, S.totals, sizeof(tot), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*M.nverts = tot[0]; *M.ntris = tot[1];
	uint64_t const nv = (tot[0] < M.vcapacity) ? tot[0] : M.vcapacity, nt = (tot[1] < M.tcapacity) ? tot[1] : M.tcapacity;
	if (nv == 0 && nt == 0) return TW_OK;
	twi_user<float> vt(M.verts, (size_t)nv*3);
	twi_user<uint32_t> ix(M.indices, (size_t)nt*3);
	rc = twi_reserve_carve(ctx, 1, [&](twi_carve &c) {vt.take(c); ix.take(c);}); if (rc) return rc;
	mesh_kernel<true><<<nblocks, MC_BLOCK, 0, ctx->stream>>>(v.d, o.d, *vp, T, n, S.words, nullptr, nullptr, S.voff, S.toff, vt.d, nv, ix.d, nt);
	TW_LAUNCH_CHECK(ctx);
	rc = vt.out(ctx); if (rc) return rc;
	rc = ix.out(ctx); if (rc) return rc;
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
	twi_user<float> v(b->vals, n); // the fill's output when vals is null
	twi_user<const uint32_t> z(b->zix_xy, nxy);
	bool const tabs = (ntab == 3);
	unsigned *cnt, *f0 = nullptr, *f1 = nullptr, *d_sums = nullptr;
	unsigned char *d_o;
	char *tab = nullptr;
	unsigned long long *d_offsets = nullptr;
	MeshScratch S;
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		cnt = c.take<unsigned>(64); // [flood counters | changed at byte 64 | triangle total at byte 128], zeroed together
		v.take(c);
		d_o = c.take<unsigned char>(n + 4);
		if (rm) {f0 = c.take<unsigned>(n + 16); f1 = c.take<unsigned>(n + 16);}
		if (tabs) {tab = c.take<char>(MC_TAB_BYTES);}
		if (mc) {d_sums = c.take<unsigned>(nblocks); d_offsets = c.take<unsigned long long>(nblocks);}
		if (b->zix_xy) {z.take(c);}
		if (wm) S = mesh_scratch(c, n, nblocks);
	}); if (rc) return rc;
	if (tab_bytes) {rc = tw_reserve(ctx, 1, tab_bytes); if (rc) return rc;}
	twi_voxel_stage *st; float *h_rdata; char *h_tab = nullptr;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		st = c.take<twi_voxel_stage>(1); h_rdata = c.take<float>(TW_N3D_RDATA); if (tabs) {h_tab = c.take<char>(MC_TAB_BYTES);} z.take_pinned(c);
	}); if (rc) return rc;
	if (fill && F.gen_mode != TW_MGEN_SINE) {rc = twi_ensure_glm3_lut(ctx); if (rc) return rc;}
	unsigned long long *d_changed = (unsigned long long *)(cnt + 16), *d_total = (unsigned long long *)(cnt + 32);
	McTables const T = tabs ? mc_tables(tab) : McTables{};
	float *const d_v = v.d;
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
		int r = fill ? twi_voxel_fill(ctx, &F, b->rdata420, d_v, h_rdata) : v.in(ctx); if (r) return r;
		r = z.in(ctx); if (r) return r;
		if (tabs) {r = mc_tables_upload(ctx, tab, b->edge_table256, b->tri_table256x16, b->edge_to_vals12x2, h_tab); if (r) return r;}
		outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(d_v, P, z.d, d_o, n);
		TW_LAUNCH_CHECK(ctx);
		if (rm) {r = enqueue_remove_unconnected(ctx, blocks, d_v, d_o, &P, f0, f1, cnt, d_changed); if (r) return r;}
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
		if (wm) {r = enqueue_mesh(ctx, d_v, d_o, P, T, S, d_mv, M.vcapacity, d_mi, M.tcapacity); if (r) return r;}
		if (fill || rm) {r = v.out(ctx); if (r) return r;}
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
// A job may run on any context of the model's family (model_begin); `ev` orders their device work on the model's memory, as a tile set's event does.
struct tw_voxel_model {
	tw_ctx *ctx = nullptr;                   // the context that created it (it owns the model)
	cudaEvent_t ev = nullptr;                // recorded after the last model job's device work, on whichever context launched it; the next one waits on it
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

__global__ void box_scatter_kernel(const twi_box *__restrict__ boxes, unsigned nboxes, const float *__restrict__ values, unsigned long long total,
	tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, BlockGrid G, float *__restrict__ raw, unsigned char *__restrict__ raw_o, float *post,
	unsigned char *post_o, unsigned char *mark)
{
	box_scatter<false>(boxes, nboxes, values, total, P, zix_xy, G, raw, raw_o, post, post_o, mark, nullptr);
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

// A model job's counts in its pinned staging
struct twi_vmodel_stage {unsigned long long nblocks, nverts, ntris, changed, nchanged;};

// A model job's slot-0 scratch: [counters (changed at byte 64, the change list's total at byte 128), zeroed together | frontiers (remove_unconnected > 0) |
// mesh scratch | table | boxes | values | change list (list: bits, chunk sums, chunk offsets)]
// and pinned staging: [twi_vmodel_stage (64 B), then the table | boxes | values | fill coefficients]
struct ChangeScratch {unsigned *bits, *sums; unsigned long long *offsets, *total; size_t nwords; unsigned nchunks;};
struct ModelScratch {
	unsigned *cnt, *f0, *f1; unsigned long long *changed; MeshScratch S; tw_voxel_block_mesh *table; twi_box *boxes; float *values; ChangeScratch L;
	twi_vmodel_stage *h_stage; tw_voxel_block_mesh *h_table; char *h_boxes, *h_values, *h_rdata;
};
int model_scratch(tw_ctx *ctx, const tw_voxel_model *m, size_t nboxes, size_t nvalues, ModelScratch *X, bool list = false) {
	size_t const n = (size_t)m->P.nx*m->P.ny*m->P.nz, ng = (size_t)m->nblocks*m->chunks;
	X->f0 = X->f1 = nullptr;
	ChangeScratch &L = X->L;
	L = ChangeScratch{};
	L.nwords = list ? (n + 31)/32 : 0; L.nchunks = (unsigned)((L.nwords + CL_BLOCK - 1)/CL_BLOCK);
	int rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		X->cnt = c.take<unsigned>(64); if (m->P.remove_unconnected > 0) {X->f0 = c.take<unsigned>(n + 16); X->f1 = c.take<unsigned>(n + 16);}
		X->S = mesh_scratch(c, ng*MC_BLOCK, (unsigned)ng); X->table = c.take<tw_voxel_block_mesh>(m->nblocks); X->boxes = c.take<twi_box>(nboxes);
		X->values = c.take<float>(nvalues);
		if (list) {L.bits = c.take<unsigned>(L.nwords); L.sums = c.take<unsigned>(L.nchunks); L.offsets = c.take<unsigned long long>(L.nchunks);}
	}); if (rc) return rc;
	L.total = (unsigned long long *)(X->cnt + 32);
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
int enqueue_block_meshes(tw_ctx *ctx, const tw_voxel_model *m, const unsigned *d_list, const ModelScratch &X, float *d_vt, uint64_t vcap, uint32_t *d_ix, uint64_t tcap) {
	twi_vmodel_stage *const st = X.h_stage;
	if (m->nblocks) {
		unsigned const ng = m->nblocks*m->chunks;
		McTables const T = mc_tables(m->tables);
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

// a model job (not cancellable: it commits the model's state) whose completion unpacks X's stage and table into o, and the change list's count into
// nchanged (optional)
twi_job model_job(const ModelScratch &X, const tw_voxel_blocks_out &o, uint64_t *nchanged = nullptr) {
	twi_job j;
	j.complete = [st = X.h_stage, table = X.h_table, o, nchanged](tw_ctx *) -> int {
		*o.nblocks = (uint32_t)st->nblocks; *o.nverts = st->nverts; *o.ntris = st->ntris;
		if (o.changed) {*o.changed = st->changed;}
		if (nchanged) {*nchanged = st->nchanged;}
		memcpy(o.blocks, table, (size_t)st->nblocks*sizeof(tw_voxel_block_mesh));
		return TW_OK;
	};
	return j;
}

// A model call on ctx: TW_ERR_ARG unless ctx and m are set and ctx is m's context, its parent or a shared context of that parent; then ctx's pending job is
// completed (never another context's)
int model_family(tw_ctx *ctx, const tw_voxel_model *m) {
	tw_ctx const *root = ctx->parent ? ctx->parent : ctx, *owner = m->ctx->parent ? m->ctx->parent : m->ctx;
	if (root != owner || ctx->device != m->ctx->device) return tw_set_error(ctx, TW_ERR_ARG, "the voxel model belongs to another family of contexts");
	return TW_OK;
}
int model_begin(tw_ctx *ctx, tw_voxel_model *m) {
	if (!ctx || !m) return TW_ERR_ARG;
	int const rc = model_family(ctx, m); if (rc) return rc;
	return twi_begin(ctx);
}

// A model job on ctx: its device work waits for the model's earlier jobs on any context of the family, and the model's event is recorded behind it
template <typename Enqueue> int launch_model_job(tw_ctx *ctx, tw_voxel_model *m, twi_job job, Enqueue &&enqueue) {
	return twi_launch_job(ctx, std::move(job), [&]() -> int {
		TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, m->ev, 0));
		int const r = enqueue(); if (r) return r;
		TW_CUDA(ctx, cudaEventRecord(m->ev, ctx->stream));
		return TW_OK;
	});
}

// The boxes of an edit or a read (TW_ERR_ARG for an empty one or one reaching outside the grid) with their values' offsets and overlaps; *total = their voxels
int model_boxes(tw_ctx *ctx, const tw_voxel_post_params &P, const tw_voxel_box *boxes, uint32_t nboxes, std::vector<twi_box> &B, unsigned long long *total) {
	*total = 0;
	B.resize(nboxes);
	for (uint32_t k = 0; k < nboxes; ++k) {
		tw_voxel_box const &b = boxes[k];
		if (b.w == 0 || b.h == 0 || b.d == 0) return tw_set_error(ctx, TW_ERR_ARG, "box %u is empty", k);
		if (b.x >= P.nx || b.w > P.nx - b.x || b.y >= P.ny || b.h > P.ny - b.y || b.z >= P.nz || b.d > P.nz - b.z)
			return tw_set_error(ctx, TW_ERR_ARG, "box %u reaches outside the %ux%ux%u grid", k, P.nx, P.ny, P.nz);
		twi_box &t = B[k];
		t.x = b.x; t.y = b.y; t.z = b.z; t.w = b.w; t.h = b.h; t.d = b.d; t.off = *total; t.later = 0; t.pad = 0;
		*total += (unsigned long long)b.w*b.h*b.d;
	}
	for (uint32_t k = 0; k < nboxes; ++k) { // overlaps: the later box's value wins
		for (uint32_t j = k + 1; j < nboxes && !B[k].later; ++j) {
			const twi_box &a = B[k], &b = B[j];
			B[k].later = (a.x < b.x + b.w && b.x < a.x + a.w && a.y < b.y + b.h && b.y < a.y + a.h && a.z < b.z + b.d && b.z < a.z + a.d);
		}
	}
	return TW_OK;
}

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
	cudaError_t const ee = cudaEventCreateWithFlags(&m->ev, cudaEventDisableTiming);
	if (ee != cudaSuccess) {delete m; return tw_set_error(ctx, TW_ERR_CUDA, "tw_voxel_model_create: event: %s", cudaGetErrorString(ee));}
	try {ctx->models.push_back(m);} catch (...) {cudaEventDestroy(m->ev); delete m; return tw_set_error(ctx, TW_ERR_CUDA, "tw_voxel_model_create: out of host memory");}
	m->ctx = ctx; m->P = P; m->bx = bx; m->by = by; m->nbx = nbx; m->nblocks = nblocks; m->chunks = (unsigned)(((size_t)bw*bh*P.nz + MC_BLOCK - 1)/MC_BLOCK);
	m->have_zix = (zix_xy != nullptr);
	auto layout = [&](twi_carve &c) {
		m->raw = c.take<float>(n); m->post = c.take<float>(n); m->work = c.take<float>(n);
		m->raw_o = c.take<unsigned char>(n + 4); m->post_o = c.take<unsigned char>(n + 4); m->work_o = c.take<unsigned char>(n + 4);
		m->zix = zix_xy ? c.take<unsigned>(nxy) : nullptr; m->tables = c.take<char>(MC_TAB_BYTES); m->mark = c.take<unsigned char>((size_t)nblocks + 1);
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
	rc = mc_tables_upload(ctx, m->tables, edge_table256, tri_table256x16, edge_to_vals12x2);
	auto up = [&](void *dst, const void *src, size_t len) {if (rc == TW_OK && cudaMemcpyAsync(dst, src, len, cudaMemcpyDefault, ctx->stream) != cudaSuccess) rc = TW_ERR_CUDA;};
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
	cudaEventSynchronize(m->ev); // and so may a job on another context of the family
	cudaEventDestroy(m->ev);
	if (m->mem) cudaFree(m->mem);
	for (size_t i = 0; i < ctx->models.size(); ++i) {if (ctx->models[i] == m) {ctx->models.erase(ctx->models.begin() + i); break;}}
	delete m;
}

extern "C" int tw_voxel_model_build_launch(tw_voxel_model *m, const tw_voxel_params *fill, const float *rdata420, const float *vals, const tw_voxel_blocks_out *out) {
	return tw_voxel_model_build_launch_on(m ? m->ctx : nullptr, m, fill, rdata420, vals, out);
}

extern "C" int tw_voxel_model_build_launch_on(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_params *fill, const float *rdata420, const float *vals,
                                              const tw_voxel_blocks_out *out) {
	int rc = model_begin(ctx, m); if (rc) return rc;
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
	rc = model_scratch(ctx, m, 0, 0, &X); if (rc) return rc;
	size_t const n = (size_t)P.nx*P.ny*P.nz;
	memset(X.h_stage, 0, sizeof(twi_vmodel_stage));
	m->built = true; // the job commits the model's state
	return launch_model_job(ctx, m, model_job(X, O), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(X.cnt, 0, 256, ctx->stream));
		if (fill) {int const r = twi_voxel_fill(ctx, &F, rdata420, m->raw, X.h_rdata); if (r) return r;}
		else {TW_CUDA(ctx, cudaMemcpyAsync(m->raw, vals, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
		outside_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(m->raw, P, m->zix, m->raw_o, n);
		TW_LAUNCH_CHECK(ctx);
		TW_CUDA(ctx, cudaMemcpyAsync(m->post, m->raw, n*sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
		TW_CUDA(ctx, cudaMemcpyAsync(m->post_o, m->raw_o, n, cudaMemcpyDeviceToDevice, ctx->stream));
		if (rm) {int const r = enqueue_remove_unconnected(ctx, blocks, m->post, m->post_o, &P, X.f0, X.f1, X.cnt, X.changed); if (r) return r;}
		return enqueue_block_meshes(ctx, m, m->all, X, d_vt, O.vcapacity, d_ix, O.tcapacity);
	});
}

namespace {
// the change list's outputs as the device addresses them
struct ChangeOut {uint32_t *index; float *vals; uint8_t *outside; unsigned long long capacity; uint64_t *nchanged;};
int validate_changes(tw_ctx *ctx, const tw_voxel_changes *ch, ChangeOut *d) {
	if (!ch->nchanged) return tw_set_error(ctx, TW_ERR_ARG, "the change list needs nchanged");
	if (ch->capacity && !ch->index) return tw_set_error(ctx, TW_ERR_ARG, "a change list capacity without index");
	if ((ch->vals || ch->outside) && !ch->index) return tw_set_error(ctx, TW_ERR_ARG, "change list vals or outside without index");
	d->index = nullptr; d->vals = nullptr; d->outside = nullptr; d->capacity = ch->capacity; d->nchanged = ch->nchanged;
	if (ch->index && !(d->index = (uint32_t *)device_view(ch->index))) return tw_set_error(ctx, TW_ERR_ARG, "change list index must be device or page-locked host memory");
	if (ch->vals && !(d->vals = (float *)device_view(ch->vals))) return tw_set_error(ctx, TW_ERR_ARG, "change list vals must be device or page-locked host memory");
	if (ch->outside && !(d->outside = (uint8_t *)device_view(ch->outside))) return tw_set_error(ctx, TW_ERR_ARG, "change list outside must be device or page-locked host memory");
	return TW_OK;
}

} // namespace

int twi_module_kernels(tw_ctx *ctx, const char *file, const char *const *names, int count, cudaKernel_t *out) {
	static std::mutex mu;
	static std::vector<std::pair<std::string, std::vector<cudaKernel_t>>> loaded; // per file, its kernels in the order of names
	std::lock_guard<std::mutex> g(mu);
	for (auto const &e : loaded) {if (e.first == file) {for (int k = 0; k < count; ++k) {out[k] = e.second[k];} return TW_OK;}}
	Dl_info info;
	if (!dladdr((void *)&tw_voxel_model_edit_launch_ex, &info) || !info.dli_fname) return tw_set_error(ctx, TW_ERR_CUDA, "cannot locate the library's file");
	std::string const lib_path = info.dli_fname, path = lib_path.substr(0, lib_path.rfind('/') + 1) + file;
	cudaLibrary_t l = nullptr;
	cudaError_t e = cudaLibraryLoadFromFile(&l, path.c_str(), nullptr, nullptr, 0, nullptr, nullptr, 0);
	std::vector<cudaKernel_t> k(count);
	for (int i = 0; i < count && e == cudaSuccess; ++i) {e = cudaLibraryGetKernel(&k[i], l, names[i]);}
	if (e != cudaSuccess) {
		cudaGetLastError();
		if (l) cudaLibraryUnload(l);
		return tw_set_error(ctx, TW_ERR_CUDA, "cannot load the kernels of %s: %s", path.c_str(), cudaGetErrorString(e));
	}
	loaded.emplace_back(file, k);
	for (int i = 0; i < count; ++i) {out[i] = k[i];}
	return TW_OK;
}

namespace {
// The change-list kernels (tw_voxel_changes.cu), from tw_voxel_changes.cubin
struct ChangeKernels {cudaKernel_t box_bits, diff_bits, count, emit;};
int change_kernels(tw_ctx *ctx, ChangeKernels *K) {
	static const char *const names[] = {"tw_box_scatter_bits_kernel", "tw_diff_bits_kernel", "tw_change_count_kernel", "tw_change_emit_kernel"};
	cudaKernel_t k[4];
	int const rc = twi_module_kernels(ctx, "tw_voxel_changes.cubin", names, 4, k); if (rc) return rc;
	*K = ChangeKernels{k[0], k[1], k[2], k[3]};
	return TW_OK;
}
// one launch of a module kernel on ctx->stream with smem bytes of dynamic shared memory; the arguments must have the kernel's parameter types exactly
template<typename... A>
int launch_module_kernel_smem(tw_ctx *ctx, cudaKernel_t k, dim3 grid, unsigned block, size_t smem, A... a) {
	void *args[] = {(void *)&a...};
	TW_CUDA(ctx, cudaLaunchKernel((const void *)k, grid, dim3(block), args, smem, ctx->stream));
	ctx->launches++;
	return TW_OK;
}
template<typename... A>
int launch_module_kernel(tw_ctx *ctx, cudaKernel_t k, unsigned grid, unsigned block, A... a) {return launch_module_kernel_smem(ctx, k, dim3(grid), block, 0, a...);}

// the list of the voxels whose bits are set (bits: every word written), its total into the pinned stage
int enqueue_change_list(tw_ctx *ctx, const tw_voxel_model *m, const ModelScratch &X, const ChangeOut &C, const ChangeKernels &K) {
	ChangeScratch const &L = X.L;
	int rc = launch_module_kernel(ctx, K.count, L.nchunks, CL_BLOCK, (const unsigned *)L.bits, L.nwords, L.sums); if (rc) return rc;
	scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(L.sums, L.nchunks, L.offsets, L.total);
	TW_LAUNCH_CHECK(ctx);
	if (C.capacity) {
		rc = launch_module_kernel(ctx, K.emit, L.nchunks, CL_BLOCK, (const unsigned *)L.bits, L.nwords, (const unsigned long long *)L.offsets, (const float *)m->post,
		                          (const unsigned char *)m->post_o, C.index, C.vals, C.outside, C.capacity);
		if (rc) return rc;
	}
	TW_CUDA(ctx, cudaMemcpyAsync(&X.h_stage->nchanged, L.total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
	return TW_OK;
}
} // namespace

extern "C" int tw_voxel_model_edit_launch(tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values, const tw_voxel_blocks_out *out) {
	return tw_voxel_model_edit_launch_ex(m, boxes, nboxes, values, out, nullptr);
}

extern "C" int tw_voxel_model_edit_launch_ex(tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values, const tw_voxel_blocks_out *out,
                                             const tw_voxel_changes *ch)
{
	return tw_voxel_model_edit_launch_on(m ? m->ctx : nullptr, m, boxes, nboxes, values, out, ch);
}

extern "C" int tw_voxel_model_edit_launch_on(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, const float *values,
                                             const tw_voxel_blocks_out *out, const tw_voxel_changes *ch)
{
	int rc = model_begin(ctx, m); if (rc) return rc;
	if (nboxes && (!boxes || !values)) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_edit_launch: null boxes or values");
	float *d_vt; uint32_t *d_ix;
	rc = validate_blocks_out(ctx, out, &d_vt, &d_ix); if (rc) return rc;
	tw_voxel_blocks_out const O = *out;
	ChangeOut CO;
	ChangeKernels K;
	if (ch) {rc = validate_changes(ctx, ch, &CO); if (rc) return rc;}
	tw_voxel_post_params const &P = m->P;
	unsigned long long total = 0;
	std::vector<twi_box> B;
	rc = model_boxes(ctx, P, boxes, nboxes, B, &total); if (rc) return rc;
	if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "the voxel model has no field yet (tw_voxel_model_build_launch)");
	bool const rm = (P.remove_unconnected > 0);
	unsigned blocks = 0;
	if (rm && total) {rc = flood_blocks(ctx, &blocks); if (rc) return rc;}
	// the change list: only an edit with boxes can change a voxel, so without them the count stays the stage's 0
	bool const list = ch && total;
	if (list) {rc = change_kernels(ctx, &K); if (rc) return rc;}
	ModelScratch X;
	rc = model_scratch(ctx, m, nboxes, total, &X, list); if (rc) return rc;
	size_t const n = (size_t)P.nx*P.ny*P.nz;
	memset(X.h_stage, 0, sizeof(twi_vmodel_stage));
	if (nboxes) {memcpy(X.h_boxes, B.data(), nboxes*sizeof(twi_box)); memcpy(X.h_values, values, total*sizeof(float));}
	return launch_model_job(ctx, m, model_job(X, O, ch ? CO.nchanged : nullptr), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(X.cnt, 0, 256, ctx->stream));
		if (total) {
			TW_CUDA(ctx, cudaMemcpyAsync(X.boxes, X.h_boxes, nboxes*sizeof(twi_box), cudaMemcpyHostToDevice, ctx->stream));
			TW_CUDA(ctx, cudaMemcpyAsync(X.values, X.h_values, total*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
			if (list && !rm) { // the boxes' voxels set their bits one by one
				TW_CUDA(ctx, cudaMemsetAsync(X.L.bits, 0, X.L.nwords*sizeof(unsigned), ctx->stream));
				int const r = launch_module_kernel(ctx, K.box_bits, stream_grid(ctx, total), 256u, (const twi_box *)X.boxes, (unsigned)nboxes, (const float *)X.values, total,
				                                   P, (const unsigned *)m->zix, block_grid(m), m->raw, m->raw_o, m->post, m->post_o, m->mark, X.L.bits);
				if (r) return r;
			}
			else {
				box_scatter_kernel<<<stream_grid(ctx, total), 256, 0, ctx->stream>>>(X.boxes, nboxes, X.values, total, P, m->zix, block_grid(m), m->raw, m->raw_o,
				                                                                     rm ? nullptr : m->post, rm ? nullptr : m->post_o, m->mark);
				TW_LAUNCH_CHECK(ctx);
			}
			if (rm) {
				TW_CUDA(ctx, cudaMemcpyAsync(m->work, m->raw, n*sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
				TW_CUDA(ctx, cudaMemcpyAsync(m->work_o, m->raw_o, n, cudaMemcpyDeviceToDevice, ctx->stream));
				int const r = enqueue_remove_unconnected(ctx, blocks, m->work, m->work_o, &P, X.f0, X.f1, X.cnt, X.changed); if (r) return r;
				if (list) {
					int const r2 = launch_module_kernel(ctx, K.diff_bits, stream_grid(ctx, n), 256u, (const float *)m->work, (const unsigned char *)m->work_o, m->post, m->post_o,
					                                    P, block_grid(m), m->mark, n, X.L.bits);
					if (r2) return r2;
				}
				else {
					diff_kernel<<<stream_grid(ctx, n), 256, 0, ctx->stream>>>(m->work, m->work_o, m->post, m->post_o, P, block_grid(m), m->mark, n);
					TW_LAUNCH_CHECK(ctx);
				}
			}
			if (list) {int const r = enqueue_change_list(ctx, m, X, CO, K); if (r) return r;}
		}
		if (m->nblocks) {list_marked_kernel<<<1, 1024, 0, ctx->stream>>>(m->mark, m->nblocks, m->marked); TW_LAUNCH_CHECK(ctx);}
		return enqueue_block_meshes(ctx, m, m->marked, X, d_vt, O.vcapacity, d_ix, O.tcapacity);
	});
}

extern "C" int tw_voxel_model_read(tw_voxel_model *m, float *raw, float *vals, uint8_t *outside) {
	tw_ctx *ctx = m ? m->ctx : nullptr;
	int rc = model_begin(ctx, m); if (rc) return rc;
	if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "the voxel model has no field yet (tw_voxel_model_build_launch)");
	size_t const n = (size_t)m->P.nx*m->P.ny*m->P.nz;
	TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, m->ev, 0)); // the model's jobs on the other contexts of the family
	if (raw) {TW_CUDA(ctx, cudaMemcpyAsync(raw, m->raw, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
	if (vals) {TW_CUDA(ctx, cudaMemcpyAsync(vals, m->post, n*sizeof(float), cudaMemcpyDefault, ctx->stream));}
	if (outside) {TW_CUDA(ctx, cudaMemcpyAsync(outside, m->post_o, n, cudaMemcpyDefault, ctx->stream));}
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return TW_OK;
}

// The read as a job: each requested array is copied from the model straight into device or page-locked memory, or into the launching context's pinned
// staging for a pageable destination, which the completing poll copies out. A box is one strided 3-D copy per array: rows of d voxels along z, w rows per
// slice (x), h slices (y), packed as the edit packs its values.
extern "C" int tw_voxel_model_read_launch(tw_ctx *ctx, tw_voxel_model *m, const tw_voxel_box *boxes, uint32_t nboxes, float *raw, float *vals, uint8_t *outside) {
	int rc = model_begin(ctx, m); if (rc) return rc;
	if (nboxes && !boxes) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_read_launch: null boxes with nboxes > 0");
	tw_voxel_post_params const &P = m->P;
	unsigned long long total = 0;
	std::vector<twi_box> B;
	rc = model_boxes(ctx, P, boxes, nboxes, B, &total); if (rc) return rc;
	if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "the voxel model has no field yet (tw_voxel_model_build_launch)");
	size_t const n = boxes ? (size_t)total : (size_t)P.nx*P.ny*P.nz;
	struct Arr {void *user; const void *src; size_t es; char *h;};
	Arr A[3] = {{raw, m->raw, sizeof(float), nullptr}, {vals, m->post, sizeof(float), nullptr}, {outside, m->post_o, 1, nullptr}};
	bool stage[3];
	for (int k = 0; k < 3; ++k) {stage[k] = A[k].user && n && !device_view(A[k].user);}
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {for (int k = 0; k < 3; ++k) {A[k].h = stage[k] ? c.take<char>(n*A[k].es) : nullptr;}}); if (rc) return rc;
	twi_job pending;
	pending.complete = [A0 = A[0], A1 = A[1], A2 = A[2], n](tw_ctx *) -> int {
		for (Arr const &a : {A0, A1, A2}) {if (a.h) memcpy(a.user, a.h, n*a.es);}
		return TW_OK;
	};
	return launch_model_job(ctx, m, std::move(pending), [&]() -> int {
		for (Arr const &a : A) {
			if (!a.user || !n) continue;
			char *dst = a.h ? a.h : (char *)a.user;
			if (!boxes) {TW_CUDA(ctx, cudaMemcpyAsync(dst, a.src, n*a.es, cudaMemcpyDefault, ctx->stream)); continue;}
			for (twi_box const &b : B) {
				cudaMemcpy3DParms q = {};
				q.srcPtr = make_cudaPitchedPtr(const_cast<void *>(a.src), (size_t)P.nz*a.es, P.nz, P.nx);
				q.srcPos = make_cudaPos((size_t)b.z*a.es, b.x, b.y);
				q.dstPtr = make_cudaPitchedPtr(dst + b.off*a.es, (size_t)b.d*a.es, b.d, b.w);
				q.extent = make_cudaExtent((size_t)b.d*a.es, b.w, b.h);
				q.kind = cudaMemcpyDefault;
				TW_CUDA(ctx, cudaMemcpy3DAsync(&q, ctx->stream));
			}
		}
		return TW_OK;
	});
}

// ------------------------------------------------------------------------------------------------ many small grids in one job (tw_voxel_build_batch_launch)
// The batch's kernels are the module tw_voxel_batch.cubin's (tw_voxel_batch.cu), each launched once over every grid through the device table of
// twi_vbatch_grid: sine tables (sine grids only), fill and flags, the flood (remove_unconnected grids only), mesh count, per-grid scan, mesh emit (grids with
// a capacity only). So a batch launches the same kernels for 1 grid as for 300.
//   device slot 0: [grid table | counts (3 per grid) | tables | sine coefficients | per grid: field (unless vals is device memory), flags, sine tables, zix_xy
//                  (host input), mesh words, block sums and offsets]
//   pinned:        [grid table | counts | tables | sine coefficients | per grid: zix_xy (host input)]
namespace {
struct BatchKernels {cudaKernel_t tables, fill, flood, count, scan, emit;};
int batch_kernels(tw_ctx *ctx, BatchKernels *K) {
	static const char *const names[] = {"tw_vbatch_tables_kernel", "tw_vbatch_fill_kernel", "tw_vbatch_flood_kernel", "tw_vbatch_mesh_count_kernel",
	                                    "tw_vbatch_mesh_scan_kernel", "tw_vbatch_mesh_emit_kernel"};
	cudaKernel_t k[6];
	int const rc = twi_module_kernels(ctx, "tw_voxel_batch.cubin", names, 6, k); if (rc) return rc;
	*K = BatchKernels{k[0], k[1], k[2], k[3], k[4], k[5]};
	return TW_OK;
}
// a refusal of entry i of a batch: the helper's message prefixed with the entry's kind and index
int entry_error(tw_ctx *ctx, const char *kind, uint32_t i, int rc) {
	std::string const msg = ctx->err;
	return tw_set_error(ctx, rc, "%s %u: %s", kind, i, msg.c_str());
}
int grid_error(tw_ctx *ctx, uint32_t i, int rc) {return entry_error(ctx, "grid", i, rc);}
// grid d's fill as the batch module reads it (F: nullptr for an input field): the mode, the epilogue and GLM parameters as twi_voxel_fill derives them, and
// in sine mode the coefficients as it stages them - at h_r (rdata420, or generated), read by the device at d_r
void vbatch_fill_params(const tw_voxel_params *F, const float *rdata420, float *h_r, const float *d_r, twi_vbatch_grid &d) {
	bool const sine = F && F->gen_mode == TW_MGEN_SINE;
	d.mode = !F ? TWI_VB_INPUT : sine ? TWI_VB_SINE : (F->gen_mode == TW_MGEN_PERLIN) ? TWI_VB_PERLIN : TWI_VB_SIMPLEX;
	memset(&d.E, 0, sizeof(d.E)); memset(&d.G, 0, sizeof(d.G));
	d.rdata = nullptr;
	for (int k = 0; k < 3; ++k) {d.s[k] = 0.0f; d.step[k] = 0.0f;}
	if (!F) return;
	d.E.zscale = F->zscale; d.E.normalize = F->normalize_to_1;
	d.E.atten_mode = F->atten_mode; d.E.atten_val = F->atten_val; d.E.inner_radius = F->atten_inner_radius;
	d.E.nx = F->nx; d.E.ny = F->ny; d.E.nz = F->nz;
	if (sine) {
		if (rdata420) {memcpy(h_r, rdata420, TW_N3D_RDATA*sizeof(float));} else {tw_noise3d_gen_sines(F->rseed1, F->rseed2, F->mag, F->freq, h_r);}
		d.rdata = d_r;
		for (int k = 0; k < 3; ++k) {d.s[k] = F->lo_pos[k] + F->offset[k]; d.step[k] = F->vsz[k];} // (lo_pos + offset), src/voxels.cpp:289
	}
	else {
		for (int k = 0; k < 3; ++k) {d.G.lo[k] = F->lo_pos[k]; d.G.vsz[k] = F->vsz[k]; d.G.off[k] = F->offset[k];}
		d.G.mag = F->mag; d.G.nfreq0 = (float)(0.25*F->freq);
		d.G.rx = F->rx; d.G.ry = F->ry; d.G.rz = F->rx - F->ry;
		d.G.octaves = F->octaves; d.G.perlin = (F->gen_mode == TW_MGEN_PERLIN);
	}
}
// the sine mode's axis tables of grid P, carved from c (none for another mode)
void vbatch_sine_tables(twi_carve &c, const tw_voxel_post_params &P, bool sine, twi_vbatch_grid &d) {
	d.xt = d.yt = d.zt = nullptr; d.xp = d.yp = d.zp = 0;
	if (!sine) return;
	d.xp = (P.nx + 31) & ~31u; d.yp = (P.ny + 31) & ~31u; d.zp = (P.nz + 31) & ~31u;
	d.xt = c.take<float>((size_t)NS*(d.xp + d.yp + d.zp)); d.yt = d.xt ? d.xt + (size_t)NS*d.xp : nullptr; d.zt = d.yt ? d.yt + (size_t)NS*d.yp : nullptr;
}
// the dynamic shared memory of the batch module's fill (the GLM tables, when a grid has a GLM fill) and flood (six bitsets of flood_words words)
int vbatch_smem(tw_ctx *ctx, const BatchKernels &K, bool any_glm, unsigned flood_words, size_t *lut_bytes, size_t *flood_bytes) {
	*lut_bytes = any_glm ? (size_t)twn2::LUT3D_N*twn2::SIMPLEX_LUT_COPIES*sizeof(float4) : 0; *flood_bytes = 6*sizeof(unsigned)*(size_t)flood_words;
	if (*lut_bytes) {TW_CUDA(ctx, cudaKernelSetAttributeForDevice(K.fill, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*lut_bytes, ctx->device));}
	if (*flood_bytes) {TW_CUDA(ctx, cudaKernelSetAttributeForDevice(K.flood, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*flood_bytes, ctx->device));}
	if (any_glm) {int const rc = twi_ensure_glm3_lut(ctx); if (rc) return rc;}
	return TW_OK;
}
} // namespace

extern "C" int tw_voxel_build_batch_launch(tw_ctx *ctx, const tw_voxel_build *grids, const tw_voxel_mesh *meshes, uint32_t n) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!grids || !meshes) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_build_batch_launch: null grids or meshes");
	if (n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_build_batch_launch: an empty batch");
	struct Grid {tw_voxel_build b; tw_voxel_post_params P; tw_voxel_params F; tw_voxel_mesh M; float *d_mv; uint32_t *d_mi; unsigned nvox, nb; bool fill, sine;};
	std::vector<Grid> G(n);
	bool any_glm = false, any_rm = false, any_cap = false;
	unsigned nsine = 0, flood_words = 0, fill_blocks = 0, mesh_blocks = 0;
	for (uint32_t i = 0; i < n; ++i) {
		Grid &g = G[i];
		g.b = grids[i];
		if (!g.b.post) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: post is required", i);
		g.P = *g.b.post;
		rc = validate(ctx, &g.P); if (rc) return grid_error(ctx, i, rc);
		if ((unsigned long long)g.P.nx*g.P.ny*g.P.nz > TWI_VB_MAX_VOXELS)
			return tw_set_error(ctx, TW_ERR_ARG, "grid %u: %ux%ux%u is more than 2^18 voxels (build it with tw_voxel_build_launch_ex)", i, g.P.nx, g.P.ny, g.P.nz);
		g.nvox = g.P.nx*g.P.ny*g.P.nz; g.nb = (g.nvox + MC_BLOCK - 1)/MC_BLOCK;
		g.fill = (g.b.fill != nullptr); g.sine = false;
		if (g.fill) {
			g.F = *g.b.fill;
			if (g.F.nx != g.P.nx || g.F.ny != g.P.ny || g.F.nz != g.P.nz)
				return tw_set_error(ctx, TW_ERR_ARG, "grid %u: the fill's grid %ux%ux%u differs from post's %ux%ux%u", i, g.F.nx, g.F.ny, g.F.nz, g.P.nx, g.P.ny, g.P.nz);
			size_t tab_bytes = 0;
			rc = twi_voxel_fill_check(ctx, &g.F, &tab_bytes); if (rc) return grid_error(ctx, i, rc);
			g.sine = (g.F.gen_mode == TW_MGEN_SINE);
			nsine += g.sine; any_glm = any_glm || !g.sine;
		}
		else if (!g.b.vals) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: vals is the input field when there is no fill", i);
		if (!g.b.edge_table256 || !g.b.tri_table256x16 || !g.b.edge_to_vals12x2) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: the welded mesh needs the three marching-cubes tables", i);
		if (g.b.edge_table256 != grids[0].edge_table256 || g.b.tri_table256x16 != grids[0].tri_table256x16 || g.b.edge_to_vals12x2 != grids[0].edge_to_vals12x2)
			return tw_set_error(ctx, TW_ERR_ARG, "grid %u: its marching-cubes tables are not grid 0's (a batch shares one set)", i);
		if (g.b.tris || g.b.capacity || g.b.ntris) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: a batch builds no triangle soup (tris, capacity and ntris must be NULL / 0)", i);
		g.M = meshes[i];
		rc = validate_mesh(ctx, &g.P, &g.M); if (rc) return grid_error(ctx, i, rc);
		g.d_mv = nullptr; g.d_mi = nullptr;
		if (g.M.verts && !(g.d_mv = (float *)device_view(g.M.verts))) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: mesh verts must be device or page-locked host memory", i);
		if (g.M.indices && !(g.d_mi = (uint32_t *)device_view(g.M.indices))) return tw_set_error(ctx, TW_ERR_ARG, "grid %u: mesh indices must be device or page-locked host memory", i);
		if (g.P.remove_unconnected > 0) {any_rm = true; flood_words = std::max(flood_words, (g.nvox + 31)/32);}
		any_cap = any_cap || g.M.vcapacity || g.M.tcapacity;
		fill_blocks += (g.nvox + TWI_VB_FILL_VOXELS - 1)/TWI_VB_FILL_VOXELS; mesh_blocks += g.nb;
	}
	BatchKernels K;
	rc = batch_kernels(ctx, &K); if (rc) return rc;
	size_t lut_bytes, flood_bytes;
	rc = vbatch_smem(ctx, K, any_glm, flood_words, &lut_bytes, &flood_bytes); if (rc) return rc;
	std::vector<twi_user<float>> V; std::vector<twi_user<const uint32_t>> Z;
	V.reserve(n); Z.reserve(n);
	for (Grid const &g : G) {V.emplace_back(g.b.vals, g.nvox); Z.emplace_back(g.b.zix_xy, (size_t)g.P.nx*g.P.ny);}
	twi_vbatch_grid *d_tab; unsigned long long *d_counts; char *tab; float *d_rdata = nullptr;
	std::vector<twi_vbatch_grid> D(n);
	rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {
		d_tab = c.take<twi_vbatch_grid>(n); d_counts = c.take<unsigned long long>(3*(size_t)n); tab = c.take<char>(MC_TAB_BYTES);
		if (nsine) {d_rdata = c.take<float>((size_t)nsine*TW_N3D_RDATA);}
		for (uint32_t i = 0; i < n; ++i) {
			Grid const &g = G[i];
			twi_vbatch_grid &d = D[i];
			V[i].take(c); d.flags = c.take<unsigned char>((size_t)g.nvox + 4);
			vbatch_sine_tables(c, g.P, g.sine, d);
			if (g.b.zix_xy) {Z[i].take(c);}
			d.words = c.take<unsigned>(g.nvox); d.vsums = c.take<unsigned>(g.nb); d.tsums = c.take<unsigned>(g.nb);
			d.voff = c.take<unsigned long long>(g.nb); d.toff = c.take<unsigned long long>(g.nb);
		}
	}); if (rc) return rc;
	twi_vbatch_grid *h_tab; unsigned long long *h_counts; char *h_mc; float *h_rdata = nullptr;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {
		h_tab = c.take<twi_vbatch_grid>(n); h_counts = c.take<unsigned long long>(3*(size_t)n); h_mc = c.take<char>(MC_TAB_BYTES);
		if (nsine) {h_rdata = c.take<float>((size_t)nsine*TW_N3D_RDATA);}
		for (twi_user<const uint32_t> &z : Z) {z.take_pinned(c);}
	}); if (rc) return rc;
	// the table: fill parameters as twi_voxel_fill derives them, sine coefficients as it stages them, the blocks' prefix sums
	unsigned fb = 0, mb = 0, si = 0;
	for (uint32_t i = 0; i < n; ++i) {
		Grid const &g = G[i];
		twi_vbatch_grid &d = D[i];
		d.P = g.P; d.n = g.nvox; d.fill_blk0 = fb; d.mesh_blk0 = mb;
		fb += (g.nvox + TWI_VB_FILL_VOXELS - 1)/TWI_VB_FILL_VOXELS; mb += g.nb;
		vbatch_fill_params(g.fill ? &g.F : nullptr, g.b.rdata420, h_rdata + (size_t)si*TW_N3D_RDATA, d_rdata + (size_t)si*TW_N3D_RDATA, d);
		si += g.sine;
		d.vals = V[i].d; d.zix = g.b.zix_xy ? Z[i].d : nullptr;
		d.verts = g.d_mv; d.vcap = g.M.vcapacity; d.indices = g.d_mi; d.tcap = g.M.tcapacity;
		d.counts = d_counts + 3*(size_t)i;
	}
	memcpy(h_tab, D.data(), (size_t)n*sizeof(twi_vbatch_grid));
	struct Out {uint64_t *nverts, *ntris, *changed;};
	std::vector<Out> outs(n);
	for (uint32_t i = 0; i < n; ++i) {outs[i] = Out{G[i].M.nverts, G[i].M.ntris, G[i].b.changed};}
	twi_job pending;
	pending.cancellable = true; // no cancellation point: a cancel changes nothing
	pending.complete = [h_counts, outs = std::move(outs)](tw_ctx *) -> int {
		for (size_t i = 0; i < outs.size(); ++i) {
			*outs[i].nverts = h_counts[3*i]; *outs[i].ntris = h_counts[3*i + 1];
			if (outs[i].changed) {*outs[i].changed = h_counts[3*i + 2];}
		}
		return TW_OK;
	};
	McTables const T = mc_tables(tab);
	twi_vbatch_grid const *const dt = d_tab;
	return twi_launch_job(ctx, std::move(pending), [&]() -> int {
		TW_CUDA(ctx, cudaMemsetAsync(d_counts, 0, 3*(size_t)n*sizeof(unsigned long long), ctx->stream));
		TW_CUDA(ctx, cudaMemcpyAsync(d_tab, h_tab, (size_t)n*sizeof(twi_vbatch_grid), cudaMemcpyHostToDevice, ctx->stream));
		if (nsine) {TW_CUDA(ctx, cudaMemcpyAsync(d_rdata, h_rdata, (size_t)nsine*TW_N3D_RDATA*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));}
		int r = mc_tables_upload(ctx, tab, grids[0].edge_table256, grids[0].tri_table256x16, grids[0].edge_to_vals12x2, h_mc); if (r) return r;
		for (uint32_t i = 0; i < n; ++i) {
			if (!G[i].fill) {r = V[i].in(ctx); if (r) return r;}
			r = Z[i].in(ctx); if (r) return r;
		}
		if (nsine) {r = launch_module_kernel_smem(ctx, K.tables, dim3(3, n), 64u, 0, dt, (const float *)ctx->d_sin_table); if (r) return r;}
		r = launch_module_kernel_smem(ctx, K.fill, dim3(fill_blocks), TWI_VB_FILL_THREADS, lut_bytes, dt, n, (const float4 *)ctx->d_glm3_lut); if (r) return r;
		if (any_rm) {r = launch_module_kernel_smem(ctx, K.flood, dim3(n), TWI_VB_FLOOD_THREADS, flood_bytes, dt); if (r) return r;}
		r = launch_module_kernel(ctx, K.count, mesh_blocks, (unsigned)MC_BLOCK, dt, n, T); if (r) return r;
		r = launch_module_kernel(ctx, K.scan, n, 1024u, dt); if (r) return r;
		if (any_cap) {r = launch_module_kernel(ctx, K.emit, mesh_blocks, (unsigned)MC_BLOCK, dt, n, T); if (r) return r;}
		for (uint32_t i = 0; i < n; ++i) {
			if (G[i].fill || G[i].P.remove_unconnected > 0) {r = V[i].out(ctx); if (r) return r;}
			if (G[i].b.outside) {TW_CUDA(ctx, cudaMemcpyAsync(G[i].b.outside, D[i].flags, G[i].nvox, cudaMemcpyDefault, ctx->stream));}
		}
		TW_CUDA(ctx, cudaMemcpyAsync(h_counts, d_counts, 3*(size_t)n*sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
		return TW_OK;
	});
}

// ------------------------------------------------------------------------------------------------ many small voxel models in one job (tw_voxel_model_*_batch_launch)
// The fill, the flags and the flood are tw_voxel_batch.cubin's kernels on twi_vbatch_grid descriptors that point at each model's own memory (raw / raw_o for
// the fill, post / post_o for the build's flood, work / work_o for an edit's); the rest is tw_voxel_model_batch.cubin's, each kernel launched once over
// every model through the device table of twi_vmb_model. Each model costs one event wait and one record: the job waits for the model's earlier jobs on any
// context of the family and orders its later ones.
//   upload (pinned -> device slot 0, one copy): [model table | batch-module table | sine coefficients | per model: boxes, values (edit), host field (build)]
//   download (device -> pinned, one copy):     [counts (8 words per model) | per model: the listed blocks' table]
//   device only:                                [per model: mesh words (slots x chunks x MC_BLOCK), launch block sums and offsets, sine tables | change bits]
namespace {
struct ModelBatchKernels {cudaKernel_t copy, scatter, diff, changes, marked, count, scan, emit;};
int model_batch_kernels(tw_ctx *ctx, ModelBatchKernels *K) {
	static const char *const names[] = {"tw_vmb_copy_kernel", "tw_vmb_box_scatter_kernel", "tw_vmb_diff_kernel", "tw_vmb_change_list_kernel",
	                                    "tw_vmb_list_marked_kernel", "tw_vmb_mesh_count_kernel", "tw_vmb_mesh_scan_kernel", "tw_vmb_mesh_emit_kernel"};
	cudaKernel_t k[8];
	int const rc = twi_module_kernels(ctx, "tw_voxel_model_batch.cubin", names, 8, k); if (rc) return rc;
	*K = ModelBatchKernels{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7]};
	return TW_OK;
}

// The refusals every entry shares: a model that is set, of ctx's family and device, at most TWI_VB_MAX_VOXELS, and not named by an earlier entry
int batch_model_check(tw_ctx *ctx, const tw_voxel_model *m, uint32_t i, std::vector<const tw_voxel_model *> &seen) {
	if (!m) return tw_set_error(ctx, TW_ERR_ARG, "model %u: model is required", i);
	int const rc = model_family(ctx, m); if (rc) return entry_error(ctx, "model", i, rc);
	tw_voxel_post_params const &P = m->P;
	if ((unsigned long long)P.nx*P.ny*P.nz > TWI_VB_MAX_VOXELS)
		return tw_set_error(ctx, TW_ERR_ARG, "model %u: %ux%ux%u is more than 2^18 voxels (use the single-model calls)", i, P.nx, P.ny, P.nz);
	if (std::find(seen.begin(), seen.end(), m) != seen.end()) return tw_set_error(ctx, TW_ERR_ARG, "model %u: the model is named twice in the batch", i);
	seen.push_back(m);
	return TW_OK;
}

// One model of a batch as the host sees it: its descriptor, its outputs and where the completing poll finds its counts and table
struct BatchModel {
	tw_voxel_model *m; twi_vmb_model d; tw_voxel_blocks_out O; uint64_t *nchanged;
	unsigned ng, nvb, nbb;                        // mesh, per-voxel and box launch blocks
	size_t table_off;                             // the model's table in the download segment, in entries
	const float *host_in;                         // a build's host field / an edit's values, staged in the upload
	std::vector<twi_box> B;
	bool sine;                                    // a build with a sine fill: its axis tables (vb) are in the device carve
	twi_vbatch_grid vb;                           // a build's fill descriptor
};

// The carve of a batch (see above) over models M with nvb batch-module descriptors and nsine sine fills; dev: the device carve (else pinned). Returns the
// upload's and download's bytes.
struct BatchCarve {twi_vmb_model *tab; twi_vbatch_grid *vb; float *rdata; unsigned long long *counts; tw_voxel_block_mesh *tables; unsigned *bits;
                   std::vector<char *> in; std::vector<twi_box *> boxes;};
void batch_carve(twi_carve &c, std::vector<BatchModel> &M, unsigned nvb, unsigned nsine, size_t ntable, size_t nwords, bool dev, BatchCarve &X,
                 size_t *up_bytes, size_t *down_bytes)
{
	size_t const n = M.size();
	X.in.assign(n, nullptr); X.boxes.assign(n, nullptr);
	X.tab = c.take<twi_vmb_model>(n); X.vb = nvb ? c.take<twi_vbatch_grid>(nvb) : nullptr; X.rdata = nsine ? c.take<float>((size_t)nsine*TW_N3D_RDATA) : nullptr;
	for (size_t i = 0; i < n; ++i) {
		BatchModel &b = M[i];
		if (!b.B.empty()) {X.boxes[i] = c.take<twi_box>(b.B.size());}
		if (b.host_in) {X.in[i] = c.take<char>((b.B.empty() ? (size_t)b.d.n : (size_t)b.d.total)*sizeof(float));}
	}
	*up_bytes = c.bytes;
	X.counts = c.take<unsigned long long>(8*n); X.tables = ntable ? c.take<tw_voxel_block_mesh>(ntable) : nullptr;
	*down_bytes = c.bytes - *up_bytes;
	X.bits = nullptr;
	if (!dev) return;
	for (BatchModel &b : M) {
		twi_vmb_model &d = b.d;
		vbatch_sine_tables(c, d.P, b.sine, b.vb);
		if (!b.ng) {d.words = d.vsums = d.tsums = nullptr; d.voff = d.toff = nullptr; continue;} // no block: the mesh kernels never reach the model
		d.words = c.take<unsigned>((size_t)b.ng*MC_BLOCK); d.vsums = c.take<unsigned>(b.ng); d.tsums = c.take<unsigned>(b.ng);
		d.voff = c.take<unsigned long long>(b.ng); d.toff = c.take<unsigned long long>(b.ng);
	}
	X.bits = nwords ? c.take<unsigned>(nwords) : nullptr;
}

// The shared part of both batch launches once the entries are validated: the models' launch blocks, the carve, the descriptors' scratch pointers, the job
// that unpacks the counts and tables. `vbatch` fills the batch-module descriptors (pinned) given the device carve; `enqueue` the kernels.
template <typename VBatch, typename Enqueue>
int launch_model_batch(tw_ctx *ctx, std::vector<BatchModel> &M, unsigned nvb, unsigned nsine, const ModelBatchKernels &K, VBatch &&vbatch, Enqueue &&enqueue) {
	size_t ntable = 0, nwords = 0;
	unsigned vb0 = 0, bb0 = 0, mb0 = 0;
	for (BatchModel &b : M) {
		twi_vmb_model &d = b.d;
		b.ng = d.nblocks*d.G.chunks; b.nvb = (d.n + TWI_VMB_VOX_PER_BLOCK - 1)/TWI_VMB_VOX_PER_BLOCK;
		b.nbb = (unsigned)((d.total + TWI_VMB_BOX_PER_BLOCK - 1)/TWI_VMB_BOX_PER_BLOCK);
		d.vox_blk0 = vb0; d.box_blk0 = bb0; d.mesh_blk0 = mb0;
		vb0 += b.nvb; bb0 += b.nbb; mb0 += b.ng;
		b.table_off = ntable; ntable += d.nblocks;
		nwords += d.nwords;
	}
	BatchCarve D, H;
	size_t up = 0, down = 0;
	int rc = twi_reserve_carve(ctx, 0, [&](twi_carve &c) {batch_carve(c, M, nvb, nsine, ntable, nwords, true, D, &up, &down);}); if (rc) return rc;
	rc = twi_reserve_carve(ctx, TWI_PINNED, [&](twi_carve &c) {batch_carve(c, M, nvb, nsine, ntable, nwords, false, H, &up, &down);}); if (rc) return rc;
	size_t bo = 0;
	for (size_t i = 0; i < M.size(); ++i) {
		BatchModel &b = M[i];
		twi_vmb_model &d = b.d;
		d.counts = D.counts + 8*i; d.table = d.nblocks ? D.tables + b.table_off : nullptr;
		if (d.nwords) {d.bits = D.bits + bo; bo += d.nwords;}
		if (!b.B.empty()) {memcpy(H.boxes[i], b.B.data(), b.B.size()*sizeof(twi_box)); d.boxes = D.boxes[i];}
		if (b.host_in) {
			size_t const nv = b.B.empty() ? (size_t)d.n : (size_t)d.total;
			memcpy(H.in[i], b.host_in, nv*sizeof(float));
			if (b.B.empty()) {d.in = (const float *)D.in[i];} else {d.values = (const float *)D.in[i];}
		}
		H.tab[i] = d;
	}
	vbatch(D, H);
	struct Out {tw_voxel_blocks_out O; uint64_t *nchanged; const unsigned long long *counts; const tw_voxel_block_mesh *table;};
	std::vector<Out> outs(M.size());
	for (size_t i = 0; i < M.size(); ++i) {outs[i] = Out{M[i].O, M[i].nchanged, H.counts + 8*i, M[i].d.nblocks ? H.tables + M[i].table_off : nullptr};}
	twi_job job; // not cancellable: it commits the models' state
	job.complete = [outs = std::move(outs)](tw_ctx *) -> int {
		for (Out const &o : outs) { // as model_job unpacks one model
			*o.O.nblocks = (uint32_t)o.counts[3]; *o.O.nverts = o.counts[0]; *o.O.ntris = o.counts[1];
			if (o.O.changed) {*o.O.changed = o.counts[2];}
			if (o.nchanged) {*o.nchanged = o.counts[4];}
			if (o.counts[3]) {memcpy(o.O.blocks, o.table, (size_t)o.counts[3]*sizeof(tw_voxel_block_mesh));}
		}
		return TW_OK;
	};
	unsigned const nm = (unsigned)M.size();
	for (BatchModel &b : M) {b.m->built = true;} // the job commits the models' state
	return twi_launch_job(ctx, std::move(job), [&]() -> int {
		for (BatchModel const &b : M) {TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, b.m->ev, 0));}
		TW_CUDA(ctx, cudaMemsetAsync(D.counts, 0, 8*M.size()*sizeof(unsigned long long), ctx->stream));
		if (nwords) {TW_CUDA(ctx, cudaMemsetAsync(D.bits, 0, nwords*sizeof(unsigned), ctx->stream));}
		TW_CUDA(ctx, cudaMemcpyAsync(D.tab, H.tab, up, cudaMemcpyHostToDevice, ctx->stream));
		int r = enqueue((const twi_vmb_model *)D.tab, nm, vb0, bb0, (const twi_vbatch_grid *)D.vb); if (r) return r;
		twi_vmb_model const *const dt = D.tab;
		if (mb0) {r = launch_module_kernel(ctx, K.count, mb0, (unsigned)MC_BLOCK, dt, nm); if (r) return r;}
		r = launch_module_kernel(ctx, K.scan, nm, 1024u, dt); if (r) return r;
		bool any_cap = false;
		for (BatchModel const &b : M) {any_cap = any_cap || b.d.vcap || b.d.tcap;}
		if (mb0 && any_cap) {r = launch_module_kernel(ctx, K.emit, mb0, (unsigned)MC_BLOCK, dt, nm); if (r) return r;}
		TW_CUDA(ctx, cudaMemcpyAsync(H.counts, D.counts, down, cudaMemcpyDeviceToHost, ctx->stream));
		for (BatchModel const &b : M) {TW_CUDA(ctx, cudaEventRecord(b.m->ev, ctx->stream));}
		return TW_OK;
	});
}

// the descriptor fields a model's build and edit share
void model_desc(tw_voxel_model *m, const tw_voxel_blocks_out &O, float *d_vt, uint32_t *d_ix, twi_vmb_model &d) {
	memset(&d, 0, sizeof(d));
	d.P = m->P; d.G = block_grid(m); d.T = mc_tables(m->tables);
	d.n = m->P.nx*m->P.ny*m->P.nz; d.nblocks = m->nblocks;
	d.raw = m->raw; d.post = m->post; d.work = m->work; d.raw_o = m->raw_o; d.post_o = m->post_o; d.work_o = m->work_o; d.mark = m->mark;
	d.zix = m->zix;
	d.verts = d_vt; d.vcap = O.vcapacity; d.indices = d_ix; d.tcap = O.tcapacity;
}
// a batch-module descriptor of model d's field vals and flags (fill_blk0, the fill and the counts set by the caller)
twi_vbatch_grid vbatch_desc(const twi_vmb_model &d, float *vals, unsigned char *flags) {
	twi_vbatch_grid g;
	memset(&g, 0, sizeof(g));
	g.P = d.P; g.n = d.n; g.vals = vals; g.flags = flags; g.zix = d.zix; g.counts = d.counts;
	return g;
}
} // namespace

extern "C" int tw_voxel_model_build_batch_launch(tw_ctx *ctx, const tw_voxel_model_build *builds, uint32_t n) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!builds) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_build_batch_launch: null builds");
	if (n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_build_batch_launch: an empty batch");
	std::vector<BatchModel> M(n);
	std::vector<tw_voxel_params> F(n);
	std::vector<const tw_voxel_model *> seen;
	bool any_glm = false;
	unsigned nsine = 0, nflood = 0, flood_words = 0, fill_blocks = 0;
	for (uint32_t i = 0; i < n; ++i) {
		tw_voxel_model_build const &e = builds[i];
		BatchModel &b = M[i];
		b.m = e.model; b.nchanged = nullptr; b.host_in = nullptr; b.sine = false;
		rc = batch_model_check(ctx, e.model, i, seen); if (rc) return rc;
		if ((e.fill != nullptr) == (e.vals != nullptr)) return tw_set_error(ctx, TW_ERR_ARG, "model %u: give either fill or vals", i);
		float *d_vt; uint32_t *d_ix;
		rc = validate_blocks_out(ctx, e.out, &d_vt, &d_ix); if (rc) return entry_error(ctx, "model", i, rc);
		b.O = *e.out;
		tw_voxel_post_params const &P = e.model->P;
		if (e.fill) {
			F[i] = *e.fill;
			if (F[i].nx != P.nx || F[i].ny != P.ny || F[i].nz != P.nz)
				return tw_set_error(ctx, TW_ERR_ARG, "model %u: the fill's grid %ux%ux%u differs from the model's %ux%ux%u", i, F[i].nx, F[i].ny, F[i].nz, P.nx, P.ny, P.nz);
			size_t tab_bytes = 0;
			rc = twi_voxel_fill_check(ctx, &F[i], &tab_bytes); if (rc) return entry_error(ctx, "model", i, rc);
			bool const sine = (F[i].gen_mode == TW_MGEN_SINE);
			nsine += sine; any_glm = any_glm || !sine; b.sine = sine;
		}
		model_desc(e.model, b.O, d_vt, d_ix, b.d);
		b.d.list = e.model->all;
		if (e.vals) {if (tw_is_device_ptr(e.vals)) {b.d.in = e.vals;} else {b.host_in = e.vals;}}
		if (P.remove_unconnected > 0) {++nflood; flood_words = std::max(flood_words, (b.d.n + 31)/32);}
		fill_blocks += (b.d.n + TWI_VB_FILL_VOXELS - 1)/TWI_VB_FILL_VOXELS;
	}
	BatchKernels VK; ModelBatchKernels K;
	rc = batch_kernels(ctx, &VK); if (rc) return rc;
	rc = model_batch_kernels(ctx, &K); if (rc) return rc;
	size_t lut_bytes, flood_bytes;
	rc = vbatch_smem(ctx, VK, any_glm, flood_words, &lut_bytes, &flood_bytes); if (rc) return rc;
	bool const any_in = std::any_of(M.begin(), M.end(), [](const BatchModel &b) {return b.d.in || b.host_in;});
	// batch-module descriptors: n for the fill (raw / raw_o), then one per flooded model (post / post_o)
	auto vbatch = [&](BatchCarve &D, BatchCarve &H) {
		unsigned fb = 0, si = 0, fl = 0;
		for (uint32_t i = 0; i < n; ++i) {
			twi_vmb_model const &d = M[i].d;
			twi_vbatch_grid g = vbatch_desc(d, M[i].m->raw, M[i].m->raw_o);
			g.counts = D.counts + 8*i;
			bool const fill = (builds[i].fill != nullptr), sine = fill && F[i].gen_mode == TW_MGEN_SINE;
			vbatch_fill_params(fill ? &F[i] : nullptr, builds[i].rdata420, H.rdata + (size_t)si*TW_N3D_RDATA, D.rdata + (size_t)si*TW_N3D_RDATA, g);
			si += sine;
			twi_vbatch_grid const &t = M[i].vb;
			g.xt = t.xt; g.yt = t.yt; g.zt = t.zt; g.xp = t.xp; g.yp = t.yp; g.zp = t.zp;
			g.fill_blk0 = fb; fb += (d.n + TWI_VB_FILL_VOXELS - 1)/TWI_VB_FILL_VOXELS;
			H.vb[i] = g;
			if (d.P.remove_unconnected > 0) {
				twi_vbatch_grid f = vbatch_desc(d, M[i].m->post, M[i].m->post_o);
				f.counts = D.counts + 8*i;
				H.vb[n + fl++] = f;
			}
		}
	};
	auto enqueue = [&](const twi_vmb_model *dt, unsigned nm, unsigned vox_blocks, unsigned, const twi_vbatch_grid *vb) -> int {
		int r;
		if (any_in) {r = launch_module_kernel(ctx, K.copy, vox_blocks, TWI_VMB_VOX_THREADS, dt, nm, (int)TWI_VMB_COPY_IN); if (r) return r;}
		if (nsine) {r = launch_module_kernel_smem(ctx, VK.tables, dim3(3, n), 64u, 0, vb, (const float *)ctx->d_sin_table); if (r) return r;}
		r = launch_module_kernel_smem(ctx, VK.fill, dim3(fill_blocks), TWI_VB_FILL_THREADS, lut_bytes, vb, n, (const float4 *)ctx->d_glm3_lut); if (r) return r;
		r = launch_module_kernel(ctx, K.copy, vox_blocks, TWI_VMB_VOX_THREADS, dt, nm, (int)TWI_VMB_COPY_POST); if (r) return r;
		if (nflood) {r = launch_module_kernel_smem(ctx, VK.flood, dim3(nflood), TWI_VB_FLOOD_THREADS, flood_bytes, vb + n); if (r) return r;}
		return TW_OK;
	};
	return launch_model_batch(ctx, M, n + nflood, nsine, K, vbatch, enqueue);
}

extern "C" int tw_voxel_model_edit_batch_launch(tw_ctx *ctx, const tw_voxel_model_edit *edits, uint32_t n) {
	int rc = twi_begin(ctx); if (rc) return rc;
	if (!edits) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_edit_batch_launch: null edits");
	if (n == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_model_edit_batch_launch: an empty batch");
	std::vector<BatchModel> M(n);
	std::vector<const tw_voxel_model *> seen;
	unsigned nflood = 0, flood_words = 0;
	bool any_list = false;
	for (uint32_t i = 0; i < n; ++i) {
		tw_voxel_model_edit const &e = edits[i];
		BatchModel &b = M[i];
		b.m = e.model; b.nchanged = nullptr; b.host_in = nullptr; b.sine = false;
		rc = batch_model_check(ctx, e.model, i, seen); if (rc) return rc;
		if (e.nboxes && (!e.boxes || !e.values)) return tw_set_error(ctx, TW_ERR_ARG, "model %u: null boxes or values", i);
		float *d_vt; uint32_t *d_ix;
		rc = validate_blocks_out(ctx, e.out, &d_vt, &d_ix); if (rc) return entry_error(ctx, "model", i, rc);
		b.O = *e.out;
		ChangeOut CO;
		if (e.ch) {rc = validate_changes(ctx, e.ch, &CO); if (rc) return entry_error(ctx, "model", i, rc);}
		tw_voxel_model *const m = e.model;
		unsigned long long total = 0;
		rc = model_boxes(ctx, m->P, e.boxes, e.nboxes, b.B, &total); if (rc) return entry_error(ctx, "model", i, rc);
		if (!m->built) return tw_set_error(ctx, TW_ERR_STATE, "model %u: the voxel model has no field yet (tw_voxel_model_build_launch)", i);
		model_desc(m, b.O, d_vt, d_ix, b.d);
		twi_vmb_model &d = b.d;
		d.list = m->marked; d.nboxes = e.nboxes; d.total = total;
		if (total) {b.host_in = e.values;}
		d.flood = (m->P.remove_unconnected > 0 && total) ? 1 : 0;
		if (d.flood) {++nflood; flood_words = std::max(flood_words, (d.n + 31)/32);}
		if (e.ch) {
			b.nchanged = CO.nchanged;
			if (total) { // only an edit with boxes can change a voxel: without them the count stays 0
				d.nwords = (d.n + 31)/32; any_list = true; // launch_model_batch carves the bits
				d.ch_index = CO.index; d.ch_vals = CO.vals; d.ch_outside = CO.outside; d.ch_cap = CO.capacity;
			}
		}
	}
	BatchKernels VK; ModelBatchKernels K;
	if (nflood) {rc = batch_kernels(ctx, &VK); if (rc) return rc;}
	rc = model_batch_kernels(ctx, &K); if (rc) return rc;
	size_t lut_bytes = 0, flood_bytes = 0;
	if (nflood) {rc = vbatch_smem(ctx, VK, false, flood_words, &lut_bytes, &flood_bytes); if (rc) return rc;}
	// batch-module descriptors: one per flooded model (work / work_o)
	auto vbatch = [&](BatchCarve &D, BatchCarve &H) {
		unsigned fl = 0;
		for (uint32_t i = 0; i < n; ++i) {
			if (!M[i].d.flood) continue;
			twi_vbatch_grid f = vbatch_desc(M[i].d, M[i].m->work, M[i].m->work_o);
			f.counts = D.counts + 8*i;
			H.vb[fl++] = f;
		}
	};
	auto enqueue = [&](const twi_vmb_model *dt, unsigned nm, unsigned vox_blocks, unsigned box_blocks, const twi_vbatch_grid *vb) -> int {
		int r;
		if (box_blocks) {r = launch_module_kernel(ctx, K.scatter, box_blocks, TWI_VMB_BOX_THREADS, dt, nm); if (r) return r;}
		if (nflood) {
			r = launch_module_kernel(ctx, K.copy, vox_blocks, TWI_VMB_VOX_THREADS, dt, nm, (int)TWI_VMB_COPY_WORK); if (r) return r;
			r = launch_module_kernel_smem(ctx, VK.flood, dim3(nflood), TWI_VB_FLOOD_THREADS, flood_bytes, vb); if (r) return r;
			r = launch_module_kernel(ctx, K.diff, vox_blocks, TWI_VMB_VOX_THREADS, dt, nm); if (r) return r;
		}
		if (any_list) {r = launch_module_kernel(ctx, K.changes, nm, 1024u, dt); if (r) return r;}
		return launch_module_kernel(ctx, K.marked, nm, 1024u, dt);
	};
	return launch_model_batch(ctx, M, nflood, 0, K, vbatch, enqueue);
}
