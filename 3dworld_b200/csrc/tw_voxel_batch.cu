// tw_voxel_batch.cu - many small voxel grids built in one job (tw_voxel_build_batch_launch): fill and outside flags, remove_unconnected and the welded mesh of
// every grid, each step one launch over all grids. Built as its own sm_90a module (build.py: tw_voxel_batch.cubin beside the library) that tw_voxel_post.cu
// loads on first use, so the library's own kernels - whose code the tests pin - stay exactly as they are. The kernels, declared in tw_voxel_batch.h, are
// extern "C" so the loader finds them by name; each walks the grids through that header's table of twi_vbatch_grid, finding a launch block's grid by a
// binary search over the grids' first blocks. The arithmetic is the library's: the fill's epilogue, sine look-up and GLM fBm come from tw_voxel_fill.cuh, the outside flag and the
// welded mesh's cube from tw_voxel_mc.cuh.
//   tw_vbatch_tables_kernel  gen_xyz_vals of the sine-mode grids, one thread per (grid, axis, term)
//   tw_vbatch_fill_kernel    per voxel: the fill (or the input field), the epilogue, the outside flag; blocks of TWI_VB_FILL_VOXELS consecutive voxels
//   tw_vbatch_flood_kernel   remove_unconnected, one CTA per grid, the flood as bitsets in shared memory (below)
//   tw_vbatch_mesh_count_kernel / tw_vbatch_mesh_scan_kernel / tw_vbatch_mesh_emit_kernel   the welded mesh: mesh_kernel's count, the block scan of
//                            each grid (one CTA per grid) and the emit
#include "tw_voxel_batch.h"
#include "tw_voxel_batch_util.cuh"

// gen_xyz_vals (tw_voxel.cu's xyz_tables_kernel) of grid blockIdx.y, axis blockIdx.x, term threadIdx.x: t[k*pitch + i] (x pre-multiplied by mag), i walked
// serially (val += step is a serial fp32 sum)
extern "C" __global__ void tw_vbatch_tables_kernel(const twi_vbatch_grid *__restrict__ grids, const float *__restrict__ sin_tab) {
	int const k = threadIdx.x, d = blockIdx.x;
	twi_vbatch_grid const &g = grids[blockIdx.y];
	if (k >= NS || g.mode != TWI_VB_SINE) return;
	unsigned const n = (d == 0) ? g.P.nx : (d == 1) ? g.P.ny : g.P.nz, pitch = (d == 0) ? g.xp : (d == 1) ? g.yp : g.zp;
	float *t = (d == 0) ? g.xt : (d == 1) ? g.yt : g.zt;
	float val = g.s[d];
	float const step = g.step[d];
	unsigned const index2 = 7*k + 2*d;
	float const f = __ldg(g.rdata + index2 + 1), ph = __ldg(g.rdata + index2 + 2), mag = __ldg(g.rdata + 7*k);
	for (unsigned i = 0; i < n; ++i) {
		float v = sinf_lut(sin_tab, f*val + ph);
		if (d == 0) {v *= mag;}
		t[(size_t)k*pitch + i] = v;
		val += step;
	}
}

// The field and the outside flags of every grid. Sine: val = sum_k (xv[k]*yv[k])*zv[k] in k order, each product rounded, as voxel_sine_kernel sums it; GLM:
// glm_value on the block's staged table (lut: the context's simplex table, the perlin table LUT3D_N entries after it), as voxel_glm_kernel. Dynamic shared
// memory: the table when the batch has a GLM grid, else none.
extern "C" __global__ void __launch_bounds__(TWI_VB_FILL_THREADS)
tw_vbatch_fill_kernel(const twi_vbatch_grid *__restrict__ grids, unsigned ngrids, const float4 *__restrict__ lut)
{
	extern __shared__ float4 lut_s[];
	unsigned const gi = find_grid(grids, ngrids, blockIdx.x, [](const twi_vbatch_grid &g) {return g.fill_blk0;});
	twi_vbatch_grid const &g = grids[gi];
	int const mode = g.mode;
	unsigned L = 0;
	if (mode == TWI_VB_SIMPLEX || mode == TWI_VB_PERLIN) { // uniform over the block
		const float4 *const src = lut + ((mode == TWI_VB_PERLIN) ? twn2::LUT3D_N : 0);
		for (int e = threadIdx.x; e < twn2::LUT3D_N*twn2::SIMPLEX_LUT_COPIES; e += blockDim.x) {lut_s[e] = __ldg(src + e/twn2::SIMPLEX_LUT_COPIES);}
		__syncthreads();
		L = twn2::simplex_lut_base(lut_s, threadIdx.x);
		asm volatile("" : "+r"(L) :: "memory"); // table loads depend on L, defined after the barrier
	}
	tw_voxel_post_params const P = g.P;
	unsigned const i0 = (blockIdx.x - g.fill_blk0)*TWI_VB_FILL_VOXELS, i1 = min(g.n, i0 + TWI_VB_FILL_VOXELS);
	for (unsigned i = i0 + threadIdx.x; i < i1; i += TWI_VB_FILL_THREADS) {
		unsigned const z = i % P.nz, xy = i / P.nz, x = xy % P.nx, y = xy / P.nx;
		float val;
		if (mode == TWI_VB_SINE) {
			float acc = 0.0f;
			for (int k = 0; k < NS; ++k) {
				float const xyv = __fmul_rn(__ldg(g.xt + (size_t)k*g.xp + x), __ldg(g.yt + (size_t)k*g.yp + y));
				acc = __fadd_rn(__fmul_rn(xyv, __ldg(g.zt + (size_t)k*g.zp + z)), acc);
			}
			val = epilogue(acc, x, y, z, g.E);
		}
		else if (mode == TWI_VB_SIMPLEX) {val = epilogue(glm_value<false>(g.G, glm_pos(g.G, 0, x), glm_pos(g.G, 1, y), glm_pos(g.G, 2, z), L), x, y, z, g.E);}
		else if (mode == TWI_VB_PERLIN)  {val = epilogue(glm_value<true >(g.G, glm_pos(g.G, 0, x), glm_pos(g.G, 1, y), glm_pos(g.G, 2, z), L), x, y, z, g.E);}
		else {val = g.vals[i];}
		if (mode != TWI_VB_INPUT) {g.vals[i] = val;}
		g.flags[i] = outside_flag(val, i, x, y, z, P, g.zix);
	}
}

// ---- remove_unconnected in one CTA per grid ----
// The reached set R of a flood is the least fixpoint of R = seeds | (dilate6(R) & claimable): every voxel joined to a seed by a 6-connected path whose voxels
// after the seed are claimable - exactly what flood_fill_kernel's generations (and the reference's stack) reach, in whatever order. Here the grid's claimable
// voxels and R are bitsets in shared memory over the linear index i = z + (x + y*nx)*nz (bit i & 31 of word i >> 5), so a z step is a shift by 1, an x step
// by nz and a y step by nx*nz. C: claimable; CU / CD: claimable and not at z = 0 / z = nz-1 (may take R from z-1 / z+1); CX0 / CX1: the same for x. Each round
// every thread ORs each of its words with its six shifted neighbours under those masks, then fills the z runs inside the word in one step (a carry chain
// up, and one down on the reversed word); rounds repeat until a __syncthreads_or sees no word change. Words another thread is writing may be read old or
// new: R only grows, so either is a subset of the fixpoint, and a round that changes nothing has read the final words.
namespace {

__device__ __forceinline__ unsigned rd(const volatile unsigned *R, int w, int W) {return (w >= 0 && w < W) ? R[w] : 0u;}
// word w of R shifted so that bit i holds bit i - s (from_lo) / bit i + s (from_hi), zeros shifted in
__device__ __forceinline__ unsigned from_lo(const volatile unsigned *R, int w, int W, unsigned s) {
	int const q = (int)(s >> 5); unsigned const r = s & 31;
	unsigned const a = rd(R, w - q, W);
	return r ? ((a << r) | (rd(R, w - q - 1, W) >> (32 - r))) : a;
}
__device__ __forceinline__ unsigned from_hi(const volatile unsigned *R, int w, int W, unsigned s) {
	int const q = (int)(s >> 5); unsigned const r = s & 31;
	unsigned const a = rd(R, w + q, W);
	return r ? ((a >> r) | (rd(R, w + q + 1, W) << (32 - r))) : a;
}
// bits of t's word reached upwards through m: bit i joins when bit i - 1 is in t or joined and bit i is in m (bit 0 never; carries out of the word are left
// to the next round's shifts). With q = m >> 1 the recurrence c_i = q_{i-1} & (t_{i-1} | c_{i-1}) is the carry chain of q + (t & q).
__device__ __forceinline__ unsigned run_up(unsigned t, unsigned m) {unsigned const q = m >> 1, b = t & q; return t | ((q + b) ^ q ^ b);}

} // namespace

// Seeds as enqueue_remove_unconnected places them: pass 0 the centre voxel (centre_seed) or the inside voxels under the mesh, and with keep_at_edge the
// scene-edge columns' voxels that are not outside; pass 1 (remove_unconnected > 2) the top plane's voxels that are not inside, and nothing at all happens in
// pass 1 without one. The finish is flood_finish_kernel's: pass 0 turns unreached inside voxels (flag 0) outside, pass 1 unreached outside voxels (flag 1)
// inside, each with the value make_voxel_outside / make_voxel_inside gives. counts[2] = the voxels flipped. Dynamic shared memory: six bitsets of the largest
// flooded grid's words.
extern "C" __global__ void __launch_bounds__(TWI_VB_FLOOD_THREADS) tw_vbatch_flood_kernel(const twi_vbatch_grid *__restrict__ grids) {
	extern __shared__ unsigned bits[];
	twi_vbatch_grid const &g = grids[blockIdx.x];
	tw_voxel_post_params const P = g.P;
	if (P.remove_unconnected <= 0) return;
	unsigned const n = g.n, nz = P.nz, nxnz = P.nx*P.nz;
	int const W = (int)((n + 31) >> 5);
	unsigned *const Rw = bits, *const C = Rw + W, *const CU = C + W, *const CD = CU + W, *const CX0 = CD + W, *const CX1 = CX0 + W;
	volatile unsigned *const R = Rw;
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	float *const vals = g.vals;
	unsigned char *const flags = g.flags;
	unsigned long long flipped = 0;
	for (int pass = 0; pass < ((P.remove_unconnected > 2) ? 2 : 1); ++pass) {
		bool any_seed = false;
		for (int w = (int)warp; w < W; w += TWI_VB_FLOOD_THREADS/32) { // a warp's lanes are one word's 32 voxels
			unsigned const i = (unsigned)w*32 + lane;
			bool const valid = (i < n);
			unsigned char const o = valid ? flags[i] : (unsigned char)0;
			unsigned const z = i % nz, xy = i / nz, x = xy % P.nx, y = xy / P.nx;
			bool seed;
			if (pass == 0) {
				seed = P.centre_seed ? (x == P.nx/2 && y == P.ny/2 && z == nz/2) : (o == TW_VOX_UNDER_MESH);
				if (P.keep_at_edge && (x == 0 || x + 1 == P.nx || y == 0 || y + 1 == P.ny) && o != 1) {seed = true;}
			}
			else {seed = (z == nz - 1 && o != 0);}
			seed = seed && valid;
			bool const claim = valid && o == (unsigned char)pass;
			unsigned const s = __ballot_sync(0xffffffffu, seed), c = __ballot_sync(0xffffffffu, claim);
			unsigned const cu = __ballot_sync(0xffffffffu, claim && z != 0), cd = __ballot_sync(0xffffffffu, claim && z != nz - 1);
			unsigned const c0 = __ballot_sync(0xffffffffu, claim && x != 0), c1 = __ballot_sync(0xffffffffu, claim && x != P.nx - 1);
			if (lane == 0) {Rw[w] = s; C[w] = c; CU[w] = cu; CD[w] = cd; CX0[w] = c0; CX1[w] = c1;}
			any_seed = any_seed || s != 0;
		}
		if (!__syncthreads_or(any_seed) && pass == 1) break; // remove_interior_holes without a seed on the top plane changes nothing
		bool grew;
		do {
			grew = false;
			for (int w = (int)threadIdx.x; w < W; w += TWI_VB_FLOOD_THREADS) {
				unsigned const r = R[w];
				unsigned t = r | (from_lo(R, w, W, 1) & CU[w]) | (from_hi(R, w, W, 1) & CD[w]) | (from_lo(R, w, W, nz) & CX0[w]) | (from_hi(R, w, W, nz) & CX1[w])
				               | ((from_lo(R, w, W, nxnz) | from_hi(R, w, W, nxnz)) & C[w]);
				t = run_up(t, CU[w]);
				t = __brev(run_up(__brev(t), __brev(CD[w])));
				if (t != r) {R[w] = t; grew = true;}
			}
		} while (__syncthreads_or(grew));
		for (unsigned i = threadIdx.x; i < n; i += TWI_VB_FLOOD_THREADS) {
			unsigned char const o = flags[i];
			if (o != (unsigned char)pass || ((R[i >> 5] >> (i & 31)) & 1u)) continue;
			if (pass == 0) {flags[i] = 1; vals[i] = P.isolevel - (P.invert ? -VOX_TOLERANCE : VOX_TOLERANCE);} // make_voxel_outside
			else           {flags[i] = 0; vals[i] = P.isolevel + (P.invert ? -VOX_TOLERANCE : VOX_TOLERANCE);} // make_voxel_inside
			++flipped;
		}
		__syncthreads(); // the flags pass 1 seeds from
	}
	for (int o = 16; o > 0; o >>= 1) {flipped += __shfl_xor_sync(0xffffffffu, flipped, o);}
	if (lane == 0 && flipped) {atomicAdd(g.counts + 2, flipped);}
}

// ---- the welded mesh ----
namespace {
// One MC_BLOCK-cube block blk of a grid's welded mesh - mesh_kernel's body (tw_voxel_post.cu) on the grid's own words, sums and offsets: count (EMIT false)
// stores the per-cube words and the block's sums at vsums[blk] / tsums[blk]; emit writes the block's vertices and triangles from voff[blk] / toff[blk],
// nothing at or past vcap / tcap.
template<bool EMIT>
__device__ __forceinline__ void mesh_block(const twi_vbatch_grid &g, const McTables &T, unsigned blk) {
	__shared__ unsigned warp_sums[MC_BLOCK/32];
	__shared__ unsigned char s_edge[12], s_look[12];
	mesh_edge_tables(T.edge_to_vals, s_edge, s_look);
	tw_voxel_post_params const P = g.P;
	size_t const n = g.n, i = (size_t)blk*MC_BLOCK + threadIdx.x;
	MeshCube m;
	m.mask = 0;
	unsigned cnt = 0; // owned vertices << 16 | kept triangles
	if (i < n) {
		unsigned const z = (unsigned)(i % P.nz);
		size_t const xy = i / P.nz;
		unsigned const nt = cube_mesh<EMIT>(g.vals, g.flags, P, T, s_edge, s_look, (unsigned)(xy % P.nx), (unsigned)(xy / P.nx), z, (unsigned)i, m);
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
		if (!EMIT && lane == 31) {g.vsums[blk] = wi >> 16; g.tsums[blk] = wi & 0xffffu;}
	}
	__syncthreads();
	unsigned const excl = warp_sums[warp] + (incl - cnt);
	if (!EMIT) {
		if (i < n) {g.words[i] = (excl & 0xffff0000u) | m.mask;}
		return;
	}
	if (i >= n) return;
	unsigned long long const vbase = g.voff[blk] + (excl >> 16);
	for (unsigned mk = m.mask; mk; mk &= mk - 1) {
		unsigned const e = __ffs(mk) - 1;
		unsigned long long const slot = vbase + __popc(m.mask & ((1u << e) - 1));
		if (slot < g.vcap) {float *o = g.verts + 3*slot; o[0] = m.vlist[e][0]; o[1] = m.vlist[e][1]; o[2] = m.vlist[e][2];}
	}
	unsigned long long const tbase = g.toff[blk] + (excl & 0xffffu);
	for (unsigned k = 0; k < (cnt & 0xffffu); ++k) {
		unsigned long long const slot = tbase + k;
		if (slot >= g.tcap) break;
		for (unsigned v = 0; v < 3; ++v) {
			unsigned const e = m.tri[k][v], owner = m.own[e], w = __ldg(g.words + owner);
			g.indices[3*slot + v] = (uint32_t)(g.voff[owner / MC_BLOCK] + (w >> 16) + __popc(w & 0xfffu & ((1u << m.oj[e]) - 1)));
		}
	}
}

} // namespace

extern "C" __global__ void __launch_bounds__(MC_BLOCK) tw_vbatch_mesh_count_kernel(const twi_vbatch_grid *__restrict__ grids, unsigned ngrids, McTables T) {
	unsigned const gi = find_grid(grids, ngrids, blockIdx.x, [](const twi_vbatch_grid &g) {return g.mesh_blk0;});
	mesh_block<false>(grids[gi], T, blockIdx.x - grids[gi].mesh_blk0);
}

// one CTA per grid: voff / toff of its blocks, counts[0] / counts[1] = its vertices and triangles
extern "C" __global__ void __launch_bounds__(1024) tw_vbatch_mesh_scan_kernel(const twi_vbatch_grid *__restrict__ grids) {
	twi_vbatch_grid const &g = grids[blockIdx.x];
	unsigned const nb = (g.n + MC_BLOCK - 1)/MC_BLOCK;
	unsigned long long const nv = scan_sums(g.vsums, nb, g.voff), nt = scan_sums(g.tsums, nb, g.toff);
	if (threadIdx.x == 0) {g.counts[0] = nv; g.counts[1] = nt;}
}

// grids without capacities write nothing, as the single build launches no emit pass for them
extern "C" __global__ void __launch_bounds__(MC_BLOCK) tw_vbatch_mesh_emit_kernel(const twi_vbatch_grid *__restrict__ grids, unsigned ngrids, McTables T) {
	unsigned const gi = find_grid(grids, ngrids, blockIdx.x, [](const twi_vbatch_grid &g) {return g.mesh_blk0;});
	twi_vbatch_grid const &g = grids[gi];
	if (g.vcap == 0 && g.tcap == 0) return;
	mesh_block<true>(g, T, blockIdx.x - g.mesh_blk0);
}
