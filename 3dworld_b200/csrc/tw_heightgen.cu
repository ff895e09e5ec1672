// tw_heightgen.cu - 2-D height generation kernels (sm_90a).
// Replaces mesh_xy_grid_cache_t::{build_arrays, enable_glaciate, eval_index} (src/mesh_gen.cpp:588-650,754-792) and
// get_noise_zval/gen_noise (src/mesh_gen.cpp:706-751) evaluated over a whole grid (or a batch of tiles).
//
// Kernels:
//   sine_tables_kernel   build_arrays sine branch (:604-626) + enable_glaciate cos terms (:640-650); k-major tables, LUT sin/cos
//   sine_grid_kernel     eval_index sine branch (:766-781): z = sum_k X[k][x]*Y[k][y], sequential fp32 sum, register-tiled 4x4 per thread,
//                        X/Y panels staged in shared memory; fused shape/postproc/glaciate/sine-bias/volcano + min/max
//   noise_grid2_kernel   eval_index noise branch (:761-764 -> get_noise_zval): fBm of simplex/perlin, optional domain warp, two cells per
//                        thread with the hash/gradient table of tw_noise2.cuh in shared memory; fused postproc/scale/
//                        glaciate/sine-bias/volcano + min/max. Pure FP32 ALU work: 4 B/cell of HBM traffic. (the shipped kernel)
//   noise_grid_kernel    the same one cell per thread in scalar arithmetic, no table: A/B reference (env TW_NOISE_SCALAR) and the
//                        literal fallback for astronomically distant lattice coordinates
//   points_kernel        eval_mesh_sin_terms / eval_mesh_sin_terms_scaled / get_exact_zval for batches of arbitrary points (:797-847)
// All arithmetic keeps the reference's rounding sequence (this TU is compiled with -fmad=false; see tw_noise.cuh).
#include "tw_internal.h"
#include <unordered_map>
#include <vector>
#include <algorithm>
#include "tw_noise.cuh"
#include "tw_noise2.cuh"
#include <stdlib.h>

namespace {

constexpr int F_TABLE = TW_F_TABLE_SIZE;

__device__ __forceinline__ float sinf_lut(const float *__restrict__ tab, float v) { // SINF, src/sinf.h:13-14
	return (v < 0.0f) ? -__ldg(tab + (tw_x86_f2i(TW_SSCALE*(-v))&(TW_TSIZE-1))) : __ldg(tab + (tw_x86_f2i(TW_SSCALE*v)&(TW_TSIZE-1)));
}
__device__ __forceinline__ float cosf_lut(const float *__restrict__ tab, float v) { // COSF, src/sinf.h:15
	return __ldg(tab + TW_TSIZE + (tw_x86_f2i(TW_SSCALE*fabsf(v))&(TW_TSIZE-1)));
}
__device__ __forceinline__ float smin(float a, float b) {return (b < a) ? b : a;} // std::min
__device__ __forceinline__ float smax(float a, float b) {return (a < b) ? b : a;} // std::max

// Everything a cell needs after the raw noise / sine sum, passed by value to the kernels (constant bank).
struct PostParams {
	tw_hmap_params h;
	int   shape;                 // apply_noise_shape_final (sine path only)
	int   need_postproc;         // hmap_params_t::need_postproc()
	int   enable_glaciate;       // do_glaciate (enable_glaciate() called)
	int   glaciate;              // GLACIATE global
	float zmax_est, zmax_est2, zmax_est2_inv, custom_exp;
	int   sine_on;               // hmap.sine_mag > 0
	float sm_scale, sm_freq, sine_offset; // sine_mag*mszi, mesh_scale*sine_freq, sine_bias*mszi
	int   volcano_on;
	float volcano_freq;          // mesh_scale/volcano_width
	float mesh_scale_z_inv;
	float mdx, mdy, dx_inv, dy_inv; // grid step, DX_VAL_INV, DY_VAL_INV
	const unsigned *tile_perm;   // tile batches: tile z of the launch is written to slot tile_perm[z] of `out` (nullptr: slot z) - the heaviest-first pipeline generates in
	                             // schedule order but stores every tile at its caller-visible index
	unsigned ngroups;            // paired noise kernels: number of chunk groups (blockDim x NCH x 2 cells each) in the band being generated
	unsigned skip_x0, skip_y0, skip_w, skip_h; // cells [skip_x0, +skip_w) x [skip_y0, +skip_h) of every grid are left unwritten (skip_w == 0: none): the
	                             // inside of an AO context grid, which calc_mesh_ao_lighting overwrites with the tile's zvals (src/tiled_mesh.cpp:627)
};

__device__ __forceinline__ float postproc_noise_zval(float z, const tw_hmap_params &h) { // src/mesh_gen.cpp:555-562
	if (z > h.plat_bot) {z = h.plat_bot + h.plat_h*(z - h.plat_bot) + smin(h.plat_max, h.plat_s*(z - h.plat_bot));}
	if (z > h.crat_h  ) {z = h.crat_h - h.crat_s*(z - h.crat_h);}
	if (z > h.crack_lo && z < h.crack_hi) {z -= h.crack_d*smin(z - h.crack_lo, h.crack_hi - z);}
	return z;
}

__device__ __forceinline__ float volcano_height(float xi, float yi, const PostParams &P, const float *__restrict__ tab) { // src/mesh_gen.cpp:364-372
	float const x = P.volcano_freq*xi, y = P.volcano_freq*yi, dist = __fsqrt_rn(x*x + y*y);
	if ((double)dist > 2.0) return 0.0f;
	float const val = cosf_lut(tab, x)*cosf_lut(tab, y);
	double const hd = 400.0*((double)val - 0.999);
	float const hole = (float)((0.0 < hd) ? hd : 0.0);
	float const peak = (float)(0.08*(double)val/(double)smax(0.04f, dist));
	return P.h.volcano_height*smax(0.0f, (peak - hole))*P.mesh_scale_z_inv;
}

// apply_glaciate (src/mesh_gen.cpp:380-385) + the sine bias / volcano terms of eval_index (src/mesh_gen.cpp:782-790).
// smx/smy: the enable_glaciate() COSF terms for this cell (sm_scale*COSF(..x..), COSF(..y..)).
__device__ __forceinline__ float glaciate_and_bias(float z, float smx, float smy, float cx, float cy, const PostParams &P, const float *__restrict__ tab) {
	if (!P.enable_glaciate) return z;
	if (P.glaciate) {
		float const relh = (z + P.zmax_est)*P.zmax_est2_inv;
		float const g = (P.custom_exp == 0.0f) ? relh*relh*relh : powf(relh, P.custom_exp); // powf: <= 2 ulp vs glibc for a custom exponent (documented)
		z = g*P.zmax_est2 - P.zmax_est;
	}
	if (P.sine_on) {
		z += smx*smy + P.sine_offset;
		if (P.volcano_on) {z += volcano_height(cx, cy, P, tab);}
	}
	return z;
}

// block-level min/max -> global ordered-uint atomics
__device__ __forceinline__ void block_minmax(float vmin, float vmax, unsigned *mm) {
	for (int o = 16; o > 0; o >>= 1) {
		vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
		vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
	}
	__shared__ float s_min[32], s_max[32];
	int const tid = threadIdx.x + blockDim.x*(threadIdx.y + blockDim.y*threadIdx.z);
	int const nw = (blockDim.x*blockDim.y*blockDim.z + 31) >> 5, w = tid >> 5, l = tid & 31;
	if (l == 0) {s_min[w] = vmin; s_max[w] = vmax;}
	__syncthreads();
	if (w == 0) {
		vmin = (l < nw) ? s_min[l] :  INFINITY;
		vmax = (l < nw) ? s_max[l] : -INFINITY;
		for (int o = 16; o > 0; o >>= 1) {
			vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
			vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
		}
		if (l == 0) {atomicMin(mm, tw_f2ord(vmin)); atomicMax(mm + 1, tw_f2ord(vmax));}
	}
}

// ------------------------------------------------------------------------------------------------ noise modes
struct NoiseParams {
	int   octaves;               // NUM_FREQ_COMP - start_eval_sin/N_RAND_SIN2
	int   gen_shape;
	float4 oct[9];               // per-octave constants of gen_noise's loop {freq, rx, ry, mag} (freq*=1.92, rx*=1.5, ry*=1.5, mag*=0.5), host-computed;
	                             // packed so that an octave reads them from the constant bank with two 64-bit loads instead of four 32-bit ones
	float xy_scale;              // MESH_SCALE_FACTOR*mesh_scale
	float hmap_scale;            // get_hmap_scale(mode)
	float freq_last, rsum_last;  // freq / (rx+ry) of the last octave: bound of the lattice coordinates (paired-path range guard)
};

template<bool SIMPLEX, int SHAPE>
__device__ __forceinline__ float gen_noise(float xv, float yv, const NoiseParams &N) { // src/mesh_gen.cpp:706-730
	float zval = 0.0f;
#pragma unroll 1
	for (int i = 0; i < N.octaves; ++i) {
		float4 const o = N.oct[i];
		float const px = o.x*xv + o.y, py = o.x*yv + o.z;
		float noise = SIMPLEX ? twn::simplex2(px, py) : twn::perlin2(px, py);
		if (SHAPE == 1) {noise = (float)((double)fabsf(noise) - 0.40);}
		if (SHAPE == 2) {noise = (float)(0.45 - (double)fabsf(noise));}
		zval = __fmaf_rn(o.w, noise, zval); // mag is a power of two: mag*noise is exact, so fused == mul-then-add
	}
	return zval;
}

template<bool SIMPLEX, bool WARP, int SHAPE>
__device__ __forceinline__ float get_noise_zval(float xval, float yval, const NoiseParams &N, const PostParams &P) { // src/mesh_gen.cpp:734-751
	float xv = N.xy_scale*xval, yv = N.xy_scale*yval; // :737-738
	if (WARP) { // domain warping, src/mesh_gen.cpp:740-747 ("xv+5.2" etc. are float+double adds rounded back to float)
		float const scale = 0.2f;
		float const dx1 = gen_noise<SIMPLEX, SHAPE>((float)((double)xv + 0.0), (float)((double)yv + 0.0), N);
		float const dy1 = gen_noise<SIMPLEX, SHAPE>((float)((double)xv + 5.2), (float)((double)yv + 1.3), N);
		float const wx = xv + scale*dx1, wy = yv + scale*dy1;
		float const dx2 = gen_noise<SIMPLEX, SHAPE>((float)((double)wx + 1.7), (float)((double)wy + 9.2), N);
		float const dy2 = gen_noise<SIMPLEX, SHAPE>((float)((double)wx + 8.3), (float)((double)wy + 2.8), N);
		xv += scale*dx2; yv += scale*dy2;
	}
	float z = gen_noise<SIMPLEX, SHAPE>(xv, yv, N);
	if (P.need_postproc) {z = postproc_noise_zval(z, P.h);}
	return z*N.hmap_scale;
}

template<bool SIMPLEX, bool WARP, int SHAPE>
__global__ void __launch_bounds__(256)
noise_grid_kernel(float *__restrict__ out, unsigned nx, unsigned ny, unsigned y_off, float mx0_single, float my0_single, const float2 *__restrict__ tile_origins,
	NoiseParams N, PostParams P, const float *__restrict__ sin_tab, unsigned *__restrict__ mm)
{
	unsigned const x = blockIdx.x*blockDim.x + threadIdx.x, y = y_off + blockIdx.y*blockDim.y + threadIdx.y, tile = blockIdx.z; // y_off: first row of this band
	float mx0 = mx0_single, my0 = my0_single;
	if (tile_origins) {float2 const o = __ldg(tile_origins + tile); mx0 = o.x; my0 = o.y;}
	float z = 0.0f;
	bool const valid = (x < nx && y < ny);
	if (valid) {
		// eval_index: xval((x*mdx + mx0)*DX_VAL_INV), src/mesh_gen.cpp:762
		float const xval = ((float)x*P.mdx + mx0)*P.dx_inv, yval = ((float)y*P.mdy + my0)*P.dy_inv;
		z = get_noise_zval<SIMPLEX, WARP, SHAPE>(xval, yval, N, P);
		float smx = 0.0f, smy = 0.0f;
		if (P.enable_glaciate && P.sine_on) { // enable_glaciate() terms, src/mesh_gen.cpp:647-649, evaluated per cell instead of tabulated
			smx = P.sm_scale*cosf_lut(sin_tab, ((float)x*P.mdx + mx0)*P.dx_inv*P.sm_freq);
			smy = cosf_lut(sin_tab, ((float)y*P.mdy + my0)*P.dy_inv*P.sm_freq);
		}
		z = glaciate_and_bias(z, smx, smy, xval, yval, P, sin_tab);
		out[(size_t)tile*nx*ny + (size_t)y*nx + x] = z;
	}
	if (mm) {block_minmax(valid ? z : INFINITY, valid ? z : -INFINITY, mm + 2*tile);}
}

#ifndef TW_NOISE2_MIN_BLOCKS
#define TW_NOISE2_MIN_BLOCKS 2   // 74 KB of table per block (79 KB with the hash table of the domain-warp kernel, tw_noise2.cuh): 2 blocks of 512 threads
                                 // = 32 warps per SM, which caps the kernel at 64 registers
#endif
#ifndef TW_NOISE2_PERSISTENT
#define TW_NOISE2_PERSISTENT 1   // k > 0: single grids launch at most k waves of resident blocks, each striding over the chunk groups (table staged once per block).
                                 // One H100, against 0: headline step 0.5 % shorter, plain simplex / Perlin 8192^2 5 % / 4 % more cells/s, e2e unchanged
                                 // (results/h100/launch_shape.txt); tile batches launch one block per chunk group either way
#endif
#ifndef TW_NOISE2_THREADS
#define TW_NOISE2_THREADS 512    // threads per block (256 x 3 blocks = 24 warps per SM at 80 registers: 0.7 % slower on the headline, results/h100/launch_shape.txt)
#endif
#ifndef TW_NOISE2_BLOCK_CELLS
// Cells per block in every mode, walked as chunks of 2*TW_NOISE2_THREADS cells: the 74 KB table fill is paid once per block (the plain modes run
// only 8 evaluations per cell), and a 258^2 tile (66564 cells) leaves 1.5 % of the cells of its last block idle. One H100, 8192^2 headline at
// 256 threads: 512 -> 9.76 ms, 1024 -> 9.31, 2048 -> 9.13, 4096 -> 9.15 (results/h100/warp_chunks.txt)
#define TW_NOISE2_BLOCK_CELLS 2048
#endif
static_assert(TW_NOISE2_BLOCK_CELLS % (2*TW_NOISE2_THREADS) == 0, "a block walks whole chunks of 2 cells per thread");
// ---- paired variant: two horizontally adjacent cells per thread (see tw_noise2.cuh) ----
// |lattice coordinate| < 2^22 for every octave of this fBm call (needed by the division-free mod); NaN-safe
__device__ __forceinline__ bool noise_lattice_in_range(float2 xv, float2 yv, const NoiseParams &N) {
	float const bx = (fabsf(xv.x) + fabsf(yv.x))*N.freq_last + N.rsum_last, by = (fabsf(xv.y) + fabsf(yv.y))*N.freq_last + N.rsum_last;
	return (bx < 2097152.0f && by < 2097152.0f); // |p + s| <= 1.37*(|px|+|py|) < 2^22, and floor(p)+1 stays in range for Perlin
}

// The domain-warp simplex kernel also stages the simplex hash table (tw_noise2.cuh): 8 instructions fewer per cell pair and octave. Its fill is
// repaid by the 40 evaluations per cell of that mode; plain simplex, 8 evaluations per cell, measured 8 % slower with the earlier (37 KB) form of it
// at one block per 2048 cells (as tile batches launch).
template<bool SIMPLEX, bool WARP> __host__ __device__ constexpr bool noise2_hash() {return SIMPLEX && WARP && TW_SIMPLEX_HASH_TABLE;}
// entries of the table a block stages: the gradient table, and the hash table behind it
template<bool HASH> __host__ __device__ constexpr int lut_entries() {return twn2::SIMPLEX_LUT_N + (HASH ? twn2::SIMPLEX_HASH_N : 0);}
// float4 slots a block stages: 8 copies of the gradient table, then SIMPLEX_HASH_COPIES of the hash table
template<bool HASH> __host__ __device__ constexpr int lut_slots() {return twn2::SIMPLEX_LUT_N*twn2::SIMPLEX_LUT_COPIES + (HASH ? twn2::SIMPLEX_HASH_N*twn2::SIMPLEX_HASH_COPIES : 0);}

// one octave of gen_noise for two cells
template<bool SIMPLEX, int SHAPE, bool HASH>
__device__ __forceinline__ float2 noise2_octave(float2 xv, float2 yv, float4 o, unsigned L, float2 zval) {
	float2 const px = twn2::add2(twn2::mul2(xv, o.x), o.y), py = twn2::add2(twn2::mul2(yv, o.x), o.z); // o = {freq, rx, ry, mag}
	float2 noise = SIMPLEX ? ((TW_SIMPLEX_LUT > 0) ? twn2::simplex2_lut<HASH>(px, py, L) : twn2::simplex2(px, py)) : ((TW_SIMPLEX_LUT > 0) ? twn2::perlin2_lut(px, py, L) : twn2::perlin2(px, py));
	if (SHAPE == 1) {noise = make_float2((float)((double)fabsf(noise.x) - 0.40), (float)((double)fabsf(noise.y) - 0.40));}
	if (SHAPE == 2) {noise = make_float2((float)(0.45 - (double)fabsf(noise.x)), (float)(0.45 - (double)fabsf(noise.y)));}
	return twn2::fma2(noise, o.w, zval); // mag is a power of two: exact product
}

template<bool SIMPLEX, int SHAPE, bool HASH>
__device__ __forceinline__ float2 gen_noise2(float2 xv, float2 yv, const NoiseParams &N, unsigned L) { // gen_noise (src/mesh_gen.cpp:706-730) for two cells; L: simplex table base (twn2::simplex_lut_base) or 0
	float2 zval = make_float2(0.0f, 0.0f);
	bool const in_range = noise_lattice_in_range(xv, yv, N);
	if (HASH && SHAPE == 0 && N.octaves == 8 && in_range) {
		// The domain-warp kernel at 8 octaves (mesh_freq_filter 1: the headline, config 5, the tile jobs) runs the same octaves in the same order
		// fully unrolled: with a constant index the octave constants need no counter, address arithmetic or branch (164 instead of 169 instructions
		// per octave). Shapes 1 and 2 keep the rolled loop: their double-precision shaping pushes the unrolled kernel past 64 registers (spills).
#pragma unroll
		for (int i = 0; i < 8; ++i) {zval = noise2_octave<SIMPLEX, SHAPE, HASH>(xv, yv, N.oct[i], L, zval);}
	}
	else if (in_range) {
#pragma unroll 1
		for (int i = 0; i < N.octaves; ++i) {zval = noise2_octave<SIMPLEX, SHAPE, HASH>(xv, yv, N.oct[i], L, zval);}
	}
	else {zval = make_float2(gen_noise<SIMPLEX, SHAPE>(xv.x, yv.x, N), gen_noise<SIMPLEX, SHAPE>(xv.y, yv.y, N));} // astronomically far out: scalar path with the literal division
	return zval;
}

#ifndef TW_NOISE2_DUAL
#define TW_NOISE2_DUAL 0   // 1: the two independent fBm evaluations of each domain-warp stage (dx1|dy1, dx2|dy2) share one octave loop (2x the ILP per thread)
#endif
// two independent gen_noise2 evaluations in one octave loop: same operations per evaluation, interleaved by the compiler
template<bool SIMPLEX, int SHAPE, bool HASH>
__device__ __forceinline__ void gen_noise2_dual(float2 xa, float2 ya, float2 xb, float2 yb, const NoiseParams &N, unsigned L, float2 &za, float2 &zb) {
	if (TW_SIMPLEX_LUT > 0 && noise_lattice_in_range(xa, ya, N) && noise_lattice_in_range(xb, yb, N)) {
		float2 zva = make_float2(0.0f, 0.0f), zvb = make_float2(0.0f, 0.0f);
#pragma unroll 1
		for (int i = 0; i < N.octaves; ++i) {
			float4 const o = N.oct[i];
			float const f = o.x, rx = o.y, ry = o.z, mag = o.w;
			float2 const pxa = twn2::add2(twn2::mul2(xa, f), rx), pya = twn2::add2(twn2::mul2(ya, f), ry);
			float2 const pxb = twn2::add2(twn2::mul2(xb, f), rx), pyb = twn2::add2(twn2::mul2(yb, f), ry);
			float2 na = SIMPLEX ? twn2::simplex2_lut<HASH>(pxa, pya, L) : twn2::perlin2_lut(pxa, pya, L);
			float2 nb = SIMPLEX ? twn2::simplex2_lut<HASH>(pxb, pyb, L) : twn2::perlin2_lut(pxb, pyb, L);
			if (SHAPE == 1) {na = make_float2((float)((double)fabsf(na.x) - 0.40), (float)((double)fabsf(na.y) - 0.40)); nb = make_float2((float)((double)fabsf(nb.x) - 0.40), (float)((double)fabsf(nb.y) - 0.40));}
			if (SHAPE == 2) {na = make_float2((float)(0.45 - (double)fabsf(na.x)), (float)(0.45 - (double)fabsf(na.y))); nb = make_float2((float)(0.45 - (double)fabsf(nb.x)), (float)(0.45 - (double)fabsf(nb.y)));}
			zva = twn2::fma2(na, mag, zva); zvb = twn2::fma2(nb, mag, zvb);
		}
		za = zva; zb = zvb;
	}
	else {za = gen_noise2<SIMPLEX, SHAPE, HASH>(xa, ya, N, L); zb = gen_noise2<SIMPLEX, SHAPE, HASH>(xb, yb, N, L);}
}

__device__ __forceinline__ float dadd(float a, double b) {return (float)((double)a + b);} // float + double literal, rounded back (src/mesh_gen.cpp:742-745)
__constant__ double2 warp_offsets[4] = {{0.0, 0.0}, {5.2, 1.3}, {1.7, 9.2}, {8.3, 2.8}}; // the domain warp's offsets per stage (src/mesh_gen.cpp:742-745)

template<bool SIMPLEX, bool WARP, int SHAPE>
__global__ void __launch_bounds__(TW_NOISE2_THREADS, TW_NOISE2_MIN_BLOCKS)
noise_grid2_kernel(float *__restrict__ out, unsigned nx, unsigned ny, unsigned y_off, unsigned y_end, float mx0_single, float my0_single, const float2 *__restrict__ tile_origins,
	NoiseParams N, PostParams P, const float *__restrict__ sin_tab, unsigned *__restrict__ mm, const float4 *__restrict__ simplex_lut)
{
	constexpr bool HASH = noise2_hash<SIMPLEX, WARP>();
	unsigned L = 0;
	if (TW_SIMPLEX_LUT > 0) { // hash/gradient table (simplex or Perlin flavour) -> shared memory, 8 interleaved copies (see tw_noise2.cuh)
		extern __shared__ float4 lut_s[]; // lut_slots<HASH>() entries (dynamic: 74 KB at level 3, + 4.6 KB of hash table)
		constexpr int G = twn2::SIMPLEX_LUT_N*twn2::SIMPLEX_LUT_COPIES;
		for (int e = threadIdx.x; e < lut_slots<HASH>(); e += blockDim.x) {
			lut_s[e] = __ldg(simplex_lut + ((e < G) ? e/twn2::SIMPLEX_LUT_COPIES : twn2::SIMPLEX_LUT_N + (e - G)/twn2::SIMPLEX_HASH_COPIES));
		}
		__syncthreads();
		L = twn2::simplex_lut_base(lut_s, threadIdx.x);
		asm volatile("" : "+r"(L) :: "memory"); // every table load depends on L, and L is defined after the barrier
	}
	// cells are numbered row-major over the band [y_off, y_end) of the grid and dealt out in pairs (2t, 2t+1): no lanes idle on widths that are
	// not a multiple of the block width (258-wide tiles wasted 27 % of a 64x8-cell block grid); a pair may straddle a row end when nx is odd
	// A block walks NCH consecutive chunks of 2*blockDim cells (TW_NOISE2_BLOCK_CELLS in all), so the table is staged once per chunk group.
	unsigned const tile = blockIdx.z;
	float mx0 = mx0_single, my0 = my0_single;
	if (tile_origins) {float2 const o = __ldg(tile_origins + tile); mx0 = o.x; my0 = o.y;}
	size_t const c_end = (size_t)y_end*nx;
	float lo = INFINITY, hi = -INFINITY;
	constexpr unsigned NCH = TW_NOISE2_BLOCK_CELLS/(2*TW_NOISE2_THREADS);
	// blocks stride over the chunk groups of the band: with gridDim.x == number of groups every block does exactly one (the default); a smaller
	// grid (TW_NOISE2_PERSISTENT: one wave of resident blocks) keeps the staged table for many chunks
	// P.ngroups = chunk groups of this band (host-computed: a 64-bit division per thread here cost 2.5 % of the whole kernel)
#pragma unroll 1
	for (unsigned grp = blockIdx.x; grp < P.ngroups; grp += gridDim.x) {
#pragma unroll 1
	for (unsigned ch = 0; ch < NCH; ++ch) {
	size_t const c0 = (size_t)y_off*nx + 2*(((size_t)grp*NCH + ch)*blockDim.x + threadIdx.x);
	unsigned y, x;
	if (c_end <= 0xffffffffull) {unsigned const c32 = (unsigned)c0; y = c32/nx; x = c32 - y*nx;} // 32-bit division for every grid below 2^32 cells
	else {y = (unsigned)(c0/nx); x = (unsigned)(c0 - (size_t)y*nx);}
	unsigned const xb = (x + 1 < nx) ? x + 1 : 0, yb = (x + 1 < nx) ? y : y + 1;
	bool const skip = (x - P.skip_x0 < P.skip_w && y - P.skip_y0 < P.skip_h && xb - P.skip_x0 < P.skip_w && yb - P.skip_y0 < P.skip_h); // both cells unread
	bool const valid0 = (c0 < c_end) && !skip, valid1 = (c0 + 1 < c_end) && !skip;
	float z0 = 0.0f, z1 = 0.0f;
	if (valid0) { // the second cell of an odd-sized band is computed and dropped
		using namespace twn2;
		float2 const xs = make_float2((float)x, (float)xb), ys = make_float2((float)y, (float)yb);
		float2 const xval = mul2(add2(mul2(xs, P.mdx), mx0), P.dx_inv);           // (x*mdx + mx0)*DX_VAL_INV, src/mesh_gen.cpp:762
		float2 const yval = mul2(add2(mul2(ys, P.mdy), my0), P.dy_inv);
		float2 xv = mul2(xval, N.xy_scale), yv = mul2(yval, N.xy_scale);          // get_noise_zval, src/mesh_gen.cpp:737-738
		float2 zz;
		if (WARP && !TW_NOISE2_DUAL) { // domain warping, src/mesh_gen.cpp:740-747: its five fBm calls as one loop around a single gen_noise2 body
			// (five inline copies of the unrolled 8-octave body measured 6 % slower than this loop: 100 KB of hot code, results/h100/octave_body.txt)
			float const scale = 0.2f;
			float2 bx = xv, by = yv, d = make_float2(0.0f, 0.0f);
#pragma unroll 1
			for (int s = 0; s < 5; ++s) { // dx1 = noise(xv + 0.0, yv + 0.0), dy1 = noise(xv + 5.2, yv + 1.3), then with w = v + scale*(dx1, dy1):
				                            // dx2 = noise(wx + 1.7, wy + 9.2), dy2 = noise(wx + 8.3, wy + 2.8), z = noise(v + scale*(dx2, dy2))
				float2 sx = xv, sy = yv;
				if (s < 4) {double2 const o = warp_offsets[s]; sx = make_float2(dadd(bx.x, o.x), dadd(bx.y, o.x)); sy = make_float2(dadd(by.x, o.y), dadd(by.y, o.y));}
				float2 const r = gen_noise2<SIMPLEX, SHAPE, HASH>(sx, sy, N, L);
				if (s == 1) {bx = add2(xv, mul2(d, scale)); by = add2(yv, mul2(r, scale));} // wx, wy
				if (s == 3) {xv = add2(xv, mul2(d, scale)); yv = add2(yv, mul2(r, scale));}
				d = r; // dx1 / dx2 for the next stage; the last stage's is the result
			}
			zz = d;
		}
		else {
		if (WARP) { // TW_NOISE2_DUAL
			float const scale = 0.2f;
			float2 dx1, dy1, dx2, dy2;
			gen_noise2_dual<SIMPLEX, SHAPE, HASH>(make_float2(dadd(xv.x, 0.0), dadd(xv.y, 0.0)), make_float2(dadd(yv.x, 0.0), dadd(yv.y, 0.0)),
			                                      make_float2(dadd(xv.x, 5.2), dadd(xv.y, 5.2)), make_float2(dadd(yv.x, 1.3), dadd(yv.y, 1.3)), N, L, dx1, dy1);
			float2 const wx = add2(xv, mul2(dx1, scale)), wy = add2(yv, mul2(dy1, scale));
			gen_noise2_dual<SIMPLEX, SHAPE, HASH>(make_float2(dadd(wx.x, 1.7), dadd(wx.y, 1.7)), make_float2(dadd(wy.x, 9.2), dadd(wy.y, 9.2)),
			                                      make_float2(dadd(wx.x, 8.3), dadd(wx.y, 8.3)), make_float2(dadd(wy.x, 2.8), dadd(wy.y, 2.8)), N, L, dx2, dy2);
			xv = add2(xv, mul2(dx2, scale)); yv = add2(yv, mul2(dy2, scale));
		}
		zz = gen_noise2<SIMPLEX, SHAPE, HASH>(xv, yv, N, L);
		}
		z0 = zz.x; z1 = zz.y;
		if (P.need_postproc) {z0 = postproc_noise_zval(z0, P.h); z1 = postproc_noise_zval(z1, P.h);}
		z0 = z0*N.hmap_scale; z1 = z1*N.hmap_scale;
		float smx0 = 0.0f, smx1 = 0.0f, smy0 = 0.0f, smy1 = 0.0f;
		if (P.enable_glaciate && P.sine_on) { // enable_glaciate() terms, src/mesh_gen.cpp:647-649
			smx0 = P.sm_scale*cosf_lut(sin_tab, xval.x*P.sm_freq);
			smx1 = P.sm_scale*cosf_lut(sin_tab, xval.y*P.sm_freq);
			smy0 = cosf_lut(sin_tab, yval.x*P.sm_freq);
			smy1 = (yb == y) ? smy0 : cosf_lut(sin_tab, yval.y*P.sm_freq);
		}
		z0 = glaciate_and_bias(z0, smx0, smy0, xval.x, yval.x, P, sin_tab);
		z1 = glaciate_and_bias(z1, smx1, smy1, xval.y, yval.y, P, sin_tab);
		float *o = out + (size_t)(P.tile_perm ? __ldg(P.tile_perm + tile) : tile)*nx*ny + c0;
		if (valid1 && ((reinterpret_cast<size_t>(o) & 7) == 0)) {*reinterpret_cast<float2 *>(o) = make_float2(z0, z1);}
		else {o[0] = z0; if (valid1) {o[1] = z1;}}
	}
	lo = fminf(lo, fminf(valid0 ? z0 : INFINITY, valid1 ? z1 : INFINITY)); hi = fmaxf(hi, fmaxf(valid0 ? z0 : -INFINITY, valid1 ? z1 : -INFINITY));
	} // chunks
	} // chunk groups
	if (mm) {block_minmax(lo, hi, mm + 2*tile);}
}

template<bool SIMPLEX, bool WARP>
void launch_noise2(int shape, dim3 grid, dim3 block, cudaStream_t st, float *out, unsigned nx, unsigned ny, unsigned y_off, unsigned y_end, float mx0, float my0,
	const float2 *origins, const NoiseParams &N, const PostParams &P, const float *tab, unsigned *mm, const float4 *lut)
{
	size_t const lut_bytes = (TW_SIMPLEX_LUT > 0) ? (size_t)lut_slots<noise2_hash<SIMPLEX, WARP>()>()*sizeof(float4) : 0;
	// more than 48 KB of dynamic shared memory needs the opt-in; set per launch (a few hundred ns) rather than cached in a static, so that
	// contexts on several devices in one process all get it
	if (lut_bytes > 48*1024) {
		switch (shape) {
		case 1:  cudaFuncSetAttribute(noise_grid2_kernel<SIMPLEX, WARP, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes); break;
		case 2:  cudaFuncSetAttribute(noise_grid2_kernel<SIMPLEX, WARP, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes); break;
		default: cudaFuncSetAttribute(noise_grid2_kernel<SIMPLEX, WARP, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes); break;
		}
	}
	switch (shape) {
	case 1:  noise_grid2_kernel<SIMPLEX, WARP, 1><<<grid, block, lut_bytes, st>>>(out, nx, ny, y_off, y_end, mx0, my0, origins, N, P, tab, mm, lut); break;
	case 2:  noise_grid2_kernel<SIMPLEX, WARP, 2><<<grid, block, lut_bytes, st>>>(out, nx, ny, y_off, y_end, mx0, my0, origins, N, P, tab, mm, lut); break;
	default: noise_grid2_kernel<SIMPLEX, WARP, 0><<<grid, block, lut_bytes, st>>>(out, nx, ny, y_off, y_end, mx0, my0, origins, N, P, tab, mm, lut); break;
	}
}

constexpr int PERLIN_LUT_OFFSET = lut_entries<true>();
__global__ void simplex_lut_kernel(float4 *__restrict__ lut) { // [0, N): simplex table, [N, N + H): simplex hash table, [N + H, 2N + H): Perlin table
	int const k = blockIdx.x*blockDim.x + threadIdx.x;
	if (k < twn2::SIMPLEX_LUT_N) {lut[k] = twn2::simplex_lut_entry((float)k); lut[PERLIN_LUT_OFFSET + k] = twn2::perlin_lut_entry((float)k);}
	if (k < twn2::SIMPLEX_HASH_N) {lut[twn2::SIMPLEX_LUT_N + k] = twn2::simplex_hash_entry((float)k);}
}
} // namespace
int twi_ensure_simplex_lut(tw_ctx *ctx) {
	if (ctx->d_simplex_lut) return TW_OK;
	static_assert(twn2::SIMPLEX_HASH_N <= twn2::SIMPLEX_LUT_N, "simplex_lut_kernel's grid covers the gradient tables");
	TW_CUDA(ctx, cudaMalloc(&ctx->d_simplex_lut, (PERLIN_LUT_OFFSET + twn2::SIMPLEX_LUT_N)*sizeof(float4)));
	simplex_lut_kernel<<<(twn2::SIMPLEX_LUT_N + 127)/128, 128, 0, ctx->stream>>>((float4 *)ctx->d_simplex_lut);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
namespace {

// ------------------------------------------------------------------------------------------------ sine-table mode
struct SineTabParams {
	float msx, msy, ms2, mesh_scale_z_inv; // mesh_scale*DX_VAL_INV, mesh_scale*DY_VAL_INV, 0.5*mesh_scale
	float dx, dy, mx0, my0;
	int   start;
	unsigned nx, ny, xpitch, ypitch;       // table row pitches (floats)
	// glaciate cos terms
	int   sine_on; float sm_scale, sm_freq, dx_inv, dy_inv;
};

// X[k][i] = SINF(xmdx*i + x_const), Y[k][j] = y_scale*SINF(ymdy*j + y_const)  (src/mesh_gen.cpp:609-625); row F_TABLE holds the
// enable_glaciate() terms (src/mesh_gen.cpp:647-649). grid = (ceil(max(nx,ny)/256), F_TABLE+1, 2[x|y]).
// Tile batches (origins != nullptr): grid.z = nux + nuy tables; table t < nux is the X table of the t-th DISTINCT tile x origin (origins[t] = its mx0), the
// others the Y tables of the distinct y origins - a W x H block of tiles needs W + H tables, not 2*W*H (the round-1 code built and launched two per tile).
__global__ void sine_tables_kernel(float *__restrict__ Xt, float *__restrict__ Yt, const float *__restrict__ T, const float *__restrict__ sin_tab, SineTabParams S,
	const float *__restrict__ origins = nullptr, unsigned nux = 0, size_t xstride = 0, size_t ystride = 0)
{
	unsigned const i = blockIdx.x*blockDim.x + threadIdx.x, k = blockIdx.y;
	bool const is_y = origins ? (blockIdx.z >= nux) : (blockIdx.z != 0);
	if (origins) {
		if (is_y) {S.my0 = __ldg(origins + blockIdx.z); Yt += (size_t)(blockIdx.z - nux)*ystride;}
		else      {S.mx0 = __ldg(origins + blockIdx.z); Xt += (size_t)blockIdx.z*xstride;}
	}
	unsigned const n = is_y ? S.ny : S.nx;
	if (i >= n) return;
	if (k == F_TABLE) { // cos terms
		if (!S.sine_on) return;
		if (!is_y) {Xt[(size_t)k*S.xpitch + i] = S.sm_scale*cosf_lut(sin_tab, ((float)i*S.dx + S.mx0)*S.dx_inv*S.sm_freq);}
		else       {Yt[(size_t)k*S.ypitch + i] = cosf_lut(sin_tab, ((float)i*S.dy + S.my0)*S.dy_inv*S.sm_freq);}
		return;
	}
	if ((int)k < S.start) return; // never read
	float const *s = T + 5*k;
	if (!is_y) {
		float const x_mult = S.msx*s[4];
		float const x_const = S.ms2*s[4] + s[2] + x_mult*S.mx0;
		float const xmdx = x_mult*S.dx;
		Xt[(size_t)k*S.xpitch + i] = sinf_lut(sin_tab, xmdx*(float)i + x_const);
	}
	else {
		float const y_mult = S.msy*s[3], y_scale = S.mesh_scale_z_inv*s[0];
		float const y_const = S.ms2*s[3] + s[1] + y_mult*S.my0;
		float const ymdy = y_mult*S.dy;
		Yt[(size_t)k*S.ypitch + i] = y_scale*sinf_lut(sin_tab, ymdy*(float)i + y_const);
	}
}

// 64x64 output tile per 256-thread block, 4x4 cells per thread (x strided by 16 so that a half-warp stores 16 consecutive floats).
constexpr int ST = 64;          // tile edge
constexpr int SK = 45;          // k-chunk staged in shared memory (2 chunks cover the 90 terms)

__global__ void __launch_bounds__(256)
sine_grid_kernel(float *__restrict__ out, unsigned nx, unsigned ny, const float *__restrict__ Xt, const float *__restrict__ Yt,
	unsigned xpitch, unsigned ypitch, int start_ix, PostParams P, float mx0, float my0, const float *__restrict__ sin_tab, unsigned *__restrict__ mm, unsigned y_off,
	const uint2 *__restrict__ tile_tabs = nullptr, const float2 *__restrict__ tile_origins = nullptr, size_t xstride = 0, size_t ystride = 0,
	const unsigned *__restrict__ tile_perm = nullptr)
{
	__shared__ float Xs[SK][ST], Ys[SK][ST];
	if (tile_tabs) { // tile batch: blockIdx.z = tile (tile_perm: tile_perm[z] of the batch, written to slot z); its X / Y tables are shared with the other tiles of its column / row
		unsigned const tz = tile_perm ? __ldg(tile_perm + blockIdx.z) : blockIdx.z;
		uint2 const tt = __ldg(tile_tabs + tz);
		float2 const o = __ldg(tile_origins + tz);
		Xt += (size_t)tt.x*xstride; Yt += (size_t)tt.y*ystride; mx0 = o.x; my0 = o.y;
		out += (size_t)blockIdx.z*nx*ny;
		if (mm) {mm += 2*(size_t)blockIdx.z;}
	}
	unsigned const x_base = blockIdx.x*ST, y_base = y_off + blockIdx.y*ST;
	int const tid = threadIdx.x, tx = tid & 15, ty = tid >> 4; // 16 x 16 threads
	float2 acc2[4][2]; // acc2[a][h] = cells (row a, columns 2h and 2h+1 of this thread): paired accumulators (see tw_noise2.cuh)
#pragma unroll
	for (int a = 0; a < 4; ++a) {acc2[a][0] = make_float2(0.0f, 0.0f); acc2[a][1] = make_float2(0.0f, 0.0f);}
	for (int k0 = start_ix; k0 < F_TABLE; k0 += SK) {
		int const kn = min(SK, F_TABLE - k0);
		__syncthreads();
		for (int e = tid; e < kn*ST; e += 256) { // stage the X and Y panels (coalesced 256-byte rows)
			int const kk = e / ST, c = e % ST;
			unsigned const gx = x_base + c, gy = y_base + c;
			Xs[kk][c] = (gx < nx) ? __ldg(Xt + (size_t)(k0 + kk)*xpitch + gx) : 0.0f;
			Ys[kk][c] = (gy < ny) ? __ldg(Yt + (size_t)(k0 + kk)*ypitch + gy) : 0.0f;
		}
		__syncthreads();
#pragma unroll 5
		for (int kk = 0; kk < kn; ++kk) {
			float xv[4];
#pragma unroll
			for (int b = 0; b < 4; ++b) {xv[b] = Xs[kk][tx + 16*b];}
			float4 const yv4 = *reinterpret_cast<const float4 *>(&Ys[kk][ty*4]);
			float const yv[4] = {yv4.x, yv4.y, yv4.z, yv4.w};
			float2 const x01 = make_float2(xv[0], xv[1]), x23 = make_float2(xv[2], xv[3]);
#pragma unroll
			for (int a = 0; a < 4; ++a) { // zval += xptr[i]*yptr[i]: product rounded, then added (two roundings, as the reference); two cells per instruction
				float2 const ya = twn2::splat(yv[a]);
				acc2[a][0] = twn2::add2(twn2::mul2(x01, ya), acc2[a][0]);
				acc2[a][1] = twn2::add2(twn2::mul2(x23, ya), acc2[a][1]);
			}
		}
	}
	float vmin = INFINITY, vmax = -INFINITY;
#pragma unroll
	for (int a = 0; a < 4; ++a) {
		unsigned const y = y_base + ty*4 + a;
		if (y >= ny) continue;
		float const smy = (P.enable_glaciate && P.sine_on) ? __ldg(Yt + (size_t)F_TABLE*ypitch + y) : 0.0f;
#pragma unroll
		for (int b = 0; b < 4; ++b) {
			unsigned const x = x_base + tx + 16*b;
			if (x >= nx) continue;
			float z = (b & 1) ? ((b >> 1) ? acc2[a][1].y : acc2[a][0].y) : ((b >> 1) ? acc2[a][1].x : acc2[a][0].x);
			if (P.shape == 1) {z = (float)((double)fabsf(z) - 2.0);}       // apply_noise_shape_final, src/mesh_gen.cpp:564-571
			else if (P.shape == 2) {z = (float)(3.5 - (double)fabsf(z));}
			if (P.need_postproc) {z = postproc_noise_zval(z, P.h);}
			float const smx = (P.enable_glaciate && P.sine_on) ? __ldg(Xt + (size_t)F_TABLE*xpitch + x) : 0.0f;
			float cx = 0.0f, cy = 0.0f;
			if (P.volcano_on) {cx = ((float)x*P.mdx + mx0)*P.dx_inv; cy = ((float)y*P.mdy + my0)*P.dy_inv;}
			z = glaciate_and_bias(z, smx, smy, cx, cy, P, sin_tab);
			out[(size_t)y*nx + x] = z;
			vmin = fminf(vmin, z); vmax = fmaxf(vmax, z);
		}
	}
	if (mm) {block_minmax(vmin, vmax, mm);}
}

__global__ void init_minmax_kernel(unsigned *mm, uint32_t n) {
	uint32_t const i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) {mm[2*i] = 0xffffffffu; mm[2*i+1] = 0u;}
}

__global__ void minmax_kernel(const float *__restrict__ v, size_t n, unsigned *mm) {
	float vmin = INFINITY, vmax = -INFINITY;
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {float const z = __ldg(v + i); vmin = fminf(vmin, z); vmax = fmaxf(vmax, z);}
	block_minmax(vmin, vmax, mm);
}

// one block per heightmap: min/max of tile t -> mm[2t], mm[2t+1] (ordered-uint encoding); perm: block b handles tile perm[b] of v and mm
__global__ void minmax_tiles_kernel(const float *__restrict__ v, size_t tile_elems, unsigned *mm, const unsigned *__restrict__ perm) {
	size_t const tile = perm ? __ldg(perm + blockIdx.x) : blockIdx.x;
	const float *t = v + tile*tile_elems;
	if (threadIdx.x == 0) {mm[2*tile] = 0xffffffffu; mm[2*tile + 1] = 0u;}
	__syncthreads();
	float vmin = INFINITY, vmax = -INFINITY;
	for (size_t i = threadIdx.x; i < tile_elems; i += blockDim.x) {float const z = __ldg(t + i); vmin = fminf(vmin, z); vmax = fmaxf(vmax, z);}
	block_minmax(vmin, vmax, mm + 2*tile);
}
// coarse work estimate of the tile pipeline: number of the C*C coarse samples of a tile above the ocean-stop level, gathered origins in schedule order
__global__ void coarse_work_kernel(const float *__restrict__ coarse, unsigned cells, unsigned nt, float level, unsigned *__restrict__ work) {
	unsigned const t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t >= nt) return;
	unsigned n = 0;
	for (unsigned i = 0; i < cells; ++i) {n += !(__ldg(coarse + (size_t)t*cells + i) < level);}
	work[t] = n;
}
__global__ void gather_origins_kernel(const float2 *__restrict__ org, const unsigned *__restrict__ order, unsigned nt, float2 *__restrict__ out) {
	unsigned const t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t < nt) {out[t] = org[order[t]];}
}

template<bool SIMPLEX, bool WARP>
void launch_noise(int shape, dim3 grid, dim3 block, cudaStream_t st, float *out, unsigned nx, unsigned ny, unsigned y_off, float mx0, float my0,
	const float2 *origins, const NoiseParams &N, const PostParams &P, const float *tab, unsigned *mm)
{
	switch (shape) {
	case 1:  noise_grid_kernel<SIMPLEX, WARP, 1><<<grid, block, 0, st>>>(out, nx, ny, y_off, mx0, my0, origins, N, P, tab, mm); break;
	case 2:  noise_grid_kernel<SIMPLEX, WARP, 2><<<grid, block, 0, st>>>(out, nx, ny, y_off, mx0, my0, origins, N, P, tab, mm); break;
	default: noise_grid_kernel<SIMPLEX, WARP, 0><<<grid, block, 0, st>>>(out, nx, ny, y_off, mx0, my0, origins, N, P, tab, mm); break;
	}
}

} // namespace

int twi_init_minmax(tw_ctx *ctx, unsigned *d_mm_ord, uint32_t n) {
	init_minmax_kernel<<<(n + 255)/256, 256, 0, ctx->stream>>>(d_mm_ord, n);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_minmax_tiles(tw_ctx *ctx, cudaStream_t st, const float *d_vals, size_t tile_elems, uint32_t nt, unsigned *d_mm_ord, const unsigned *d_perm) {
	minmax_tiles_kernel<<<nt, 256, 0, st>>>(d_vals, tile_elems, d_mm_ord, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_coarse_work(tw_ctx *ctx, const float *d_coarse, unsigned cells, uint32_t nt, float level, unsigned *d_work) {
	coarse_work_kernel<<<(nt + 127)/128, 128, 0, ctx->stream>>>(d_coarse, cells, nt, level, d_work);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_gather_origins(tw_ctx *ctx, const void *d_org, const unsigned *d_order, uint32_t nt, void *d_out) {
	gather_origins_kernel<<<(nt + 255)/256, 256, 0, ctx->stream>>>((const float2 *)d_org, d_order, nt, (float2 *)d_out);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_minmax(tw_ctx *ctx, const float *d_vals, size_t n, unsigned *d_mm_ord) {
	int const blocks = (int)((n + 255)/256 < ctx->num_sms*8 ? (n + 255)/256 : ctx->num_sms*8);
	minmax_kernel<<<blocks > 0 ? blocks : 1, 256, 0, ctx->stream>>>(d_vals, n, d_mm_ord);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// Height generation for one grid (ntiles==0/1, d_tile_origins==nullptr) or a batch of equally sized tiles (noise modes only).
// rows per band: whole grid unless the result goes to a host buffer and is large enough to be worth overlapping (>= 32 MB); bands are
// multiples of 64 rows (the sine kernel's tile) and there are at most 16 of them
static unsigned band_rows_for(tw_ctx *ctx, unsigned ny, unsigned nx, bool to_host) {
	if (!to_host || (size_t)nx*ny*sizeof(float) < ((size_t)32 << 20) || !ctx->aux_stream[0]) return ny;
	unsigned rows = ((ny + 15)/16 + 63) & ~63u;
	return rows < 64 ? 64 : rows;
}
static int band_join(tw_ctx *ctx) { // ctx->stream waits for the band copies
	cudaEvent_t ev;
	TW_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
	TW_CUDA(ctx, cudaEventRecord(ev, ctx->aux_stream[0]));
	TW_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev, 0));
	TW_CUDA(ctx, cudaEventDestroy(ev));
	return TW_OK;
}

// After the kernel of a row band has been issued on ctx->stream: copy that band to the host buffer on the copy stream (overlaps the next band)
static int band_copy(tw_ctx *ctx, float *h_out, const float *d_out, unsigned nx, unsigned r0, unsigned r1) {
	cudaEvent_t ev;
	TW_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
	TW_CUDA(ctx, cudaEventRecord(ev, ctx->stream));
	TW_CUDA(ctx, cudaStreamWaitEvent(ctx->aux_stream[0], ev, 0));
	TW_CUDA(ctx, cudaEventDestroy(ev));
	TW_CUDA(ctx, cudaMemcpyAsync(h_out + (size_t)r0*nx, d_out + (size_t)r0*nx, (size_t)(r1 - r0)*nx*sizeof(float), cudaMemcpyDeviceToHost, ctx->aux_stream[0]));
	return TW_OK;
}

// h_out_bands != nullptr (single grid only): the grid is issued in row bands and each finished band is copied to the host buffer on a second
// stream while the next band computes; ctx->stream finally waits for the copies, so an event recorded on it covers the whole result.
static PostParams make_post_params(const tw_height_params *p, int enable_glaciate, float dx, float dy) {
	PostParams P;
	memset(&P, 0, sizeof(P));
	P.h = p->hmap;
	P.shape = p->gen_shape;
	P.need_postproc = 1; // get_noise_zval (:749) and apply_noise_shape_final (:570) call postproc_noise_zval unconditionally (3 compares at defaults)
	P.enable_glaciate = (enable_glaciate != 0);
	P.glaciate = (p->glaciate != 0);
	P.zmax_est = p->zmax_est;
	P.zmax_est2 = (float)(2.0*p->zmax_est);           // set_zmax_est, src/mesh_gen.cpp:162-167
	P.zmax_est2_inv = (float)(1.0/P.zmax_est2);
	P.custom_exp = p->custom_glaciate_exp;
	P.sine_on = (p->hmap.sine_mag > 0.0f);
	P.sm_scale = p->hmap.sine_mag*p->mesh_scale_z_inv;
	P.sm_freq = p->mesh_scale*p->hmap.sine_freq;
	P.sine_offset = p->hmap.sine_bias*p->mesh_scale_z_inv;
	P.volcano_on = (p->hmap.volcano_width > 0.0f && p->hmap.volcano_height > 0.0f);
	P.volcano_freq = P.volcano_on ? p->mesh_scale/p->hmap.volcano_width : 0.0f;
	P.mesh_scale_z_inv = p->mesh_scale_z_inv;
	P.mdx = dx; P.mdy = dy; P.dx_inv = p->dx_val_inv; P.dy_inv = p->dy_val_inv;
	return P;
}

static bool make_noise_params(const tw_height_params *p, NoiseParams &N, bool &simplex) {
	memset(&N, 0, sizeof(N));
	int const start = p->start_eval_sin;
	if (start < 0 || start > F_TABLE) return false;
	N.octaves = 9 - start/10;
	N.gen_shape = p->gen_shape;
	float mag = 1.0f, freq = 1.0f, rx = p->rx, ry = p->ry;
	for (int i = 0; i < 9; ++i) { // loop-carried constants of gen_noise, src/mesh_gen.cpp:725-728
		N.oct[i] = make_float4(freq, rx, ry, mag);
		mag *= 0.5f; freq *= 1.92f; rx *= 1.5f; ry *= 1.5f;
	}
	float4 const last = N.oct[N.octaves > 0 ? N.octaves - 1 : 0];
	N.freq_last = last.x; N.rsum_last = last.y + last.z;
	N.xy_scale = 0.0007f*p->mesh_scale; // MESH_SCALE_FACTOR, src/mesh_gen.cpp:23,737
	simplex = (p->gen_mode == TW_MGEN_SIMPLEX || p->gen_mode == TW_MGEN_SIMPLEX_GPU || p->gen_mode == TW_MGEN_DWARP_GPU);
	N.hmap_scale = (simplex ? 16.0f : 32.0f)*p->mesh_height*p->mesh_height_scale*p->mesh_scale_z_inv; // get_hmap_scale, :550-553
	return true;
}

size_t twi_heightgen_slot1_bytes(const tw_grid2d *g, const tw_height_params *p) { // the sine-table mode's X / Y tables below
	if (p->gen_mode != TW_MGEN_SINE) return 0;
	unsigned const xpitch = (g->nx + 63) & ~63u, ypitch = (g->ny + 63) & ~63u;
	return (size_t)(F_TABLE + 1)*(xpitch + ypitch)*sizeof(float);
}

int twi_heightgen(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin,
                  const float2 *d_tile_origins, uint32_t ntiles, float *d_out, unsigned *d_mm_ord, float *h_out_bands)
{
	unsigned const nx = g->nx, ny = g->ny;
	float const dx = g->dx, dy = g->dy;
	float const mx0 = dx*g->x0, my0 = dy*g->y0; // src/mesh_gen.cpp:591
	if (ntiles == 0) ntiles = 1;

	PostParams P = make_post_params(p, enable_glaciate, dx, dy);
	P.skip_x0 = ctx->skip_rect[0]; P.skip_y0 = ctx->skip_rect[1]; P.skip_w = ctx->skip_rect[2]; P.skip_h = ctx->skip_rect[3];
	P.tile_perm = ctx->tile_perm;
	if (P.tile_perm && (p->gen_mode == TW_MGEN_SINE || getenv("TW_NOISE_SCALAR"))) return tw_set_error(ctx, TW_ERR_STATE, "internal: tile_perm is only wired into the paired noise kernels");

	if (p->gen_mode != TW_MGEN_SINE) {
		NoiseParams N;
		bool simplex = false;
		if (!make_noise_params(p, N, simplex)) return tw_set_error(ctx, TW_ERR_ARG, "start_eval_sin %d out of range", p->start_eval_sin);
		bool const warp = (p->gen_mode == TW_MGEN_DWARP_GPU);
		{int const rc = twi_ensure_simplex_lut(ctx); if (rc) return rc;}
		const float4 *lut = (const float4 *)ctx->d_simplex_lut + (simplex ? 0 : PERLIN_LUT_OFFSET);
		unsigned const band_rows = band_rows_for(ctx, ny, nx, h_out_bands != nullptr && ntiles == 1);
		for (unsigned r0 = 0; r0 < ny; r0 += band_rows) {
			unsigned const r1 = (ny - r0 < band_rows) ? ny : r0 + band_rows;
			static bool const use_scalar = (getenv("TW_NOISE_SCALAR") != nullptr); // A/B switch: one cell per thread, scalar FMUL/FADD
			if (!use_scalar) { // two cells per thread
				size_t const band_cells = (size_t)(r1 - r0)*nx;
				unsigned gx = (unsigned)((band_cells + TW_NOISE2_BLOCK_CELLS - 1)/TW_NOISE2_BLOCK_CELLS);
				P.ngroups = gx;
#if TW_NOISE2_PERSISTENT
				{unsigned const wave = ctx->num_sms*TW_NOISE2_MIN_BLOCKS*TW_NOISE2_PERSISTENT; if (ntiles == 1 && gx > wave) gx = wave;} // TW_NOISE2_PERSISTENT waves' worth of resident blocks
#endif
				dim3 const block(TW_NOISE2_THREADS, 1, 1), grid(gx, 1, ntiles);
				if (p->gen_mode == TW_MGEN_PERLIN) {launch_noise2<false, false>(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, r1, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord, lut);}
				else if (warp) {launch_noise2<true, true >(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, r1, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord, lut);}
				else           {launch_noise2<true, false>(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, r1, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord, lut);}
				TW_LAUNCH_CHECK(ctx);
				if (h_out_bands) {int const rc = band_copy(ctx, h_out_bands, d_out, nx, r0, r1); if (rc) return rc;}
				continue;
			}
			dim3 const block(32, 8, 1), grid((nx + 31)/32, (r1 - r0 + 7)/8, ntiles);
			if (p->gen_mode == TW_MGEN_PERLIN) {launch_noise<false, false>(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord);}
			else if (warp) {launch_noise<true, true >(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord);}
			else           {launch_noise<true, false>(p->gen_shape, grid, block, ctx->stream, d_out, nx, ny, r0, mx0, my0, d_tile_origins, N, P, ctx->d_sin_table, d_mm_ord);}
			TW_LAUNCH_CHECK(ctx);
			if (h_out_bands) {int const rc = band_copy(ctx, h_out_bands, d_out, nx, r0, r1); if (rc) return rc;}
		}
		return h_out_bands ? band_join(ctx) : TW_OK;
	}

	// ---- sine-table mode ----
	if (!ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called");
	if (d_tile_origins && ntiles > 1) return tw_set_error(ctx, TW_ERR_ARG, "internal: sine mode tiles are issued one grid at a time");
	unsigned const xpitch = (nx + 63) & ~63u, ypitch = (ny + 63) & ~63u;
	size_t const tab_floats = (size_t)(F_TABLE + 1)*(xpitch + ypitch);
	int rc = tw_reserve(ctx, 1, tab_floats*sizeof(float));
	if (rc) return rc;
	float *Xt = (float *)ctx->d_scratch[1], *Yt = Xt + (size_t)(F_TABLE + 1)*xpitch;
	SineTabParams S;
	memset(&S, 0, sizeof(S));
	S.msx = p->mesh_scale*p->dx_val_inv; S.msy = p->mesh_scale*p->dy_val_inv; S.ms2 = (float)(0.5*p->mesh_scale);
	S.mesh_scale_z_inv = p->mesh_scale_z_inv;
	S.dx = dx; S.dy = dy; S.mx0 = mx0; S.my0 = my0;
	S.start = p->start_eval_sin;
	S.nx = nx; S.ny = ny; S.xpitch = xpitch; S.ypitch = ypitch;
	S.sine_on = (enable_glaciate && p->hmap.sine_mag != 0.0f); S.sm_scale = P.sm_scale; S.sm_freq = P.sm_freq; S.dx_inv = p->dx_val_inv; S.dy_inv = p->dy_val_inv;
	{
		unsigned const nmax = nx > ny ? nx : ny;
		dim3 const grid((nmax + 255)/256, F_TABLE + 1, 2);
		sine_tables_kernel<<<grid, 256, 0, ctx->stream>>>(Xt, Yt, ctx->d_sine_params, ctx->d_sin_table, S);
		TW_LAUNCH_CHECK(ctx);
	}
	int const start_ix = (p->start_eval_sin > min_start_sin) ? p->start_eval_sin : min_start_sin; // src/mesh_gen.cpp:769
	unsigned const band_rows = band_rows_for(ctx, ny, nx, h_out_bands != nullptr);
	for (unsigned r0 = 0; r0 < ny; r0 += band_rows) {
		unsigned const r1 = (ny - r0 < band_rows) ? ny : r0 + band_rows;
		dim3 const grid((nx + ST - 1)/ST, (r1 - r0 + ST - 1)/ST, 1);
		sine_grid_kernel<<<grid, 256, 0, ctx->stream>>>(d_out, nx, ny, Xt, Yt, xpitch, ypitch, start_ix, P, mx0, my0, ctx->d_sin_table, d_mm_ord, r0);
		TW_LAUNCH_CHECK(ctx);
		if (h_out_bands) {int const rc = band_copy(ctx, h_out_bands, d_out, nx, r0, r1); if (rc) return rc;}
	}
	return h_out_bands ? band_join(ctx) : TW_OK;
}

// Sine-mode tile batch (tile_t::create_zvals / create_texture in force_sine_mode): tables once per distinct tile column / row (twi_sine_tiles_setup), then
// ONE grid launch per <= 65535 tiles (twi_sine_tiles_grid). h_org = ntiles (mx0, my0) pairs (HOST; mx0 = dx*float(x1 - MESH_X_SIZE/2) as build_arrays computes it).
size_t twi_sine_tiles_stage_bytes(uint32_t ntiles) {return (size_t)ntiles*(2*sizeof(float) + sizeof(uint2) + sizeof(float2));} // distinct origins (<= 2 per tile), table indices, origins

namespace {
// a sine batch's device memory: the tables (nux X tables, then nuy Y tables), the distinct origins, the tiles' table indices and origins
struct SineTilesMem {float *Xt, *uorg; uint2 *tabs; float2 *torg;};
SineTilesMem sine_tiles_layout(twi_carve &c, const tw_grid2d *g, size_t nux, size_t nuy, uint32_t ntiles) {
	size_t const xstride = (size_t)(F_TABLE + 1)*((g->nx + 63) & ~63u), ystride = (size_t)(F_TABLE + 1)*((g->ny + 63) & ~63u);
	SineTilesMem M;
	M.Xt = c.take<float>(nux*xstride + nuy*ystride); M.uorg = c.take<float>(nux + nuy); M.tabs = c.take<uint2>(ntiles); M.torg = c.take<float2>(ntiles);
	return M;
}
} // namespace

size_t twi_sine_tiles_plan(const tw_grid2d *g, const float2 *h_org, uint32_t ntiles, twi_sine_batch *b) { // distinct origins (bit patterns) -> table indices
	std::unordered_map<uint32_t, unsigned> mx, my;
	std::vector<float> uy;
	b->uorg.clear(); b->tabs.resize(ntiles);
	for (uint32_t t = 0; t < ntiles; ++t) {
		uint32_t bx, by;
		memcpy(&bx, &h_org[t].x, 4); memcpy(&by, &h_org[t].y, 4);
		auto ix = mx.find(bx); if (ix == mx.end()) {ix = mx.emplace(bx, (unsigned)b->uorg.size()).first; b->uorg.push_back(h_org[t].x);}
		auto iy = my.find(by); if (iy == my.end()) {iy = my.emplace(by, (unsigned)uy.size()).first; uy.push_back(h_org[t].y);}
		b->tabs[t] = make_uint2(ix->second, iy->second);
	}
	b->nux = (unsigned)b->uorg.size(); b->nuy = (unsigned)uy.size();
	b->uorg.insert(b->uorg.end(), uy.begin(), uy.end()); // [distinct x origins | distinct y origins]
	twi_carve c; sine_tiles_layout(c, g, b->nux, b->nuy, ntiles);
	return c.bytes;
}

int twi_sine_tiles_setup(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, const float2 *h_org, uint32_t ntiles,
                         void *d_mem, void *h_stage, twi_sine_batch *b)
{
	if (!ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called");
	unsigned const nx = g->nx, ny = g->ny;
	PostParams const P = make_post_params(p, enable_glaciate, g->dx, g->dy);
	unsigned const nux = b->nux, nuy = b->nuy;
	if (nux + nuy > 65535) return tw_set_error(ctx, TW_ERR_ARG, "more than 65535 distinct tile rows + columns in one batch"); // gridDim.z of the table launch
	unsigned const xpitch = (nx + 63) & ~63u, ypitch = (ny + 63) & ~63u;
	size_t const xstride = (size_t)(F_TABLE + 1)*xpitch, ystride = (size_t)(F_TABLE + 1)*ypitch;
	SineTilesMem M;
	auto layout = [&](twi_carve &c) {M = sine_tiles_layout(c, g, nux, nuy, ntiles);};
	if (d_mem) {twi_carve c{(char *)d_mem}; layout(c);}
	else {int const rc = twi_reserve_carve(ctx, 1, layout); if (rc) return rc;}
	float *Xt = M.Xt, *Yt = Xt + nux*xstride, *d_uorg = M.uorg; uint2 *d_tabs = M.tabs; float2 *d_torg = M.torg;
	std::vector<float> const &uorg = b->uorg;
	const void *src_uorg = uorg.data(), *src_tabs = b->tabs.data(), *src_org = h_org;
	if (h_stage) { // pinned copies that outlive this call: nothing below has to wait for the uploads
		char *hs = (char *)h_stage;
		memcpy(hs, uorg.data(), uorg.size()*sizeof(float)); src_uorg = hs; hs += (size_t)2*ntiles*sizeof(float);
		memcpy(hs, b->tabs.data(), (size_t)ntiles*sizeof(uint2)); src_tabs = hs; hs += (size_t)ntiles*sizeof(uint2);
		memcpy(hs, h_org, (size_t)ntiles*sizeof(float2)); src_org = hs;
	}
	TW_CUDA(ctx, cudaMemcpyAsync(d_uorg, src_uorg, uorg.size()*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(d_tabs, src_tabs, (size_t)ntiles*sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
	TW_CUDA(ctx, cudaMemcpyAsync(d_torg, src_org, (size_t)ntiles*sizeof(float2), cudaMemcpyHostToDevice, ctx->stream));
	SineTabParams S;
	memset(&S, 0, sizeof(S));
	S.msx = p->mesh_scale*p->dx_val_inv; S.msy = p->mesh_scale*p->dy_val_inv; S.ms2 = (float)(0.5*p->mesh_scale);
	S.mesh_scale_z_inv = p->mesh_scale_z_inv;
	S.dx = g->dx; S.dy = g->dy;
	S.start = p->start_eval_sin;
	S.nx = nx; S.ny = ny; S.xpitch = xpitch; S.ypitch = ypitch;
	S.sine_on = (enable_glaciate && p->hmap.sine_mag != 0.0f); S.sm_scale = P.sm_scale; S.sm_freq = P.sm_freq; S.dx_inv = p->dx_val_inv; S.dy_inv = p->dy_val_inv;
	unsigned const nmax = nx > ny ? nx : ny;
	sine_tables_kernel<<<dim3((nmax + 255)/256, F_TABLE + 1, nux + nuy), 256, 0, ctx->stream>>>(Xt, Yt, ctx->d_sine_params, ctx->d_sin_table, S, d_uorg, nux, xstride, ystride);
	TW_LAUNCH_CHECK(ctx);
	if (!h_stage) {TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));} // the async copies read the plan's host vectors
	b->g = *g; b->p = *p; b->enable_glaciate = enable_glaciate; b->min_start_sin = min_start_sin;
	b->Xt = Xt; b->Yt = Yt; b->d_tabs = d_tabs; b->d_torg = d_torg; b->xstride = xstride; b->ystride = ystride; b->xpitch = xpitch; b->ypitch = ypitch;
	return TW_OK;
}

int twi_sine_tiles_grid(tw_ctx *ctx, const twi_sine_batch *b, uint32_t t0, uint32_t nt, const unsigned *d_perm, float *d_out, unsigned *d_mm_ord) {
	unsigned const nx = b->g.nx, ny = b->g.ny;
	PostParams const P = make_post_params(&b->p, b->enable_glaciate, b->g.dx, b->g.dy);
	int const start_ix = (b->p.start_eval_sin > b->min_start_sin) ? b->p.start_eval_sin : b->min_start_sin; // src/mesh_gen.cpp:769
	for (uint32_t c0 = 0; c0 < nt; c0 += 65535) {
		uint32_t const cn = std::min<uint32_t>(65535u, nt - c0);
		size_t const s = (size_t)t0 + c0; // batch index of the launch's first tile (through d_perm when given)
		sine_grid_kernel<<<dim3((nx + ST - 1)/ST, (ny + ST - 1)/ST, cn), 256, 0, ctx->stream>>>(d_out + (size_t)c0*nx*ny, nx, ny, b->Xt, b->Yt, b->xpitch, b->ypitch, start_ix, P, 0.0f, 0.0f,
			ctx->d_sin_table, d_mm_ord ? d_mm_ord + 2*(size_t)c0 : nullptr, 0, d_perm ? b->d_tabs : b->d_tabs + s, d_perm ? b->d_torg : b->d_torg + s, b->xstride, b->ystride,
			d_perm ? d_perm + s : nullptr);
		TW_LAUNCH_CHECK(ctx);
	}
	return TW_OK;
}

int twi_heightgen_sine_tiles(tw_ctx *ctx, const tw_grid2d *g, const tw_height_params *p, int enable_glaciate, int min_start_sin, const float2 *h_org, uint32_t ntiles,
                             float *d_out, unsigned *d_mm_ord, void *h_stage)
{
	twi_sine_batch b;
	twi_sine_tiles_plan(g, h_org, ntiles, &b);
	int rc = twi_sine_tiles_setup(ctx, g, p, enable_glaciate, min_start_sin, h_org, ntiles, nullptr, h_stage, &b); if (rc) return rc;
	return twi_sine_tiles_grid(ctx, &b, 0, ntiles, nullptr, d_out, d_mm_ord);
}

// ------------------------------------------------------------------------------------------------ point queries (SURVEY 8a row a9)
// eval_mesh_sin_terms (src/mesh_gen.cpp:797-805), eval_mesh_sin_terms_scaled (:807-813) and the procedural branch of get_exact_zval
// (:816-847) for a batch of arbitrary points: one thread per point; the 90 sine-table rows are read from constant-like global memory
// (uniform across the warp), the two SINF look-ups per term hit the 256 KB table in L1/L2.
struct PointParams {
	int   kind, sine_mode, start, glaciate;
	float xy_scale, mesh_scale, x_scene_size, y_scene_size;
	float half_mx, half_my;      // float(MESH_X_SIZE >> 1), float(MESH_Y_SIZE >> 1)
	float xoff, yoff;            // float(xoff2), float(yoff2) or 0 when no_xyoff
	float sine_mag, sine_bias, sine_freq; // apply_mesh_sine: hmap.sine_mag, hmap.sine_bias, mesh_scale*hmap.sine_freq
};

__device__ __forceinline__ float eval_mesh_sin_terms(float xv, float yv, const float *__restrict__ T, const float *__restrict__ tab, int start) {
	float zval = 0.0f;
	for (int k = start; k < F_TABLE; ++k) { // zval += stk[0]*SINF(stk[3]*yv + stk[1])*SINF(stk[4]*xv + stk[2]), left to right
		const float *stk = T + 5*k;
		float const t = __ldg(stk)*sinf_lut(tab, __ldg(stk + 3)*yv + __ldg(stk + 1));
		zval += t*sinf_lut(tab, __ldg(stk + 4)*xv + __ldg(stk + 2));
	}
	return zval;
}

template<bool SIMPLEX, bool WARP, int SHAPE>
__global__ void __launch_bounds__(256)
points_kernel(const float2 *__restrict__ xy, size_t n, float *__restrict__ out, PointParams Q, NoiseParams N, PostParams P,
	const float *__restrict__ T, const float *__restrict__ tab)
{
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	float2 const pt = __ldg(xy + i);
	if (Q.kind == TW_PQ_SIN_TERMS) {out[i] = eval_mesh_sin_terms(pt.x, pt.y, T, tab, Q.start); return;}
	float xval = pt.x, yval = pt.y;
	if (Q.kind == TW_PQ_EXACT_ZVAL) { // real -> index space, src/mesh_gen.cpp:818-819,826-829 (the "+ 0.5" double add rounds like the float add)
		xval = (pt.x + Q.x_scene_size)*P.dx_inv + 0.5f + Q.xoff;
		yval = (pt.y + Q.y_scene_size)*P.dy_inv + 0.5f + Q.yoff;
	}
	float const xv = Q.xy_scale*(xval - Q.half_mx), yv = Q.xy_scale*(yval - Q.half_my); // :808
	float z;
	if (!Q.sine_mode) {z = get_noise_zval<SIMPLEX, WARP, SHAPE>(xv, yv, N, P);}
	else {
		z = eval_mesh_sin_terms(Q.mesh_scale*xv, Q.mesh_scale*yv, T, tab, Q.start)*P.mesh_scale_z_inv;
		if (P.shape == 1) {z = (float)((double)fabsf(z) - 2.0);}       // apply_noise_shape_final, src/mesh_gen.cpp:564-571
		else if (P.shape == 2) {z = (float)(3.5 - (double)fabsf(z));}
		z = postproc_noise_zval(z, P.h);
	}
	if (Q.kind == TW_PQ_EXACT_ZVAL) {
		if (Q.glaciate) { // apply_glaciate, :380-385
			float const relh = (z + P.zmax_est)*P.zmax_est2_inv;
			float const g = (P.custom_exp == 0.0f) ? relh*relh*relh : powf(relh, P.custom_exp);
			z = g*P.zmax_est2 - P.zmax_est;
		}
		if (P.sine_on) { // apply_mesh_sine, :373-379
			float const x = xval - Q.half_mx, y = yval - Q.half_my;
			z += (Q.sine_mag*cosf_lut(tab, x*Q.sine_freq)*cosf_lut(tab, y*Q.sine_freq) + Q.sine_bias)*P.mesh_scale_z_inv;
			if (P.volcano_on) {z += volcano_height(x, y, P, tab);}
		}
	}
	out[i] = z;
}

template<bool SIMPLEX, bool WARP>
static void launch_points(int shape, unsigned grid, cudaStream_t st, const float2 *xy, size_t n, float *out, const PointParams &Q, const NoiseParams &N,
	const PostParams &P, const float *T, const float *tab)
{
	switch (shape) {
	case 1:  points_kernel<SIMPLEX, WARP, 1><<<grid, 256, 0, st>>>(xy, n, out, Q, N, P, T, tab); break;
	case 2:  points_kernel<SIMPLEX, WARP, 2><<<grid, 256, 0, st>>>(xy, n, out, Q, N, P, T, tab); break;
	default: points_kernel<SIMPLEX, WARP, 0><<<grid, 256, 0, st>>>(xy, n, out, Q, N, P, T, tab); break;
	}
}

int twi_eval_points(tw_ctx *ctx, const float *d_xy, size_t n, const tw_height_params *p, const tw_point_query *q, float *d_out) {
	if (q->kind < TW_PQ_SIN_TERMS || q->kind > TW_PQ_EXACT_ZVAL) return tw_set_error(ctx, TW_ERR_ARG, "tw_eval_points: bad kind %d", q->kind);
	bool const sine_mode = (p->gen_mode == TW_MGEN_SINE || q->kind == TW_PQ_SIN_TERMS);
	if (sine_mode && !ctx->have_sine_params) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sine_params() has not been called");
	if (p->start_eval_sin < 0 || p->start_eval_sin > F_TABLE) return tw_set_error(ctx, TW_ERR_ARG, "start_eval_sin %d out of range", p->start_eval_sin);
	if (n > (size_t)0x7fffffff*256) return tw_set_error(ctx, TW_ERR_ARG, "tw_eval_points: too many points");
	PostParams const P = make_post_params(p, 1, 0.0f, 0.0f);
	NoiseParams N;
	bool simplex = true;
	memset(&N, 0, sizeof(N));
	if (!sine_mode && !make_noise_params(p, N, simplex)) return tw_set_error(ctx, TW_ERR_ARG, "start_eval_sin out of range");
	PointParams Q;
	memset(&Q, 0, sizeof(Q));
	Q.kind = q->kind; Q.sine_mode = sine_mode; Q.start = p->start_eval_sin; Q.glaciate = (p->glaciate != 0);
	Q.xy_scale = (q->kind == TW_PQ_EXACT_ZVAL) ? 1.0f : q->xy_scale;
	Q.mesh_scale = p->mesh_scale; Q.x_scene_size = q->x_scene_size; Q.y_scene_size = q->y_scene_size;
	Q.half_mx = (float)(q->mesh_x_size >> 1); Q.half_my = (float)(q->mesh_y_size >> 1);
	Q.xoff = q->no_xyoff ? 0.0f : (float)q->xoff2; Q.yoff = q->no_xyoff ? 0.0f : (float)q->yoff2;
	Q.sine_mag = p->hmap.sine_mag; Q.sine_bias = p->hmap.sine_bias; Q.sine_freq = p->mesh_scale*p->hmap.sine_freq;
	unsigned const grid = (unsigned)((n + 255)/256);
	const float2 *xy = reinterpret_cast<const float2 *>(d_xy);
	bool const warp = (p->gen_mode == TW_MGEN_DWARP_GPU);
	if (sine_mode)                           {launch_points<true,  false>(p->gen_shape, grid, ctx->stream, xy, n, d_out, Q, N, P, ctx->d_sine_params, ctx->d_sin_table);}
	else if (p->gen_mode == TW_MGEN_PERLIN)  {launch_points<false, false>(p->gen_shape, grid, ctx->stream, xy, n, d_out, Q, N, P, ctx->d_sine_params, ctx->d_sin_table);}
	else if (warp)                           {launch_points<true,  true >(p->gen_shape, grid, ctx->stream, xy, n, d_out, Q, N, P, ctx->d_sine_params, ctx->d_sin_table);}
	else                                     {launch_points<true,  false>(p->gen_shape, grid, ctx->stream, xy, n, d_out, Q, N, P, ctx->d_sine_params, ctx->d_sin_table);}
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
