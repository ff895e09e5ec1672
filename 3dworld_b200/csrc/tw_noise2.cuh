// tw_noise2.cuh - two-cells-per-thread versions of glm::simplex(vec2) / glm::perlin(vec2), their table-driven forms (simplex2_lut /
// perlin2_lut: hash and gradient from a shared-memory table, the shipped path) and the table-driven one-voxel-per-thread 3-D forms
// (simplex3_lut / perlin3_lut).
// A thread evaluates two horizontally adjacent cells: the two evaluations are independent chains of the same instructions (twice the
// instruction-level parallelism per thread), and they share the per-thread table base and the per-octave scalars.
//
// Every operation is the same IEEE round-to-nearest op as in tw_noise.cuh, element-wise (see that file for the exactness arguments of the
// hand-placed fused forms). The element-wise primitives below use the explicitly rounded intrinsics (__fmul_rn / __fadd_rn / __fsub_rn),
// which the compiler never contracts into a fused multiply-add: a fused multiply-add rounds once where the reference rounds twice.
// floor() stays on FRND.
// The caller guarantees |lattice coordinate| < 2^22 (noise_lattice_in_range, needed by the division-free mod); otherwise it uses the
// scalar path of tw_noise.cuh.
#pragma once
#include <cuda_runtime.h>
#include "tw_noise.cuh"

namespace twn2 {

typedef float2 f2;

__device__ __forceinline__ f2 splat(float v) {return make_float2(v, v);}
__device__ __forceinline__ f2 raw_fma(f2 a, f2 b, f2 c) {return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));}
__device__ __forceinline__ f2 mul2(f2 a, f2 b) {return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));}
__device__ __forceinline__ f2 mul2(f2 a, float b) {return mul2(a, splat(b));}
__device__ __forceinline__ f2 add2(f2 a, f2 b) {return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));}
__device__ __forceinline__ f2 add2(f2 a, float b) {return add2(a, splat(b));}
__device__ __forceinline__ f2 sub2(f2 a, f2 b) {return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));}
__device__ __forceinline__ f2 rsub2(float a, f2 b) {return sub2(splat(a), b);}   // a - b, scalar a
// a*b + c*d, unfused
__device__ __forceinline__ f2 sumprod2(f2 a, f2 b, f2 c, f2 d) {return add2(mul2(a, b), mul2(c, d));}
__device__ __forceinline__ f2 sumprod2(f2 a, float b, f2 c, float d) {return sumprod2(a, splat(b), c, splat(d));}
// genuine fused multiply-adds: only where the product is exact, so fused == unfused (see tw_noise.cuh); `a` is never itself a product
__device__ __forceinline__ f2 fma2(f2 a, float b, f2 c) {return raw_fma(a, splat(b), c);}
__device__ __forceinline__ f2 fma2(f2 a, float b, float c) {return raw_fma(a, splat(b), splat(c));}
__device__ __forceinline__ f2 abs2(f2 a) {return make_float2(fabsf(a.x), fabsf(a.y));}
__device__ __forceinline__ f2 max0_2(f2 a) {return make_float2(fmaxf(a.x, 0.0f), fmaxf(a.y, 0.0f));} // see twn::gmax0
// max(a - d, 0) as one saturating subtract (FADD.SAT) for the simplex falloff terms, d a sum of squares, a = 0.5 or 0.6: the same bits as
// fmaxf(a - d, 0.0f) for every d. The saturation clamps to [0, 1]; d >= 0 keeps a - d <= a < 1, so only the lower clamp can act, and it is max(., 0).
// A NaN saturates to +0, as fmaxf(NaN, 0) returns +0; an exact zero difference is +0 under round-to-nearest either way.
__device__ __forceinline__ float rsub_max0(float a, float d) {float r; asm("sub.rn.sat.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(d)); return r;}
__device__ __forceinline__ f2 rsub_max0_2(float a, f2 d) {return make_float2(rsub_max0(a, d.x), rsub_max0(a, d.y));}
__device__ __forceinline__ f2 floor2(f2 x) {return make_float2(floorf(x.x), floorf(x.y));}

__device__ __forceinline__ f2 mod289(f2 x)  {f2 const t = floor2(mul2(x, 1.0f/289.0f)); return fma2(t, -289.0f, x);}
__device__ __forceinline__ f2 permute(f2 x) {return mod289(mul2(fma2(x, 34.0f, 1.0f), x));}
// glm::mod(a, 289) for integer |a| < 2^22 (see twn::mod_int289): q = floor(a*RN(1/289)) can be one short only when a is a multiple of 289,
// leaving r = 289, which one conditional subtract folds back to 0.
__device__ __forceinline__ f2 mod_int289(f2 a) {
	f2 const r = fma2(floor2(mul2(a, 1.0f/289.0f)), -289.0f, a);
	return make_float2((r.x >= 289.0f) ? r.x - 289.0f : r.x, (r.y >= 289.0f) ? r.y - 289.0f : r.y);
}
// Same without the fold: r in [0, 289], with 289 standing for 0 (only for exact multiples of 289). Sufficient wherever r only feeds exact
// integer arithmetic modulo 289 - permute(r + c) (arguments stay below 2^24, so the float hash is the exact integer hash and
// permute(289 + c) == permute(c)) - or a table whose entries 289 and 290 repeat 0 and 1 by the same arithmetic. Used by the table variants.
__device__ __forceinline__ f2 mod_int289_lazy(f2 a) {return fma2(floor2(mul2(a, 1.0f/289.0f)), -289.0f, a);}
__device__ __forceinline__ f2 fract2(f2 x) {return sub2(x, floor2(x));}
__device__ __forceinline__ f2 tinvsqrt(f2 r) {return rsub2(1.79284291400159f, mul2(r, 0.85373472095314f));}
__device__ __forceinline__ f2 mix2(f2 x, f2 y, f2 a) {return add2(x, mul2(a, sub2(y, x)));}
__device__ __forceinline__ f2 fade2(f2 t) { // (t*t*t)*(t*(t*6 - 15) + 10)
	f2 const t3 = mul2(mul2(t, t), t);
	return mul2(t3, add2(mul2(t, add2(mul2(t, 6.0f), -15.0f)), 10.0f));
}

// glm::simplex(vec2) for two positions (v.x = first cell, v.y = second cell of each operand)
__device__ __forceinline__ f2 simplex2(f2 vx, f2 vy) {
	float const Cx = 0.211324865405187f, Cy = 0.366025403784439f, Cz = -0.577350269189626f, Cw = 0.024390243902439f;
	f2 const s = add2(mul2(vx, Cy), mul2(vy, Cy));
	f2 ix = floor2(add2(vx, s)), iy = floor2(add2(vy, s));
	f2 const t = add2(mul2(ix, Cx), mul2(iy, Cx));
	f2 const x0x = add2(sub2(vx, ix), t), x0y = add2(sub2(vy, iy), t);
	f2 const i1x = make_float2((x0x.x > x0y.x) ? 1.0f : 0.0f, (x0x.y > x0y.y) ? 1.0f : 0.0f);
	f2 const i1y = rsub2(1.0f, i1x); // (1,0) or (0,1)
	f2 const x12x = sub2(add2(x0x, Cx), i1x), x12y = sub2(add2(x0y, Cx), i1y), x12z = add2(x0x, Cz), x12w = add2(x0y, Cz);
	ix = mod_int289(ix); iy = mod_int289(iy);
	f2 const q0 = permute(iy), q1 = permute(add2(iy, i1y)), q2 = permute(add2(iy, 1.0f));
	f2 const p0 = permute(add2(q0, ix)), p1 = permute(add2(add2(q1, ix), i1x)), p2 = permute(add2(add2(q2, ix), 1.0f));
	f2 m0 = max0_2(rsub2(0.5f, add2(mul2(x0x, x0x), mul2(x0y, x0y))));
	f2 m1 = max0_2(rsub2(0.5f, add2(mul2(x12x, x12x), mul2(x12y, x12y))));
	f2 m2 = max0_2(rsub2(0.5f, add2(mul2(x12z, x12z), mul2(x12w, x12w))));
	m0 = mul2(m0, m0); m1 = mul2(m1, m1); m2 = mul2(m2, m2);
	m0 = mul2(m0, m0); m1 = mul2(m1, m1); m2 = mul2(m2, m2);
	f2 const t0 = mul2(p0, Cw), t1 = mul2(p1, Cw), t2 = mul2(p2, Cw);
	f2 const X0 = fma2(sub2(t0, floor2(t0)), 2.0f, -1.0f), X1 = fma2(sub2(t1, floor2(t1)), 2.0f, -1.0f), X2 = fma2(sub2(t2, floor2(t2)), 2.0f, -1.0f);
	f2 const h0 = add2(abs2(X0), -0.5f), h1 = add2(abs2(X1), -0.5f), h2 = add2(abs2(X2), -0.5f);
	f2 const a0 = sub2(X0, floor2(add2(X0, 0.5f))), a1 = sub2(X1, floor2(add2(X1, 0.5f))), a2 = sub2(X2, floor2(add2(X2, 0.5f)));
	m0 = mul2(m0, tinvsqrt(add2(mul2(a0, a0), mul2(h0, h0))));
	m1 = mul2(m1, tinvsqrt(add2(mul2(a1, a1), mul2(h1, h1))));
	m2 = mul2(m2, tinvsqrt(add2(mul2(a2, a2), mul2(h2, h2))));
	f2 const gx = add2(mul2(a0, x0x), mul2(h0, x0y)), gy = add2(mul2(a1, x12x), mul2(h1, x12y)), gz = add2(mul2(a2, x12z), mul2(h2, x12w));
	return mul2(add2(add2(mul2(m0, gx), mul2(m1, gy)), mul2(m2, gz)), 130.0f);
}

// ---- simplex with tabulated hash/gradient (TW_SIMPLEX_LUT) ----
// After `i = mod(i, 289)` everything between the lattice index and the gradient is a function of small integers:
//   q = permute(iy + {0, i1.y, 1})       argument in [0, 290]  -> value in [0, 288]
//   p = permute(q + ix + {0, i1.x, 1})   argument in [0, 578]  -> value in [0, 288]   (exhaustively: the float arithmetic is exact there)
//   x = 2*fract(p*C.w) - 1, h = |x| - 0.5, a0 = x - floor(x + 0.5), n = taylorInvSqrt(a0*a0 + h*h)   depend on p only.
// simplex_lut_entry() evaluates exactly those reference operations once per integer; at levels 1/2 the kernel keeps a 291-entry table
// {a0, h, n, permute(k)} in shared memory and replaces 22 instructions + 8 floors per cell pair and corner (level 1: gradient) plus 8 + 4 per
// corner (level 2: the first permute) by one 16-byte load each. Random indices would collide on the 32 banks, so the table is stored as 8
// interleaved copies: entry k of copy c sits at float4 index 8*k + c and lane l reads copy l & 7 - the 8 lanes of every quarter-warp phase
// of an LDS.128 then hit 8 different 16-byte bank groups by construction (conflict-free, 4 cycles per warp load).
// Level 3 folds the second permute into the gradient entries: entry k = {gradient of permute(k), permute(k)} for every reachable argument
// k = permute(iy') + ix' <= 578, so the gradient is fetched at k directly and the second hash (8 instructions + 4 floors per cell pair and corner)
// disappears at no extra load; the table grows to 580 entries (74 KB with the 8 copies; 3 blocks of 256 threads per SM measured the same as 5
// before it: the kernel is bound by instruction issue).
#ifndef TW_SIMPLEX_LUT
#define TW_SIMPLEX_LUT 3
#endif
constexpr int SIMPLEX_LUT_COPIES = 8;
constexpr int LUT3D_N = 580;                                  // 3-D tables (tw_voxel.cu): same folding of the LAST permute, arguments <= 578
constexpr int SIMPLEX_LUT_N = (TW_SIMPLEX_LUT >= 3) ? 580 : 291; // 2-D tables

__device__ __forceinline__ float4 simplex_lut_entry(float k) { // scalar restatement of twn::simplex2's per-corner gradient and of permute()
	float const Cw = 0.024390243902439f;
	float const pk = twn::permute(k);
	float const gi = (TW_SIMPLEX_LUT >= 3) ? pk : k; // level 3: the entry holds the gradient of the hashed index
	float const X = twn::two_f_minus_1(twn::fract(gi*Cw));
	float const h = fabsf(X) - 0.5f, a0 = X - floorf(X + 0.5f);
	float const n = 1.79284291400159f - 0.85373472095314f*(a0*a0 + h*h);
	return make_float4(a0, h, n, pk);
}

// Table addressing without integer arithmetic on the index: for an exact small non-negative integer k held in a float,
// k*128 + 1.5*2^23 is exact (one genuine FFMA per cell) and its bit pattern is 0x4B400000 + 128*k, i.e. a byte offset into the
// 8-copy table (8 copies * 16 bytes per entry) plus a constant. The constant and the lane's copy are folded into the per-thread base
// `Lb` (32-bit shared-memory address), so a look-up is one integer add and one LDS - no F2I (XU pipe), no shift, no mask.
// k is in range by construction (see above; NaN and far-out inputs never get here: noise_lattice_in_range sends them to the scalar path).
// TW_LUT_DENORM (default): the magic number is a DENORMAL. k*(128*2^-149) + (A*2^-149) is exact for integers k*128 + A < 2^23, and the bit pattern of the
// denormal result IS the integer 128*k + A. With A = the shared-memory address of the lane's copy of entry 0 (< 2^18), one genuine FFMA per cell turns the
// cell's index into its LDS address - no integer add at all (fp32 denormals run at full rate on the FMA pipe; nothing here is compiled with -ftz).
// Without it (TW_LUT_DENORM=0, the round-1 form): magic 1.5*2^23, bits 0x4B400000 + 128*k, and one IADD per look-up to rebase.
#ifndef TW_LUT_DENORM
#define TW_LUT_DENORM 1
#endif
#ifndef TW_HASH_Q1_ARITH
#define TW_HASH_Q1_ARITH 0   // 1: the middle corner's hash by exact integer arithmetic instead of a third table load. It trades two table loads per cell pair
                             // for two more FMA-pipe instructions on the hash chain.
#endif
constexpr unsigned SIMPLEX_LUT_MAGIC_BITS = 0x4B400000u; // bits of 12582912.0f = 1.5*2^23
constexpr unsigned LUT_ENTRY_BYTES = 16u*SIMPLEX_LUT_COPIES;

// Simplex hash table (level 3 with the denormal addressing): SIMPLEX_HASH_N entries staged right behind the 8 copies of the gradient table. Its
// entries are the second-permute arguments already turned into gradient-table byte offsets: with P = permute and B(v) = the float whose bit
// pattern is the integer v (a denormal, v*2^-149),
//   entry k = {B(128*P(k)), B(128*(P(k) + 1)), B(128*(P(k + 1) + 1)), 0}.
// With bx = lut_offsets(ix) (bits 128*ix + Lb), the three gradient addresses of a cell are one add each:
//   k0 = [iy].x + bx = lut_offsets(P(iy) + ix)              (p0 = q0 + ix)
//   k2 = [iy].z + bx = lut_offsets(P(iy + 1) + ix + 1)      (p2 = q2 + ix + 1)
//   k1 = [iy].y + bx (i1.y = 0) or [iy + 1].x + bx (i1.y = 1) = lut_offsets(P(iy + i1.y) + ix + i1.x)   (p1 = q1 + ix + i1.x, i1.x = 1 - i1.y):
//        the word at entry iy's address + 4 + (pitch - 4)*i1.y.
// Exact, bit for bit: every operand is a non-negative integer multiple of 2^-149 below 2^23*2^-149, where float adds are exact (denormals are
// fixed point; nothing here is compiled with -ftz). ix, iy come from mod_int289_lazy (<= 289) and P <= 288, so the largest offset is
// 128*578 + Lb < 2^19. Entries up to 290 are read; entry 290 needs permute(291), which the float arithmetic of permute() evaluates exactly
// (= permute(2)). Against the hash values of the table's earlier form this saves the three address FMAs of lut_offsets per cell for one (bx).
#define TW_SIMPLEX_HASH_TABLE (TW_SIMPLEX_LUT >= 3 && TW_LUT_DENORM && !TW_HASH_Q1_ARITH)
constexpr int SIMPLEX_HASH_N = TW_SIMPLEX_HASH_TABLE ? 291 : 0;
// The hash table is ONE copy (16-byte pitch), not 8 interleaved ones like the gradient table: the lattice row iy is nearly uniform across a warp, so
// its look-ups mostly broadcast, and the block stages 4.6 KB instead of 37 KB (headline 0.7 % faster than 8 copies, results/h100/octave_body.txt).
constexpr int SIMPLEX_HASH_COPIES = 1;
constexpr unsigned SIMPLEX_HASH_OFFSET = SIMPLEX_LUT_N*LUT_ENTRY_BYTES; // byte distance from the start of the gradient table to the hash table
__device__ __forceinline__ float4 simplex_hash_entry(float k) {
	unsigned const p0 = (unsigned)twn::permute(k), p1 = (unsigned)twn::permute(k + 1.0f);
	return make_float4(__uint_as_float(LUT_ENTRY_BYTES*p0), __uint_as_float(LUT_ENTRY_BYTES*(p0 + 1)), __uint_as_float(LUT_ENTRY_BYTES*(p1 + 1)), 0.0f);
}
__device__ __forceinline__ unsigned simplex_lut_base(const float4 *lut_s, unsigned lane) {
	unsigned const a = (unsigned)__cvta_generic_to_shared(lut_s) + (lane & (SIMPLEX_LUT_COPIES - 1))*16u;
	return TW_LUT_DENORM ? a : a - SIMPLEX_LUT_MAGIC_BITS;
}
// offsets for two cells; with TW_LUT_DENORM their bits are the LDS addresses themselves
__device__ __forceinline__ f2 lut_offsets(f2 k, unsigned Lb) {
	if (TW_LUT_DENORM) {return raw_fma(k, splat(__uint_as_float(LUT_ENTRY_BYTES)), splat(__uint_as_float(Lb)));}
	return fma2(k, 16.0f*SIMPLEX_LUT_COPIES, 12582912.0f);
}
__device__ __forceinline__ unsigned lut_addr(unsigned Lb, float off) {return TW_LUT_DENORM ? __float_as_uint(off) : Lb + __float_as_uint(off);}
__device__ __forceinline__ float4 lut_load4(unsigned Lb, float off) {
	float4 v; asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(lut_addr(Lb, off)));
	return v;
}
__device__ __forceinline__ float lut_load_w_addr(unsigned addr) {
	float v; asm("ld.shared.f32 %0, [%1+12];" : "=f"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ float lut_load_w_addr_next(unsigned addr) { // .w of the following entry
	float v; asm("ld.shared.f32 %0, [%1+140];" : "=f"(v) : "r"(addr));
	return v;
}
__device__ __forceinline__ float lut_load_w(unsigned Lb, float off) {return lut_load_w_addr(lut_addr(Lb, off));}
template<unsigned OFF> __device__ __forceinline__ float lut_load_f32(unsigned addr) { // one word at a constant byte offset (an LDS immediate)
	float v; asm("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(OFF));
	return v;
}

// Domain-warp windows (the headline kernel, tw_heightgen.cu): one launch of the domain-warp kernel only reaches a small window of lattice indices
// per fBm stage and octave, [ix_lo, ix_lo + span] x [iy_lo, iy_lo + span], which the host evaluates exactly. With c = 289*floor(lo/289), the shifted
// index i - c lies in [0, 288 + span]; tables that repeat themselves every 289 entries then give, at i - c, the bits the 580-entry tables give at
// mod 289 of i, and the octave needs no reduction (12 instructions per cell pair: FMUL, FRND, FFMA per coordinate and cell). The shift is folded into
// the table bases (one exact denormal add each, shared by the two cells). Octaves 0 .. DWARP_WIN_OCTAVES-1 take this form; the last octaves' windows
// would need larger tables and keep the reduction.
//   gradient table: entry k = simplex_lut_entry(k mod 289), k <= P + (i - c) + 1 <= 577 + span
//   hash table:     entry r = simplex_hash_entry(r mod 289), r <= (i - c) + 1 <= 289 + span
// Both are built from k mod 289: permute() is exact only while (34k + 1)k < 2^24.
// TW_DWARP_WIN_OCTAVES 7: 161 KB of tables, one block of 1024 threads per SM; 5: 101 KB, two blocks of 512 (both 32 warps at 64 registers).
#ifndef TW_DWARP_WIN_OCTAVES
#define TW_DWARP_WIN_OCTAVES 7
#endif
constexpr int DWARP_WIN_OCTAVES = TW_DWARP_WIN_OCTAVES;
constexpr int DWARP_WIN_SPAN = (DWARP_WIN_OCTAVES > 5) ? 600 : 170;   // widest window the tables hold (8192^2 headline: 576 at octave 6, 157 at octave 4)
constexpr int SIMPLEX_WLUT_N = 578 + DWARP_WIN_SPAN;
constexpr int SIMPLEX_WHASH_N = 290 + DWARP_WIN_SPAN;
static_assert(DWARP_WIN_OCTAVES >= 1 && DWARP_WIN_OCTAVES <= 8, "windowed octaves of the 8-octave body");

// gradient-table offsets of the three corners of two cells from the simplex hash table (ix, iy: lattice indices after mod_int289_lazy, or shifted into
// a window). H: byte distance from the gradient table to the hash table; gb: denormal whose bits are the address of the lane's copy of gradient
// entry 0 (Lb), hb: the same for hash entry 0, less H; a window's shift is folded into both.
template<unsigned H>
__device__ __forceinline__ void simplex_hash_offsets(f2 ix, f2 iy, f2 i1y, float gb, float hb, f2 &k0, f2 &k1, f2 &k2) {
	constexpr unsigned PITCH = 16u*SIMPLEX_HASH_COPIES;
	f2 const j0 = raw_fma(iy, splat(__uint_as_float(PITCH)), splat(hb));   // address of entry iy of the hash table, less H (exact, as lut_offsets)
	f2 const j1 = raw_fma(i1y, splat(__uint_as_float(PITCH - 4)), j0);     // + pitch - 4 bytes when i1.y = 1 (see simplex_hash_entry)
	unsigned const ja = __float_as_uint(j0.x), jb = __float_as_uint(j0.y), j1a = __float_as_uint(j1.x), j1b = __float_as_uint(j1.y);
	f2 const bx = raw_fma(ix, splat(__uint_as_float(LUT_ENTRY_BYTES)), splat(gb));
	k0 = add2(make_float2(lut_load_f32<H>(ja), lut_load_f32<H>(jb)), bx);
	k1 = add2(make_float2(lut_load_f32<H + 4>(j1a), lut_load_f32<H + 4>(j1b)), bx);
	k2 = add2(make_float2(lut_load_f32<H + 8>(ja), lut_load_f32<H + 8>(jb)), bx);
}

// glm::simplex(vec2) for two positions with the table; Lb = simplex_lut_base(); HASH: the block staged the simplex hash table too, H bytes behind
// the gradient table; WIN: ix, iy stay unreduced and wb = {gb, hb} of simplex_hash_offsets with the octave's window shift folded in
template<bool HASH, unsigned H = SIMPLEX_HASH_OFFSET, bool WIN = false>
__device__ __forceinline__ f2 simplex2_lut(f2 vx, f2 vy, unsigned Lb, f2 wb = f2()) {
	static_assert(!HASH || TW_SIMPLEX_HASH_TABLE, "the hash table exists at level 3 with the denormal addressing only");
	static_assert(!WIN || HASH, "the windowed form addresses through the hash table");
	float const Cx = 0.211324865405187f, Cy = 0.366025403784439f, Cz = -0.577350269189626f;
	f2 const s = sumprod2(vx, Cy, vy, Cy);
	f2 ix = floor2(add2(vx, s)), iy = floor2(add2(vy, s));
	f2 const t = sumprod2(ix, Cx, iy, Cx);
	f2 const x0x = add2(sub2(vx, ix), t), x0y = add2(sub2(vy, iy), t);
	f2 const i1x = make_float2((x0x.x > x0y.x) ? 1.0f : 0.0f, (x0x.y > x0y.y) ? 1.0f : 0.0f);
	f2 const i1y = rsub2(1.0f, i1x); // (1,0) or (0,1)
	f2 const x12x = sub2(add2(x0x, Cx), i1x), x12y = sub2(add2(x0y, Cx), i1y), x12z = add2(x0x, Cz), x12w = add2(x0y, Cz);
	f2 k0, k1, k2;
	if constexpr (WIN) {simplex_hash_offsets<H>(ix, iy, i1y, wb.x, wb.y, k0, k1, k2);}
	else if constexpr (HASH) { // the hash table's one copy starts at Lb without the lane's copy offset
		unsigned const base = Lb - (threadIdx.x & (SIMPLEX_LUT_COPIES - 1))*16u;
		simplex_hash_offsets<H>(mod_int289_lazy(ix), mod_int289_lazy(iy), i1y, __uint_as_float(Lb), __uint_as_float(base), k0, k1, k2);
	}
	else {
	f2 p0, p1, p2;
#if TW_SIMPLEX_LUT >= 2
	ix = mod_int289_lazy(ix); iy = mod_int289_lazy(iy);
	// permute(iy), permute(iy + i1.y), permute(iy + 1): consecutive table entries, so the second and third addresses are the first plus 0/128/256 bytes
	f2 const j0 = lut_offsets(iy, Lb);
	unsigned const ja = lut_addr(Lb, j0.x), jb = lut_addr(Lb, j0.y);
	static_assert(LUT_ENTRY_BYTES == 128, "lut_load_w_addr_next hard-codes the entry pitch");
	f2 const q0 = make_float2(lut_load_w_addr(ja), lut_load_w_addr(jb));
#if TW_HASH_Q1_ARITH && TW_SIMPLEX_LUT >= 3
	// no load for q1 (see p1 below)
#elif TW_LUT_DENORM
	f2 const j1 = raw_fma(i1y, splat(__uint_as_float(LUT_ENTRY_BYTES)), j0); // entry iy + i1.y: one FMA per cell instead of a select and an add
	f2 const q1 = make_float2(lut_load_w_addr(__float_as_uint(j1.x)), lut_load_w_addr(__float_as_uint(j1.y)));
#else
	f2 const q1 = make_float2(lut_load_w_addr(ja + ((x0x.x > x0y.x) ? 0u : LUT_ENTRY_BYTES)), lut_load_w_addr(jb + ((x0x.y > x0y.y) ? 0u : LUT_ENTRY_BYTES)));
#endif
	f2 const q2 = make_float2(lut_load_w_addr_next(ja), lut_load_w_addr_next(jb));
#else
	ix = mod_int289(ix); iy = mod_int289(iy);
	f2 const q0 = permute(iy), q1 = permute(add2(iy, i1y)), q2 = permute(add2(iy, 1.0f));
#endif
#if TW_SIMPLEX_LUT >= 3 && TW_HASH_Q1_ARITH
	// q1 = permute(iy + i1.y) is q0 or q2, so the three table indices are p0 = q0 + ix, p2 = q2 + ix + 1 and p1 = i1.y ? q2 + ix : q0 + ix + 1 (i1.x = 1 - i1.y).
	// All of these are small non-negative integers, exact in fp32 in any order: with d = q2 - q0 and e = p0 + 1, p2 = e + d and p1 = e + i1.y*(d - 1)
	// (a product by 0 or 1 plus an integer: fused or not, the same number). Two table loads fewer per pair of cells - the shared-memory pipe is the
	// second-busiest unit of this kernel - for one more FMA per cell.
	p0 = add2(q0, ix); f2 const dq = sub2(q2, q0), e1 = add2(p0, 1.0f); p2 = add2(e1, dq); p1 = raw_fma(i1y, add2(dq, -1.0f), e1);
#elif TW_SIMPLEX_LUT >= 3
	p0 = add2(q0, ix); p1 = add2(add2(q1, ix), i1x); p2 = add2(add2(q2, ix), 1.0f); // the table is indexed by the argument of the second permute (q: table values, ix: an fma result)
#else
	p0 = permute(add2(q0, ix)); p1 = permute(add2(add2(q1, ix), i1x)); p2 = permute(add2(add2(q2, ix), 1.0f));
#endif
	k0 = lut_offsets(p0, Lb); k1 = lut_offsets(p1, Lb); k2 = lut_offsets(p2, Lb);
	}
	f2 m0 = rsub_max0_2(0.5f, sumprod2(x0x, x0x, x0y, x0y));
	f2 m1 = rsub_max0_2(0.5f, sumprod2(x12x, x12x, x12y, x12y));
	f2 m2 = rsub_max0_2(0.5f, sumprod2(x12z, x12z, x12w, x12w));
	m0 = mul2(m0, m0); m1 = mul2(m1, m1); m2 = mul2(m2, m2);
	m0 = mul2(m0, m0); m1 = mul2(m1, m1); m2 = mul2(m2, m2);
	float4 const g0a = lut_load4(Lb, k0.x), g0b = lut_load4(Lb, k0.y), g1a = lut_load4(Lb, k1.x), g1b = lut_load4(Lb, k1.y), g2a = lut_load4(Lb, k2.x), g2b = lut_load4(Lb, k2.y);
	// the table values arrive one cell per register quad (same IEEE operations; the file is compiled with -fmad=false)
	m0 = make_float2(m0.x*g0a.z, m0.y*g0b.z); m1 = make_float2(m1.x*g1a.z, m1.y*g1b.z); m2 = make_float2(m2.x*g2a.z, m2.y*g2b.z);
	f2 const gx = make_float2(g0a.x*x0x.x  + g0a.y*x0y.x,  g0b.x*x0x.y  + g0b.y*x0y.y);
	f2 const gy = make_float2(g1a.x*x12x.x + g1a.y*x12y.x, g1b.x*x12x.y + g1b.y*x12y.y);
	f2 const gz = make_float2(g2a.x*x12z.x + g2a.y*x12w.x, g2b.x*x12z.y + g2b.y*x12w.y);
	return mul2(add2(add2(mul2(m0, gx), mul2(m1, gy)), mul2(m2, gz)), 130.0f);
}

__device__ __forceinline__ void perlin2_corner(f2 ix, f2 iy, f2 &gx, f2 &gy) {
	f2 const i = permute(add2(permute(ix), iy));
	float const c41 = 1.0f/41.0f;
	f2 const q0 = mul2(i, c41);
	f2 const q = fma2(fma2(q0, -41.0f, i), c41, q0); // i/41, see twn::div41_small (fma(-q0,41,i) == fma(q0,-41,i)); both are genuine fmas
	f2 const g = fma2(fract2(q), 2.0f, -1.0f);
	gy = add2(abs2(g), -0.5f);
	gx = sub2(g, floor2(add2(g, 0.5f)));
	f2 const n = tinvsqrt(add2(mul2(gx, gx), mul2(gy, gy)));
	gx = mul2(gx, n); gy = mul2(gy, n);
}

// glm::perlin(vec2) for two positions
__device__ __forceinline__ f2 perlin2(f2 Px, f2 Py) {
	f2 const flx = floor2(Px), fly = floor2(Py);
	f2 const frx = sub2(Px, flx), fry = sub2(Py, fly);
	f2 const Pfz = add2(frx, -1.0f), Pfw = add2(fry, -1.0f);
	f2 const Pix = mod_int289(flx), Piy = mod_int289(fly), Piz = mod_int289(add2(flx, 1.0f)), Piw = mod_int289(add2(fly, 1.0f));
	f2 g00x, g00y, g10x, g10y, g01x, g01y, g11x, g11y;
	perlin2_corner(Pix, Piy, g00x, g00y);
	perlin2_corner(Piz, Piy, g10x, g10y);
	perlin2_corner(Pix, Piw, g01x, g01y);
	perlin2_corner(Piz, Piw, g11x, g11y);
	f2 const n00 = add2(mul2(g00x, frx), mul2(g00y, fry));
	f2 const n10 = add2(mul2(g10x, Pfz), mul2(g10y, fry));
	f2 const n01 = add2(mul2(g01x, frx), mul2(g01y, Pfw));
	f2 const n11 = add2(mul2(g11x, Pfz), mul2(g11y, Pfw));
	f2 const fdx = fade2(frx), fdy = fade2(fry);
	f2 const nx0 = mix2(n00, n10, fdx), nx1 = mix2(n01, n11, fdx);
	return mul2(mix2(nx0, nx1, fdy), 2.3f);
}

// ---- Perlin with the same kind of table: {gx*n, gy*n, 0, permute(k)} for the hashed lattice index k (gradient of glm::perlin(vec2):
// g = 2*fract(k/41) - 1, gy = |g| - 0.5, gx = g - floor(g + 0.5), both scaled by taylorInvSqrt(gx*gx + gy*gy)), k in [0, 288]; .w as above ----
__device__ __forceinline__ float4 perlin_lut_entry(float k) {
	float const pk = twn::permute(k);
	float const g = twn::two_f_minus_1(twn::fract(twn::div41_small((TW_SIMPLEX_LUT >= 3) ? pk : k)));
	float gy = fabsf(g) - 0.5f, gx = g - floorf(g + 0.5f);
	float const n = twn::tinvsqrt(gx*gx + gy*gy);
	gx *= n; gy *= n;
	return make_float4(gx, gy, 0.0f, pk);
}

// glm::perlin(vec2) for two positions with the table
__device__ __forceinline__ f2 perlin2_lut(f2 Px, f2 Py, unsigned Lb) {
	f2 const flx = floor2(Px), fly = floor2(Py);
	f2 const frx = sub2(Px, flx), fry = sub2(Py, fly);
	f2 const Pfz = add2(frx, -1.0f), Pfw = add2(fry, -1.0f);
	f2 const Pix = mod_int289_lazy(flx), Piy = mod_int289_lazy(fly), Piz = mod_int289_lazy(add2(flx, 1.0f)), Piw = mod_int289_lazy(add2(fly, 1.0f));
	f2 const jx = lut_offsets(Pix, Lb), jz = lut_offsets(Piz, Lb);
	f2 const qx = make_float2(lut_load_w(Lb, jx.x), lut_load_w(Lb, jx.y)), qz = make_float2(lut_load_w(Lb, jz.x), lut_load_w(Lb, jz.y)); // permute(ix)
#if TW_SIMPLEX_LUT >= 3
	f2 const k00 = lut_offsets(add2(qx, Piy), Lb), k10 = lut_offsets(add2(qz, Piy), Lb), k01 = lut_offsets(add2(qx, Piw), Lb), k11 = lut_offsets(add2(qz, Piw), Lb);
#else
	f2 const k00 = lut_offsets(permute(add2(qx, Piy)), Lb), k10 = lut_offsets(permute(add2(qz, Piy)), Lb);
	f2 const k01 = lut_offsets(permute(add2(qx, Piw)), Lb), k11 = lut_offsets(permute(add2(qz, Piw)), Lb);
#endif
	float4 const a00 = lut_load4(Lb, k00.x), b00 = lut_load4(Lb, k00.y), a10 = lut_load4(Lb, k10.x), b10 = lut_load4(Lb, k10.y);
	float4 const a01 = lut_load4(Lb, k01.x), b01 = lut_load4(Lb, k01.y), a11 = lut_load4(Lb, k11.x), b11 = lut_load4(Lb, k11.y);
	// products with the table values (see simplex2_lut)
	f2 const n00 = make_float2(a00.x*frx.x + a00.y*fry.x, b00.x*frx.y + b00.y*fry.y);
	f2 const n10 = make_float2(a10.x*Pfz.x + a10.y*fry.x, b10.x*Pfz.y + b10.y*fry.y);
	f2 const n01 = make_float2(a01.x*frx.x + a01.y*Pfw.x, b01.x*frx.y + b01.y*Pfw.y);
	f2 const n11 = make_float2(a11.x*Pfz.x + a11.y*Pfw.x, b11.x*Pfz.y + b11.y*Pfw.y);
	f2 const fdx = fade2(frx), fdy = fade2(fry);
	f2 const nx0 = mix2(n00, n10, fdx), nx1 = mix2(n01, n11, fdx);
	return mul2(mix2(nx0, nx1, fdy), 2.3f);
}

// ---- 3-D noise (voxel density) with the same tables, one voxel per thread (scalar arithmetic) ----
// simplex(vec3): entry k = {P.x*n, P.y*n, P.z*n, permute(k)}, the normalised gradient that glm::simplex(vec3) derives from the hashed index
// (gtc/noise.inl:680-709: x_, y_, h, the sign fix-up s*sh, taylorInvSqrt); perlin(vec3): entry k = {g.x*n, g.y*n, g.z*n, permute(k)}
// (gtc/noise.inl:90-118). The lattice indices here come from mod289() (the multiply form), which can return exactly 289 for a multiple of
// 289, hence 291 entries; callers guard |lattice coordinate| < 2^20 (mod289 then stays within [0, 289]) and use twn::simplex3/perlin3 beyond.
__device__ __forceinline__ float4 simplex3_lut_entry(float k) { // gradient of the hashed index permute(k) (the last of the three permutes is folded in)
	float X, Y, H;
	float const pk = twn::permute(k);
	twn::simplex3_xyh(pk, X, Y, H);
	float const sh = -twn::step(H, 0.0f);
	float Px = X + (floorf(X)*2.0f + 1.0f)*sh, Py = Y + (floorf(Y)*2.0f + 1.0f)*sh, Pz = H;
	float const n = twn::tinvsqrt(Px*Px + Py*Py + Pz*Pz);
	Px *= n; Py *= n; Pz *= n;
	return make_float4(Px, Py, Pz, pk);
}
__device__ __forceinline__ float4 perlin3_lut_entry(float k) {
	float gx, gy, gz;
	float const pk = twn::permute(k);
	twn::perlin3_grad(pk, gx, gy, gz);
	return make_float4(gx, gy, gz, pk);
}
__device__ __forceinline__ float lut_offset1(float k, unsigned Lb) { // exact, see lut_offsets
	return TW_LUT_DENORM ? __fmaf_rn(k, __uint_as_float(LUT_ENTRY_BYTES), __uint_as_float(Lb)) : __fmaf_rn(k, 16.0f*SIMPLEX_LUT_COPIES, 12582912.0f);
}

__device__ __forceinline__ float simplex3_lut(float vx, float vy, float vz, unsigned Lb) {
	float const Cx = (float)(1.0/6.0), Cy = (float)(1.0/3.0);
	float const s = vx*Cy + vy*Cy + vz*Cy;
	float i0 = floorf(vx + s), i1_ = floorf(vy + s), i2_ = floorf(vz + s);
	float const t = i0*Cx + i1_*Cx + i2_*Cx;
	float const x0x = vx - i0 + t, x0y = vy - i1_ + t, x0z = vz - i2_ + t;
	float const gx = twn::step(x0y, x0x), gy = twn::step(x0z, x0y), gz = twn::step(x0x, x0z);
	float const lx = 1.0f - gx, ly = 1.0f - gy, lz = 1.0f - gz;
	float const i1x = twn::gmin(gx, lz), i1y = twn::gmin(gy, lx), i1z = twn::gmin(gz, ly);
	float const i2x = twn::gmax(gx, lz), i2y = twn::gmax(gy, lx), i2z = twn::gmax(gz, ly);
	float const x1x = x0x - i1x + Cx, x1y = x0y - i1y + Cx, x1z = x0z - i1z + Cx;
	float const x2x = x0x - i2x + Cy, x2y = x0y - i2y + Cy, x2z = x0z - i2z + Cy;
	float const x3x = x0x - 0.5f, x3y = x0y - 0.5f, x3z = x0z - 0.5f;
	i0 = twn::mod289(i0); i1_ = twn::mod289(i1_); i2_ = twn::mod289(i2_);
	float const q0 = lut_load_w(Lb, lut_offset1(i2_, Lb)), q1 = lut_load_w(Lb, lut_offset1(i2_ + i1z, Lb)), q2 = lut_load_w(Lb, lut_offset1(i2_ + i2z, Lb)),
	            q3 = lut_load_w(Lb, lut_offset1(i2_ + 1.0f, Lb)); // twn::permute(i.z + ...)
	float const p0 = twn::permute(q0 + i1_)        + i0;        // arguments of the last permute: the table holds the gradient of permute(argument)
	float const p1 = twn::permute(q1 + i1_ + i1y)  + i0 + i1x;
	float const p2 = twn::permute(q2 + i1_ + i2y)  + i0 + i2x;
	float const p3 = twn::permute(q3 + i1_ + 1.0f) + i0 + 1.0f;
	float4 const P0 = lut_load4(Lb, lut_offset1(p0, Lb)), P1 = lut_load4(Lb, lut_offset1(p1, Lb)), P2 = lut_load4(Lb, lut_offset1(p2, Lb)), P3 = lut_load4(Lb, lut_offset1(p3, Lb));
	float m0 = rsub_max0(0.6f, x0x*x0x + x0y*x0y + x0z*x0z), m1 = rsub_max0(0.6f, x1x*x1x + x1y*x1y + x1z*x1z);
	float m2 = rsub_max0(0.6f, x2x*x2x + x2y*x2y + x2z*x2z), m3 = rsub_max0(0.6f, x3x*x3x + x3y*x3y + x3z*x3z);
	m0 = m0*m0; m1 = m1*m1; m2 = m2*m2; m3 = m3*m3;
	float const d0 = P0.x*x0x + P0.y*x0y + P0.z*x0z, d1 = P1.x*x1x + P1.y*x1y + P1.z*x1z;
	float const d2 = P2.x*x2x + P2.y*x2y + P2.z*x2z, d3 = P3.x*x3x + P3.y*x3y + P3.z*x3z;
	return 42.0f*(((m0*m0)*d0 + (m1*m1)*d1) + ((m2*m2)*d2 + (m3*m3)*d3));
}

__device__ __forceinline__ float perlin3_lut(float Px, float Py, float Pz, unsigned Lb) {
	float const flx = floorf(Px), fly = floorf(Py), flz = floorf(Pz);
	float const Pi0x = twn::mod289(flx), Pi0y = twn::mod289(fly), Pi0z = twn::mod289(flz);
	float const Pi1x = twn::mod289(flx + 1.0f), Pi1y = twn::mod289(fly + 1.0f), Pi1z = twn::mod289(flz + 1.0f);
	float const f0x = Px - flx, f0y = Py - fly, f0z = Pz - flz;
	float const f1x = f0x - 1.0f, f1y = f0y - 1.0f, f1z = f0z - 1.0f;
	float const px0 = lut_load_w(Lb, lut_offset1(Pi0x, Lb)), px1 = lut_load_w(Lb, lut_offset1(Pi1x, Lb)); // twn::permute(Pi.x)
	float const ixy00 = twn::permute(px0 + Pi0y), ixy10 = twn::permute(px1 + Pi0y), ixy01 = twn::permute(px0 + Pi1y), ixy11 = twn::permute(px1 + Pi1y);
	float4 g;
	g = lut_load4(Lb, lut_offset1(ixy00 + Pi0z, Lb)); float const n000 = g.x*f0x + g.y*f0y + g.z*f0z;
	g = lut_load4(Lb, lut_offset1(ixy10 + Pi0z, Lb)); float const n100 = g.x*f1x + g.y*f0y + g.z*f0z;
	g = lut_load4(Lb, lut_offset1(ixy01 + Pi0z, Lb)); float const n010 = g.x*f0x + g.y*f1y + g.z*f0z;
	g = lut_load4(Lb, lut_offset1(ixy11 + Pi0z, Lb)); float const n110 = g.x*f1x + g.y*f1y + g.z*f0z;
	g = lut_load4(Lb, lut_offset1(ixy00 + Pi1z, Lb)); float const n001 = g.x*f0x + g.y*f0y + g.z*f1z;
	g = lut_load4(Lb, lut_offset1(ixy10 + Pi1z, Lb)); float const n101 = g.x*f1x + g.y*f0y + g.z*f1z;
	g = lut_load4(Lb, lut_offset1(ixy01 + Pi1z, Lb)); float const n011 = g.x*f0x + g.y*f1y + g.z*f1z;
	g = lut_load4(Lb, lut_offset1(ixy11 + Pi1z, Lb)); float const n111 = g.x*f1x + g.y*f1y + g.z*f1z;
	float const fx = twn::fade(f0x), fy = twn::fade(f0y), fz = twn::fade(f0z);
	float const nz0 = twn::mix(n000, n001, fz), nz1 = twn::mix(n100, n101, fz), nz2 = twn::mix(n010, n011, fz), nz3 = twn::mix(n110, n111, fz);
	float const nyz0 = twn::mix(nz0, nz2, fy), nyz1 = twn::mix(nz1, nz3, fy);
	return 2.2f*twn::mix(nyz0, nyz1, fx);
}

} // namespace twn2
