// tw_voxel_edit.cuh - the pieces of a voxel model edit shared by tw_voxel_post.cu (the library) and tw_voxel_changes.cu (the change-list module, which
// tw_voxel_post.cu loads at run time): the block grid, the blocks that read a voxel, the edit's boxes and the box scatter. Included by each at file scope;
// everything here but the module's kernel declarations has internal linkage, so each translation unit keeps its own copy and its own kernels' names.
#pragma once
#include "../../include/tw3d.h"

namespace {

struct BlockGrid {unsigned bx, by, nbx, chunks;};

// every block whose cubes read voxel column (x, y): the cubes x-1, x and y-1, y that exist
__device__ __forceinline__ void mark_readers(unsigned char *mark, const tw_voxel_post_params &P, const BlockGrid &G, unsigned x, unsigned y) {
	for (unsigned cy = (y ? y - 1 : 0); cy <= y && cy + 1 < P.ny; ++cy) {
		for (unsigned cx = (x ? x - 1 : 0); cx <= x && cx + 1 < P.nx; ++cx) {mark[(cy / G.by)*G.nbx + cx / G.bx] = 1;}
	}
}

// an edit's box and the index of its first value among the packed values; later: a later box overlaps it
struct twi_box {unsigned x, y, z, w, h, d; unsigned long long off; unsigned later, pad;};

// the edit's values into the raw field, with the raw flags of outside_kernel; post (rm == 0, where the post field is the raw one): also compared with the
// model's field and flags, which take the new values, marking the blocks that read a changed voxel; with BITS also setting the voxel's change bit
template<bool BITS>
__device__ __forceinline__ void box_scatter(const twi_box *__restrict__ boxes, unsigned nboxes, const float *__restrict__ values, unsigned long long total,
	tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, BlockGrid G, float *__restrict__ raw, unsigned char *__restrict__ raw_o, float *post,
	unsigned char *post_o, unsigned char *mark, unsigned *bits)
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
		if (post && (__float_as_uint(post[i]) != __float_as_uint(val) || post_o[i] != o)) {
			post[i] = val; post_o[i] = o; mark_readers(mark, P, G, x, y);
			if (BITS) {atomicOr(bits + (i >> 5), 1u << (i & 31));} // a box row need not start on a word
		}
	}
}

// the change list's chunk: CL_BLOCK bitmask words, one per thread of change_count_kernel / change_emit_kernel
constexpr int CL_BLOCK = 256;

} // namespace

// The change-list module's kernels (tw_voxel_changes.cu), declared once for the module's definitions and the host's launches (tw_voxel_post.cu)
extern "C" __global__ void tw_box_scatter_bits_kernel(const twi_box *boxes, unsigned nboxes, const float *values, unsigned long long total,
	tw_voxel_post_params P, const unsigned *zix_xy, BlockGrid G, float *raw, unsigned char *raw_o, float *post, unsigned char *post_o, unsigned char *mark,
	unsigned *bits);
extern "C" __global__ void tw_diff_bits_kernel(const float *nv, const unsigned char *no, float *ov, unsigned char *oo, tw_voxel_post_params P, BlockGrid G,
	unsigned char *mark, size_t n, unsigned *bits);
extern "C" __global__ void tw_change_count_kernel(const unsigned *bits, size_t nwords, unsigned *sums);
extern "C" __global__ void tw_change_emit_kernel(const unsigned *bits, size_t nwords, const unsigned long long *offsets, const float *post,
	const unsigned char *post_o, uint32_t *index, float *vals, uint8_t *outside, unsigned long long capacity);
