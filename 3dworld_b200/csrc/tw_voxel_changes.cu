// tw_voxel_changes.cu - the change list of a voxel model edit (tw_voxel_model_edit_launch_ex): one change bit per voxel, then the changed voxels in
// ascending index order. Built as its own sm_90a module (build.py: tw_voxel_changes.cubin beside the library) that tw_voxel_post.cu loads on first use
// with cudaLibraryLoadFromFile, so the library's own kernels - whose code the tests pin, kernel by kernel - stay exactly as they are. The kernels are
// extern "C" so the loader finds them by name, and declared in tw_voxel_edit.cuh, which the host's launches also read.
#include "tw_voxel_edit.cuh"

// rm == 0: box_scatter_kernel that also sets each changed voxel's bit; post is the model's field, bits are zeroed before
extern "C" __global__ void tw_box_scatter_bits_kernel(const twi_box *__restrict__ boxes, unsigned nboxes, const float *__restrict__ values,
	unsigned long long total, tw_voxel_post_params P, const unsigned *__restrict__ zix_xy, BlockGrid G, float *__restrict__ raw,
	unsigned char *__restrict__ raw_o, float *post, unsigned char *post_o, unsigned char *mark, unsigned *__restrict__ bits)
{
	box_scatter<true>(boxes, nboxes, values, total, P, zix_xy, G, raw, raw_o, post, post_o, mark, bits);
}

// rm > 0: diff_kernel with the change bits. Every word of bits (ceil(n/32)) is written - a warp holds 32 consecutive voxels (the block size and the
// stride are multiples of 32), whose change bits it gathers with one ballot - so no word needs zeroing first and no atomic is needed
extern "C" __global__ void tw_diff_bits_kernel(const float *__restrict__ nv, const unsigned char *__restrict__ no, float *__restrict__ ov,
	unsigned char *__restrict__ oo, tw_voxel_post_params P, BlockGrid G, unsigned char *__restrict__ mark, size_t n, unsigned *__restrict__ bits)
{
	size_t const stride = (size_t)gridDim.x*blockDim.x, n32 = (n + 31) & ~(size_t)31;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n32; i += stride) { // uniform over the warp
		bool changed = false;
		if (i < n) {
			float const v = nv[i];
			unsigned char const o = no[i];
			changed = (__float_as_uint(v) != __float_as_uint(ov[i]) || o != oo[i]);
			if (changed) {
				ov[i] = v; oo[i] = o;
				size_t const xy = i / P.nz;
				mark_readers(mark, P, G, (unsigned)(xy % P.nx), (unsigned)(xy / P.nx));
			}
		}
		unsigned const word = __ballot_sync(0xffffffffu, changed);
		if ((threadIdx.x & 31) == 0) {bits[i >> 5] = word;}
	}
}

// The list from the bits: a chunk is CL_BLOCK words, one per thread. change_count_kernel counts each chunk's set bits into sums; scan_blocks_kernel (the
// library's) turns them into offsets and the total; change_emit_kernel writes each set bit's voxel - index, and the model's new value and flags when asked -
// at its chunk's offset plus its rank within the chunk, so the list is in ascending index order. Slots at or past the capacity are not written.
namespace {
template<bool EMIT>
__device__ __forceinline__ void change_list(const unsigned *__restrict__ bits, size_t nwords, unsigned *__restrict__ sums,
	const unsigned long long *__restrict__ offsets, const float *__restrict__ post, const unsigned char *__restrict__ post_o, uint32_t *__restrict__ index,
	float *__restrict__ vals, uint8_t *__restrict__ outside, unsigned long long capacity)
{
	__shared__ unsigned warp_sums[CL_BLOCK/32];
	size_t const w = (size_t)blockIdx.x*CL_BLOCK + threadIdx.x;
	unsigned word = (w < nwords) ? bits[w] : 0u;
	unsigned const cnt = __popc(word), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += v;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned const ws = (lane < CL_BLOCK/32) ? warp_sums[lane] : 0u;
		unsigned wi = ws;
		for (int o = 1; o < CL_BLOCK/32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
		if (lane < CL_BLOCK/32) {warp_sums[lane] = wi - ws;}
		if (!EMIT && lane == CL_BLOCK/32 - 1) {sums[blockIdx.x] = wi;}
	}
	if (!EMIT) return;
	__syncthreads();
	unsigned long long slot = offsets[blockIdx.x] + warp_sums[warp] + (incl - cnt);
	for (; word && slot < capacity; word &= word - 1, ++slot) {
		size_t const i = w*32 + (unsigned)(__ffs(word) - 1);
		index[slot] = (uint32_t)i;
		if (vals) {vals[slot] = post[i];}
		if (outside) {outside[slot] = post_o[i];}
	}
}
} // namespace

extern "C" __global__ void __launch_bounds__(CL_BLOCK) tw_change_count_kernel(const unsigned *__restrict__ bits, size_t nwords, unsigned *__restrict__ sums) {
	change_list<false>(bits, nwords, sums, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
}
extern "C" __global__ void __launch_bounds__(CL_BLOCK) tw_change_emit_kernel(const unsigned *__restrict__ bits, size_t nwords,
	const unsigned long long *__restrict__ offsets, const float *__restrict__ post, const unsigned char *__restrict__ post_o, uint32_t *__restrict__ index,
	float *__restrict__ vals, uint8_t *__restrict__ outside, unsigned long long capacity)
{
	change_list<true>(bits, nwords, nullptr, offsets, post, post_o, index, vals, outside, capacity);
}
