// tw_voxel_batch_util.cuh - device helpers of the batch modules (tw_voxel_batch.cu, tw_voxel_model_batch.cu), whose kernels walk many grids through a table
// of per-grid descriptors: the descriptor of a launch block, and a CTA's scan of one grid's per-block sums. Included at file scope; everything here has
// internal linkage, so each module keeps its own copy.
#pragma once

namespace {

// the entry of launch block b: the last entry whose first block is <= b (entry 0's first block is 0; an entry of no blocks shares its first block with
// the next one, which is found instead)
template<typename D, typename F>
__device__ __forceinline__ unsigned find_grid(const D *__restrict__ g, unsigned ngrids, unsigned b, F first) {
	unsigned lo = 0, hi = ngrids - 1;
	while (lo < hi) {unsigned const mid = (lo + hi + 1) >> 1; if (first(g[mid]) <= b) lo = mid; else hi = mid - 1;}
	return lo;
}

// exclusive scan of sums[0, nb) into 64-bit offsets by the whole CTA (1024 threads); returns the total to every thread
__device__ __forceinline__ unsigned long long scan_sums(const unsigned *__restrict__ sums, unsigned nb, unsigned long long *__restrict__ offsets) {
	__shared__ unsigned long long warp_sums[32];
	__shared__ unsigned long long carry;
	if (threadIdx.x == 0) {carry = 0;}
	__syncthreads();
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (unsigned base = 0; base < nb; base += 1024) {
		unsigned const i = base + threadIdx.x;
		unsigned long long const v = (i < nb) ? sums[i] : 0ull;
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
		if (i < nb) {offsets[i] = excl;}
		__syncthreads();
		if (threadIdx.x == 1023) {carry = excl + v;}
		__syncthreads();
	}
	unsigned long long const total = carry;
	__syncthreads(); // carry is reused by the next scan
	return total;
}

} // namespace
