// tw_hmap_ao.cu - the AO map of heightmap-texture tiles (tw_hmap_tile_ao_launch): tile_t::calc_mesh_ao_lighting (src/tiled_mesh.cpp:586-662) with the
// rays reading the tile's final zvals inside the tile and get_clamped_height of the context's image outside it. Built as its own sm_90a module (build.py:
// tw_hmap_ao.cubin beside the library) that the library loads on first use, so the library's own kernels - whose code the tests pin, kernel by kernel - stay
// exactly as they are. For the same reason the sampler's device helpers are copied here from tw_streaming.cu (hmap_scale_val, hmap_raw_height and
// hmap_sample_tiles_kernel's cell body) rather than shared; the index arithmetic is tw_hmap_index.cuh's, which the host-only tw_hmap_tiles_touched
// also uses. The kernel is extern "C" so the loader finds it by name.
#include "tw_hmap_ao.h"
#include "tw_hmap_index.cuh"

namespace {
__device__ __forceinline__ float hmap_scale_val(float val, const tw_hmap_sampler &H) { // scale_mh_texture_val, src/mesh_gen.cpp:120
	return (H.h_scale*H.mesh_file_scale*val + H.mesh_file_tz)*H.mesh_scale_z_inv;
}
__device__ __forceinline__ float hmap_raw_height(const uint8_t *__restrict__ d, int x, int y, const tw_hmap_sampler &H) { // get_raw_height
	size_t const ix = (size_t)H.width*y + x;
	unsigned const px = __ldg(reinterpret_cast<const unsigned short *>(d) + ix); // little endian: low byte = data[2ix] (fraction), high = data[2ix+1]
	float const v = (float)((double)(px & 255u)/256.0 + (double)(px >> 8)); // get_heightmap_value: exact in fp32 (16 significant bits)
	return hmap_scale_val(v, H);
}
// get_clamped_height(x, y): hmap_sample_tiles_kernel's value at cell (x, y), expression for expression
__device__ __forceinline__ float hmap_height(const uint8_t *__restrict__ data16, const tw_hmap_sampler &H, int x, int y) {
	if (H.mesh_scale < 1.0f) { // interpolate_height(float(x), float(y)), src/heightmap.cpp:394-402
		int xlo, ylo, xhi, yhi;
		float const sx = twh::lerp_index(H.mesh_scale, x, xlo, xhi), sy = twh::lerp_index(H.mesh_scale, y, ylo, yhi);
		float const xv = sx - (float)xlo, yv = sy - (float)ylo;
		bool const ok_lo = twh::clamp_no_scale(xlo, ylo, H);
		bool const ok = ok_lo && twh::clamp_no_scale(xhi, yhi, H); // the reference short-circuits the same way
		if (!ok) return hmap_scale_val(0.0f, H);
		return yv*(xv*hmap_raw_height(data16, xhi, yhi, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, yhi, H)) +
		       (1.0f - yv)*(xv*hmap_raw_height(data16, xhi, ylo, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, ylo, H));
	}
	x = twh::near_index(H.mesh_scale, x); y = twh::near_index(H.mesh_scale, y); // clamp_xy, src/heightmap.cpp:309-313
	return twh::clamp_no_scale(x, y, H) ? hmap_raw_height(data16, x, y, H) : hmap_scale_val(0.0f, H);
}
} // namespace

// One CTA per (tile, sub-square): it stages the (nx + 72) x (ny + 72) window of heights its rays can reach in shared memory - the tile's zvals inside the
// tile, image samples outside - then runs tile_ao_kernel's 8 x 8 ray march for each of its nx x ny cells from there, with tile_ao_kernel's arithmetic
// (fp32 z0 += dz, built without FMA contraction, and the same double expression for the byte). A thread's ray samples of a warp are consecutive cells of
// a window row for each step, so the reads are free of bank conflicts.
extern "C" __global__ void __launch_bounds__(TWI_AO_THREADS) tw_hmap_ao_kernel(twi_hmap_ao_args A) {
	extern __shared__ float win[];
	unsigned const per = A.nsub*A.nsub, t = blockIdx.x/per, sub = blockIdx.x - t*per;
	int const zv = (int)A.zvsize, stride = zv - 1, R = TWI_AO_RAY_LEN;
	int const sx0 = (int)((sub % A.nsub)*A.side), sy0 = (int)((sub / A.nsub)*A.side);
	int const nx = min((int)A.side, stride - sx0), ny = min((int)A.side, stride - sy0), W = nx + 2*R, H = ny + 2*R;
	int const x1 = __ldg(A.origins + 2*t), y1 = __ldg(A.origins + 2*t + 1);
	const float *z = A.zvals + (size_t)(A.slots ? __ldg(A.slots + t) : (int)t)*zv*zv;
	for (int i = threadIdx.x; i < W*H; i += blockDim.x) {
		int const wy = i/W, vx = sx0 - R + (i - wy*W), vy = sy0 - R + wy; // the window cell's tile coordinates
		win[i] = ((unsigned)vx < (unsigned)zv && (unsigned)vy < (unsigned)zv) ? __ldg(z + vy*zv + vx) : hmap_height(A.img, A.H, x1 + vx, y1 + vy);
	}
	__syncthreads();
	unsigned char *ao = A.ao + (size_t)t*stride*stride;
	for (int i = threadIdx.x; i < nx*ny; i += blockDim.x) {
		int const ly = i/nx, lx = i - ly*nx;
		const float *c = win + (ly + R)*W + lx + R;
		float const zc = *c;
		unsigned atten = 0;
#pragma unroll
		for (int d = 0; d < 8; ++d) {
			int const k = (d < 4) ? d : d + 1, step = (k%3 - 1) + (k/3 - 1)*W; // ao_dirs order: y = -1..1 outer, x = -1..1 inner, skipping (0,0)
			float z0 = zc;
			int o = 0, so = step;
#pragma unroll
			for (int s = 0; s < 8; ++s) {
				o += so; z0 += A.dz; so += step;
				if (c[o] > z0) {atten += 8 - s; break;} // hit a higher point
			}
		}
		float const ao_scale = (float)(1.0 - (double)((float)atten/(float)64));
		ao[(size_t)(sy0 + ly)*stride + sx0 + lx] = (unsigned char)(255.0*(double)ao_scale);
	}
}
