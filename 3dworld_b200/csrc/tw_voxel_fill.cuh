// tw_voxel_fill.cuh - the arithmetic of the voxel density fill shared by tw_voxel.cu (the library's fill kernels) and tw_voxel_batch.cu (the batch module,
// which tw_voxel_post.cu loads at run time): the sine-table look-up, the fused epilogue with its attenuation, and one voxel's GLM fBm. Both fill the
// same values from this one source. Included at file scope; everything here has internal linkage.
#pragma once
#include "tw_internal.h"
#include "tw_noise.cuh"
#include "tw_noise2.cuh"
#include "tw_voxel_math.cuh"

namespace {

constexpr int NS = TW_N3D_SINES; // 60

__device__ __forceinline__ float sinf_lut(const float *__restrict__ tab, float v) {
	return (v < 0.0f) ? -__ldg(tab + (tw_x86_f2i(TW_SSCALE*(-v))&(TW_TSIZE-1))) : __ldg(tab + (tw_x86_f2i(TW_SSCALE*v)&(TW_TSIZE-1)));
}

struct VoxEpilogue {
	float zscale; int normalize;
	int atten_mode; float atten_val, inner_radius;
	unsigned nx, ny, nz;
};

// val += z*zscale; CLIP_TO_pm1; then the attenuation pass that voxel_model::build applies afterwards (src/voxels.cpp:1517-1525)
__device__ __forceinline__ float epilogue(float val, unsigned x, unsigned y, unsigned z, const VoxEpilogue &E) {
	val += (float)z*E.zscale;
	if (E.normalize) {val = smax(-1.0f, smin(1.0f, val));}
	if (E.atten_mode == 2) { // atten_at_edges, src/voxels.cpp:403-419
		float const vy = (float)(1.0 - 2.0*fabs((double)(int)y - 0.5*(double)E.ny)/(double)(float)E.ny);
		float const vx = (float)(1.0 - 2.0*fabs((double)x - 0.5*(double)E.nx)/(double)(float)E.nx);
		float const vz = (float)(1.0 - 2.0*fabs((double)z - 0.5*(double)E.nz)/(double)(float)E.nz), v = 0.25f - vx*vy*vz;
		if (v > 0.0f) {val = (float)((double)val + 8.0*(double)E.atten_val*(double)v);}
	}
	else if (E.atten_mode == 1) { // atten_at_top_only with atten_top_mode 0, src/voxels.cpp:447-450
		float const z_atten = (float)((double)((float)z/(float)E.nz) - 0.75);
		if (z_atten > 0.0f) {val += E.atten_val*z_atten;}
	}
	else if (E.atten_mode >= 3) { // atten_to_sphere, src/voxels.cpp:457-482
		float const two_nz_inv = (float)(2.0/(double)(float)E.nz);
		float const vy = (float)(2.0*fabs((double)(int)y - 0.5*(double)E.ny)/(double)(float)E.ny);
		float const vx = (float)(2.0*fabs((double)x - 0.5*(double)E.nx)/(double)(float)E.nx);
		float const deltaz = (float)((double)z - 0.5*(double)E.nz), zval = (E.atten_mode == 5) ? smax(0.0f, deltaz) : fabsf(deltaz);
		float const vz = zval*two_nz_inv, radius = __fsqrt_rn(vx*vx + vy*vy + vz*vz);
		float adj = 0.0f;
		if (radius > E.inner_radius) {adj = __fdiv_rn(radius - E.inner_radius, 1.0f - E.inner_radius);}
		else if (E.atten_mode >= 4) {adj = __fdiv_rn(radius - E.inner_radius, E.inner_radius);}
		val += E.atten_val*adj;
	}
	return val;
}

struct GlmParams {
	float lo[3], vsz[3], off[3];
	float mag, nfreq0, rx, ry, rz; // nfreq0 = 0.25*freq, rz = rx - ry
	int octaves, perlin;
};

// get_pt_at(c) + offset on axis d = (c*vsz + lo_pos) + offset, src/voxels.h:149, src/voxels.cpp:328
__device__ __forceinline__ float glm_pos(const GlmParams &G, int d, unsigned c) {return ((float)c*G.vsz[d] + G.lo[d]) + G.off[d];}

// the GLM perlin / simplex fBm at (px, py, pz) (src/voxels.cpp:327-339); L = twn2::simplex_lut_base of the block's staged table
template<bool PERLIN>
__device__ __forceinline__ float glm_value(const GlmParams &G, float px, float py, float pz, unsigned L) {
	float val = 0.0f, nmag = G.mag, nfreq = G.nfreq0;
	for (int n = 0; n < G.octaves; ++n) {
		float const nvx = nfreq*px + G.rx, nvy = nfreq*py + G.ry, nvz = nfreq*pz + G.rz;
		float nz_;
		if (fabsf(nvx) + fabsf(nvy) + fabsf(nvz) < 262144.0f) { // lattice coordinates stay below 2^20: table domain (NaN-safe: goes to the literal path)
			nz_ = PERLIN ? twn2::perlin3_lut(nvx, nvy, nvz, L) : twn2::simplex3_lut(nvx, nvy, nvz, L);
		}
		else {nz_ = PERLIN ? twn::perlin3(nvx, nvy, nvz) : twn::simplex3(nvx, nvy, nvz);}
		val   = val + nmag*nz_;
		nmag  = nmag*0.5f;
		nfreq = nfreq*1.92f;
	}
	return val;
}

} // namespace
