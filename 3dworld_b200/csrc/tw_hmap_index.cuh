// tw_hmap_index.cuh - the texel index arithmetic of get_clamped_height (src/heightmap.cpp:309-341,385-402): which texels a cell of a heightmap-texture tile
// reads. Shared by hmap_sample_tiles_kernel (tw_streaming.cu) and the host-only tw_hmap_tiles_touched, so that the texels the host names as read are the ones
// the kernel reads, expression for expression (both are compiled without FMA contraction); hmap_points_kernel uses the float forms below.
#pragma once
#include "../../include/tw3d.h"
#include <math.h>
#include <stdlib.h>
#ifdef __CUDACC__
#define TWH_HD __host__ __device__ __forceinline__
#else
#define TWH_HD inline
#endif

namespace twh {

TWH_HD int round_fp(float v) {return (v > 0.0f) ? (int)(v + 0.5f) : (int)(v - 0.5f);} // src/inlines.h:63 (values are small: no x86 overflow semantics needed)

// clamp_no_scale, src/heightmap.cpp:315-341: false = "off the texture" (cliff mode only)
TWH_HD bool clamp_no_scale(int &x, int &y, const tw_hmap_sampler &H) {
	x += H.width/2; y += H.height/2;
	if (x >= 0 && y >= 0 && x < H.width && y < H.height) return true;
	switch (H.edge_mode) {
	case 0: x = (x < 0) ? 0 : ((x > H.width - 1) ? H.width - 1 : x); y = (y < 0) ? 0 : ((y > H.height - 1) ? H.height - 1 : y); break;
	case 1: return false;
	default: {
		int const xmod = abs(x)%H.width, ymod = abs(y)%H.height, xdiv = x/H.width, ydiv = y/H.height;
		x = (xdiv & 1) ? (H.width  - xmod - 1) : xmod;
		y = (ydiv & 1) ? (H.height - ymod - 1) : ymod;
		}
	}
	return true;
}

// mesh_scale >= 1: clamp_xy's nearest texel round_fp(mesh_scale*(x + 0.0f)), before clamp_no_scale (src/heightmap.cpp:309-313)
TWH_HD int near_index(float mesh_scale, int x) {return round_fp(mesh_scale*((float)x + 0.0f));}
// mesh_scale < 1: interpolate_height's scaled coordinate and its two taps floor / ceil, before clamp_no_scale (src/heightmap.cpp:394-402)
TWH_HD float lerp_index(float mesh_scale, int x, int &lo, int &hi) {
	float const s = mesh_scale*(float)x;
	lo = (int)floorf(s); hi = (int)ceilf(s);
	return s;
}

// The same at a fractional cell (hmap_points_kernel: an object between cells), the library's extension of the integer-cell function. At an integer x with
// |mesh_scale*x| < 2^30 (every |x| < 2^24 at a mesh_scale below 64) both forms give the int forms' results bit for bit: (float)x is then exact and the
// arithmetic is the same. The scaled coordinate is held to [-2^30, 2^30] (NaN goes to -2^30), so the texel index and clamp_no_scale's
// x + width/2 stay inside int range for any float a caller passes.
TWH_HD float clamp_scaled(float s) {return fminf(fmaxf(s, -1073741824.0f), 1073741824.0f);}
TWH_HD int near_index(float mesh_scale, float x) {return round_fp(clamp_scaled(mesh_scale*(x + 0.0f)));}
TWH_HD float lerp_index(float mesh_scale, float x, int &lo, int &hi) {
	float const s = clamp_scaled(mesh_scale*x);
	lo = (int)floorf(s); hi = (int)ceilf(s);
	return s;
}

} // namespace twh
