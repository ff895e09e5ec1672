// tw_streaming.cu - HBM-bound element-wise passes on the far side of the height path (SURVEY.md section 8f N2):
//   heightmap_t::from_floats / to_floats 16-bit pack (src/heightmap.cpp:191-215, texture_t::write_pixel_16_bits src/Textures.cpp:1889-1893).
// One float4 (16 B) in, 8 B out per thread; grid sized to a multiple of the SM count.
#include "tw_internal.h"

namespace {

__device__ __forceinline__ unsigned pack16(float h, float val_add, float val_div, unsigned &bad) {
	float const v = (h - val_add)*val_div;                 // src/heightmap.cpp:210
	if (!(v >= 0.0f && v < 256.0f)) {bad = 1; return 0;}   // the reference asserts here (:211)
	unsigned const high_bits = (unsigned)v & 0xffu;        // (unsigned char)val - truncate
	unsigned const low_bits  = (unsigned)(256.0f*(v - (float)high_bits)) & 0xffu;
	return low_bits | (high_bits << 8);                    // data[2i] = low, data[2i+1] = high
}

__global__ void from_floats_u16_kernel(const float *__restrict__ vals, size_t n, float val_add, float val_div, uint16_t *__restrict__ out, unsigned *__restrict__ bad_count) {
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	unsigned bad = 0;
	size_t const n4 = n/4;
	bool const aligned = ((((uintptr_t)vals) & 15) == 0) && ((((uintptr_t)out) & 7) == 0);
	if (aligned) {
		for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n4; i += stride) {
			float4 const v = __ldg(reinterpret_cast<const float4 *>(vals) + i);
			unsigned const a = pack16(v.x, val_add, val_div, bad) | (pack16(v.y, val_add, val_div, bad) << 16);
			unsigned const b = pack16(v.z, val_add, val_div, bad) | (pack16(v.w, val_add, val_div, bad) << 16);
			reinterpret_cast<uint2 *>(out)[i] = make_uint2(a, b);
		}
		for (size_t i = 4*n4 + (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {out[i] = (uint16_t)pack16(__ldg(vals + i), val_add, val_div, bad);}
	}
	else {
		for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {out[i] = (uint16_t)pack16(__ldg(vals + i), val_add, val_div, bad);}
	}
	if (bad) {atomicAdd(bad_count, 1u);}
}

__global__ void to_floats_u16_kernel(const uint16_t *__restrict__ data, size_t n, float val_mult, float val_add, float *__restrict__ vals) {
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {
		unsigned const p = __ldg(data + i);
		float const v = (float)((double)(p & 0xffu)/256.0 + (double)(p >> 8)); // data[i<<1]/256.0 + data[(i<<1)+1], src/heightmap.cpp:199
		vals[i] = val_mult*v + val_add;
	}
}

int grid_for(const tw_ctx *ctx, size_t n) {size_t b = (n + 1023)/1024; if (b > ctx->num_sms*16) b = ctx->num_sms*16; if (b < 1) b = 1; return (int)b;}

} // namespace

int twi_from_floats_u16(tw_ctx *ctx, const float *d_vals, size_t n, float val_mult, float val_add, uint8_t *d_out, unsigned *d_bad) {
	float const val_div = (float)(1.0/(double)val_mult); // src/heightmap.cpp:206
	from_floats_u16_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(d_vals, n, val_add, val_div, reinterpret_cast<uint16_t *>(d_out), d_bad);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_to_floats_u16(tw_ctx *ctx, const uint8_t *d_data, size_t n, float val_mult, float val_add, float *d_vals) {
	to_floats_u16_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(reinterpret_cast<const uint16_t *>(d_data), n, val_mult, val_add, d_vals);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ heightmap-texture tiles (N2)
namespace {
__device__ __forceinline__ int round_fp(float v) {return (v > 0.0f) ? (int)(v + 0.5f) : (int)(v - 0.5f);} // src/inlines.h:63 (values are small: no x86 overflow semantics needed)

// clamp_no_scale, src/heightmap.cpp:315-341
__device__ __forceinline__ bool hmap_clamp_no_scale(int &x, int &y, const tw_hmap_sampler &H) {
	x += H.width/2; y += H.height/2;
	if (x >= 0 && y >= 0 && x < H.width && y < H.height) return true;
	switch (H.edge_mode) {
	case 0: x = max(0, min(H.width - 1, x)); y = max(0, min(H.height - 1, y)); break;
	case 1: return false;
	default: {
		int const xmod = abs(x)%H.width, ymod = abs(y)%H.height, xdiv = x/H.width, ydiv = y/H.height;
		x = (xdiv & 1) ? (H.width  - xmod - 1) : xmod;
		y = (ydiv & 1) ? (H.height - ymod - 1) : ymod;
		}
	}
	return true;
}
__device__ __forceinline__ float hmap_scale_val(float val, const tw_hmap_sampler &H) { // scale_mh_texture_val, src/mesh_gen.cpp:120
	return (H.h_scale*H.mesh_file_scale*val + H.mesh_file_tz)*H.mesh_scale_z_inv;
}
__device__ __forceinline__ float hmap_raw_height(const uint8_t *__restrict__ d, int x, int y, const tw_hmap_sampler &H) { // get_raw_height
	size_t const ix = (size_t)H.width*y + x;
	unsigned const px = __ldg(reinterpret_cast<const unsigned short *>(d) + ix); // little endian: low byte = data[2ix] (fraction), high = data[2ix+1]
	float const v = (float)((double)(px & 255u)/256.0 + (double)(px >> 8)); // get_heightmap_value: exact in fp32 (16 significant bits)
	return hmap_scale_val(v, H);
}

__global__ void __launch_bounds__(256)
hmap_sample_tiles_kernel(const uint8_t *__restrict__ data16, tw_hmap_sampler H, const int2 *__restrict__ origins, unsigned zvsize, float *__restrict__ out,
                         const unsigned *__restrict__ perm, int cstep) {
	unsigned const i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= zvsize*zvsize) return;
	unsigned const tile = perm ? __ldg(perm + blockIdx.y) : blockIdx.y;
	int2 const o = __ldg(origins + tile);
	int x = o.x + cstep*(int)(i % zvsize), y = o.y + cstep*(int)(i / zvsize);
	float z;
	if (H.mesh_scale < 1.0f) { // interpolate_height(float(x), float(y)), src/heightmap.cpp:394-402
		float const sx = H.mesh_scale*(float)x, sy = H.mesh_scale*(float)y;
		int xlo = (int)floorf(sx), ylo = (int)floorf(sy), xhi = (int)ceilf(sx), yhi = (int)ceilf(sy);
		float const xv = sx - (float)xlo, yv = sy - (float)ylo;
		bool const ok_lo = hmap_clamp_no_scale(xlo, ylo, H);
		bool const ok = ok_lo && hmap_clamp_no_scale(xhi, yhi, H); // the reference short-circuits the same way
		if (!ok) {z = hmap_scale_val(0.0f, H);}
		else {
			z = yv*(xv*hmap_raw_height(data16, xhi, yhi, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, yhi, H)) +
			    (1.0f - yv)*(xv*hmap_raw_height(data16, xhi, ylo, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, ylo, H));
		}
	}
	else { // clamp_xy(x, y): x = round_fp(mesh_scale*(x + 0.0f)), src/heightmap.cpp:309-313
		x = round_fp(H.mesh_scale*((float)x + 0.0f)); y = round_fp(H.mesh_scale*((float)y + 0.0f));
		z = hmap_clamp_no_scale(x, y, H) ? hmap_raw_height(data16, x, y, H) : hmap_scale_val(0.0f, H);
	}
	out[(size_t)tile*zvsize*zvsize + i] = z;
}
} // namespace

int twi_hmap_sample_tiles(tw_ctx *ctx, const uint8_t *d_data16, const tw_hmap_sampler *hs, const void *d_origins, uint32_t ntiles, uint32_t zvsize, float *d_out,
                          cudaStream_t st, const unsigned *d_perm, uint32_t cstep) {
	size_t const tile_elems = (size_t)zvsize*zvsize;
	for (uint32_t t0 = 0; t0 < ntiles; t0 += 65535) { // gridDim.y limit
		uint32_t const nt = (ntiles - t0 < 65535) ? ntiles - t0 : 65535;
		const int2 *org = (const int2 *)d_origins + (d_perm ? 0 : t0);
		float *out = d_out + (d_perm ? 0 : (size_t)t0*tile_elems);
		hmap_sample_tiles_kernel<<<dim3((zvsize*zvsize + 255)/256, nt), 256, 0, st ? st : ctx->stream>>>(d_data16, *hs, org, zvsize, out, d_perm ? d_perm + t0 : nullptr, (int)cstep);
		TW_LAUNCH_CHECK(ctx);
	}
	return TW_OK;
}
