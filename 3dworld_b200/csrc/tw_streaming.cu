// tw_streaming.cu - HBM-bound element-wise passes on the far side of the height path (SURVEY.md section 8f N2):
//   heightmap_t::from_floats / to_floats 16-bit pack (src/heightmap.cpp:191-215, texture_t::write_pixel_16_bits src/Textures.cpp:1889-1893).
// One float4 (16 B) in, 8 B out per thread; grid sized to a multiple of the SM count.
#include "tw_internal.h"
#include "tw_hmap_index.cuh"
#include <algorithm>
#include <map>

namespace {

__device__ __forceinline__ unsigned pack16(float h, float val_add, float val_div, unsigned &bad) {
	float const v = (h - val_add)*val_div;                 // src/heightmap.cpp:210
	if (!(v >= 0.0f && v < 256.0f)) {bad = 1; return 0;}   // the reference asserts here (:211)
	unsigned const high_bits = (unsigned)v & 0xffu;        // (unsigned char)val - truncate
	unsigned const low_bits  = (unsigned)(256.0f*(v - (float)high_bits)) & 0xffu;
	return low_bits | (high_bits << 8);                    // data[2i] = low, data[2i+1] = high
}

// stage (optional): val_add / val_div come from the device (tw_proc_gen_heightmap_launch) instead of the arguments
__global__ void from_floats_u16_kernel(const float *__restrict__ vals, size_t n, float val_add, float val_div, uint16_t *__restrict__ out, unsigned *__restrict__ bad_count,
                                       const twi_hmap_stage *__restrict__ stage = nullptr) {
	if (stage) {val_add = stage->val_add; val_div = stage->val_div;}
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

// the host code of tw_proc_gen_heightmap's scalars, operation for operation (every TU is built with -fmad=false; the _rn intrinsics pin the rest):
// set_mesh_height_scales_for_zval_range(min_z, dz/255.0) and get_mh_texture_mult/add (src/mesh_gen.cpp:124-131), val_div as twi_from_floats_u16 forms it
__global__ void hmap_scales_kernel(const unsigned *__restrict__ mm, float mhs, float mszi, twi_hmap_stage *__restrict__ st) {
	float const TOLERANCE = 1.0E-12, READ_MESH_H_SCALE = 0.0008; // src/3DWorld.h:50, src/mesh_gen.cpp:22
	float const min_z = tw_ord2f(mm[0]), max_z = tw_ord2f(mm[1]);
	float const dzr = __fsub_rn(max_z, min_z), dz = (TOLERANCE < dzr) ? dzr : TOLERANCE;
	float const dz255 = __double2float_rn(__ddiv_rn((double)dz, 255.0));
	float const rh = __fmul_rn(READ_MESH_H_SCALE, mhs);
	float const mesh_file_scale = __fdiv_rn(dz255, __fmul_rn(rh, mszi));
	float const mesh_file_tz = __fdiv_rn(min_z, mszi);
	float const val_mult = __fmul_rn(__fmul_rn(rh, mesh_file_scale), mszi);
	st->min_z = min_z; st->max_z = max_z; st->val_mult = val_mult; st->val_add = __fmul_rn(mesh_file_tz, mszi);
	st->mesh_file_scale = mesh_file_scale; st->mesh_file_tz = mesh_file_tz;
	st->val_div = __double2float_rn(__ddiv_rn(1.0, (double)val_mult)); // src/heightmap.cpp:206
}

__global__ void ord_min_kernel(const unsigned *__restrict__ mm, float *__restrict__ out) {*out = tw_ord2f(mm[0]);}

int grid_for(const tw_ctx *ctx, size_t n) {size_t b = (n + 1023)/1024; if (b > ctx->num_sms*16) b = ctx->num_sms*16; if (b < 1) b = 1; return (int)b;}

} // namespace

int twi_from_floats_u16(tw_ctx *ctx, const float *d_vals, size_t n, float val_mult, float val_add, uint8_t *d_out, unsigned *d_bad) {
	float const val_div = (float)(1.0/(double)val_mult); // src/heightmap.cpp:206
	from_floats_u16_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(d_vals, n, val_add, val_div, reinterpret_cast<uint16_t *>(d_out), d_bad);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_hmap_scales(tw_ctx *ctx, const unsigned *d_mm, float mesh_height_scale, float mesh_scale_z_inv, twi_hmap_stage *d_stage) {
	hmap_scales_kernel<<<1, 1, 0, ctx->stream>>>(d_mm, mesh_height_scale, mesh_scale_z_inv, d_stage);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_from_floats_u16_dev(tw_ctx *ctx, const float *d_vals, size_t n, const twi_hmap_stage *d_stage, uint8_t *d_out) {
	from_floats_u16_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(d_vals, n, 0.0f, 0.0f, reinterpret_cast<uint16_t *>(d_out), const_cast<unsigned *>(&d_stage->bad), d_stage);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_ord_min(tw_ctx *ctx, const unsigned *d_mm, float *d_min) {
	ord_min_kernel<<<1, 1, 0, ctx->stream>>>(d_mm, d_min);
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
		int xlo, ylo, xhi, yhi;
		float const sx = twh::lerp_index(H.mesh_scale, x, xlo, xhi), sy = twh::lerp_index(H.mesh_scale, y, ylo, yhi);
		float const xv = sx - (float)xlo, yv = sy - (float)ylo;
		bool const ok_lo = twh::clamp_no_scale(xlo, ylo, H);
		bool const ok = ok_lo && twh::clamp_no_scale(xhi, yhi, H); // the reference short-circuits the same way
		if (!ok) {z = hmap_scale_val(0.0f, H);}
		else {
			z = yv*(xv*hmap_raw_height(data16, xhi, yhi, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, yhi, H)) +
			    (1.0f - yv)*(xv*hmap_raw_height(data16, xhi, ylo, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, ylo, H));
		}
	}
	else { // clamp_xy(x, y): x = round_fp(mesh_scale*(x + 0.0f)), src/heightmap.cpp:309-313
		x = twh::near_index(H.mesh_scale, x); y = twh::near_index(H.mesh_scale, y);
		z = twh::clamp_no_scale(x, y, H) ? hmap_raw_height(data16, x, y, H) : hmap_scale_val(0.0f, H);
	}
	out[(size_t)tile*zvsize*zvsize + i] = z;
}

// get_clamped_height at n arbitrary cells (x, y) of the tiles' index space, one thread per point: hmap_sample_tiles_kernel's expressions with the float index
// forms, so an integer cell gives that kernel's value bit for bit and a fractional one takes the float directly
__global__ void __launch_bounds__(256)
hmap_points_kernel(const uint8_t *__restrict__ data16, tw_hmap_sampler H, const float2 *__restrict__ xy, size_t n, float *__restrict__ out) {
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	float2 const pt = __ldg(xy + i);
	float z;
	if (H.mesh_scale < 1.0f) {
		int xlo, ylo, xhi, yhi;
		float const sx = twh::lerp_index(H.mesh_scale, pt.x, xlo, xhi), sy = twh::lerp_index(H.mesh_scale, pt.y, ylo, yhi);
		float const xv = sx - (float)xlo, yv = sy - (float)ylo;
		bool const ok_lo = twh::clamp_no_scale(xlo, ylo, H);
		bool const ok = ok_lo && twh::clamp_no_scale(xhi, yhi, H);
		if (!ok) {z = hmap_scale_val(0.0f, H);}
		else {
			z = yv*(xv*hmap_raw_height(data16, xhi, yhi, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, yhi, H)) +
			    (1.0f - yv)*(xv*hmap_raw_height(data16, xhi, ylo, H) + (1.0f - xv)*hmap_raw_height(data16, xlo, ylo, H));
		}
	}
	else {
		int x = twh::near_index(H.mesh_scale, pt.x), y = twh::near_index(H.mesh_scale, pt.y);
		z = twh::clamp_no_scale(x, y, H) ? hmap_raw_height(data16, x, y, H) : hmap_scale_val(0.0f, H);
	}
	out[i] = z;
}
} // namespace

int twi_hmap_points(tw_ctx *ctx, const uint8_t *d_data16, const tw_hmap_sampler *hs, const float *d_xy, size_t n, float *d_out) {
	hmap_points_kernel<<<(unsigned)((n + 255)/256), 256, 0, ctx->stream>>>(d_data16, *hs, reinterpret_cast<const float2 *>(d_xy), n, d_out);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

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

// ------------------------------------------------------------------------------------------------ heightmap image edits (tw_update_heightmap)
namespace {
// Row r copies rows[r].w texels from data + rows[r].src to img + rows[r].dst. The host packs every row so that its source has the destination's phase
// modulo 16 bytes, so the row's body moves as 16-byte words and only its head and tail as single texels. One warp per row.
__global__ void __launch_bounds__(256)
hmap_scatter_kernel(const twi_hmap_row *__restrict__ rows, uint32_t nrows, const uint16_t *__restrict__ data, uint16_t *__restrict__ img) {
	unsigned const lane = threadIdx.x & 31u;
	for (uint32_t r = (blockIdx.x*blockDim.x + threadIdx.x) >> 5; r < nrows; r += (gridDim.x*blockDim.x) >> 5) {
		twi_hmap_row const R = rows[r];
		uint16_t *d = img + R.dst;
		const uint16_t *s = data + R.src;
		unsigned const head = min(R.w, (8u - (unsigned)(R.dst & 7u)) & 7u), n16 = (R.w - head) >> 3, tail = head + 8u*n16;
		for (unsigned i = lane; i < head; i += 32) {d[i] = s[i];}
		const uint4 *s4 = reinterpret_cast<const uint4 *>(s + head);
		uint4 *d4 = reinterpret_cast<uint4 *>(d + head);
		for (unsigned i = lane; i < n16; i += 32) {d4[i] = __ldg(s4 + i);}
		for (unsigned i = tail + lane; i < R.w; i += 32) {d[i] = s[i];}
	}
}
} // namespace

int twi_hmap_scatter(tw_ctx *ctx, cudaStream_t st, const twi_hmap_row *d_rows, uint32_t nrows, const uint8_t *d_data, uint8_t *d_img) {
	unsigned const blocks = std::max(1u, std::min((nrows + 7u)/8u, ctx->num_sms*16u));
	hmap_scatter_kernel<<<blocks, 256, 0, st>>>(d_rows, nrows, reinterpret_cast<const uint16_t *>(d_data), reinterpret_cast<uint16_t *>(d_img));
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// The sampler's index arithmetic is separable: clamp, mirror and the cliff test act on each axis alone, and a tile's cells are the product of its columns and
// rows. So the texels a tile reads are the product of the texels its columns read and the texels its rows read (cliff mode: of the columns and rows that stay
// on the texture), and a tile reads a texel of a rect exactly when both axis sets meet the rect's ranges.
extern "C" int tw_hmap_tiles_touched(const tw_hmap_sampler *hs, const int32_t *origins_xy, uint32_t ntiles, uint32_t zvsize, const tw_hmap_rect *rects,
                                     uint32_t nrects, uint8_t *touched) {
	if (!hs || hs->edge_mode < 0 || hs->edge_mode > 2 || hs->width <= 0 || hs->height <= 0 || zvsize < 2) return TW_ERR_ARG;
	if ((ntiles && (!origins_xy || !touched)) || (nrects && !rects)) return TW_ERR_ARG;
	tw_hmap_sampler const H = *hs;
	// the sorted texels the cells o .. o + zvsize - 1 of one axis read; the other axis is held at the image's first texel, which is always on the texture
	auto axis = [&](int o, bool is_x) {
		std::vector<int> out;
		out.reserve(2*(size_t)zvsize);
		for (uint32_t i = 0; i < zvsize; ++i) {
			int const v = o + (int)i;
			int const fixed = is_x ? -(H.height/2) : -(H.width/2);
			if (H.mesh_scale < 1.0f) {
				int lo, hi;
				twh::lerp_index(H.mesh_scale, v, lo, hi);
				int lx = is_x ? lo : fixed, ly = is_x ? fixed : lo, hx = is_x ? hi : fixed, hy = is_x ? fixed : hi;
				if (twh::clamp_no_scale(lx, ly, H) && twh::clamp_no_scale(hx, hy, H)) {out.push_back(is_x ? lx : ly); out.push_back(is_x ? hx : hy);}
			}
			else {
				int const t = twh::near_index(H.mesh_scale, v);
				int x = is_x ? t : fixed, y = is_x ? fixed : t;
				if (twh::clamp_no_scale(x, y, H)) {out.push_back(is_x ? x : y);}
			}
		}
		std::sort(out.begin(), out.end());
		out.erase(std::unique(out.begin(), out.end()), out.end());
		return out;
	};
	auto meets = [](std::vector<int> const &s, int a, int n) {auto const it = std::lower_bound(s.begin(), s.end(), a); return it != s.end() && (long long)*it < (long long)a + n;};
	std::map<int, std::vector<int>> cols, rows; // tiles of one grid column (row) share their column (row) texels
	for (uint32_t t = 0; t < ntiles; ++t) {
		int const x1 = origins_xy[2*t], y1 = origins_xy[2*t + 1];
		auto cx = cols.find(x1);
		if (cx == cols.end()) cx = cols.emplace(x1, axis(x1, true)).first;
		auto cy = rows.find(y1);
		if (cy == rows.end()) cy = rows.emplace(y1, axis(y1, false)).first;
		uint8_t hit = 0;
		for (uint32_t r = 0; r < nrects && !hit; ++r) {hit = meets(cx->second, rects[r].x, rects[r].w) && meets(cy->second, rects[r].y, rects[r].h);}
		touched[t] = hit;
	}
	return TW_OK;
}
