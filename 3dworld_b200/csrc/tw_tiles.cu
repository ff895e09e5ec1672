// tw_tiles.cu - the pieces of the reference's callers that sit right next to the generators (sm_90a):
//   tile_bounds_kernel     tail of tile_t::create_zvals (src/tiled_mesh.cpp:517-540): 4x4 sub-block min/max (inclusive ends), water bbox
//   glaciate_mesh_kernel   glaciate() of the ground-mode mesh (src/mesh_gen.cpp:388-404): apply_glaciate + apply_mesh_sine per cell + zbottom/ztop
//   probe_absmax_kernel,   the z estimate of gen_mesh (estimate_zminmax + set_zvals, src/mesh_gen.cpp:447-504) for tw_gen_mesh_launch, into its device record
//   gen_mesh_zvals_kernel
//   tile_normals_kernel    tile_t::upload_normal_texture (src/tiled_mesh.cpp:865-880, get_norm src/tiled_mesh.h:281-284): RGBA8 normal map + min_normal_z
//   tile_ao_kernel         tile_t::calc_mesh_ao_lighting (src/tiled_mesh.cpp:586-662): 8 directions x 8 steps of growing stride over the
//                          tile's zvals and the (stride+72)^2 context generated around it
// All are single streaming passes over data that is already resident (4 B/cell read, glaciate also 4 B/cell written): HBM/L2-bound.
#include "tw_internal.h"
#include <algorithm>

namespace {

__device__ __forceinline__ float cosf_lut(const float *__restrict__ tab, float v) { // COSF, src/sinf.h:15
	return __ldg(tab + TW_TSIZE + (tw_x86_f2i(TW_SSCALE*fabsf(v))&(TW_TSIZE-1)));
}
__device__ __forceinline__ float smin(float a, float b) {return (b < a) ? b : a;}
__device__ __forceinline__ float smax(float a, float b) {return (a < b) ? b : a;}

struct SubBounds {float zmin, zmax; int wx1, wy1, wx2, wy2;};

// grid (16 sub-blocks, ntiles), 256 threads: min/max and under-water bbox of the (block_size+1)^2 cells of one sub-block; perm (optional): block row y
// handles tile perm[y] of zvals and out
__global__ void __launch_bounds__(256)
tile_bounds_kernel(const float *__restrict__ zvals, unsigned zvsize, float wpz_max, SubBounds *__restrict__ out, const unsigned *__restrict__ perm) {
	unsigned const sb = blockIdx.x, tile = perm ? __ldg(perm + blockIdx.y) : blockIdx.y, xx = sb & 3, yy = sb >> 2, bs = zvsize/4, w = bs + 1;
	const float *z = zvals + (size_t)tile*zvsize*zvsize;
	float vmin = 100.0f, vmax = -100.0f; // FAR_DISTANCE, src/3DWorld.h:116
	int wx1 = 2147483647, wy1 = 2147483647, wx2 = -1, wy2 = -1;
	for (unsigned i = threadIdx.x; i < w*w; i += blockDim.x) {
		unsigned const x = xx*bs + i % w, y = yy*bs + i / w;
		float const v = __ldg(z + (size_t)y*zvsize + x);
		vmin = smin(vmin, v); vmax = smax(vmax, v);
		if (v < wpz_max) {wx1 = min(wx1, (int)x); wy1 = min(wy1, (int)y); wx2 = max(wx2, (int)x); wy2 = max(wy2, (int)y);}
	}
	for (int o = 16; o > 0; o >>= 1) {
		vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o)); vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
		wx1 = min(wx1, __shfl_xor_sync(0xffffffffu, wx1, o)); wy1 = min(wy1, __shfl_xor_sync(0xffffffffu, wy1, o));
		wx2 = max(wx2, __shfl_xor_sync(0xffffffffu, wx2, o)); wy2 = max(wy2, __shfl_xor_sync(0xffffffffu, wy2, o));
	}
	__shared__ SubBounds s[8];
	int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (lane == 0) {s[warp] = SubBounds{vmin, vmax, wx1, wy1, wx2, wy2};}
	__syncthreads();
	if (threadIdx.x == 0) {
		SubBounds r = s[0];
		for (int i = 1; i < 8; ++i) {
			r.zmin = fminf(r.zmin, s[i].zmin); r.zmax = fmaxf(r.zmax, s[i].zmax);
			r.wx1 = min(r.wx1, s[i].wx1); r.wy1 = min(r.wy1, s[i].wy1); r.wx2 = max(r.wx2, s[i].wx2); r.wy2 = max(r.wy2, s[i].wy2);
		}
		out[(size_t)tile*16 + sb] = r;
	}
}

struct GlacParams {
	int   glaciate; float zmax_est, zmax_est2, zmax_est2_inv, custom_exp;
	int   sine_on; float sine_mag, sine_bias, freq, mszi;
	int   volcano_on; float volcano_freq, volcano_height;
	int   nx, ny, x_shift, y_shift; // x_shift = xoff2 - MESH_X_SIZE/2
};

__device__ __forceinline__ float volcano_height(float xi, float yi, const GlacParams &P, const float *__restrict__ tab) { // src/mesh_gen.cpp:364-372
	float const x = P.volcano_freq*xi, y = P.volcano_freq*yi, dist = __fsqrt_rn(x*x + y*y);
	if ((double)dist > 2.0) return 0.0f;
	float const val = cosf_lut(tab, x)*cosf_lut(tab, y);
	double const hd = 400.0*((double)val - 0.999);
	float const hole = (float)((0.0 < hd) ? hd : 0.0);
	float const peak = (float)(0.08*(double)val/(double)smax(0.04f, dist));
	return P.volcano_height*smax(0.0f, (peak - hole))*P.mszi;
}

// REC (tw_gen_mesh_launch): zmax_est, zmax_est2 and zmax_est2_inv come from the job's device record instead of P
template<bool REC>
__global__ void __launch_bounds__(256)
glaciate_mesh_kernel(float *__restrict__ mesh, GlacParams P, const float *__restrict__ tab, unsigned *__restrict__ mm, const twi_gen_mesh_rec *__restrict__ rec) {
	if (REC) {P.zmax_est = rec->zmax_est; P.zmax_est2 = rec->zmax_est2; P.zmax_est2_inv = rec->zmax_est2_inv;}
	int const j = blockIdx.x*blockDim.x + threadIdx.x, i = blockIdx.y;
	float vmin = INFINITY, vmax = -INFINITY;
	if (j < P.nx) {
		float z = mesh[(size_t)i*P.nx + j];
		if (P.glaciate) { // apply_glaciate, src/mesh_gen.cpp:380-385
			float const relh = (z + P.zmax_est)*P.zmax_est2_inv;
			float const g = (P.custom_exp == 0.0f) ? relh*relh*relh : powf(relh, P.custom_exp);
			z = g*P.zmax_est2 - P.zmax_est;
		}
		if (P.sine_on) { // apply_mesh_sine(zval, float(j + xoff2 - MESH_X_SIZE/2), float(i + yoff2 - MESH_Y_SIZE/2)), src/mesh_gen.cpp:373-379,398
			float const x = (float)(j + P.x_shift), y = (float)(i + P.y_shift);
			z += (P.sine_mag*cosf_lut(tab, x*P.freq)*cosf_lut(tab, y*P.freq) + P.sine_bias)*P.mszi;
			if (P.volcano_on) {z += volcano_height(x, y, P, tab);}
		}
		mesh[(size_t)i*P.nx + j] = z;
		vmin = vmax = z;
	}
	for (int o = 16; o > 0; o >>= 1) {
		vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o)); vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
	}
	if (mm && (threadIdx.x & 31) == 0 && vmin <= vmax) {atomicMin(mm, tw_f2ord(vmin)); atomicMax(mm + 1, tw_f2ord(vmax));}
}

// estimate_zminmax's loop over the probe (src/mesh_gen.cpp:474-478): zmax_est = (zmax_est < |z|) ? |z| : zmax_est, so a NaN never wins. |z| is never negative, so
// its float bits order as integers and the largest non-NaN |z| is one atomicMax; folding that into zmax_est (> 0, or NaN) gives the loop's result.
__global__ void __launch_bounds__(256)
probe_absmax_kernel(const float *__restrict__ v, size_t n, unsigned *__restrict__ absmax) {
	unsigned m = 0u;
	size_t const stride = (size_t)gridDim.x*blockDim.x;
	for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride) {float const a = fabsf(__ldg(v + i)); if (a == a) {m = max(m, __float_as_uint(a));}}
	for (int o = 16; o > 0; o >>= 1) {m = max(m, __shfl_xor_sync(0xffffffffu, m, o));}
	if ((threadIdx.x & 31) == 0 && m) {atomicMax(absmax, m);}
}

// calc_zminmax -> estimate_zminmax -> set_zvals of gen_mesh (src/mesh_gen.cpp:447-504) on one thread, with the host chain's operation types: the double products
// rounded to float, and water_plane_z = get_water_z_height's tail, wpz (its zmax_est-free head) computed on the host
__global__ void gen_mesh_zvals_kernel(twi_gen_mesh_rec *rec, bool sine_mode, float wpz, float water_h_off, float prev_zbottom, float prev_ztop, float prev_wpz) {
	float const zmin = tw_ord2f(rec->mm[0]), zmax = tw_ord2f(rec->mm[1]);
	float zmax_est = (zmax < -zmin) ? -zmin : zmax;                  // set_zmax_est(max(zmax, -zmin))
	if (zmax == zmin) { // flat mesh: estimate_zminmax returns before set_zvals (src/mesh_gen.cpp:463-466)
		zmax_est = (float)((double)zmax_est + 1.0E-6);
		rec->zmin = zmin; rec->zmax = zmax; rec->zbottom = prev_zbottom; rec->ztop = prev_ztop; rec->water_plane_z = prev_wpz;
	}
	else {
		float const a = __uint_as_float(rec->absmax);
		zmax_est = (zmax_est < a) ? a : zmax_est;
		if (!sine_mode) {zmax_est = (float)((double)zmax_est*1.2);}
		zmax_est = (float)(1.1*(double)zmax_est);
		rec->zbottom = zmin; rec->ztop = zmax; rec->zmin = -zmax_est; rec->zmax = zmax_est; // set_zvals
		float const zmax_est2 = (float)(2.0*(double)zmax_est);           // get_water_z_height (src/mesh_gen.cpp:507-512)
		rec->water_plane_z = wpz*zmax_est2 - zmax_est + water_h_off;
	}
	rec->zmax_est = zmax_est;
	rec->zmax_est2 = (float)(2.0*(double)zmax_est); rec->zmax_est2_inv = (float)(1.0/(double)rec->zmax_est2); // set_zmax_est, as twi_glaciate_mesh derives them
	rec->mm[0] = 0xffffffffu; rec->mm[1] = 0u; // for the glaciated mesh's min/max
}

__global__ void gen_mesh_zbottom_kernel(twi_gen_mesh_rec *rec) {rec->zbottom = tw_ord2f(rec->mm[0]); rec->ztop = tw_ord2f(rec->mm[1]);} // glaciate(), :399-403


// One thread per cell of the stride^2 normal map (stride = zvsize-1). get_norm_not_normalized(ix) = (DY_VAL*(z[ix] - z[ix+1]),
// DX_VAL*(z[ix] - z[ix+zvsize]), dxdy), normalised by pointT::get_norm (src/3DWorld.h:297-300: unchanged when |v| < TOLERANCE), stored as
// (unsigned char)(127.0*(n + 1.0)) (double arithmetic as in the reference), alpha 0. perm (optional) as for tile_bounds_kernel.
__global__ void __launch_bounds__(256)
tile_normals_kernel(const float *__restrict__ zvals, unsigned zvsize, float dx_val, float dy_val, float dxdy, uchar4 *__restrict__ rgba, unsigned *__restrict__ min_nz,
                    const unsigned *__restrict__ perm) {
	unsigned const stride = zvsize - 1, tile = perm ? __ldg(perm + blockIdx.y) : blockIdx.y, i = blockIdx.x*blockDim.x + threadIdx.x;
	float nzv = INFINITY;
	if (i < stride*stride) {
		unsigned const y = i/stride, x = i - y*stride, ix2 = y*zvsize + x;
		const float *z = zvals + (size_t)tile*zvsize*zvsize;
		float const z0 = __ldg(z + ix2);
		float vx = dy_val*(z0 - __ldg(z + ix2 + 1)), vy = dx_val*(z0 - __ldg(z + ix2 + zvsize)), vz = dxdy;
		float const vmag = __fsqrt_rn(vx*vx + vy*vy + vz*vz);
		if (!(vmag < 1.0E-12f)) {vx = __fdiv_rn(vx, vmag); vy = __fdiv_rn(vy, vmag); vz = __fdiv_rn(vz, vmag);}
		uchar4 o;
		o.x = (unsigned char)(127.0*((double)vx + 1.0)); o.y = (unsigned char)(127.0*((double)vy + 1.0)); o.z = (unsigned char)(127.0*((double)vz + 1.0)); o.w = 0;
		rgba[(size_t)tile*stride*stride + i] = o;
		nzv = vz;
	}
	for (int o = 16; o > 0; o >>= 1) {nzv = fminf(nzv, __shfl_xor_sync(0xffffffffu, nzv, o));} // min(min_normal_z, norm.z): a NaN never replaces the minimum
	if (min_nz && (threadIdx.x & 31) == 0 && nzv < INFINITY) {atomicMin(min_nz + tile, tw_f2ord(nzv));}
}

// One thread per cell of the stride^2 AO map. Heights inside the tile come from zvals, outside from the context grid czv
// ((stride + 2*AO_RAY_LEN)^2, origin (x1 - AO_RAY_LEN, y1 - AO_RAY_LEN), generated by the same height function); the ray in direction d visits
// v += step, step += dir (offsets 1, 3, 6, ... 36 cells) with z0 += dz per step, and the first higher point ends it: atten += 8 - s.
// ctx_inside: the reference's GPU-gen-mode flow (mesh_gen_mode >= MGEN_SIMPLEX_GPU with AO on): create_zvals generated the context ONCE, cut zvals out
// of it and kept the un-eroded grid in ao_zvals (src/tiled_mesh.cpp:479-487,505); calc_mesh_ao_lighting swaps it in as czv and does NOT substitute
// zvals inside the tile (:604,620), so every ray sample comes from the un-eroded context and only the ray origin z0 is the (eroded) zval.
constexpr int AO_DIRS = 8, AO_STEPS = 8, AO_RAY_LEN = AO_STEPS*(AO_STEPS + 1)/2; // src/tiled_mesh.cpp:41-43
__global__ void __launch_bounds__(256)
tile_ao_kernel(const float *__restrict__ zvals, const float *__restrict__ czv, unsigned zvsize, float dz, bool ctx_inside, unsigned char *__restrict__ ao,
               const unsigned *__restrict__ perm) {
	unsigned const stride = zvsize - 1, csz = stride + 2*AO_RAY_LEN, tile = perm ? __ldg(perm + blockIdx.y) : blockIdx.y, i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= stride*stride) return;
	int const y = i/stride, x = i - y*stride;
	const float *z = zvals + (size_t)tile*zvsize*zvsize, *c = czv + (size_t)blockIdx.y*csz*csz; // the context grids stay in launch order
	float const zc = __ldg(z + y*zvsize + x);
	unsigned atten = 0;
#pragma unroll
	for (int d = 0; d < AO_DIRS; ++d) {
		int const k = (d < 4) ? d : d + 1, dx = k%3 - 1, dy = k/3 - 1; // ao_dirs order: y = -1..1 outer, x = -1..1 inner, skipping (0,0)
		float z0 = zc;
		int vx = x, vy = y, sx = dx, sy = dy;
#pragma unroll
		for (int s = 0; s < AO_STEPS; ++s) {
			vx += sx; vy += sy; z0 += dz; sx += dx; sy += dy;
			bool const inside = (!ctx_inside && (unsigned)vx < zvsize && (unsigned)vy < zvsize);
			float const h = inside ? __ldg(z + vy*(int)zvsize + vx) : __ldg(c + (vy + AO_RAY_LEN)*(int)csz + vx + AO_RAY_LEN);
			if (h > z0) {atten += AO_STEPS - s; break;} // hit a higher point
		}
	}
	float const ao_scale = (float)(1.0 - (double)((float)atten/(float)(AO_DIRS*AO_STEPS)));
	ao[(size_t)tile*stride*stride + i] = (unsigned char)(255.0*(double)ao_scale);
}

} // namespace

int twi_tile_bounds(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, uint32_t ntiles, uint32_t zvsize, float wpz_max, void *d_sub /* ntiles*16*24 bytes */, const unsigned *d_perm) {
	tile_bounds_kernel<<<dim3(16, ntiles), 256, 0, st>>>(d_zvals, zvsize, wpz_max, (SubBounds *)d_sub, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

static GlacParams glac_params(int nx, int ny, int xoff2, int yoff2, int MX, int MY, const tw_height_params *p) {
	GlacParams P;
	memset(&P, 0, sizeof(P));
	P.glaciate = (p->glaciate != 0);
	P.zmax_est = p->zmax_est; P.zmax_est2 = (float)(2.0*p->zmax_est); P.zmax_est2_inv = (float)(1.0/P.zmax_est2); P.custom_exp = p->custom_glaciate_exp;
	P.sine_on = (p->hmap.sine_mag > 0.0f); P.sine_mag = p->hmap.sine_mag; P.sine_bias = p->hmap.sine_bias;
	P.freq = p->mesh_scale*p->hmap.sine_freq; P.mszi = p->mesh_scale_z_inv;
	P.volcano_on = (p->hmap.volcano_width > 0.0f && p->hmap.volcano_height > 0.0f);
	P.volcano_freq = P.volcano_on ? p->mesh_scale/p->hmap.volcano_width : 0.0f; P.volcano_height = p->hmap.volcano_height;
	P.nx = nx; P.ny = ny; P.x_shift = xoff2 - MX/2; P.y_shift = yoff2 - MY/2;
	return P;
}

int twi_glaciate_mesh(tw_ctx *ctx, float *d_mesh, int nx, int ny, int xoff2, int yoff2, int MX, int MY, const tw_height_params *p, unsigned *d_mm) {
	glaciate_mesh_kernel<false><<<dim3((nx + 255)/256, ny), 256, 0, ctx->stream>>>(d_mesh, glac_params(nx, ny, xoff2, yoff2, MX, MY, p), ctx->d_sin_table, d_mm, nullptr);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_glaciate_mesh_rec(tw_ctx *ctx, float *d_mesh, int nx, int ny, int xoff2, int yoff2, int MX, int MY, const tw_height_params *p, twi_gen_mesh_rec *d_rec) {
	glaciate_mesh_kernel<true><<<dim3((nx + 255)/256, ny), 256, 0, ctx->stream>>>(d_mesh, glac_params(nx, ny, xoff2, yoff2, MX, MY, p), ctx->d_sin_table, d_rec->mm, d_rec);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_gen_mesh_zbottom(tw_ctx *ctx, twi_gen_mesh_rec *d_rec) {
	gen_mesh_zbottom_kernel<<<1, 1, 0, ctx->stream>>>(d_rec);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_gen_mesh_zvals(tw_ctx *ctx, twi_gen_mesh_rec *d_rec, const float *d_probe, size_t n, bool sine_mode, float wpz, float water_h_off,
                       float prev_zbottom, float prev_ztop, float prev_water_plane_z) {
	unsigned const blocks = (unsigned)std::min<size_t>((n + 255)/256, (size_t)ctx->num_sms*8);
	probe_absmax_kernel<<<blocks ? blocks : 1, 256, 0, ctx->stream>>>(d_probe, n, &d_rec->absmax);
	TW_LAUNCH_CHECK(ctx);
	gen_mesh_zvals_kernel<<<1, 1, 0, ctx->stream>>>(d_rec, sine_mode, wpz, water_h_off, prev_zbottom, prev_ztop, prev_water_plane_z);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_tile_normals(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, uint32_t ntiles, uint32_t zvsize, float dx_val, float dy_val, unsigned char *d_rgba, unsigned *d_min_nz_ord,
                     const unsigned *d_perm) {
	unsigned const stride = zvsize - 1;
	tile_normals_kernel<<<dim3((stride*stride + 255)/256, ntiles), 256, 0, st>>>(d_zvals, zvsize, dx_val, dy_val, dx_val*dy_val /* dxdy, src/matrix_ops.cpp:80 */,
		(uchar4 *)d_rgba, d_min_nz_ord, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

__global__ void fill_u32_kernel(unsigned *__restrict__ v, size_t n, unsigned value) {
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) {v[i] = value;}
}
int twi_fill_u32(tw_ctx *ctx, cudaStream_t st, unsigned *d_vals, size_t n, unsigned value) {
	fill_u32_kernel<<<(unsigned)((n + 255)/256), 256, 0, st>>>(d_vals, n, value);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_tile_ao(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, const float *d_czv, uint32_t ntiles, uint32_t zvsize, float half_dxy, bool ctx_inside, unsigned char *d_ao,
                const unsigned *d_perm) {
	unsigned const stride = zvsize - 1;
	float const dz = (float)(0.5*half_dxy); // src/tiled_mesh.cpp:612
	tile_ao_kernel<<<dim3((stride*stride + 255)/256, ntiles), 256, 0, st>>>(d_zvals, d_czv, zvsize, dz, ctx_inside, d_ao, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// zvals = the zvsize^2 interior of the (stride + 72)^2 context grid: zval = ao_zvals[(y + AO_RAY_LEN)*context_sz + (x + AO_RAY_LEN)] (src/tiled_mesh.cpp:505);
// perm (optional): context z is cut into tile perm[z] of zvals
__global__ void tile_cut_kernel(const float *__restrict__ czv, unsigned zvsize, float *__restrict__ zvals, const unsigned *__restrict__ perm) {
	unsigned const csz = zvsize - 1 + 2*AO_RAY_LEN, x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y;
	size_t const tile = blockIdx.z, out_tile = perm ? __ldg(perm + blockIdx.z) : blockIdx.z;
	if (x < zvsize) {zvals[out_tile*zvsize*zvsize + (size_t)y*zvsize + x] = __ldg(czv + tile*csz*csz + (size_t)(y + AO_RAY_LEN)*csz + x + AO_RAY_LEN);}
}
int twi_tile_cut(tw_ctx *ctx, cudaStream_t st, const float *d_czv, uint32_t ntiles, uint32_t zvsize, float *d_zvals, const unsigned *d_perm) {
	tile_cut_kernel<<<dim3((zvsize + 127)/128, zvsize, ntiles), 128, 0, st>>>(d_czv, zvsize, d_zvals, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ terrain weights texture (tw_tile_weights_batch)
#include "tw_weights.cuh"
namespace {
// one thread per texel; rand = the force-sine-mode noise grid of the tile (stride^2, un-scaled); flags[tile] |= "a texel has grass"; perm (optional): launch tile z
// handles tile perm[z] of zvals, tile_params, out and flags (rand stays in launch order)
__global__ void tile_weights_kernel(const float *__restrict__ zvals, const float *__restrict__ rand, unsigned zvsize, const float *__restrict__ tile_params, tw_weight_params W,
	uchar4 *__restrict__ out, unsigned char *__restrict__ flags, const unsigned *__restrict__ perm)
{
	unsigned const stride = zvsize - 1, x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y, tile = perm ? __ldg(perm + blockIdx.z) : blockIdx.z;
	bool grass = false;
	if (x < stride) {
		unsigned char rgba[4];
		float const rand_offset = W.noise_scale*__ldg(rand + ((size_t)blockIdx.z*stride + y)*stride + x);
		grass = tww::weights_texel(zvals + (size_t)tile*zvsize*zvsize, zvsize, x, y, rand_offset, tile_params + (size_t)tile*8, W, rgba);
		out[((size_t)tile*stride + y)*stride + x] = make_uchar4(rgba[0], rgba[1], rgba[2], rgba[3]);
	}
	if (flags && __any_sync(0xffffffffu, grass) && (threadIdx.x & 31) == 0) {flags[tile] = 1;} // benign race: every writer stores 1
}
}

int twi_tile_weights(tw_ctx *ctx, cudaStream_t st, const float *d_zvals, const float *d_rand, uint32_t ntiles, uint32_t zvsize, const float *d_tile_params, const tw_weight_params *W,
                     uint8_t *d_out, uint8_t *d_flags, const unsigned *d_perm) {
	unsigned const stride = zvsize - 1;
	for (uint32_t t0 = 0; t0 < ntiles; t0 += 65535) { // gridDim.z limit
		uint32_t const nt = (ntiles - t0 < 65535) ? ntiles - t0 : 65535;
		size_t const r0 = d_perm ? 0 : t0; // first tile the launch addresses directly; with a permutation every tile-indexed access goes through it
		tile_weights_kernel<<<dim3((stride + 127)/128, stride, nt), 128, 0, st>>>(d_zvals + r0*zvsize*zvsize, d_rand + (size_t)t0*stride*stride, zvsize,
			d_tile_params + r0*8, *W, (uchar4 *)d_out + r0*stride*stride, d_flags ? d_flags + r0 : nullptr, d_perm ? d_perm + t0 : nullptr);
		TW_LAUNCH_CHECK(ctx);
	}
	return TW_OK;
}

