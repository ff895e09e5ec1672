// tw_voxel.cu - 3-D voxel density fill (sm_90a). Replaces the fill loop of voxel_manager::create_procedural
// (src/voxels.cpp:278-346), noise_gen_3d::{gen_xyz_vals,get_val} (src/upsurface.cpp:41-70) and the atten_* passes (src/voxels.cpp:403-482).
// Output layout is the reference's: out[z + (x + y*nx)*nz] (src/voxels.h:141-144), z fastest => lanes run along z, stores coalesce.
//
//   xyz_tables_kernel   gen_xyz_vals: per-axis tables SINF(f*pos + phase) (x table pre-multiplied by mag). The position is the
//                       reference's running sum val += step (:53), so each (axis) is a short serial prefix done by one thread per k.
//   voxel_sine_kernel   get_val(x,y,z,tables): val = sum_k (xv[k]*yv[k])*zv[k], sequential fp32 sum; the x*y product is shared by the
//                       whole z column, the z table is staged k-major in shared memory. 2 flops/term/voxel + 4 B store.
//   voxel_glm_kernel    GLM perlin/simplex fBm (:327-339), one voxel per thread.
//   fused epilogue      val += z*zscale; clamp to [-1,1] (:340-341); optional attenuation (atten_at_edges / top / sphere).
#include "tw_voxel_fill.cuh"

namespace {

// tables: xt[k*xpitch + i] (x pre-multiplied by mag), yt, zt; one thread per (axis, k) walks i serially (val += step is a serial fp32 sum)
__global__ void xyz_tables_kernel(float *__restrict__ xt, float *__restrict__ yt, float *__restrict__ zt, unsigned xpitch, unsigned ypitch, unsigned zpitch,
	unsigned nx, unsigned ny, unsigned nz, float sx, float sy, float sz, float dxs, float dys, float dzs, const float *__restrict__ rdata, const float *__restrict__ sin_tab)
{
	int const k = threadIdx.x, d = blockIdx.x;
	if (k >= NS) return;
	unsigned const n = (d == 0) ? nx : (d == 1) ? ny : nz, pitch = (d == 0) ? xpitch : (d == 1) ? ypitch : zpitch;
	float *t = (d == 0) ? xt : (d == 1) ? yt : zt;
	float val = (d == 0) ? sx : (d == 1) ? sy : sz;
	float const step = (d == 0) ? dxs : (d == 1) ? dys : dzs;
	unsigned const index2 = 7*k + 2*d;
	float const f = __ldg(rdata + index2 + 1), ph = __ldg(rdata + index2 + 2), mag = __ldg(rdata + 7*k);
	for (unsigned i = 0; i < n; ++i) {
		float v = sinf_lut(sin_tab, f*val + ph);
		if (d == 0) {v *= mag;}
		t[(size_t)k*pitch + i] = v;
		val += step;
	}
}

// block = VZ threads along z for one y and a range of VXB x columns (VX at a time); the z-table slice is staged once per block.
constexpr int VZ  = 128;  // z per block (threads)
constexpr int VX  = 8;    // x per thread per pass
constexpr int VXB = 64;   // x per block

__global__ void __launch_bounds__(VZ)
voxel_sine_kernel(float *__restrict__ out, const float *__restrict__ xt, const float *__restrict__ yt, const float *__restrict__ zt,
	unsigned xpitch, unsigned ypitch, unsigned zpitch, VoxEpilogue E)
{
	__shared__ float zs[NS][VZ];                    // z table slice, k-major
	__shared__ __align__(16) float xy[NS][VX];      // xv[k]*yv[k] for the current x pass (shared by the whole z column)
	__shared__ float ys[NS];
	unsigned const z0 = blockIdx.x*VZ, xb = blockIdx.y*VXB, y = blockIdx.z;
	unsigned const tz = threadIdx.x, z = z0 + tz;
	for (int e = tz; e < NS*VZ; e += VZ) {
		int const k = e / VZ, c = e % VZ;
		zs[k][c] = (z0 + c < E.nz) ? __ldg(zt + (size_t)k*zpitch + z0 + c) : 0.0f;
	}
	if (tz < NS) {ys[tz] = __ldg(yt + (size_t)tz*ypitch + y);}
	for (unsigned x0 = xb; x0 < min(xb + VXB, E.nx); x0 += VX) {
		__syncthreads();
		for (int e = tz; e < NS*VX; e += VZ) {
			int const k = e / VX, c = e % VX;
			xy[k][c] = (x0 + c < E.nx) ? __ldg(xt + (size_t)k*xpitch + x0 + c)*ys[k] : 0.0f;
		}
		__syncthreads();
		float2 acc2[VX/2]; // paired accumulators: two x columns per step (see tw_noise2.cuh)
#pragma unroll
		for (int c = 0; c < VX/2; ++c) {acc2[c] = make_float2(0.0f, 0.0f);}
#pragma unroll 4
		for (int k = 0; k < NS; ++k) {
			float2 const zv = twn2::splat(zs[k][tz]);
			float4 const a = *reinterpret_cast<const float4 *>(&xy[k][0]), b = *reinterpret_cast<const float4 *>(&xy[k][4]);
			// val += xv[k]*yv[k]*zv[k]: (xv*yv)*zv rounded, then added (no contraction)
			acc2[0] = twn2::add2(twn2::mul2(make_float2(a.x, a.y), zv), acc2[0]);
			acc2[1] = twn2::add2(twn2::mul2(make_float2(a.z, a.w), zv), acc2[1]);
			acc2[2] = twn2::add2(twn2::mul2(make_float2(b.x, b.y), zv), acc2[2]);
			acc2[3] = twn2::add2(twn2::mul2(make_float2(b.z, b.w), zv), acc2[3]);
		}
		float const acc[VX] = {acc2[0].x, acc2[0].y, acc2[1].x, acc2[1].y, acc2[2].x, acc2[2].y, acc2[3].x, acc2[3].y};
		if (z < E.nz) {
#pragma unroll
			for (int c = 0; c < VX; ++c) {
				unsigned const x = x0 + c;
				if (x < E.nx) {out[z + ((size_t)x + (size_t)y*E.nx)*E.nz] = epilogue(acc[c], x, y, z, E);}
			}
		}
	}
}

// One voxel per thread, lanes along z (the layout's fastest dimension); a block walks VGX consecutive x columns so that the 74 KB
// hash/gradient table (tw_noise2.cuh: gradient of permute(k) for every reachable argument k of the last permute) is staged once per
// VGX*blockDim voxels.
constexpr unsigned VGX = 32;
template<bool PERLIN>
__global__ void __launch_bounds__(256, 3)
voxel_glm_kernel(float *__restrict__ out, GlmParams G, VoxEpilogue E, const float4 *__restrict__ lut)
{
	extern __shared__ float4 lut_s[]; // LUT3D_N*SIMPLEX_LUT_COPIES entries (74 KB)
	for (int e = threadIdx.x; e < twn2::LUT3D_N*twn2::SIMPLEX_LUT_COPIES; e += blockDim.x) {lut_s[e] = __ldg(lut + e/twn2::SIMPLEX_LUT_COPIES);}
	__syncthreads();
	unsigned L = twn2::simplex_lut_base(lut_s, threadIdx.x);
	asm volatile("" : "+r"(L) :: "memory"); // table loads depend on L, defined after the barrier
	unsigned const z = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.z;
	if (z >= E.nz) return;
	float const py = glm_pos(G, 1, y), pz = glm_pos(G, 2, z);
	for (unsigned x = blockIdx.y*VGX; x < min(E.nx, (blockIdx.y + 1)*VGX); ++x) {
		float const val = glm_value<PERLIN>(G, glm_pos(G, 0, x), py, pz, L);
		out[z + ((size_t)x + (size_t)y*E.nx)*E.nz] = epilogue(val, x, y, z, E);
	}
}

__global__ void glm3_lut_kernel(float4 *__restrict__ lut) { // [0, N): simplex(vec3) table, [N, 2N): perlin(vec3) table
	int const k = blockIdx.x*blockDim.x + threadIdx.x;
	if (k < twn2::LUT3D_N) {lut[k] = twn2::simplex3_lut_entry((float)k); lut[twn2::LUT3D_N + k] = twn2::perlin3_lut_entry((float)k);}
}

} // namespace

int twi_ensure_glm3_lut(tw_ctx *ctx) {
	if (ctx->d_glm3_lut) return TW_OK;
	TW_CUDA(ctx, cudaMalloc(&ctx->d_glm3_lut, 2*twn2::LUT3D_N*sizeof(float4)));
	glm3_lut_kernel<<<(twn2::LUT3D_N + 127)/128, 128, 0, ctx->stream>>>((float4 *)ctx->d_glm3_lut);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

int twi_voxel_fill_check(tw_ctx *ctx, const tw_voxel_params *vp, size_t *tab_bytes)
{
	if (!ctx->have_sin) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	if (vp->gen_mode < 0 || vp->gen_mode > TW_MGEN_DWARP_GPU) return tw_set_error(ctx, TW_ERR_ARG, "bad gen_mode");
	unsigned const nx = vp->nx, ny = vp->ny, nz = vp->nz;
	if (nx == 0 || ny == 0 || nz == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_fill: empty grid");
	if (ny > 65535 || (vp->gen_mode != TW_MGEN_SINE && nx > 65535)) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_fill: nx/ny > 65535 not supported");
	unsigned const xp = (nx + 31) & ~31u, yp = (ny + 31) & ~31u, zp = (nz + 31) & ~31u;
	*tab_bytes = (vp->gen_mode == TW_MGEN_SINE) ? (size_t)NS*(xp + yp + zp)*sizeof(float) + TW_N3D_RDATA*sizeof(float) : 0;
	return TW_OK;
}

int twi_voxel_fill(tw_ctx *ctx, const tw_voxel_params *vp, const float *rdata420, float *d_out, void *h_stage)
{
	unsigned const nx = vp->nx, ny = vp->ny, nz = vp->nz;
	if (nx == 0 || ny == 0 || nz == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_fill: empty grid");
	if (ny > 65535 || (vp->gen_mode != TW_MGEN_SINE && nx > 65535)) return tw_set_error(ctx, TW_ERR_ARG, "tw_voxel_fill: nx/ny > 65535 not supported");
	VoxEpilogue E;
	E.zscale = vp->zscale; E.normalize = vp->normalize_to_1;
	E.atten_mode = vp->atten_mode; E.atten_val = vp->atten_val; E.inner_radius = vp->atten_inner_radius;
	E.nx = nx; E.ny = ny; E.nz = nz;
	if (vp->gen_mode == TW_MGEN_SINE) {
		unsigned const xp = (nx + 31) & ~31u, yp = (ny + 31) & ~31u, zp = (nz + 31) & ~31u;
		size_t const tab_bytes = (size_t)NS*(xp + yp + zp)*sizeof(float) + TW_N3D_RDATA*sizeof(float);
		int rc = tw_reserve(ctx, 1, tab_bytes);
		if (rc) return rc;
		float *xt = (float *)ctx->d_scratch[1], *yt = xt + (size_t)NS*xp, *zt = yt + (size_t)NS*yp, *d_rdata = zt + (size_t)NS*zp;
		float stack_rdata[TW_N3D_RDATA];
		float *const rdata = h_stage ? (float *)h_stage : stack_rdata;
		if (rdata420) {memcpy(rdata, rdata420, sizeof(stack_rdata));} else {tw_noise3d_gen_sines(vp->rseed1, vp->rseed2, vp->mag, vp->freq, rdata);}
		TW_CUDA(ctx, cudaMemcpyAsync(d_rdata, rdata, sizeof(stack_rdata), cudaMemcpyHostToDevice, ctx->stream));
		if (!h_stage) {TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));} // rdata is a stack buffer
		float const sx = vp->lo_pos[0] + vp->offset[0], sy = vp->lo_pos[1] + vp->offset[1], sz = vp->lo_pos[2] + vp->offset[2]; // (lo_pos + offset), src/voxels.cpp:289
		xyz_tables_kernel<<<3, 64, 0, ctx->stream>>>(xt, yt, zt, xp, yp, zp, nx, ny, nz, sx, sy, sz, vp->vsz[0], vp->vsz[1], vp->vsz[2], d_rdata, ctx->d_sin_table);
		TW_LAUNCH_CHECK(ctx);
		dim3 const grid((nz + VZ - 1)/VZ, (nx + VXB - 1)/VXB, ny);
		voxel_sine_kernel<<<grid, VZ, 0, ctx->stream>>>(d_out, xt, yt, zt, xp, yp, zp, E);
		TW_LAUNCH_CHECK(ctx);
		return TW_OK;
	}
	GlmParams G;
	for (int d = 0; d < 3; ++d) {G.lo[d] = vp->lo_pos[d]; G.vsz[d] = vp->vsz[d]; G.off[d] = vp->offset[d];}
	G.mag = vp->mag; G.nfreq0 = (float)(0.25*vp->freq);
	G.rx = vp->rx; G.ry = vp->ry; G.rz = vp->rx - vp->ry;
	G.octaves = vp->octaves; G.perlin = (vp->gen_mode == TW_MGEN_PERLIN);
	{int const rc = twi_ensure_glm3_lut(ctx); if (rc) return rc;}
	unsigned const bz = (nz > 128) ? 256 : 128;
	dim3 const grid((nz + bz - 1)/bz, (nx + VGX - 1)/VGX, ny);
	size_t const lut_bytes = (size_t)twn2::LUT3D_N*twn2::SIMPLEX_LUT_COPIES*sizeof(float4);
	if (G.perlin) {cudaFuncSetAttribute(voxel_glm_kernel<true >, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes);} // > 48 KB opt-in, per launch (any device)
	else          {cudaFuncSetAttribute(voxel_glm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes);}
	if (G.perlin) {voxel_glm_kernel<true ><<<grid, bz, lut_bytes, ctx->stream>>>(d_out, G, E, (const float4 *)ctx->d_glm3_lut + twn2::LUT3D_N);}
	else          {voxel_glm_kernel<false><<<grid, bz, lut_bytes, ctx->stream>>>(d_out, G, E, (const float4 *)ctx->d_glm3_lut);}
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
