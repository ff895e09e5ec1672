// tw_voxel_batch.h - one grid of a voxel batch (tw_voxel_build_batch_launch) as the batch module's kernels read it: tw_voxel_post.cu builds a table of these
// in pinned staging and copies it to the device, and every kernel of tw_voxel_batch.cu walks all grids through it, so a batch's kernel count does not
// depend on its size.
#pragma once
#include "tw_voxel_fill.cuh"
#include "tw_voxel_mc.cuh"

// the fill of a grid: none (vals holds the input field), the sine sum, or GLM fBm
enum {TWI_VB_INPUT = 0, TWI_VB_SINE = 1, TWI_VB_SIMPLEX = 2, TWI_VB_PERLIN = 3};
constexpr unsigned TWI_VB_FILL_THREADS = 256, TWI_VB_FILL_VOXELS = 8192;    // a fill block: 32 voxels per thread, consecutive indices
constexpr unsigned TWI_VB_MAX_VOXELS = 1u << 18;                            // per grid: the flood's six bitsets fill 192 KB of one SM's shared memory
constexpr unsigned TWI_VB_FLOOD_THREADS = 1024;

struct twi_vbatch_grid {
	tw_voxel_post_params P;
	VoxEpilogue E; GlmParams G;                      // the fill's epilogue and GLM parameters
	int mode;                                        // TWI_VB_*
	unsigned n;                                      // nx*ny*nz <= TWI_VB_MAX_VOXELS
	unsigned fill_blk0, mesh_blk0;                   // the grid's first block of the fill / mesh launches (prefix sums over the grids before it)
	float *vals; unsigned char *flags;               // the field (the caller's device vals, or scratch) and the outside flags
	const unsigned *zix;                             // zix_xy on the device, or nullptr
	float *xt, *yt, *zt; unsigned xp, yp, zp;        // sine mode: the axis tables and their pitches
	float s[3], step[3]; const float *rdata;         // sine mode: lo_pos + offset, vsz, the 420 coefficients on the device
	unsigned *words, *vsums, *tsums;                 // the welded mesh's per-cube words and per-block sums
	unsigned long long *voff, *toff;                 // and the per-block offsets within the grid's mesh
	float *verts; unsigned long long vcap;           // the caller's outputs as the device addresses them
	uint32_t *indices; unsigned long long tcap;
	unsigned long long *counts;                      // [vertices, triangles, voxels flipped by remove_unconnected], zeroed before the batch
};

// The module's kernels (tw_voxel_batch.cu), declared once for the module's definitions and the host's launches (tw_voxel_post.cu)
extern "C" __global__ void tw_vbatch_tables_kernel(const twi_vbatch_grid *grids, const float *sin_tab);
extern "C" __global__ void tw_vbatch_fill_kernel(const twi_vbatch_grid *grids, unsigned ngrids, const float4 *lut);
extern "C" __global__ void tw_vbatch_flood_kernel(const twi_vbatch_grid *grids);
extern "C" __global__ void tw_vbatch_mesh_count_kernel(const twi_vbatch_grid *grids, unsigned ngrids, McTables T);
extern "C" __global__ void tw_vbatch_mesh_scan_kernel(const twi_vbatch_grid *grids);
extern "C" __global__ void tw_vbatch_mesh_emit_kernel(const twi_vbatch_grid *grids, unsigned ngrids, McTables T);
