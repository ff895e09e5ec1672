// tw_voxel_model_batch.h - one voxel model of a model batch (tw_voxel_model_build_batch_launch / tw_voxel_model_edit_batch_launch) as the kernels of
// tw_voxel_model_batch.cu read it: tw_voxel_post.cu builds a table of these in pinned staging and copies it to the device with the batch's other inputs,
// and every kernel walks all models through it, so a batch's kernel count does not depend on its size. Every pointer is the model's own memory or the
// launching context's scratch.
#pragma once
#include "tw_voxel_edit.cuh"
#include "tw_voxel_mc.cuh"

constexpr unsigned TWI_VMB_VOX_THREADS = 256, TWI_VMB_VOX_PER_BLOCK = 2048;  // the per-voxel kernels: 8 consecutive-warp voxels per thread
constexpr unsigned TWI_VMB_BOX_THREADS = 256, TWI_VMB_BOX_PER_BLOCK = 1024;  // the box scatter: 4 box voxels per thread
// what the per-voxel copy does (tw_vmb_copy_kernel): the input field into raw, raw into post (build), raw into work (edit of a flooded model)
enum {TWI_VMB_COPY_IN = 0, TWI_VMB_COPY_POST = 1, TWI_VMB_COPY_WORK = 2};

struct twi_vmb_model {
	tw_voxel_post_params P;
	BlockGrid G; McTables T;                          // the model's blocks and its marching-cubes tables
	unsigned n, nblocks;                              // voxels, blocks
	unsigned vox_blk0, box_blk0, mesh_blk0;           // the model's first block of the per-voxel, box and mesh launches (prefix sums)
	int flood;                                        // an edit with boxes and remove_unconnected > 0: raw -> work, the flood on work, work diffed into post
	float *raw, *post, *work; unsigned char *raw_o, *post_o, *work_o, *mark;
	const unsigned *zix;                              // zix_xy on the device, or nullptr
	const float *in;                                  // a build from vals: the field as the device reads it (nullptr: a fill)
	unsigned *list;                                   // the blocks to mesh, {count, blocks...}: every block (build) or the marked ones (edit, written by the job)
	const twi_box *boxes; const float *values;        // an edit's boxes and packed values (scratch)
	unsigned nboxes; unsigned long long total;        // and its voxel count
	unsigned *bits; unsigned nwords;                  // the change list's bits (nullptr: no list)
	unsigned *words, *vsums, *tsums;                  // the mesh's per-cube words (slots x chunks x MC_BLOCK) and per launch block sums
	unsigned long long *voff, *toff;                  // and offsets within the model's outputs
	float *verts; unsigned long long vcap;            // the caller's outputs as the device addresses them
	uint32_t *indices; unsigned long long tcap;
	tw_voxel_block_mesh *table;                       // the listed blocks' table (scratch, copied back with the counts)
	uint32_t *ch_index; float *ch_vals; uint8_t *ch_outside; unsigned long long ch_cap; // the change list's outputs
	unsigned long long *counts;                       // [vertices, triangles, voxels flipped, blocks listed, voxels changed], zeroed before the job
};

// The module's kernels (tw_voxel_model_batch.cu), declared once for the module's definitions and the host's launches (tw_voxel_post.cu)
extern "C" __global__ void tw_vmb_copy_kernel(const twi_vmb_model *models, unsigned nmodels, int what);
extern "C" __global__ void tw_vmb_box_scatter_kernel(const twi_vmb_model *models, unsigned nmodels);
extern "C" __global__ void tw_vmb_diff_kernel(const twi_vmb_model *models, unsigned nmodels);
extern "C" __global__ void tw_vmb_change_list_kernel(const twi_vmb_model *models);
extern "C" __global__ void tw_vmb_list_marked_kernel(const twi_vmb_model *models);
extern "C" __global__ void tw_vmb_mesh_count_kernel(const twi_vmb_model *models, unsigned nmodels);
extern "C" __global__ void tw_vmb_mesh_scan_kernel(const twi_vmb_model *models);
extern "C" __global__ void tw_vmb_mesh_emit_kernel(const twi_vmb_model *models, unsigned nmodels);
