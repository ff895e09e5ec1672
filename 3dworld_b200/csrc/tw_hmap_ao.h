// tw_hmap_ao.h - the launch record of the heightmap-tile AO kernel (tw_hmap_ao.cu, module tw_hmap_ao.cubin), shared by the module and the host code that
// launches it (tw_api.cu, tw_hmap_tile_ao_launch), so both see one layout
#pragma once
#include <stdint.h>
#include "../../include/tw3d.h"

// One CTA per (tile, sub-square of side `side`): tile t = blockIdx.x / (nsub*nsub). Tile t's zvals are zvsize^2 floats at zvals + s*zvsize^2 with
// s = slots ? slots[t] : t (a tile set's slab, or the caller's array); its origin is (origins[2t], origins[2t + 1]); its stride^2 AO bytes go to
// ao + t*stride^2. img is the context's 16-bit image, sampled under H outside the tile.
struct twi_hmap_ao_args {
	const uint8_t *img;
	const int32_t *origins;
	const float *zvals;
	const int *slots;
	unsigned char *ao;
	tw_hmap_sampler H;
	unsigned zvsize, side, nsub;
	float dz;                 // 0.5*half_dxy, the ray's z step (tile_ao_kernel's)
};
constexpr int TWI_AO_RAY_LEN = 36;          // AO_RAY_LEN: 8 steps of growing stride, 1 + 2 + ... + 8 cells
constexpr unsigned TWI_AO_MAX_SIDE = 160;   // (160 + 72)^2 floats = 210.25 KB of shared memory, inside sm_90a's 227 KB opt-in
constexpr unsigned TWI_AO_THREADS = 1024;
