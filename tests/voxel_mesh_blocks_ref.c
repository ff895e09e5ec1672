/* voxel_mesh_blocks_ref.c - the welded mesh of tests/voxel_mesh_ref.c per block, as a voxel model keeps one mesh and one vertex cache per block
 * (voxel_model::create_block, src/voxels.cpp:1077-1108): the reference that tests/test_voxel_model_host.py, tests/test_gpu_voxel_model.py and
 * tools/bench_voxel_edit.py hold the tw_voxel_model_* block meshes to. The cube loop is voxel_mesh_ref.c's, run over one block's cubes at a time with the
 * cache cleared at each block's start. Built by tests/voxel_mesh_blocks_ref.py with -ffp-contract=off. */
#include "tw3d.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

static inline float std_min(float a, float b) {return (b < a) ? b : a;} /* std::min */
static inline float std_max(float a, float b) {return (a < b) ? b : a;} /* std::max */
/* interpolate_pt, ref: :485-493 */
static void interpolate_pt(float isolevel, const float *pt1, const float *pt2, float val1, float val2, float *pt) {
	float const TOLERANCE = 1.0E-12f;
	if (fabsf(isolevel - val1) < TOLERANCE) {pt[0] = pt1[0]; pt[1] = pt1[1]; pt[2] = pt1[2]; return;}
	if (fabsf(isolevel - val2) < TOLERANCE) {pt[0] = pt2[0]; pt[1] = pt2[1]; pt[2] = pt2[2]; return;}
	if (fabsf(val1     - val2) < TOLERANCE) {pt[0] = pt1[0]; pt[1] = pt1[1]; pt[2] = pt1[2]; return;}
	float const mu = std_max(0.0f, std_min(1.0f, (isolevel - val1)/(val2 - val1))); /* CLIP_TO_01 */
	for (int i = 0; i < 3; ++i) {pt[i] = pt1[i] + mu*(pt2[i] - pt1[i]);}
}

/* The welded mesh: the loop of to_voxel_triangles, but the vertices go through a cache as in create_block - a cube looks each crossing edge up (grid
 * point of its low end, axis) and, on a miss, interpolates it with its own corners in its own edge_to_vals order and appends it. The cache holds two
 * layers of grid points in y: a cube of row y touches the edges at y and y + 1, so the slot of y + 1 is cleared when row y starts.
 * Per block (bx, by >= 1 cubes): block (i, j) = the cubes x in [i*bx, min((i+1)*bx, nx-1)), y in [j*by, min((j+1)*by, ny-1)), every z, numbered j*nbx + i;
 * each block is welded with a cache of its own, its vertices and indices local to it and appended block after block. table (optional) gets
 * {block, voff, nverts, toff, ntris} per block as 5 uint64 (voff / toff: the block's first vertex / triangle in the whole output). One block covering
 * the grid is the mesh of voxel_mesh_ref.c's ref_voxel_mesh. */
void ref_voxel_mesh_blocks(const float *vals, const unsigned char *outside, const tw_voxel_post_params *vp, const unsigned *edge_table, const int *tri_table,
                          const unsigned *edge_to_vals, unsigned bx, unsigned by, float *verts, unsigned long long vcap, unsigned *indices,
                          unsigned long long tcap, unsigned long long *table, unsigned long long *nverts, unsigned long long *ntris)
{
	unsigned const nx = vp->nx, ny = vp->ny, nz = vp->nz;
	size_t const layer = (size_t)nx*nz*3;
	unsigned *cache = (unsigned *)malloc(2*layer*sizeof(unsigned));
	memset(cache, 0xff, 2*layer*sizeof(unsigned));
	unsigned long long nv = 0, nt = 0, vmax = 0;
	float *pos = NULL; /* every vertex: the triangle test needs positions past vcap */
	unsigned const ncx = (nx > 1) ? nx - 1 : 0, ncy = (ny > 1) ? ny - 1 : 0, nbx = (ncx + bx - 1)/bx, nby = (ncy + by - 1)/by;
	for (unsigned b = 0; b < nbx*nby; ++b) {
		unsigned const x0 = (b % nbx)*bx, y0 = (b / nbx)*by, x1 = (x0 + bx < ncx) ? x0 + bx : ncx, y1 = (y0 + by < ncy) ? y0 + by : ncy;
		unsigned long long const nv0 = nv, nt0 = nt;
		memset(cache, 0xff, 2*layer*sizeof(unsigned));
		for (unsigned y = y0; y < y1; ++y) {
			memset(cache + ((y + 1) & 1)*layer, 0xff, layer*sizeof(unsigned));
			for (unsigned x = x0; x < x1; ++x) {
				for (unsigned z = 0; z < nz; ++z) {
					unsigned const x2 = (x+1 < nx-1) ? x+1 : nx-1, y2 = (y+1 < ny-1) ? y+1 : ny-1, z2 = (z+1 < nz-1) ? z+1 : nz-1;
					unsigned const xv[2] = {x, x2}, yv[2] = {y, y2}, zv[2] = {z, z2};
					if (x2 <= x || y2 <= y || z2 <= z) continue;
					unsigned cix = 0;
					int all_under_mesh = (vp->skip_under_mesh != 0);
					for (unsigned yhi = 0; yhi < 2; ++yhi) {
						for (unsigned xhi = 0; xhi < 2; ++xhi) {
							size_t const ix = z + ((size_t)xv[xhi] + (size_t)yv[yhi]*nx)*nz;
							if (all_under_mesh) {all_under_mesh = ((outside[ix] & TW_VOX_UNDER_MESH) != 0);}
							for (unsigned zhi = 0; zhi < 2; ++zhi) {if (outside[ix + zv[zhi]-z] & 7) {cix |= 1u << ((xhi^yhi) + 2*yhi + 4*zhi);}}
						}
					}
					if (all_under_mesh) continue;
					unsigned const edge_val = edge_table[cix];
					if (edge_val == 0) continue;
					const int *t = tri_table + 16*cix;
					float const cube[3][2] = {{x*vp->vsz[0] + vp->lo_pos[0], x2*vp->vsz[0] + vp->lo_pos[0]}, {y*vp->vsz[1] + vp->lo_pos[1], y2*vp->vsz[1] + vp->lo_pos[1]},
					                          {z*vp->vsz[2] + vp->lo_pos[2], z2*vp->vsz[2] + vp->lo_pos[2]}};
					unsigned vix[12];
					for (unsigned i = 0; i < 12; ++i) {
						if (!(edge_val & (1u << i))) continue;
						unsigned hi[2][3];
						for (unsigned d = 0; d < 2; ++d) {
							unsigned const e = edge_to_vals[2*i + d];
							hi[d][1] = (e & 2) >> 1; hi[d][0] = hi[d][1] ^ (e & 1); hi[d][2] = e >> 2;
						}
						unsigned const axis = (hi[0][0] != hi[1][0]) ? 0 : ((hi[0][1] != hi[1][1]) ? 1 : 2);
						unsigned lo[3];
						for (unsigned k = 0; k < 3; ++k) {lo[k] = (hi[0][k] < hi[1][k]) ? hi[0][k] : hi[1][k];}
						unsigned const gy = y + lo[1];
						unsigned *slot = cache + (gy & 1)*layer + ((size_t)(x + lo[0])*nz + z + lo[2])*3 + axis;
						if (*slot == 0xffffffffu) {
							float v2[2], pts[2][3], p[3];
							for (unsigned d = 0; d < 2; ++d) {
								size_t const ix = zv[hi[d][2]] + ((size_t)xv[hi[d][0]] + (size_t)yv[hi[d][1]]*nx)*nz;
								v2[d] = ((outside[ix] & 7) == TW_VOX_ON_EDGE) ? vp->isolevel : vals[ix];
								pts[d][0] = cube[0][hi[d][0]]; pts[d][1] = cube[1][hi[d][1]]; pts[d][2] = cube[2][hi[d][2]];
							}
							interpolate_pt(vp->isolevel, pts[0], pts[1], v2[0], v2[1], p);
							if (nv == vmax) {vmax = vmax ? 2*vmax : 4096; pos = (float *)realloc(pos, vmax*3*sizeof(float));}
							memcpy(pos + 3*nv, p, sizeof(p));
							*slot = (unsigned)(nv++ - nv0);
						}
						vix[i] = *slot + (unsigned)nv0;
					}
					for (unsigned i = 0; t[i] >= 0; i += 3) { /* the reference's get_normal on the cached points */
						const float *p0 = pos + 3*(size_t)vix[t[i]], *p1 = pos + 3*(size_t)vix[t[i+1]], *p2 = pos + 3*(size_t)vix[t[i+2]];
						float const a[3] = {p1[0]-p0[0], p1[1]-p0[1], p1[2]-p0[2]}, b[3] = {p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2]};
						float const cx = a[1]*b[2] - a[2]*b[1], cy = a[2]*b[0] - a[0]*b[2], cz = a[0]*b[1] - a[1]*b[0];
						if (cx == 0.0f && cy == 0.0f && cz == 0.0f) continue;
						if (nt < tcap) {for (unsigned k = 0; k < 3; ++k) {indices[3*nt + k] = vix[t[i+k]] - (unsigned)nv0;}}
						++nt;
					}
				}
			}
		}
		if (table) {unsigned long long *r = table + 5*(size_t)b; r[0] = b; r[1] = nv0; r[2] = nv - nv0; r[3] = nt0; r[4] = nt - nt0;}
	}
	if (vcap) {memcpy(verts, pos, 3*sizeof(float)*(size_t)(nv < vcap ? nv : vcap));}
	free(pos);
	free(cache);
	*nverts = nv; *ntris = nt;
}

