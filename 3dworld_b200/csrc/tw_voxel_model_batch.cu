// tw_voxel_model_batch.cu - many small voxel models built or edited in one job (tw_voxel_model_build_batch_launch / tw_voxel_model_edit_batch_launch). Built
// as its own sm_90a module (build.py: tw_voxel_model_batch.cubin beside the library) that tw_voxel_post.cu loads on first use, so the library's own kernels -
// whose code the tests pin - stay exactly as they are. The fill, the outside flags and the flood are tw_voxel_batch.cubin's kernels, launched on descriptors
// that point at the models' own memory; the kernels here are the rest of the single-model path (tw_voxel_post.cu), each launched once over every model
// through the table of twi_vmb_model (tw_voxel_model_batch.h), a launch block finding its model by a binary search over the models' first blocks.
//   tw_vmb_copy_kernel          per voxel: the input field into raw, raw into post (build) or into work (edit of a flooded model)
//   tw_vmb_box_scatter_kernel   box_scatter_kernel / tw_box_scatter_bits_kernel of each model's boxes
//   tw_vmb_diff_kernel          diff_kernel / tw_diff_bits_kernel of each flooded model
//   tw_vmb_change_list_kernel   the change list of each model that asks for one, one CTA per model
//   tw_vmb_list_marked_kernel   list_marked_kernel, one CTA per model
//   tw_vmb_mesh_count_kernel / tw_vmb_mesh_scan_kernel / tw_vmb_mesh_emit_kernel   block_mesh_kernel's count, the scans of the model's launch blocks with
//                               block_table_kernel (one CTA per model), and the emit
#include "tw_voxel_model_batch.h"
#include "tw_voxel_batch_util.cuh"

namespace {
// value t of an edit's packed values (box_scatter's loop body, tw_voxel_edit.cuh; kept apart so the library's box_scatter_kernel keeps its SASS): into the
// raw field with its raw flags unless a later box overwrites the voxel; post (rm == 0): also compared with the model's field and flags, which take the new
// value, marking the blocks that read a changed voxel, with BITS also setting its change bit
template<bool BITS>
__device__ __forceinline__ void box_voxel(const twi_box *__restrict__ boxes, unsigned nboxes, const float *__restrict__ values, unsigned long long t,
	const tw_voxel_post_params &P, const unsigned *__restrict__ zix_xy, const BlockGrid &G, float *__restrict__ raw, unsigned char *__restrict__ raw_o, float *post,
	unsigned char *post_o, unsigned char *mark, unsigned *bits)
{
	unsigned lo = 0, hi = nboxes - 1;
	while (lo < hi) {unsigned const mid = (lo + hi + 1) >> 1; if (boxes[mid].off <= t) lo = mid; else hi = mid - 1;}
	twi_box const B = boxes[lo];
	unsigned long long const r = t - B.off, xy = r / B.d;
	unsigned const z = B.z + (unsigned)(r - xy*B.d), x = B.x + (unsigned)(xy % B.w), y = B.y + (unsigned)(xy / B.w);
	bool overwritten = false;
	for (unsigned k = lo + 1; B.later && k < nboxes && !overwritten; ++k) {
		twi_box const &C = boxes[k];
		overwritten = (x - C.x < C.w && y - C.y < C.h && z - C.z < C.d);
	}
	if (overwritten) return;
	size_t const i = z + ((size_t)x + (size_t)y*P.nx)*P.nz;
	float const val = values[t];
	unsigned char const o = outside_flag(val, i, x, y, z, P, zix_xy);
	raw[i] = val; raw_o[i] = o;
	if (post && (__float_as_uint(post[i]) != __float_as_uint(val) || post_o[i] != o)) {
		post[i] = val; post_o[i] = o; mark_readers(mark, P, G, x, y);
		if (BITS) {atomicOr(bits + (i >> 5), 1u << (i & 31));} // a box row need not start on a word
	}
}

__device__ __forceinline__ unsigned vox_model(const twi_vmb_model *m, unsigned nm) {return find_grid(m, nm, blockIdx.x, [](const twi_vmb_model &d) {return d.vox_blk0;});}
} // namespace

// what (TWI_VMB_COPY_*): the models with an input field, every model, or the flooded models; a warp's 32 lanes copy 32 consecutive voxels
extern "C" __global__ void __launch_bounds__(TWI_VMB_VOX_THREADS) tw_vmb_copy_kernel(const twi_vmb_model *__restrict__ models, unsigned nmodels, int what) {
	twi_vmb_model const &m = models[vox_model(models, nmodels)];
	if ((what == TWI_VMB_COPY_IN && !m.in) || (what == TWI_VMB_COPY_WORK && !m.flood)) return;
	unsigned const i0 = (blockIdx.x - m.vox_blk0)*TWI_VMB_VOX_PER_BLOCK, i1 = min(m.n, i0 + TWI_VMB_VOX_PER_BLOCK);
	for (unsigned i = i0 + threadIdx.x; i < i1; i += TWI_VMB_VOX_THREADS) {
		if (what == TWI_VMB_COPY_IN) {m.raw[i] = m.in[i]; continue;}
		float *const dv = (what == TWI_VMB_COPY_POST) ? m.post : m.work;
		unsigned char *const doo = (what == TWI_VMB_COPY_POST) ? m.post_o : m.work_o;
		dv[i] = m.raw[i]; doo[i] = m.raw_o[i];
	}
}

// Each model's boxes: value t of the model is box_voxel's t. A flooded model's scatter writes the raw field only; the others' also compare with the model's
// field (rm == 0, where it is the raw one), with the change bits when the model has a list (zeroed before).
extern "C" __global__ void __launch_bounds__(TWI_VMB_BOX_THREADS) tw_vmb_box_scatter_kernel(const twi_vmb_model *__restrict__ models, unsigned nmodels) {
	twi_vmb_model const &m = models[find_grid(models, nmodels, blockIdx.x, [](const twi_vmb_model &d) {return d.box_blk0;})];
	unsigned long long const t0 = (unsigned long long)(blockIdx.x - m.box_blk0)*TWI_VMB_BOX_PER_BLOCK;
	unsigned long long const t1 = min(m.total, t0 + TWI_VMB_BOX_PER_BLOCK);
	bool const rm = (m.P.remove_unconnected > 0);
	float *const post = rm ? nullptr : m.post;
	unsigned char *const post_o = rm ? nullptr : m.post_o;
	for (unsigned long long t = t0 + threadIdx.x; t < t1; t += TWI_VMB_BOX_THREADS) {
		if (m.bits && !rm) {box_voxel<true>(m.boxes, m.nboxes, m.values, t, m.P, m.zix, m.G, m.raw, m.raw_o, post, post_o, m.mark, m.bits);}
		else               {box_voxel<false>(m.boxes, m.nboxes, m.values, t, m.P, m.zix, m.G, m.raw, m.raw_o, post, post_o, m.mark, nullptr);}
	}
}

// A flooded model's field and flags (post, post_o) take the flood's (work, work_o) where they differ, marking the blocks that read a changed voxel; with a
// list, every word of the bits is written from one ballot per warp (a block's voxels start on a word)
extern "C" __global__ void __launch_bounds__(TWI_VMB_VOX_THREADS) tw_vmb_diff_kernel(const twi_vmb_model *__restrict__ models, unsigned nmodels) {
	twi_vmb_model const &m = models[vox_model(models, nmodels)];
	if (!m.flood) return;
	unsigned const i0 = (blockIdx.x - m.vox_blk0)*TWI_VMB_VOX_PER_BLOCK, i1 = min((m.n + 31) & ~31u, i0 + TWI_VMB_VOX_PER_BLOCK);
	tw_voxel_post_params const &P = m.P;
	for (unsigned i = i0 + threadIdx.x; i < i1; i += TWI_VMB_VOX_THREADS) { // uniform over the warp
		bool changed = false;
		if (i < m.n) {
			float const v = m.work[i];
			unsigned char const o = m.work_o[i];
			changed = (__float_as_uint(v) != __float_as_uint(m.post[i]) || o != m.post_o[i]);
			if (changed) {
				m.post[i] = v; m.post_o[i] = o;
				unsigned const xy = i / P.nz;
				mark_readers(m.mark, P, m.G, xy % P.nx, xy / P.nx);
			}
		}
		unsigned const word = __ballot_sync(0xffffffffu, changed);
		if (m.bits && (threadIdx.x & 31) == 0) {m.bits[i >> 5] = word;}
	}
}

namespace {
// exclusive scan of v over the CTA (1024 threads) after carry, which then holds the running total; warp_sums: 33 words of shared memory
__device__ __forceinline__ unsigned cta_scan(unsigned v, unsigned &carry, unsigned *warp_sums) {
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = v;
	for (int o = 1; o < 32; o <<= 1) {unsigned const u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += u;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned w = warp_sums[lane], wi = w;
		for (int o = 1; o < 32; o <<= 1) {unsigned const u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += u;}
		warp_sums[lane] = wi - w;
		if (lane == 31) {warp_sums[32] = wi;}
	}
	__syncthreads();
	unsigned const excl = carry + warp_sums[warp] + (incl - v);
	carry += warp_sums[32];
	__syncthreads(); // warp_sums is reused by the next call
	return excl;
}
} // namespace

// One CTA per model with a list: the voxels whose bits are set, in ascending index order - index, and the new value and flags when asked - the first ch_cap
// of them written; counts[4] = their number
extern "C" __global__ void __launch_bounds__(1024) tw_vmb_change_list_kernel(const twi_vmb_model *__restrict__ models) {
	twi_vmb_model const &m = models[blockIdx.x];
	if (!m.bits) return;
	__shared__ unsigned warp_sums[33];
	unsigned carry = 0;
	for (unsigned base = 0; base < m.nwords; base += 1024) {
		unsigned const w = base + threadIdx.x;
		unsigned word = (w < m.nwords) ? m.bits[w] : 0u;
		unsigned long long slot = cta_scan(__popc(word), carry, warp_sums);
		for (; word && slot < m.ch_cap; word &= word - 1, ++slot) {
			unsigned const i = w*32 + (unsigned)(__ffs(word) - 1);
			m.ch_index[slot] = i;
			if (m.ch_vals) {m.ch_vals[slot] = m.post[i];}
			if (m.ch_outside) {m.ch_outside[slot] = m.post_o[i];}
		}
	}
	if (threadIdx.x == 0) {m.counts[4] = carry;}
}

// One CTA per model: list = {count, the marked blocks in ascending order}; clears the marks
extern "C" __global__ void __launch_bounds__(1024) tw_vmb_list_marked_kernel(const twi_vmb_model *__restrict__ models) {
	twi_vmb_model const &m = models[blockIdx.x];
	__shared__ unsigned warp_sums[33];
	unsigned carry = 0;
	for (unsigned base = 0; base < m.nblocks; base += 1024) {
		unsigned const i = base + threadIdx.x;
		bool const f = (i < m.nblocks) && m.mark[i];
		if (f) {m.mark[i] = 0;}
		unsigned const s = cta_scan(f ? 1u : 0u, carry, warp_sums);
		if (f) {m.list[1 + s] = i;}
	}
	if (threadIdx.x == 0) {m.list[0] = carry;}
}

// ---- the welded mesh of each model's listed blocks: block_mesh_kernel (tw_voxel_post.cu) over (model, list slot, chunk) ----
namespace {
__device__ __forceinline__ CubeRange block_range(const tw_voxel_post_params &P, const BlockGrid &G, unsigned b) {
	CubeRange R;
	R.x0 = (b % G.nbx)*G.bx; R.y0 = (b / G.nbx)*G.by;
	R.x1 = min(R.x0 + G.bx, P.nx - 1); R.y1 = min(R.y0 + G.by, P.ny - 1);
	return R;
}

// launch block k of model m (k = slot*chunks + chunk): count (EMIT false) stores the per-cube words and the launch block's sums at vsums[k] / tsums[k];
// emit writes its vertices and triangles from voff[k] / toff[k], nothing at or past vcap / tcap
template<bool EMIT>
__device__ __forceinline__ void mesh_block(const twi_vmb_model &m, unsigned k) {
	tw_voxel_post_params const &P = m.P;
	BlockGrid const &G = m.G;
	unsigned const slot = k / G.chunks;
	if (slot >= __ldg(m.list)) { // not listed: nothing to count (the scans read zeros), nothing to emit
		if (!EMIT && threadIdx.x == 0) {m.vsums[k] = 0; m.tsums[k] = 0;}
		return;
	}
	__shared__ unsigned warp_sums[MC_BLOCK/32];
	__shared__ unsigned char s_edge[12], s_look[12];
	mesh_edge_tables(m.T.edge_to_vals, s_edge, s_look);
	CubeRange const R = block_range(P, G, __ldg(m.list + 1 + slot));
	unsigned const w = R.x1 - R.x0, ncubes = (R.y1 - R.y0)*w*P.nz;
	unsigned const l = (k - slot*G.chunks)*MC_BLOCK + threadIdx.x;
	MeshCube c;
	c.mask = 0;
	unsigned cnt = 0;
	if (l < ncubes) {
		unsigned const xy = l / P.nz;
		unsigned const nt = cube_mesh<EMIT, true>(m.post, m.post_o, P, m.T, s_edge, s_look, R.x0 + xy % w, R.y0 + xy / w, l - xy*P.nz, l, c, R);
		cnt = ((unsigned)__popc(c.mask) << 16) | nt;
	}
	unsigned const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += v;}
	if (lane == 31) {warp_sums[warp] = incl;}
	__syncthreads();
	if (warp == 0) {
		unsigned ws = warp_sums[lane], wi = ws;
		for (int o = 1; o < 32; o <<= 1) {unsigned const v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (unsigned)o) wi += v;}
		warp_sums[lane] = wi - ws;
		if (!EMIT && lane == 31) {m.vsums[k] = wi >> 16; m.tsums[k] = wi & 0xffffu;}
	}
	__syncthreads();
	unsigned const excl = warp_sums[warp] + (incl - cnt);
	unsigned *const bw = m.words + (size_t)slot*G.chunks*MC_BLOCK;
	if (!EMIT) {
		if (l < ncubes) {bw[l] = (excl & 0xffff0000u) | c.mask;}
		return;
	}
	if (l >= ncubes) return;
	const unsigned long long *const bvoff = m.voff + (size_t)slot*G.chunks;
	unsigned long long const vbase = m.voff[k] + (excl >> 16);
	for (unsigned mk = c.mask; mk; mk &= mk - 1) {
		unsigned const e = __ffs(mk) - 1;
		unsigned long long const s = vbase + __popc(c.mask & ((1u << e) - 1));
		if (s < m.vcap) {float *o = m.verts + 3*s; o[0] = c.vlist[e][0]; o[1] = c.vlist[e][1]; o[2] = c.vlist[e][2];}
	}
	unsigned long long const tbase = m.toff[k] + (excl & 0xffffu);
	for (unsigned t = 0; t < (cnt & 0xffffu); ++t) {
		unsigned long long const s = tbase + t;
		if (s >= m.tcap) break;
		for (unsigned v = 0; v < 3; ++v) {
			unsigned const e = c.tri[t][v], owner = c.own[e], ow = bw[owner];
			m.indices[3*s + v] = (uint32_t)(bvoff[owner / MC_BLOCK] - bvoff[0] + (ow >> 16) + __popc(ow & 0xfffu & ((1u << c.oj[e]) - 1)));
		}
	}
}
__device__ __forceinline__ unsigned mesh_model(const twi_vmb_model *m, unsigned nm) {return find_grid(m, nm, blockIdx.x, [](const twi_vmb_model &d) {return d.mesh_blk0;});}
} // namespace

extern "C" __global__ void __launch_bounds__(MC_BLOCK) tw_vmb_mesh_count_kernel(const twi_vmb_model *__restrict__ models, unsigned nmodels) {
	twi_vmb_model const &m = models[mesh_model(models, nmodels)];
	mesh_block<false>(m, blockIdx.x - m.mesh_blk0);
}

// One CTA per model: voff / toff of its launch blocks, the table of its listed blocks (block_table_kernel), counts[0, 1, 3] = its vertices, triangles and
// listed blocks
extern "C" __global__ void __launch_bounds__(1024) tw_vmb_mesh_scan_kernel(const twi_vmb_model *__restrict__ models) {
	twi_vmb_model const &m = models[blockIdx.x];
	if (m.nblocks == 0) return; // no cube: the counts stay 0
	unsigned const ng = m.nblocks*m.G.chunks, chunks = m.G.chunks;
	unsigned long long const nv = scan_sums(m.vsums, ng, m.voff), nt = scan_sums(m.tsums, ng, m.toff);
	unsigned const listed = __ldg(m.list);
	for (unsigned s = threadIdx.x; s < listed; s += 1024) {
		size_t const a = (size_t)s*chunks, b = a + chunks;
		unsigned long long const v1 = (s + 1 < m.nblocks) ? m.voff[b] : nv, t1 = (s + 1 < m.nblocks) ? m.toff[b] : nt;
		tw_voxel_block_mesh e;
		e.block = m.list[1 + s]; e.pad = 0; e.voff = m.voff[a]; e.nverts = v1 - m.voff[a]; e.toff = m.toff[a]; e.ntris = t1 - m.toff[a];
		m.table[s] = e;
	}
	if (threadIdx.x == 0) {m.counts[0] = nv; m.counts[1] = nt; m.counts[3] = listed;}
}

// models without capacities write nothing, as the single job launches no emit pass for them
extern "C" __global__ void __launch_bounds__(MC_BLOCK) tw_vmb_mesh_emit_kernel(const twi_vmb_model *__restrict__ models, unsigned nmodels) {
	twi_vmb_model const &m = models[mesh_model(models, nmodels)];
	if (m.vcap == 0 && m.tcap == 0) return;
	mesh_block<true>(m, blockIdx.x - m.mesh_blk0);
}
