// tw_erosion.cu - droplet hydraulic erosion (sm_90a). Replaces apply_erosion() (src/erosion.cpp:14-164).
//
// The reference algorithm is a Lagrangian droplet walk: droplet k sees every height written by droplets < k, so one heightmap is a
// serial dependency chain (SURVEY.md section 7 "erosion order dependence"). The parallelism the reference's callers expose is ACROSS
// heightmaps: tile_t::create_zvals erodes every tile independently with the same droplet seeds (src/tiled_mesh.cpp:515). Mapping:
//   pad_kernel      (:31-37)   clamped PAD=4 border copy, fully parallel, coalesced
//   droplet_kernel  (:66-155)  ONE WARP PER HEIGHTMAP, droplets in the reference's serial order. The scalar droplet state is kept
//                              redundantly in all 32 lanes (uniform control flow, no shuffles); the 2x2 bilinear deposit is done by
//                              lanes 0-3 and the 4x4 erode brush by lanes 0-15, one cell each, so a brush costs 4 row-coalesced
//                              read-modify-writes instead of 16 serial ones. Heights live in global memory and are served from L2/L1.
//   unpad_kernel    (:158-162) remove border, clamp to min_zval
// Bit-exactness: IEEE sqrt/div, no FMA contraction (-fmad=false), std::min/max argument order preserved (NaN semantics, SURVEY A.6),
// the random-direction fallback (:84-87) reads cos/sin from a 1e6-entry table built with the HOST libm (rand_float() has only 1e6 values).
#include "tw_internal.h"
#include <cooperative_groups.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

namespace {

constexpr int PAD = 4;

__device__ __forceinline__ float smin(float a, float b) {return (b < a) ? b : a;} // std::min
__device__ __forceinline__ float smax(float a, float b) {return (a < b) ? b : a;} // std::max
__device__ __forceinline__ int clampi(int v, int hi) {return max(min(v, hi), 0);}

struct EParams {
	float erode_amount, wpz_minus_half_dxy, zmin, zrange, relh_adj_tex, clip_hd1;
	float rock_min;   // get_bare_ls_tid(nh) == ROCK_TEX  <=>  nh >= rock_min (see make_eparams); rock_exact == 0: evaluate the reference expression per move
	int   rock_exact;
};

// Also counts, per heightmap, the cells above the ocean-stop level (src/erosion.cpp:98): droplets that start below it die in one move, the
// others walk downhill, so this count predicts the heightmap's total droplet work (correlation 0.95 on the BASELINE terrain) and is used to
// schedule the heaviest heightmaps first (the work per heightmap is heavy-tailed: median 3, mean 26, max > 140 moves per droplet).
// perm (optional): heightmap z of this batch lives at slot perm[z] of `in` (the tile pipeline's schedule order -> caller's tile index)
__global__ void pad_kernel(const float *__restrict__ in, float *__restrict__ out, int xsize, int ysize, int NX, int NY, float work_level, unsigned *__restrict__ work,
	const unsigned *__restrict__ perm = nullptr) {
	int const x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y;
	size_t const tile = blockIdx.z, src_tile = perm ? __ldg(perm + blockIdx.z) : blockIdx.z;
	bool above = false;
	if (x < NX) {
		int const sx = clampi(x - PAD, xsize - 1), sy = clampi(y - PAD, ysize - 1);
		float const v = __ldg(in + src_tile*xsize*ysize + (size_t)sy*xsize + sx);
		out[tile*NX*NY + (size_t)y*NX + x] = v;
		above = !(v < work_level);
	}
	unsigned const n = __popc(__ballot_sync(0xffffffffu, above));
	if (work && n && (threadIdx.x & 31) == 0) {atomicAdd(work + tile, n);}
}

// counting sort of the heightmap indices by descending work estimate (256 bins; order within a bin is irrelevant: heightmaps are independent)
constexpr int WORK_BINS = 256;
__global__ void order_hist_kernel(const unsigned *__restrict__ work, unsigned nt, unsigned max_work, unsigned *__restrict__ hist) {
	unsigned const t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t >= nt) return;
	unsigned const bin = (WORK_BINS - 1) - min((unsigned)(WORK_BINS - 1), (unsigned)(((unsigned long long)work[t]*(WORK_BINS - 1))/max_work));
	atomicAdd(hist + bin, 1u);
}
__global__ void order_scan_kernel(unsigned *__restrict__ hist) { // exclusive prefix sum of 256 bins, one warp
	unsigned const lane = threadIdx.x;
	unsigned v[WORK_BINS/32], sum = 0;
	for (int i = 0; i < WORK_BINS/32; ++i) {v[i] = hist[lane*(WORK_BINS/32) + i]; sum += v[i];}
	unsigned incl = sum;
	for (int o = 1; o < 32; o <<= 1) {unsigned const n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += n;}
	unsigned run = incl - sum;
	for (int i = 0; i < WORK_BINS/32; ++i) {hist[lane*(WORK_BINS/32) + i] = run; run += v[i];}
}
__global__ void order_scatter_kernel(const unsigned *__restrict__ work, unsigned nt, unsigned max_work, unsigned *__restrict__ cursor, unsigned *__restrict__ order) {
	unsigned const t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t >= nt) return;
	unsigned const bin = (WORK_BINS - 1) - min((unsigned)(WORK_BINS - 1), (unsigned)(((unsigned long long)work[t]*(WORK_BINS - 1))/max_work));
	order[atomicAdd(cursor + bin, 1u)] = t;
}

__global__ void unpad_kernel(const float *__restrict__ padded, float *__restrict__ out, int xsize, int ysize, int NX, int NY,
	const float *__restrict__ min_zvals, float min_zval_all, const unsigned *__restrict__ perm = nullptr)
{
	int const x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y;
	size_t const tile = blockIdx.z, dst_tile = perm ? __ldg(perm + blockIdx.z) : blockIdx.z;
	if (x >= xsize) return;
	float const mz = min_zvals ? __ldg(min_zvals + tile) : min_zval_all;
	out[dst_tile*xsize*ysize + (size_t)y*xsize + x] = smax(mz, padded[tile*NX*NY + (size_t)(y + PAD)*NX + x + PAD]);
}

// M_FROZEN in a job: the end of the sweep that starts at droplet it0 (the last sweep of n droplets may be short)
__device__ __forceinline__ unsigned fz_end(unsigned it0, unsigned sweep, unsigned n) {return (n - it0 < sweep) ? n : it0 + sweep;}

// rand_gen_t core (src/rand_gen.h:22-26) in 32-bit: all intermediates fit (Schrage factorisation), states stay in [0, 2^31)
struct Rng {
	int s1, s2;
	__device__ __forceinline__ int rand() {
		if ((s1 = 40014*(s1%53668) - 12211*(s1/53668)) < 0) s1 += 2147483563;
		if ((s2 = 40692*(s2%52774) - 3791 *(s2/52774)) < 0) s2 += 2147483399;
		int r = s1 - s2;
		if (r < 1) r += 2147483562;
		return r;
	}
};

// One heightmap per group of G lanes (G = 1, 2, 4, 8, 16, 32; 32/G heightmaps per warp). The droplet's scalar state is replicated in the
// G lanes of its group (group-uniform control flow, no shuffles); the 4 deposit corners and the 16 brush cells are dealt round-robin to
// the lanes of the group (c = sub, sub+G, ...: ascending c is the reference's z-outer/x-inner order, so G == 1 is literally the serial
// loop). The droplet loop is flattened into one state machine per group (init-droplet / step) so that groups whose droplets end at
// different times stay converged at the top of the loop. G trades redundant ALU work (G = 32: every lane repeats the ~250-instruction
// step for ONE map) against memory coalescing and in-flight parallelism (G = 1: no redundancy, but 32 unrelated maps per load
// instruction and 32x more maps needed to fill the machine); twi_erode picks G from the number of heightmaps.
//
// Where the heights live (MODE):
//   M_GLOBAL  padded copy in global memory, served by L1/L2: the THROUGHPUT mode - thousands of maps in flight hide the two dependent L2
//             round trips of a move; a single map runs at ~0.75 us per move.
//   M_ATOMIC  (tw_erode_parallel) the reference's multi-threaded mode, `#pragma omp parallel for schedule(dynamic,1)` over the droplets of ONE
//             heightmap (src/erosion.cpp:66): `ntiles` groups play the OpenMP threads, each takes the next droplet index from an atomic counter
//             (the dynamic,1 schedule), reads bypass L1 (the CPU's caches are coherent) and the read-modify-writes are float atomics (the
//             reference's are unsynchronised). One group => exactly the serial order.
//   M_WINDOW  LATENCY mode for maps that do not fit on chip (258^2 tiles, the 8192^2 map): each lane group keeps a WX x WY window of the padded
//             map around its droplet in SHARED MEMORY. Reads hit the window (29-cycle LDS instead of a ~250-cycle L2 round trip), writes go
//             through to the window AND to global memory, so the global copy is always current: the window is a pure read cache, any access
//             outside it simply falls back to global memory, and re-centring is a plain re-load (ld.global.cg) ahead of the droplet's heading.
//   M_WHOLE   LATENCY mode for maps that fit on chip (130^2 tiles = 76 KB padded; the reference's default mesh_size 128): the whole padded map
//             is built in shared memory straight from the caller's un-padded tile (the PAD = 4 clamped border, src/erosion.cpp:31-37, is
//             replicated in shared memory), all droplets walk it there, and the interior is written back once with the min_zval clamp
//             (:158-162). No padded scratch copy, no pad/unpad kernels: DRAM traffic = read the tile once + write it once.
//   M_FROZEN  (tw_erode_sweeps*) the coherent batched variant for ONE map sharded over GPUs (SURVEY.md 8e, north_star "halo exchange between erosion
//             sweeps"; no reference counterpart): the droplets of a sweep all read the map as it was at the start of the sweep and accumulate
//             their deposits/erosions into a 64-bit FIXED-POINT delta buffer (2^-40 units, integer atomics: associative, hence independent of
//             thread order AND of how the rows are split over devices); the host adds the deltas to the map between sweeps. A droplet must
//             still see its OWN writes (the walk relies on that feedback: a droplet in a pit fills it and stops - on a frozen map it would
//             bounce for thousands of moves): it keeps a private VIEW x VIEW window in shared memory = sweep-start heights + its own writes,
//             re-read from the sweep-start map (re-centred ahead of its heading, exactly as M_WINDOW does) whenever it walks out of it. A device stores the
//             padded rows [row0, row0 + rows) (its band +- halo), walks only droplets that start in its own rows [own0, own1), and a droplet
//             ends once it is more than halo_rule rows from its start row (so it never leaves the band +- halo) - a rule of the algorithm
//             itself, applied on one GPU too, which makes the sharded result bit-identical to the single-GPU one.
//   M_SPEC    (twi_erode_spec) the reference's SERIAL droplet order on ONE big map, executed speculatively in parallel and committed in order - exact, bit for
//             bit the serial result. A window of B consecutive droplets is in flight. Every droplet is walked by one warp against the COMMITTED map, seeing its
//             own writes through a private view (the M_FROZEN machinery) and keeping what it did to itself: a log of (cell, final value) for the cells it changed
//             and the list of 4x4-cell tiles it touched (read or written). After each round of walks the tiles are stamped with the lowest droplet index that
//             touched them; a droplet CONFLICTS if a lower-indexed droplet of the window touched one of its tiles. The prefix of the window up to the first
//             conflict is committed (the logs are copied into the map: disjoint tiles, so any order), droplets whose tiles were touched by a committed one are
//             walked again against the new map, the window slides. The head of the window never conflicts, so every round commits at least one droplet; on an
//             8192^2 map the first conflict among random droplets sits a few hundred droplets in (birthday bound on ~1e6 tiles). A droplet that outgrows its log
//             / tile list / view count, or whose position becomes non-finite (the reference then reads the map's corner), is walked IN PLACE on the map when it
//             is the head of the window (the plain M_GLOBAL walk of one droplet, alone on the device).
enum {M_GLOBAL = 0, M_ATOMIC = 1, M_WINDOW = 2, M_WHOLE = 3, M_FROZEN = 4, M_SPEC = 5};
enum {SP_EMPTY = 0, SP_DIRTY = 1, SP_VALID = 2, SP_HUGE = 3, SP_INPLACE = 4, SP_WALKING = 5}; // state of a window slot
constexpr unsigned SP_STATE_WORDS = 32; // saved registers of a suspended walk
#ifndef TW_SPEC_TILE_SHIFT
#define TW_SPEC_TILE_SHIFT 2
#endif
constexpr int SP_TILE_SHIFT = TW_SPEC_TILE_SHIFT; // conflict tiles of (1 << shift)^2 cells, >= 4x4 (a move's 4 x 4 footprint then spans at most 2 x 2 tiles)
static_assert(SP_TILE_SHIFT >= 2, "a move may touch at most 2 x 2 tiles");
constexpr unsigned SP_NONE = 0xffffffffu;
constexpr unsigned SP_CTL_ROUND = 16; // ctl word of the round counter: the round kernel advances it, so one graph body serves every round
struct SpecArgs { // M_SPEC: the window of in-flight droplets (slot = droplet index % B)
	unsigned B, W, T, R;            // slots, log entries / tile ids / view segments per slot
	unsigned *it, *status, *nlog, *ntiles, *nseg, *minw, *steps; // [B]
	unsigned *cells; float *vals;   // [B][W] log: packed cell (z << 16 | x) and its final value
	unsigned *tiles;                // [B][T] touched tile ids (duplicates allowed)
	unsigned *seg;                  // [B][R][3] per flush segment: its end in the log, the bounding box of its cells (a cell appears at most once per segment; later segments win)
	unsigned *stamps;               // [tile] lowest droplet index that touched the tile this round (SP_NONE: none)
	unsigned *state;                // [B][SP_STATE_WORDS] registers of a walk suspended after `cap` moves in one round (a round must not wait for a 900-move droplet)
	unsigned *ctl;                  // {lo[0], lo[1], first conflict, done, in-place round, statistics ..., [SP_CTL_ROUND] rounds run}
	unsigned cap;
	int TNX;                        // tiles per row
};
constexpr int TW_SWEEP_VIEW = 32; // M_FROZEN: side of a droplet's private view (part of the algorithm's definition, see tw3d.h)
constexpr double FIXED_ONE = 1099511627776.0; // 2^40 delta units per height unit

struct DArgs {
	float *padded;              // M_GLOBAL / M_ATOMIC / M_WINDOW: padded heightmaps [tile][NY][NX] (M_ATOMIC: the one map)
	float *maps;                // M_WHOLE: the caller's un-padded heightmaps [tile][ysize][xsize], read once and written once
	const float *min_zvals;     // M_WHOLE: per-map lower clamp of the write-back (nullptr => min_zval_all)
	float min_zval_all;
	unsigned ntiles;            // M_ATOMIC: number of lane groups; otherwise unused
	unsigned slot0, nslots;     // this launch walks the schedule slots [slot0, slot0 + nslots)
	int xsize, ysize;
	unsigned num_iters;
	EParams E;
	const float2 *dir_table;
	unsigned long long *steps_out;
	const unsigned *order;      // heaviest-first schedule (slot -> map) or nullptr
	const unsigned *perm;       // M_WHOLE: map t of this batch lives at slot perm[t] of `maps` (nullptr: slot t)
	unsigned *next_droplet;     // M_ATOMIC: the dynamic,1 droplet counter
	int WX, WY, P;              // M_WINDOW / M_WHOLE: window extent and row pitch in floats (M_WHOLE: WX = NX, WY = NY)
	unsigned win_elems;         // floats of shared memory per lane group
	unsigned win_min_moves;     // M_WINDOW: a droplet gets a window once it has survived this many moves (ocean droplets die in one)
	// M_FROZEN: this device's band of the padded map
	long long *delta;           // fixed-point deltas, same layout as `padded` (rows [row0, row0 + band rows))
	int row0, own0, own1;       // first stored padded row; droplets starting in padded rows [own0, own1) are walked here
	int halo_rule;              // a droplet ends when |zi - start row| exceeds this
	unsigned it0, it1;          // droplets [it0, it1) = this sweep
	SpecArgs S;                 // M_SPEC; M_GLOBAL with S.ctl != nullptr: walk the window's head in place if it is SP_HUGE
	twi_job_words *jw;          // in a job: the context's job words (tw_cancel), M_GLOBAL / M_ATOMIC / M_WINDOW / M_WHOLE start no droplet once it is cancelled; nullptr otherwise
	const unsigned *sweep_it0;  // M_FROZEN in a job (twi_erode_sweeps_enqueue): the device word holding it0; the sweep is [it0, fz_end(it0, sweep, num_iters))
	unsigned sweep;
};

// CANCEL: the variant with the cancellation point, for jobs (see launch_droplets); synchronous calls and short latency-mode walks run the one without it, whose
// code is the same as before tw_cancel existed (the check's branch makes ptxas lay the loop out differently, which costs a serial chain about 4 %).
// M_FROZEN's job variant (CANCEL = true) has no check in the walk: it reads its sweep's bounds from A.sweep_it0, so one graph body serves every sweep, and
// the loop's cancellation point is sweep_advance_kernel. The flags are spelled out in the expressions below rather than named: even an unused constexpr local
// changes how the front end orders the code, and the SASS of the other instantiations is meant to stay as it was.
template<int G, int MODE, bool CANCEL>
__global__ void __launch_bounds__(128)
droplet_kernel(DArgs const A)
{
	constexpr bool SHARED = (MODE == M_ATOMIC), FROZEN = (MODE == M_FROZEN), SPEC = (MODE == M_SPEC), WIN = (MODE == M_WINDOW || MODE == M_FROZEN || MODE == M_SPEC), WHOLE = (MODE == M_WHOLE);
	static_assert(!CANCEL || !SPEC, "M_SPEC stops at its round boundary (spec_round_kernel)");
	static_assert(!SPEC || G == 32, "M_SPEC: one droplet per warp");
	// M_FROZEN shares M_WINDOW's machinery: the window is the droplet's PRIVATE view (sweep-start heights + its own writes); see hadd
	constexpr int TPW = 32/G; // heightmaps per warp
	extern __shared__ __align__(16) float tw_smem[];
	// the thread index is passed through a warp shuffle once: a shuffle result cannot be rematerialised, so ptxas keeps lane / sub in registers instead of
	// re-reading SR_TID.X (S2R, ~25 cycles) three times per move on the droplet's serial chain, as the round-1 SASS did
	unsigned const tid_once = (unsigned)__shfl_sync(0xffffffffu, (int)threadIdx.x, (int)(threadIdx.x & 31));
	int const lane = tid_once & 31, sub = lane % G, grp = lane / G;
	unsigned const wib = tid_once >> 5;
	unsigned const gslot = (blockIdx.x*(blockDim.x >> 5) + wib)*TPW + grp;       // position in this launch's part of the heaviest-first schedule
	bool active = (gslot < A.nslots);
	unsigned const tile = active ? (A.order ? __ldg(A.order + A.slot0 + gslot) : (A.slot0 + gslot)) : 0u;
	unsigned const gmask = (G == 32) ? 0xffffffffu : (((1u << (G & 31)) - 1u) << (grp*G));
	int const xsize = A.xsize, ysize = A.ysize;
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	float *mh = (MODE == M_WHOLE) ? nullptr : (FROZEN ? A.padded - (ptrdiff_t)A.row0*NX : A.padded + ((SHARED || SPEC) ? (size_t)0 : (size_t)tile*NX*NY)); // FROZEN: indexed by global padded row; M_SPEC: every slot walks the ONE map
	long long *dl64 = FROZEN ? A.delta - (ptrdiff_t)A.row0*NX : nullptr;
	unsigned const fz_stride = FROZEN ? A.nslots : 0u;
	int zstart = 0;
	float const Kq=10, Kw=0.001f, Kr=0.9f, Kd=0.02f, Ki=0.1f, minSlope=0.05f, g=20, Kg=g*2;
	unsigned const MAX_PATH_LEN = 4u*(unsigned)NX*(unsigned)NY;
	float const erode_amount = A.E.erode_amount;
	EParams const E = A.E;
	unsigned num_iters = A.num_iters;
	unsigned long long steps = 0;
	bool const have_tile = active;
	bool in_droplet = false;
	unsigned iter = (MODE == M_FROZEN) ? ((CANCEL && FROZEN) ? *A.sweep_it0 : A.it0) + gslot : 0u, numMoves = 0; // M_FROZEN: group g walks droplets it0 + g, it0 + g + groups, ... of the sweep
	// M_SPEC: this warp's slot of the window; the log it writes
	unsigned sp_nlog = 0, sp_nseg = 0, sp_ntiles = 0;
	int sp_ax = -1, sp_az = -1, sp_bx = -1, sp_bz = -1; // tile rectangle of the previous move (most moves stay inside it)
	bool sp_overflow = false, sp_started = false, sp_tile0 = false, sp_nonfinite = false, sp_resume = false;
	unsigned sp_launch_moves = 0;
	unsigned sp_why = 0; // statistics: why the walk outgrew its log (bit 0 log, 1 views, 2 tiles, 3 write outside the view, 4 non-finite near the corner)
	unsigned *sp_cells = nullptr, *sp_tiles = nullptr, *sp_seg = nullptr; float *sp_vals = nullptr;
	bool sp_inplace = false; // M_SPEC: this warp walks the window's HEAD directly on the map (nothing earlier is uncommitted, so its writes are final as they happen)
	if (SPEC) {
		unsigned const lo = A.S.ctl[A.S.ctl[SP_CTL_ROUND] & 1u];
		unsigned const st0 = active ? A.S.status[gslot] : SP_EMPTY;
		if (!active || A.S.it[gslot] >= num_iters) return;
		iter = A.S.it[gslot];
		bool const head = (iter == lo);
		// walk this slot's droplet if it needs walking: fresh (SP_DIRTY), suspended (SP_WALKING), or outsized and now at the head (SP_HUGE)
		if (!(st0 == SP_DIRTY || st0 == SP_WALKING || (st0 == SP_HUGE && head))) return;
		sp_resume = (st0 == SP_WALKING);
		sp_inplace = head && !sp_resume; // (a suspended head goes on the way it started: its state word says which)
		sp_cells = A.S.cells + (size_t)gslot*A.S.W; sp_vals = A.S.vals + (size_t)gslot*A.S.W; sp_tiles = A.S.tiles + (size_t)gslot*A.S.T; sp_seg = A.S.seg + (size_t)gslot*A.S.R*3;
	}
	Rng rgen; rgen.s1 = rgen.s2 = 1;
	int xi = 0, zi = 0;
	float xp=0, zp=0, xf=0, zf=0, s=0, v=0, w=1, dx=0, dz=0, h=0, h00=0, h10=0, h01=0, h11=0;
	// shared-memory window of this lane group
	int const WX = A.WX, WY = A.WY, P = A.P;
	float *win = (WIN || WHOLE) ? tw_smem + (size_t)(wib*TPW + grp)*A.win_elems : nullptr;
	unsigned *sp_dirty = SPEC ? reinterpret_cast<unsigned *>(win + (size_t)P*WY) : nullptr; // M_SPEC: one word of dirty bits per view row (WX <= 32), after the view
	int wx0 = 0, wz0 = 0;           // padded coordinates of the window's first cell
	bool have_win = WHOLE;
	// M_SPEC: append the view's changed cells to the droplet's log as one segment (row-major; a cell at most once per segment) and clear the dirty bits
	auto sp_flush = [&]() {
		if (!SPEC || !have_win) return;
		__syncwarp();
		unsigned orw = 0; int zlo = -1, zhi = -1;
		for (int r = 0; r < WY; ++r) {
			unsigned const word = sp_dirty[r];
			if (word == 0u) continue; // warp-uniform
			bool const mine = (lane < WX) && ((word >> lane) & 1u);
			unsigned const pos = sp_nlog + __popc(word & ((1u << lane) - 1u));
			if (mine && pos < A.S.W) {sp_cells[pos] = ((unsigned)(wz0 + r) << 16) | (unsigned)(wx0 + lane); sp_vals[pos] = win[r*P + lane];}
			sp_nlog += __popc(word);
			orw |= word; if (zlo < 0) {zlo = r;} zhi = r;
		}
		__syncwarp();
		if (lane < WY) {sp_dirty[lane] = 0u;}
		if (orw != 0u) { // one segment: its end in the log and the bounding box of its cells (sp_overlay only looks at segments that reach into the view)
			if (sp_nlog > A.S.W || sp_nseg >= A.S.R) {sp_overflow = true; sp_why |= (sp_nlog > A.S.W) ? 1u : 2u; sp_nlog = min(sp_nlog, A.S.W);}
			else {
				if (lane == 0) {
					sp_seg[3*sp_nseg] = sp_nlog;
					sp_seg[3*sp_nseg + 1] = (unsigned)(wx0 + __ffs(orw) - 1) | ((unsigned)(wx0 + 31 - __clz(orw)) << 16);
					sp_seg[3*sp_nseg + 2] = (unsigned)(wz0 + zlo) | ((unsigned)(wz0 + zhi) << 16);
				}
				++sp_nseg;
			}
		}
		__syncwarp();
	};
	// M_SPEC: after a view (re)load from the committed map, put the droplet's own earlier writes back on top: the segments whose bounding box reaches into the view,
	// in the order they were written (later segments win). A steadily moving droplet has dozens of segments but only the last one or two matter.
	auto sp_overlay = [&]() {
		if (!SPEC) return;
		unsigned prev_end = 0;
		for (unsigned base = 0; base < sp_nseg; base += 32) {
			unsigned const idx = base + lane;
			bool const in = (idx < sp_nseg);
			unsigned const e = in ? sp_seg[3*idx] : 0u, bx = in ? sp_seg[3*idx + 1] : 0u, bz = in ? sp_seg[3*idx + 2] : 0u;
			unsigned start = __shfl_up_sync(0xffffffffu, e, 1);
			if (lane == 0) {start = prev_end;}
			bool const hit = in && (int)(bx & 0xffffu) < wx0 + WX && (int)(bx >> 16) >= wx0 && (int)(bz & 0xffffu) < wz0 + WY && (int)(bz >> 16) >= wz0;
			unsigned mask = __ballot_sync(0xffffffffu, hit);
			while (mask) {
				int const l = __ffs(mask) - 1;
				mask &= mask - 1u;
				unsigned const b = __shfl_sync(0xffffffffu, start, l), ee = __shfl_sync(0xffffffffu, e, l);
				for (unsigned k = b + lane; k < ee; k += 32) {
					unsigned const c = sp_cells[k];
					unsigned const rx = (c & 0xffffu) - (unsigned)wx0, rz = (c >> 16) - (unsigned)wz0;
					if (rx < (unsigned)WX && rz < (unsigned)WY) {win[rz*P + rx] = sp_vals[k];}
				}
				__syncwarp();
			}
			prev_end = __shfl_sync(0xffffffffu, e, (int)min(31u, sp_nseg - 1u - base));
		}
	};

	auto load_view = [&]() { // the WX x WY cells at (wx0, wz0) of the (committed / sweep-start / current) map -> shared memory
		__syncwarp(gmask); // the group's earlier write-throughs are ordered before the loads below
#pragma unroll 4
		for (int r = 0; r < WY; ++r) {
			const float *src = mh + ((size_t)NX*(wz0 + r) + wx0);
			float *dst = win + r*P;
			for (int c = sub; c < WX; c += G) {dst[c] = FROZEN ? __ldg(src + c) : __ldcg(src + c);}
		}
		__syncwarp(gmask);
		have_win = true;
		sp_overlay();
	};
	if (SPEC && sp_resume) { // pick a suspended walk up again: registers from the slot's state, the view re-read from the committed map + the droplet's own log
		const unsigned *q = A.S.state + (size_t)gslot*SP_STATE_WORDS;
		xi = (int)q[0]; zi = (int)q[1]; wx0 = (int)q[2]; wz0 = (int)q[3]; numMoves = q[4]; rgen.s1 = (int)q[5]; rgen.s2 = (int)q[6];
		sp_ax = (int)q[7]; sp_az = (int)q[8]; sp_bx = (int)q[9]; sp_bz = (int)q[10];
		unsigned const fl = q[11]; sp_tile0 = (fl & 2u) != 0u; sp_nonfinite = (fl & 4u) != 0u; sp_inplace = (fl & 8u) != 0u;
		steps = q[12];
		xp = __uint_as_float(q[13]); zp = __uint_as_float(q[14]); xf = __uint_as_float(q[15]); zf = __uint_as_float(q[16]); s = __uint_as_float(q[17]); v = __uint_as_float(q[18]);
		w = __uint_as_float(q[19]); dx = __uint_as_float(q[20]); dz = __uint_as_float(q[21]); h = __uint_as_float(q[22]);
		h00 = __uint_as_float(q[23]); h10 = __uint_as_float(q[24]); h01 = __uint_as_float(q[25]); h11 = __uint_as_float(q[26]);
		sp_nlog = A.S.nlog[gslot]; sp_nseg = A.S.nseg[gslot]; sp_ntiles = A.S.ntiles[gslot];
		in_droplet = true; sp_started = true; ++iter;
		if (lane < WY) {sp_dirty[lane] = 0u;}
		if (fl & 1u) {load_view();}
	}

	if (WHOLE) { // build the padded map in shared memory from the caller's tile (src/erosion.cpp:31-37)
		if (active) {
			const float *src = A.maps + (size_t)(A.perm ? __ldg(A.perm + tile) : tile)*xsize*ysize;
#pragma unroll 4
			for (int y = 0; y < NY; ++y) {
				const float *row = src + (size_t)clampi(y - PAD, ysize - 1)*xsize;
				float *dst = win + y*P;
				for (int x = sub; x < NX; x += G) {dst[x] = __ldcs(row + clampi(x - PAD, xsize - 1));}
			}
		}
		__syncwarp(gmask);
	}

	// HREAD(x, y): HMAP(x, y) of the reference = clamped read
	auto hread = [&](int x, int z) -> float {
		int const cx = clampi(x, NX-1), cz = clampi(z, NY-1);
		if (WHOLE) {return win[cz*P + cx];}
		if (WIN && have_win) {
			unsigned const rx = (unsigned)(cx - wx0), rz = (unsigned)(cz - wz0);
			if (rx < (unsigned)WX && rz < (unsigned)WY) {return win[rz*P + rx];}
		}
		float const *p = mh + ((size_t)NX*cz + cx);
		return SHARED ? __ldcg(p) : *p;
	};
	// hadd(x, z, delta, pred): read-modify-write of the in-array cell (x, z) where pred holds. In the plain modes EVERY lane computes the address and loads
	// (x, z are valid for all lanes) and only the store is predicated: no divergent region around the 4 deposit / 16 brush lanes, which in the round-1
	// kernel cost a BSSY/BSYNC pair and two branches per read-modify-write on the droplet's serial chain. Window modes write through to global memory.
	auto hadd = [&](int x, int z, float delta, bool pred) {
		if (WHOLE) {float *q = win + (z*P + x); float const nv = *q + delta; if (pred) {*q = nv;} return;}
		float *p = mh + ((size_t)NX*z + x);
		if (MODE == M_GLOBAL) {float const nv = *p + delta; if (pred) {*p = nv;} return;}
		if (!pred) return;
		if (SPEC && sp_inplace) {*p = *p + delta; return;} // the head of the window: straight into the map
		if (SPEC) { // the write stays private: view + dirty bit (the log is written when the view moves on or the droplet ends)
			unsigned const rx = (unsigned)(x - wx0), rz = (unsigned)(z - wz0);
			if (have_win && rx < (unsigned)WX && rz < (unsigned)WY) {float *q = win + (rz*P + rx); *q = *q + delta; atomicOr(sp_dirty + rz, 1u << rx);}
			else {sp_overflow = true; sp_why |= 8u;} // cannot happen (the view covers every cell a move touches); if it did, the droplet is walked in place instead
			return;
		}
		if (WIN && have_win) {
			unsigned const rx = (unsigned)(x - wx0), rz = (unsigned)(z - wz0);
			if (rx < (unsigned)WX && rz < (unsigned)WY) {
				float *q = win + (rz*P + rx); float const nv = *q + delta; *q = nv; // the droplet sees its own write
				if (!FROZEN) {*p = nv; return;}                                     // M_WINDOW: write through
			}
		}
		if (FROZEN) { // everybody else sees it after the sweep: fixed-point accumulation; NaN / inf / absurd deltas contribute nothing (same rule in the oracle)
			long long const q = (fabsf(delta) < 1048576.0f) ? __double2ll_rn((double)delta*FIXED_ONE) : 0ll;
			if (q) {atomicAdd((unsigned long long *)(dl64 + ((size_t)NX*z + x)), (unsigned long long)q);}
			return;
		}
		if (SHARED) {atomicAdd(p, delta);} else {*p += delta;}
	};
	// DEPOSIT(H): src/erosion.cpp:42-54; corner c of the 2x2 cell goes to lane c % G (inside cells are distinct => no aliasing between lanes)
	// corner c of the 2x2 cell: lanes c, c + DG, ... of the group with DG = min(G, 4); lanes >= 4 of a wide group shadow lanes 0-3 with the store predicated off
#define DEPOSIT(H) { \
	constexpr int DG = (G < 4) ? G : 4; \
	_Pragma("unroll") \
	for (int c0 = 0; c0 < 4; c0 += DG) { \
		int const c = c0 + (sub & (DG - 1)); \
		int const X = xi + (c & 1), Z = zi + (c >> 1); \
		float const W = ((c & 1) ? xf : (1-xf))*((c >> 1) ? zf : (1-zf)); \
		float const delta = ds*erode_amount*W; \
		bool const inside = ((unsigned)X < (unsigned)NX && (unsigned)Z < (unsigned)NY); \
		hadd(clampi(X, NX-1), clampi(Z, NY-1), delta, inside && (G <= 4 || sub < 4)); \
	} \
	if (G > 1) {__syncwarp(gmask);} \
	(H) += ds; }

	for (;;) {
		if (active && !in_droplet) { // next droplet of this group's heightmap (src/erosion.cpp:67-73)
			if (SHARED) { // schedule(dynamic,1): the group's leader draws the next droplet
				unsigned nd = 0;
				if (sub == 0) {nd = atomicAdd(A.next_droplet, 1u);}
				iter = __shfl_sync(gmask, nd, grp*G);
			}
			if (SPEC && sp_started) { // the slot's one droplet has ended: close the log
				sp_flush();
				if (lane == 0) {
					A.S.nlog[gslot] = sp_nlog; A.S.nseg[gslot] = sp_nseg; A.S.ntiles[gslot] = sp_ntiles; A.S.steps[gslot] = (unsigned)steps;
					A.S.status[gslot] = sp_inplace ? ((sp_overflow || A.S.ctl[14] != 0u) ? SP_INPLACE : SP_VALID) : (sp_overflow ? SP_HUGE : SP_VALID);
					if (sp_inplace) {A.S.ctl[14] = 0u; sp_nlog = 0; sp_nseg = 0;} // nothing to commit: the map has it all already
					if (sp_inplace) {atomicAdd(A.S.ctl + 5, 1u);}
					atomicAdd(A.S.ctl + 6, 1u); if (sp_overflow) {atomicAdd(A.S.ctl + 7, 1u);} // statistics: walks, walks that outgrew their log
					for (unsigned b = 0; b < 5; ++b) {if (sp_why & (1u << b)) {atomicAdd(A.S.ctl + 8 + b, 1u);}}
					atomicMax(A.S.ctl + 13, numMoves);
				}
				active = false;
			}
			else if (iter >= (FROZEN ? ((CANCEL && FROZEN) ? fz_end(*A.sweep_it0, A.sweep, num_iters) : A.it1) : num_iters)) {active = false;}
			// cancelled (tw_cancel): the group stops as if num_iters had been reached. Its leader reads the job words before every 8th droplet only (the
			// droplet index, group-uniform), which keeps the read's latency off nearly every droplet of the serial chain
			else if (CANCEL && !FROZEN && (iter & 7u) == 0u && __shfl_sync(gmask, (sub == 0 && twi_cancelled(A.jw)) ? 1u : 0u, grp*G)) {
				if (sub == 0) {twi_mark_stopped(A.jw);}
				active = false;
			}
			else {
				rgen.s1 = (int)iter + 11; rgen.s2 = 79*(int)iter + 121;
				xi = PAD + (rgen.rand()%xsize);
				zi = PAD + (rgen.rand()%ysize);
				if (FROZEN && (zi < A.own0 || zi >= A.own1)) {iter += fz_stride;} // another device's droplet
				else {
					xp=xi; zp=zi; xf=0; zf=0; s=0; v=0; w=1; dx=0; dz=0;
					if (FROZEN) {have_win = false;} // M_FROZEN: a new droplet knows nothing of the previous one's writes - its first reads included
					if (SPEC) {sp_started = true; if (lane < WY) {sp_dirty[lane] = 0u;}}
					h=hread(xi, zi); h00=h; h10=hread(xi+1, zi); h01=hread(xi, zi+1); h11=hread(xi+1, zi+1);
					numMoves = 0; in_droplet = true; zstart = zi;
					if (FROZEN) {iter += fz_stride;} else {++iter;}
				}
			}
		}
		if (!__any_sync(0xffffffffu, active)) break;
		if (!active || !in_droplet) continue;
		if (FROZEN && (unsigned)(zi - zstart + A.halo_rule) > 2u*(unsigned)A.halo_rule) {in_droplet = false; continue;} // left the band +- halo: the droplet ends (rule of the batched algorithm)
		if (numMoves >= MAX_PATH_LEN) {in_droplet = false; continue;} // "droplet path is too long" (src/erosion.cpp:153)
		if (SPEC && sp_overflow && !sp_inplace) {in_droplet = false; continue;} // outgrew its log: it will be walked in place as the head, no point in finishing this walk
		if (SPEC && sp_launch_moves >= (sp_inplace ? 2u*A.S.cap : A.S.cap)) { // enough for this round (the in-place head moves at twice the speed): the walk goes on in the next one (a round must not wait for a 900-move droplet)
			unsigned const had_win = have_win ? 1u : 0u;
			sp_flush();
			if (lane == 0) {
				unsigned *q = A.S.state + (size_t)gslot*SP_STATE_WORDS;
				q[0] = (unsigned)xi; q[1] = (unsigned)zi; q[2] = (unsigned)wx0; q[3] = (unsigned)wz0; q[4] = numMoves; q[5] = (unsigned)rgen.s1; q[6] = (unsigned)rgen.s2;
				q[7] = (unsigned)sp_ax; q[8] = (unsigned)sp_az; q[9] = (unsigned)sp_bx; q[10] = (unsigned)sp_bz;
				q[11] = had_win | (sp_tile0 ? 2u : 0u) | (sp_nonfinite ? 4u : 0u) | (sp_inplace ? 8u : 0u);
				q[12] = (unsigned)steps;
				q[13] = __float_as_uint(xp); q[14] = __float_as_uint(zp); q[15] = __float_as_uint(xf); q[16] = __float_as_uint(zf); q[17] = __float_as_uint(s); q[18] = __float_as_uint(v);
				q[19] = __float_as_uint(w); q[20] = __float_as_uint(dx); q[21] = __float_as_uint(dz); q[22] = __float_as_uint(h);
				q[23] = __float_as_uint(h00); q[24] = __float_as_uint(h10); q[25] = __float_as_uint(h01); q[26] = __float_as_uint(h11);
				A.S.nlog[gslot] = sp_nlog; A.S.nseg[gslot] = sp_nseg; A.S.ntiles[gslot] = sp_ntiles;
				A.S.status[gslot] = (sp_overflow && !sp_inplace) ? SP_HUGE : SP_WALKING;
				if (sp_overflow && sp_inplace) {A.S.ctl[14] = 1u;} // the head's tile list is incomplete: remember it across the suspension
			}
			return;
		}
		++numMoves; ++steps; ++sp_launch_moves;
		if (WIN && !(SPEC && sp_inplace)) { // keep the cells one move can touch - brush [xi-1, xi+2], next corners within +-2 of xi - inside the window
			int const cx = clampi(xi, NX-1), cz = clampi(zi, NY-1);
			bool const covered = have_win && max(cx - 2, 0) >= wx0 && min(cx + 3, NX-1) < wx0 + WX && max(cz - 2, 0) >= wz0 && min(cz + 3, NY-1) < wz0 + WY;
			if (!covered && (FROZEN || SPEC || numMoves > A.win_min_moves)) { // re-centre ahead of the droplet's heading (dx, dz = unit direction of the last move) and re-load
				sp_flush();
				wx0 = max(0, min(cx - WX/2 + __float2int_rn(dx*(float)(WX/2 - 5)), NX - WX));
				wz0 = max(0, min(cz - WY/2 + __float2int_rn(dz*(float)(WY/2 - 5)), NY - WY));
				load_view();
			}
		}
		if (SPEC && !sp_nonfinite) { // the conflict tiles this move can read or write (after a non-finite position: only cell (0, 0) is read any more, nothing written)
			int const qx = clampi(xi, NX-1), qz = clampi(zi, NY-1); // (a droplet that has left the map sits at INT_MIN: clamp before the +-)
			// exactly the cells a move at (xi, zi) can read or write: the 2 x 2 cells at the next position (nxi in xi-1 .. xi+1), the deposit at xi .. xi+1, the brush xi-1 .. xi+2
			int const ax = clampi(qx - 1, NX-1) >> SP_TILE_SHIFT, bx = clampi(qx + 2, NX-1) >> SP_TILE_SHIFT, az = clampi(qz - 1, NY-1) >> SP_TILE_SHIFT, bz = clampi(qz + 2, NY-1) >> SP_TILE_SHIFT;
			if (ax == 0 && az == 0) {sp_tile0 = true;}
			if (ax != sp_ax || az != sp_az || bx != sp_bx || bz != sp_bz) {
				sp_ax = ax; sp_az = az; sp_bx = bx; sp_bz = bz;
				if (sp_ntiles + 4 > A.S.T) {sp_overflow = true; sp_why |= 4u;} // (in place: the walk goes on, see below)
				else {
					if (lane < 4) {
						int const tx = (lane & 1) ? bx : ax, tz = (lane & 2) ? bz : az; // up to 2 x 2 tiles; duplicates are harmless
						sp_tiles[sp_ntiles + lane] = (unsigned)(tz*A.S.TNX + tx);
					}
					sp_ntiles += 4;
				}
			}
		}
		{ // ---- one move of the droplet (src/erosion.cpp:76-152) ----
			float const gx=h00+h01-h10-h11, gz=h00+h10-h01-h11;
			dx=(dx-gx)*Ki+gx;
			dz=(dz-gz)*Ki+gz;
			float const dl=__fsqrt_rn(dx*dx+dz*dz);
			if (dl<=FLT_EPSILON) { // pick random dir: a = rand_float()*TWO_PI, rand_float() = 1e-6*(rand()%1000000)
				float2 const cs = __ldg(A.dir_table + (rgen.rand()%1000000));
				dx=cs.x; dz=cs.y;
			}
			else {dx=__fdiv_rn(dx, dl); dz=__fdiv_rn(dz, dl);}
			float const nxp=xp+dx, nzp=zp+dz;
			int nxi=__float2int_rd(nxp), nzi=__float2int_rd(nzp); // (int)floor(.)
			// M_FROZEN: a droplet whose next position is not a finite in-range number ends here (rule of the batched algorithm, same in the oracle): the reference would
			// read the map at the clamp of INT_MIN, i.e. row 0 - a row a device that holds only its band +- halo does not have
			if (FROZEN && !(fabsf(nxp) < 2147483648.0f && fabsf(nzp) < 2147483648.0f)) {in_droplet = false; continue;}
			if (SPEC && !(fabsf(nxp) < 2147483648.0f && fabsf(nzp) < 2147483648.0f)) {
				// a NaN of the droplet's own making (2 % of the droplets on the BASELINE terrain): the reference goes on to read the map at the clamp of INT_MIN - cell
				// (0, 0), four times - before the droplet ends as "outside" on its next move. That cell comes straight from the committed map (hread's fall-back), so
				// tile 0 joins the droplet's tiles; only if the droplet itself has been there (its own write may sit in its log, not in the map) it is walked in place.
				if (!sp_nonfinite) { // (the droplet passes here once more on its last move, from "outside")
					sp_nonfinite = true;
					if (sp_tile0 && !sp_inplace) {sp_overflow = true; sp_why |= 16u; in_droplet = false; continue;}
					if (sp_ntiles + 4 > A.S.T) {sp_overflow = true; sp_why |= 4u; if (!sp_inplace) {in_droplet = false; continue;}}
					else {
						if (lane < 4) {sp_tiles[sp_ntiles + lane] = 0u;}
						sp_ntiles += 4;
					}
				}
			}
			if (!(fabsf(nxp) < 2147483648.0f && fabsf(nzp) < 2147483648.0f)) { // NaN / out of int range: x86 cvttss2si yields INT_MIN -> "outside" next step
				nxi=tw_x86_f2i(floorf(nxp)); nzi=tw_x86_f2i(floorf(nzp));
			}
			float const nxf=nxp-(float)nxi, nzf=nzp-(float)nzi;
			float nh00, nh10, nh01, nh11;
			if (WHOLE || WIN) { // common case: the 2x2 cell lies inside the window (which lies inside the array: no clamping)
				unsigned const rx = (unsigned)(nxi - wx0), rz = (unsigned)(nzi - wz0);
				if (have_win && rx < (unsigned)(WX-1) && rz < (unsigned)(WY-1)) {
					float const *q = win + (rz*P + rx);
					nh00 = q[0]; nh10 = q[1]; nh01 = q[P]; nh11 = q[P+1];
				}
				else {nh00=hread(nxi, nzi); nh10=hread(nxi+1, nzi); nh01=hread(nxi, nzi+1); nh11=hread(nxi+1, nzi+1);}
			}
			else if ((unsigned)nxi < (unsigned)(NX-1) && (unsigned)nzi < (unsigned)(NY-1)) { // common case: no clamping needed
				float const *q = mh + (nzi*NX + nxi);
				if (SHARED) {nh00 = __ldcg(q); nh10 = __ldcg(q + 1); q += NX; nh01 = __ldcg(q); nh11 = __ldcg(q + 1);}
				else        {nh00 = *q; nh10 = q[1]; q += NX; nh01 = *q; nh11 = q[1];}
			}
			else {nh00=hread(nxi, nzi); nh10=hread(nxi+1, nzi); nh01=hread(nxi, nzi+1); nh11=hread(nxi+1, nzi+1);}
			float const nh=(nh00*(1-nxf)+nh10*nxf)*(1-nzf)+(nh01*(1-nxf)+nh11*nxf)*nzf;
			if (smax(smax(nh00, nh10), smax(nh01, nh11)) < E.wpz_minus_half_dxy) {in_droplet = false; continue;} // reached ocean water

			bool const outside = ((unsigned)xi >= (unsigned)NX || (unsigned)zi >= (unsigned)NY);
			if (nh>=h || outside) {
				float ds=(nh-h)+0.001f;
				if (ds>=s || outside) {
					ds=s;
					DEPOSIT(h)
					s=0;
					in_droplet = false; continue;
				}
				DEPOSIT(h)
				s-=ds;
				v=0;
			}
			float dh=h-nh;
			float const q=smax(dh, minSlope)*v*w*Kq;
			float ds=s-q;
			if (ds>=0) { // deposit
				ds*=Kd;
				DEPOSIT(dh)
				s-=ds;
			}
			else { // erode
				ds*=-Kr;
				ds=smin(ds, dh*0.99f);
				{ // get_bare_ls_tid(nh) == ROCK_TEX ? 0.5 : 2.0 (src/Textures.cpp:1284-1287); x0.5 / x2 are exact in fp32
					bool rock;
					if (E.rock_exact) {rock = (nh >= E.rock_min);} // the reference predicate is monotone in nh: one compare against its host-found threshold
					else {float const relh = E.relh_adj_tex + __fdiv_rn(nh - E.zmin, E.zrange); rock = (relh > E.clip_hd1);}
					ds *= rock ? 0.5f : 2.0f;
				}
				bool const interior = ((unsigned)(xi - 1) < (unsigned)(NX - 3) && (unsigned)(zi - 1) < (unsigned)(NY - 3));
				if (interior || G == 1) { // 16 distinct cells dealt to the lanes of the group (G == 1: the reference's serial loop, clamped); uniform control flow, predicated stores
					constexpr int BG = (G < 16) ? G : 16;
#pragma unroll
					for (int c0 = 0; c0 < 16; c0 += BG) {
						int const c = c0 + (sub & (BG - 1));
						int const x = xi + (c & 3) - 1, z = zi + (c >> 2) - 1;
						float const zo=(float)z-zp, zo2=zo*zo, xo=(float)x-xp;
						float wgt=1-(xo*xo+zo2)*0.25f;
						bool const on = !(wgt<=0) && (G <= 16 || sub < 16);
						wgt*=0.1591549430918953f;
						float const delta=ds*erode_amount*wgt;
						if (interior) {hadd(x, z, -delta, on);} else {hadd(clampi(x, NX-1), clampi(z, NY-1), -delta, on);}
					}
				}
				else if (sub == 0) { // border: clamped indices may alias, keep the reference's serial order
					for (int z=zi-1; z<=zi+2; ++z) {
						float const zo=(float)z-zp, zo2=zo*zo;
						for (int x=xi-1; x<=xi+2; ++x) {
							float const xo=(float)x-xp;
							float wgt=1-(xo*xo+zo2)*0.25f;
							if (wgt<=0) continue;
							wgt*=0.1591549430918953f;
							float const delta=ds*erode_amount*wgt;
							hadd(clampi(x, NX-1), clampi(z, NY-1), -delta, true);
						}
					}
				}
				if (G > 1) {__syncwarp(gmask);}
				dh-=ds;
				s+=ds;
			}
			v=__fsqrt_rn(v*v+Kg*dh);
			w*=1-Kw;
			xp=nxp; zp=nzp; xi=nxi; zi=nzi; xf=nxf; zf=nzf;
			h=nh; h00=nh00; h10=nh10; h01=nh01; h11=nh11;
		}
	}
#undef DEPOSIT
	if (WHOLE && have_tile) { // remove padding and clamp to min_zval (src/erosion.cpp:158-162)
		__syncwarp(gmask);
		float const mz = A.min_zvals ? __ldg(A.min_zvals + tile) : A.min_zval_all;
		float *dst = A.maps + (size_t)(A.perm ? __ldg(A.perm + tile) : tile)*xsize*ysize;
#pragma unroll 4
		for (int y = 0; y < ysize; ++y) {
			float const *srow = win + (y + PAD)*P + PAD;
			for (int x = sub; x < xsize; x += G) {dst[(size_t)y*xsize + x] = smax(mz, srow[x]);}
		}
	}
	if (sub == 0 && A.steps_out && steps) {atomicAdd(A.steps_out, steps);}
}

constexpr size_t SMEM_MAX_BLOCK = 227u*1024u; // sm_90: 227 KB of dynamic shared memory per block

template<int G, int MODE, bool CANCEL>
void launch_droplets_c(cudaStream_t st, DArgs const &A, unsigned warps_per_block, size_t smem_per_group) {
	unsigned const groups_per_block = warps_per_block*(32/G);
	size_t const smem = smem_per_group*groups_per_block;
	if (smem > 48*1024) {cudaFuncSetAttribute(droplet_kernel<G, MODE, CANCEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);}
	droplet_kernel<G, MODE, CANCEL><<<(A.nslots + groups_per_block - 1)/groups_per_block, 32*warps_per_block, smem, st>>>(A);
}

// The variant with the cancellation point runs for a job's erosion (A.jw set: twi_erode_enqueue / twi_erode_parallel_enqueue inside twi_launch_job) in the
// throughput mode, and in the latency modes for walks of at least CANCEL_MIN_DROPLETS droplets per map. A shorter latency-mode walk is not worth the
// check: the checking loop's layout costs a serial chain about 4 % (tools/bench_frame_tiles.py's 16-tile frame, 1000 droplets per tile: ready after
// 23.0-23.7 ms against 22.1 ms), while the whole walk is over in under 0.1 s (22 ms for 1000 droplets in that frame). In M_GLOBAL the cost hides behind
// thousands of walks in flight (bench.py's fused 16384-tile row is unchanged). DESIGN §4g.
constexpr unsigned CANCEL_MIN_DROPLETS = 4096;
template<int G, int MODE>
void launch_droplets(cudaStream_t st, DArgs const &A, unsigned warps_per_block, size_t smem_per_group) {
	if constexpr (MODE != M_SPEC && MODE != M_FROZEN) {
		if (A.jw && (MODE == M_GLOBAL || A.num_iters >= CANCEL_MIN_DROPLETS)) {launch_droplets_c<G, MODE, true>(st, A, warps_per_block, smem_per_group); return;}
	}
	if constexpr (MODE == M_FROZEN) {
		if (A.sweep_it0) {launch_droplets_c<G, MODE, true>(st, A, warps_per_block, smem_per_group); return;}
	}
	launch_droplets_c<G, MODE, false>(st, A, warps_per_block, smem_per_group);
}

template<int MODE>
void launch_droplets_g(int G, cudaStream_t st, DArgs const &A, unsigned warps_per_block, size_t smem_per_group) {
	while (G < 32 && (size_t)(32/G)*warps_per_block*smem_per_group > SMEM_MAX_BLOCK) {G *= 2;} // fewer maps per warp until their windows fit in one block's shared memory
	switch (G) {
	case 1:  launch_droplets<1,  MODE>(st, A, warps_per_block, smem_per_group); break;
	case 2:  launch_droplets<2,  MODE>(st, A, warps_per_block, smem_per_group); break;
	case 4:  launch_droplets<4,  MODE>(st, A, warps_per_block, smem_per_group); break;
	case 8:  launch_droplets<8,  MODE>(st, A, warps_per_block, smem_per_group); break;
	case 16: launch_droplets<16, MODE>(st, A, warps_per_block, smem_per_group); break;
	default: launch_droplets<32, MODE>(st, A, warps_per_block, smem_per_group); break;
	}
}

int env_int(const char *name, int dflt) {const char *e = getenv(name); return e ? atoi(e) : dflt;}

// lanes per heightmap: the smallest group of at least 16 lanes that still keeps 16384 warps in flight, see the kernel comment
int pick_group(unsigned ntiles) {
	int const g = env_int("TW_EROSION_LANES", 0);
	if (g == 1 || g == 2 || g == 4 || g == 8 || g == 16 || g == 32) return g;
	// With many warps in flight the kernel is issue-bound, so sharing a warp between maps pays; below that it is latency/tail-bound and one warp
	// per map is fastest. tools/bench_erosion.py on one H100, 258^2 tiles, 1000 droplets: 8192 / 16384 maps fastest at G=32 (0.163 / 0.198 s),
	// 32768 / 65536 maps at G=16 (0.264 / 0.535 s; G=8 0.294 / 0.584 s). => smallest G >= 16 that keeps 16384 warps.
	for (int gg = 16; gg < 32; gg *= 2) {if ((unsigned long long)ntiles*gg >= 32ull*16384ull) return gg;}
	return 32;
}

// lanes per heightmap of the shared-memory modes: 16 lanes cover the 4x4 brush; 32 keeps one map per warp (default)
int pick_smem_group() {
	int const g = env_int("TW_EROSION_SMEM_LANES", 32);
	return (g == 1 || g == 2 || g == 4 || g == 8 || g == 16) ? g : 32;
}


// row pitch of the whole-map layout: the smallest P >= NX whose four brush rows start >= 4 banks apart (the 4x4 brush is then conflict-free);
// kept at NX when padding would push the map over the shared-memory budget
int whole_pitch(int NX, int NY) {
	for (int P = NX; P < NX + 8; ++P) {
		bool ok = true;
		for (int a = 0; a < 4 && ok; ++a) for (int b = a + 1; b < 4 && ok; ++b) {
			int d = ((b - a)*P) % 32; if (d > 16) d = 32 - d;
			if (d < 4) ok = false;
		}
		// three 1-warp blocks per SM (228 KB per SM, 1 KB reserved per block) are worth more than conflict-free rows
		bool const fits3_before = ((size_t)NX*NY*4 + 1024)*3 <= 228u*1024u, fits3_after = ((size_t)P*NY*4 + 1024)*3 <= 228u*1024u;
		if (ok && (size_t)P*NY*4 <= SMEM_MAX_BLOCK && (fits3_after || !fits3_before)) return P;
	}
	return NX;
}

enum {EM_AUTO = 0, EM_GLOBAL = 1, EM_WINDOW = 2, EM_WHOLE = 3, EM_SPEC = 4};
int env_mode() { // TW_EROSION_MODE = global | window | whole | spec (tests and tuning; default: chosen from the batch shape)
	const char *e = getenv("TW_EROSION_MODE");
	if (!e) return EM_AUTO;
	if (!strcmp(e, "global")) return EM_GLOBAL;
	if (!strcmp(e, "window")) return EM_WINDOW;
	if (!strcmp(e, "whole"))  return EM_WHOLE;
	if (!strcmp(e, "spec"))   return EM_SPEC;
	return EM_AUTO;
}

} // namespace

// get_bare_ls_tid(z) == ROCK_TEX  <=>  relh_adj_tex + (z - zmin)/(zmax - zmin) > clip_hd1 (src/Textures.cpp:1284-1287), evaluated in fp32 with the
// reference's operation order. For zmax > zmin every step (rounded subtraction of a constant, rounded division by a positive constant, rounded addition
// of a constant) is monotone non-decreasing in z, so the predicate is a step function of z: false below some float T, true from T on. T is found on the
// host by bisection over the ordered bit patterns of ALL floats (-inf .. +inf) with the same IEEE operations (this file is compiled without FMA
// contraction or fast-math, host side included); the kernel then tests z >= T - one compare instead of FADD, FCHK + MUFU.RCP + 5 FFMA (+ slow path), FADD,
// FSETP on the droplet's dependency chain. NaN z: both forms are false. Anything not provably monotone (zmax <= zmin, NaN parameters) keeps the expression.
static inline bool rock_pred(float z, float adj, float zmin, float zrange, float clip) {
	volatile float d = z - zmin;      // volatile: no algebraic simplification across the three rounded steps
	volatile float q = d/zrange;
	volatile float r = adj + q;
	return r > clip;
}
static inline float ord2float(uint32_t u) { // order-preserving bijection uint32 -> float (inverse of tw_f2ord), NaNs excluded by the search range
	uint32_t const b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
	float f; memcpy(&f, &b, 4); return f;
}
static EParams make_eparams(const tw_erosion_params *p) {
	EParams E;
	E.erode_amount = p->erode_amount;
	E.wpz_minus_half_dxy = p->water_plane_z - p->half_dxy;
	E.zmin = p->zmin; E.zrange = p->zmax - p->zmin;
	E.relh_adj_tex = p->relh_adj_tex; E.clip_hd1 = p->clip_hd1;
	E.rock_min = 0.0f; E.rock_exact = 0;
	if (E.zrange > 0.0f && E.zrange < INFINITY && E.zmin == E.zmin && fabsf(E.zmin) < INFINITY && E.relh_adj_tex == E.relh_adj_tex && E.clip_hd1 == E.clip_hd1) {
		uint32_t const lo_u = tw_f2ord(-INFINITY), hi_u = tw_f2ord(INFINITY); // ordered keys: lo_u < hi_u, every float in between is a non-NaN
		if (!rock_pred(INFINITY, E.relh_adj_tex, E.zmin, E.zrange, E.clip_hd1)) {E.rock_min = NAN; E.rock_exact = 1;} // never rock: z >= NaN is always false
		else {
			uint32_t lo = lo_u, hi = hi_u; // invariant: pred(hi) true; smallest true key in [lo, hi]
			while (lo < hi) {
				uint32_t const mid = lo + (hi - lo)/2;
				if (rock_pred(ord2float(mid), E.relh_adj_tex, E.zmin, E.zrange, E.clip_hd1)) {hi = mid;} else {lo = mid + 1;}
			}
			E.rock_min = ord2float(hi); E.rock_exact = 1;
			// -0.0 and +0.0 are distinct keys but equal floats: if the step sits between them, z >= +0.0 also accepts -0.0 - keep the expression then
			if (E.rock_min == 0.0f && rock_pred(-0.0f, E.relh_adj_tex, E.zmin, E.zrange, E.clip_hd1) != rock_pred(0.0f, E.relh_adj_tex, E.zmin, E.zrange, E.clip_hd1)) {E.rock_exact = 0;}
		}
	}
	if (getenv("TW_EROSION_NO_ROCK_THRESHOLD")) {E.rock_exact = 0;}
	return E;
}

// ---- which mode walks a batch (see the kernel comment) ----
// M_WHOLE for batches of on-chip-sized maps up to 4 waves of resident walkers (SMs x 3 resident 76 KB maps; the streaming case - the reference
// creates <= 16 tiles per frame, src/tiled_mesh.cpp:2403-2417): no padded scratch copy and no pad/unpad passes - each tile is read once and written
// once; larger batches go to M_GLOBAL, whose thousands of resident warps hide the latency of the serial chains (tools/bench_erosion_modes.py).
static bool plan_whole(unsigned num_sms, uint32_t nt, int xsize, int ysize) {
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD, mode = env_mode();
	if ((size_t)whole_pitch(NX, NY)*NY*sizeof(float) > SMEM_MAX_BLOCK) return false;
	if (mode == EM_WHOLE) return true;
	return (mode == EM_AUTO && nt <= (uint32_t)env_int("TW_EROSION_WHOLE_MAX", (int)num_sms*3*4));
}
// M_WINDOW for the `heavy` first slots of the heaviest-first schedule, M_GLOBAL for the rest. One move is ~233 dependent instructions of ONE warp:
// the serial chain is bound by instruction latency, not by where the heights live, and the window's bookkeeping adds instructions to it. So the
// default is 0 (never); the mode stays selectable (TW_EROSION_MODE=window, TW_EROSION_HEAVY, TW_EROSION_WINDOW_ALL) and parity-tested.
static uint32_t plan_heavy(uint32_t nt) {
	int const mode = env_mode();
	if (mode == EM_GLOBAL) return 0;
	if (mode == EM_WINDOW) return nt;
	uint32_t const all_below = (uint32_t)env_int("TW_EROSION_WINDOW_ALL", 0), heavy = (uint32_t)env_int("TW_EROSION_HEAVY", 0);
	return (nt <= all_below) ? nt : (heavy < nt ? heavy : nt);
}

int twi_ensure_heavy(tw_ctx *ctx, int lane) {
	if (ctx->heavy_stream[lane]) return TW_OK;
	int lo = 0, hi = 0;
	TW_CUDA(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
	TW_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->heavy_stream[lane], cudaStreamNonBlocking, hi)); // the serial chains of the heaviest maps go first
	TW_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork[lane], cudaEventDisableTiming));
	TW_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_join[lane], cudaEventDisableTiming));
	return TW_OK;
}

// twi_erode_enqueue's scratch for `capacity` padded maps: the maps, then the schedule's [work | hist | order] words
static void erode_layout(twi_carve &c, uint32_t capacity, int xsize, int ysize, float *&d_pad, unsigned *&d_work) {
	d_pad = c.take<float>((size_t)capacity*(xsize + 2*PAD)*(ysize + 2*PAD)); d_work = c.take<unsigned>((size_t)capacity*2 + WORK_BINS);
}

size_t twi_erode_scratch_bytes(const tw_ctx *ctx, uint32_t chunk, int xsize, int ysize) {
	if (plan_whole(ctx->num_sms, chunk, xsize, ysize)) return 256; // no padded copy
	twi_carve c; float *d_pad; unsigned *d_work; erode_layout(c, chunk, xsize, ysize, d_pad, d_work);
	return c.bytes;
}

// Enqueue the erosion of nt <= 65535 heightmaps on `st`, using `scratch` (twi_erode_scratch_bytes(capacity,..) bytes). `lane` (0..2) selects
// the context's fork/join stream for the heavy part. No synchronisation; d_steps (device counter) accumulates the droplet moves.
int twi_erode_enqueue(tw_ctx *ctx, cudaStream_t st, int lane, void *scratch, uint32_t capacity, float *maps, uint32_t nt, int xsize, int ysize,
                      const float *d_min_zvals, float min_zval_all, uint32_t num_iters, const tw_erosion_params *p, unsigned long long *d_steps,
                      const unsigned *d_perm)
{
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	size_t const padded_elems = (size_t)NX*NY;
	DArgs A;
	memset(&A, 0, sizeof(A));
	A.E = make_eparams(p);
	A.xsize = xsize; A.ysize = ysize; A.num_iters = num_iters; A.dir_table = ctx->d_dir_table; A.steps_out = d_steps;
	A.min_zvals = d_min_zvals; A.min_zval_all = min_zval_all; A.jw = ctx->in_job ? ctx->d_job_words : nullptr;
	if (plan_whole(ctx->num_sms, nt, xsize, ysize)) { // whole maps in shared memory, straight from / to the caller's tiles
		A.maps = maps; A.slot0 = 0; A.nslots = nt; A.perm = d_perm;
		A.WX = NX; A.WY = NY; A.P = whole_pitch(NX, NY); A.win_elems = (unsigned)A.P*NY;
		launch_droplets_g<M_WHOLE>(pick_smem_group(), st, A, 1, (size_t)A.win_elems*sizeof(float));
		TW_LAUNCH_CHECK(ctx);
		return TW_OK;
	}
	twi_carve c{(char *)scratch}; float *d_pad; unsigned *d_work; erode_layout(c, capacity, xsize, ysize, d_pad, d_work);
	unsigned *d_hist = d_work + capacity, *d_order = d_hist + WORK_BINS;
	bool const schedule = (nt > ctx->num_sms*4u); // with few heightmaps everything is resident at once anyway
	if (schedule) {TW_CUDA(ctx, cudaMemsetAsync(d_work, 0, ((size_t)capacity + WORK_BINS)*sizeof(unsigned), st));}
	pad_kernel<<<dim3((NX + 255)/256, NY, nt), 256, 0, st>>>(maps, d_pad, xsize, ysize, NX, NY, A.E.wpz_minus_half_dxy, schedule ? d_work : nullptr, d_perm);
	TW_LAUNCH_CHECK(ctx);
	if (schedule) {int const rc = twi_order_by_work(ctx, st, d_work, nt, (unsigned)padded_elems, d_hist, d_order); if (rc) return rc;}
	else {d_order = nullptr;}
	A.padded = d_pad; A.order = d_order;
	uint32_t const heavy = plan_heavy(nt);
	bool const fork = (heavy > 0 && heavy < nt);
	if (heavy > 0) { // latency mode: shared-memory windows for the maps with the longest serial chains
		DArgs W = A;
		int const wsz = env_int("TW_EROSION_WIN", 32);
		W.slot0 = 0; W.nslots = heavy;
		W.WX = std::min(std::max(wsz, 8), NX); W.WY = std::min(std::max(wsz, 8), NY);
		W.P = whole_pitch(W.WX, W.WY); W.win_elems = (unsigned)W.P*W.WY;
		W.win_min_moves = (unsigned)env_int("TW_EROSION_WIN_MIN_MOVES", (nt == 1) ? 0 : 2);
		cudaStream_t hs = st;
		if (fork) {
			int const rc = twi_ensure_heavy(ctx, lane); if (rc) return rc;
			hs = ctx->heavy_stream[lane];
			TW_CUDA(ctx, cudaEventRecord(ctx->ev_fork[lane], st));
			TW_CUDA(ctx, cudaStreamWaitEvent(hs, ctx->ev_fork[lane], 0));
		}
		launch_droplets_g<M_WINDOW>(pick_smem_group(), hs, W, 2, (size_t)W.win_elems*sizeof(float));
		TW_LAUNCH_CHECK(ctx);
		if (fork) {TW_CUDA(ctx, cudaEventRecord(ctx->ev_join[lane], hs));}
	}
	if (heavy < nt) { // throughput mode for the rest
		DArgs T = A;
		T.slot0 = heavy; T.nslots = nt - heavy;
		launch_droplets_g<M_GLOBAL>(pick_group(nt - heavy), st, T, 2, 0);
		TW_LAUNCH_CHECK(ctx);
	}
	if (fork) {TW_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_join[lane], 0));}
	unpad_kernel<<<dim3((xsize + 255)/256, ysize, nt), 256, 0, st>>>(d_pad, maps, xsize, ysize, NX, NY, d_min_zvals, min_zval_all, d_perm);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// heaviest-first order of nt items by their work estimate (counting sort, 256 bins); d_hist256 is zeroed by the caller
int twi_order_by_work(tw_ctx *ctx, cudaStream_t st, const unsigned *d_work, uint32_t nt, unsigned max_work, unsigned *d_hist256, unsigned *d_order) {
	order_hist_kernel<<<(nt + 255)/256, 256, 0, st>>>(d_work, nt, max_work, d_hist256);
	TW_LAUNCH_CHECK(ctx);
	order_scan_kernel<<<1, 32, 0, st>>>(d_hist256);
	TW_LAUNCH_CHECK(ctx);
	order_scatter_kernel<<<(nt + 255)/256, 256, 0, st>>>(d_work, nt, max_work, d_hist256, d_order);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// largest chunk (heightmaps per enqueue) whose scratch fits in `budget` bytes
uint32_t twi_erode_chunk_for(size_t budget, uint32_t ntiles, int xsize, int ysize) {
	size_t const per = (size_t)(xsize + 2*PAD)*(ysize + 2*PAD)*sizeof(float) + 2*sizeof(unsigned);
	size_t c = budget/per;
	if (c < 1) c = 1;
	if (c > ntiles) c = ntiles;
	if (c > 65535) c = 65535; // gridDim.z limit
	return (uint32_t)c;
}

size_t twi_erode_parallel_scratch_bytes(int xsize, int ysize) {return (size_t)(xsize + 2*PAD)*(ysize + 2*PAD)*sizeof(float);}

// tw_erode_parallel's work on ctx->stream, nothing waits: pad into `scratch` (twi_erode_parallel_scratch_bytes), the droplets, unpad with the lower clamp
// *d_min_zval (nullptr: min_zval). d_steps accumulates the droplet moves (the caller zeroes it); d_next is the droplet counter, zeroed here.
int twi_erode_parallel_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zval, float min_zval, uint32_t num_iters,
                               const tw_erosion_params *p, uint32_t num_threads, unsigned long long *d_steps, unsigned *d_next) {
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	float *d_pad = (float *)scratch;
	cudaStream_t const st = ctx->stream;
	TW_CUDA(ctx, cudaMemsetAsync(d_next, 0, sizeof(unsigned), st));
	DArgs A;
	memset(&A, 0, sizeof(A));
	A.E = make_eparams(p);
	pad_kernel<<<dim3((NX + 255)/256, NY, 1), 256, 0, st>>>(d_map, d_pad, xsize, ysize, NX, NY, A.E.wpz_minus_half_dxy, nullptr);
	TW_LAUNCH_CHECK(ctx);
	unsigned groups = num_threads ? num_threads : 65536u; // auto: the 65536-map operating point of pick_group() (8 lanes per droplet)
	if (groups > num_iters) {groups = num_iters;}
	A.padded = d_pad; A.ntiles = groups; A.slot0 = 0; A.nslots = groups; A.xsize = xsize; A.ysize = ysize; A.num_iters = num_iters;
	A.dir_table = ctx->d_dir_table; A.steps_out = d_steps; A.next_droplet = d_next; A.jw = ctx->in_job ? ctx->d_job_words : nullptr;
	launch_droplets_g<M_ATOMIC>(pick_group(groups), st, A, 2, 0);
	TW_LAUNCH_CHECK(ctx);
	unpad_kernel<<<dim3((xsize + 255)/256, ysize, 1), 256, 0, st>>>(d_pad, d_map, xsize, ysize, NX, NY, d_min_zval, min_zval);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// tw_erode_parallel: `num_threads` droplets of ONE heightmap in flight (0 = as many groups as keep the GPU busy)
int twi_erode_parallel(tw_ctx *ctx, float *d_map, int xsize, int ysize, float min_zval, uint32_t num_iters, const tw_erosion_params *p, uint32_t num_threads) {
	ctx->last_erosion_steps = 0;
	if (num_iters == 0 || p->erode_amount <= 0.0) return TW_OK; // erosion disabled, src/erosion.cpp:16
	if (xsize <= 0 || ysize <= 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_erode_parallel: empty heightmap");
	if (!ctx->d_dir_table) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	int rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words));
	if (rc) return rc;
	unsigned long long *d_steps = &twi_slot2(ctx)->steps;
	TW_CUDA(ctx, cudaMemsetAsync(d_steps, 0, sizeof(unsigned long long), ctx->stream));
	rc = tw_reserve(ctx, 1, twi_erode_parallel_scratch_bytes(xsize, ysize));
	if (rc) return rc;
	rc = twi_erode_parallel_enqueue(ctx, ctx->d_scratch[1], d_map, xsize, ysize, nullptr, min_zval, num_iters, p, num_threads, d_steps, &twi_slot2(ctx)->next);
	if (rc) return rc;
	cudaStream_t const st = ctx->stream;
	unsigned long long h_steps = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&h_steps, d_steps, sizeof(h_steps), cudaMemcpyDeviceToHost, st));
	TW_CUDA(ctx, cudaStreamSynchronize(st));
	ctx->last_erosion_steps = h_steps;
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ M_SPEC: exact serial order, speculatively parallel
namespace {
__global__ void spec_init_kernel(SpecArgs S, unsigned num_iters, size_t ntile_stamps) {
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i < ntile_stamps) {S.stamps[i] = SP_NONE;}
	if (i < S.B) {
		unsigned const s = (unsigned)i;
		S.it[s] = s; S.status[s] = (s < num_iters) ? SP_DIRTY : SP_EMPTY; // slot s starts with droplet s
		S.nlog[s] = 0; S.ntiles[s] = 0; S.nseg[s] = 0; S.minw[s] = SP_NONE; S.steps[s] = 0;
	}
	if (i == 0) {S.ctl[0] = 0; S.ctl[1] = 0; S.ctl[2] = SP_NONE; S.ctl[3] = 0; S.ctl[4] = 0; for (int k = 5; k <= (int)SP_CTL_ROUND; ++k) {S.ctl[k] = 0;}}
}
// The bookkeeping of one round: ONE thread-block cluster of 8 x 1024 threads = 256 warps, one warp per slot, cluster.sync() between the phases (a hardware
// barrier: the blocks of a cluster are co-scheduled, so unlike a grid-wide barrier it cannot dead-lock). Every slot's chain of dependent loads runs beside
// the others'; as three kernels this cost three launches per round, as one block 8-16 slots per warp one after the other.
//   stamp     every walked, uncommitted droplet (finished or suspended) stamps its tiles with its index; the lowest index wins
//   validate  a droplet conflicts if a lower-indexed droplet of the window touched one of its tiles; f = the first droplet that cannot be committed
//   commit    the prefix [lo, f): the logs go into the map (disjoint tiles: any order), the slots get their next droplets; behind f, droplets whose tiles a
//             committed droplet touched are walked again from the start; every stamping droplet takes its stamps back
// The kernel advances the round counter. In the graph form (spec_loop_graph: the body of a conditional WHILE node) it also ends the loop once every droplet is
// committed, or - with *fail = the rounds run - after max_rounds + 1 rounds without finishing; the host-driven form passes max_rounds = UINT_MAX. In the graph
// form a cancelled job (tw_cancel, the job words jw) also ends the loop after the round; the host-driven form (tw_erode) is never cancelled.
constexpr unsigned SPEC_CLUSTER = 8, SPEC_MAX_SLOTS = SPEC_CLUSTER*32;
__global__ void __cluster_dims__(SPEC_CLUSTER, 1, 1) __launch_bounds__(1024) spec_round_kernel(SpecArgs S, unsigned num_iters, float *__restrict__ padded, int NX, unsigned long long *__restrict__ steps_total,
                                                                                               unsigned max_rounds, unsigned *__restrict__ fail, cudaGraphConditionalHandle loop, bool in_graph,
                                                                                               twi_job_words *jw) {
	namespace cg = cooperative_groups;
	cg::cluster_group cluster = cg::this_cluster();
	unsigned const s = (blockIdx.x*blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	unsigned const round = S.ctl[SP_CTL_ROUND]; // written below only after the last cluster.sync(), when every thread has read it
	unsigned const lo = S.ctl[round & 1u], hi = (num_iters - lo < S.B) ? num_iters : lo + S.B, hs = lo % S.B;
	bool const mine = (s < S.B);
	unsigned const st = mine ? S.status[s] : SP_EMPTY, it = mine ? S.it[s] : SP_NONE, nt = mine ? S.ntiles[s] : 0u;
	bool const live = mine && st != SP_EMPTY && it < num_iters, stamps = live && (st == SP_VALID || st == SP_WALKING);
	bool const inplace_round = (lo < num_iters && S.status[hs] == SP_INPLACE && S.it[hs] == lo); // in-place head with an incomplete tile list: everything else is stale
	const unsigned *t = S.tiles + (size_t)s*S.T;
	// ctl[2] (first uncommittable droplet) was reset by the previous round's kernel (or the init kernel)
	if (stamps) {for (unsigned k = lane; k < nt; k += 32) {atomicMin(S.stamps + t[k], it);}} // ---- stamp
	cluster.sync();
	unsigned m = SP_NONE;
	if (live) { // ---- validate
		if (inplace_round) {if (lane == 0 && it != lo) {atomicMin(S.ctl + 2, lo + 1u);}}
		else if (!stamps) {if (lane == 0) {atomicMin(S.ctl + 2, it);}} // not walked yet, or outsized and waiting to become the head
		else {
			for (unsigned k = lane; k < nt; k += 32) {m = min(m, S.stamps[t[k]]);}
			for (int o = 16; o; o >>= 1) {m = min(m, __shfl_xor_sync(0xffffffffu, m, o));}
			if (lane == 0 && (m < it || st == SP_WALKING)) {atomicMin(S.ctl + 2, it);} // an unfinished walk cannot be committed either
		}
	}
	cluster.sync();
	unsigned const f = min(S.ctl[2], hi);
	if (stamps) {for (unsigned k = lane; k < nt; k += 32) {S.stamps[t[k]] = SP_NONE;}} // take the stamps back: the array is clean for the next round
	if (live) { // ---- commit / invalidate
		if (it < f) {
			if (st == SP_VALID) {
				const unsigned *cells = S.cells + (size_t)s*S.W; const float *vals = S.vals + (size_t)s*S.W; const unsigned *seg = S.seg + (size_t)s*S.R*3;
				unsigned b = 0;
				for (unsigned g = 0, ng = S.nseg[s]; g < ng; ++g) { // segment by segment: a cell logged twice gets its later value
					unsigned const e = seg[3*g]; // (end of the segment, bounding box x, bounding box z)
					for (unsigned k = b + lane; k < e; k += 32) {unsigned const cc = cells[k]; padded[(size_t)(cc >> 16)*NX + (cc & 0xffffu)] = vals[k];}
					b = e;
					__syncwarp();
				}
			}
			if (lane == 0) {
				if (st == SP_VALID || st == SP_INPLACE) {atomicAdd(steps_total, (unsigned long long)S.steps[s]);}
				unsigned const nit = it + S.B; S.it[s] = nit; S.status[s] = (nit < num_iters) ? SP_DIRTY : SP_EMPTY;
			}
		}
		else if (stamps && lane == 0 && (inplace_round || m < f)) {S.status[s] = SP_DIRTY;} // finished or not: walked again from the start
	}
	cluster.sync(); // everybody has read ctl[2] and the head's header
	if (s == 0 && lane == 0) {
		S.ctl[(round + 1u) & 1u] = f; S.ctl[2] = SP_NONE; S.ctl[SP_CTL_ROUND] = round + 1u;
		bool const done = (f >= num_iters);
		if (done) {S.ctl[3] = 1u;}
		else if (round >= max_rounds) {*fail = round + 1u;}
		bool const cancel = in_graph && !done && round < max_rounds && twi_cancelled(jw);
		if (cancel) {twi_mark_stopped(jw);}
		if (in_graph && (done || round >= max_rounds || cancel)) {cudaGraphSetConditional(loop, 0u);}
	}
}

bool spec_eligible(uint32_t nt, int xsize, int ysize, uint32_t num_iters) {
	int const mode = env_mode();
	size_t const NX = (size_t)xsize + 2*PAD, NY = (size_t)ysize + 2*PAD;
	if (nt != 1 || NX > 65535 || NY > 65535) return false;
	if (mode == EM_SPEC) return true;
	// auto: a round costs ~150 us and commits the window up to the first conflict. With t tiles of 4x4 cells and ~30 tiles per droplet the first conflict among
	// random droplets sits ~sqrt(2*t/900) droplets in: ~12 on a 1024^2 map (twice the one-warp walk's 3.5e4 droplets/s), ~6 on 512^2 (no gain), 25-45 measured
	// on 8192^2 (4x). Hence: from 2^20 cells on, and only when there are enough droplets to fill a few rounds
	return (mode == EM_AUTO && NX*NY >= ((size_t)1 << 20) && num_iters >= 64);
}
} // namespace

// M_SPEC's window: sizes from the TW_SPEC_* overrides, arrays carved by c
static void spec_layout(twi_carve &c, int xsize, int ysize, SpecArgs &S, float *&d_pad, size_t &ntile) {
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	memset(&S, 0, sizeof(S));
	S.B = (unsigned)std::max(32, std::min(env_int("TW_SPEC_WINDOW", 256), (int)SPEC_MAX_SLOTS)); S.B &= ~31u; // <= 256: the round kernel is one cluster with a warp per slot
	S.W = (unsigned)std::max(64, env_int("TW_SPEC_LOG", 8192));
	S.T = (unsigned)std::max(16, env_int("TW_SPEC_TILES", 4096)) & ~3u;
	S.R = (unsigned)std::max(2, env_int("TW_SPEC_VIEWS", 256));
	S.TNX = ((NX - 1) >> SP_TILE_SHIFT) + 1;
	S.cap = (unsigned)std::max(1, env_int("TW_SPEC_MOVES", 64));
	ntile = (size_t)S.TNX*(((NY - 1) >> SP_TILE_SHIFT) + 1);
	d_pad = c.take<float>((size_t)NX*NY);
	unsigned **slot_arrays[7] = {&S.it, &S.status, &S.nlog, &S.ntiles, &S.nseg, &S.minw, &S.steps};
	for (auto a : slot_arrays) {*a = c.take<unsigned>(S.B);}
	S.cells = c.take<unsigned>((size_t)S.B*S.W); S.vals = c.take<float>((size_t)S.B*S.W); S.tiles = c.take<unsigned>((size_t)S.B*S.T);
	S.seg = c.take<unsigned>((size_t)S.B*S.R*3); S.state = c.take<unsigned>((size_t)S.B*SP_STATE_WORDS); S.stamps = c.take<unsigned>(ntile); S.ctl = c.take<unsigned>(64);
}

// The rounds as one CUDA graph: a conditional WHILE node whose body is the walker launch and the round kernel, which clears the condition. The graph's kernel
// arguments are fixed, so it is kept in the context and rebuilt only when they change (another map size, scratch address or droplet count).
static int spec_loop_graph(tw_ctx *ctx, cudaStream_t st, DArgs const &W, unsigned num_iters, float *d_pad, int NX, unsigned long long *d_steps, unsigned max_rounds, unsigned *d_fail) {
	struct Key {DArgs W; unsigned num_iters, max_rounds; int NX; float *pad; unsigned long long *steps; unsigned *fail;} k;
	memset(&k, 0, sizeof(k));
	k.W = W; k.num_iters = num_iters; k.max_rounds = max_rounds; k.NX = NX; k.pad = d_pad; k.steps = d_steps; k.fail = d_fail;
	if (ctx->spec_graph && ctx->spec_key.size() == sizeof(k) && !memcmp(ctx->spec_key.data(), &k, sizeof(k))) return TW_OK;
	if (ctx->spec_graph) {cudaGraphExecDestroy(ctx->spec_graph); ctx->spec_graph = nullptr; ctx->spec_key.clear();} // a launch still in flight keeps its copy until it ends
	cudaGraph_t g = nullptr;
	cudaGraphExec_t ex = nullptr;
	cudaGraphConditionalHandle h = 0;
	cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
	cudaError_t e = cudaGraphCreate(&g, 0);
	if (e == cudaSuccess) {e = cudaGraphConditionalHandleCreate(&h, g, 1u, cudaGraphCondAssignDefault);}
	if (e == cudaSuccess) {
		cudaGraphNode_t node;
		np.conditional.handle = h; np.conditional.type = cudaGraphCondTypeWhile; np.conditional.size = 1;
		e = cudaGraphAddNode(&node, g, nullptr, 0, &np);
	}
	if (e == cudaSuccess) {e = cudaStreamBeginCaptureToGraph(st, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed);}
	if (e == cudaSuccess) {
		launch_droplets<32, M_SPEC>(st, W, 4, (size_t)W.win_elems*sizeof(float));
		spec_round_kernel<<<SPEC_CLUSTER, 1024, 0, st>>>(W.S, num_iters, d_pad, NX, d_steps, max_rounds, d_fail, h, true, W.jw);
		cudaError_t const le = cudaGetLastError();
		cudaGraph_t body = nullptr;
		e = cudaStreamEndCapture(st, &body);
		if (e == cudaSuccess) {e = le;}
	}
	if (e == cudaSuccess) {e = cudaGraphInstantiate(&ex, g, 0);}
	if (g) {cudaGraphDestroy(g);}
	if (e != cudaSuccess) {cudaGetLastError(); return tw_set_error(ctx, TW_ERR_CUDA, "speculative erosion graph: %s", cudaGetErrorString(e));}
	ctx->spec_graph = ex;
	ctx->spec_key.assign((const unsigned char *)&k, (const unsigned char *)&k + sizeof(k));
	return TW_OK;
}

bool twi_erode_spec_eligible(uint32_t nt, int xsize, int ysize, uint32_t num_iters) {return spec_eligible(nt, xsize, ysize, num_iters);}

size_t twi_erode_spec_scratch_bytes(int xsize, int ysize) {
	twi_carve c; SpecArgs S; float *d_pad; size_t ntile; spec_layout(c, xsize, ysize, S, d_pad, ntile);
	return c.bytes;
}

// One heightmap, the reference's serial droplet order, bit for bit (see M_SPEC at the top), on ctx->stream: pad, window set-up, the rounds, unpad with the lower
// clamp *d_min_zvals (nullptr: min_zval). scratch: twi_erode_spec_scratch_bytes() bytes. d_steps accumulates the committed moves.
// host_rounds = false: the rounds are one graph launch that ends on the device and nothing waits; *d_fail becomes the number of rounds run if the window stopped
// making progress (0 otherwise). host_rounds = true (tw_erode): the rounds are queued from the host, which reads the "done" flag every 8 rounds and returns the
// no-progress error itself; on the BASELINE 8192^2 map this was 1-2 % faster than the graph with 1000 droplets and equal with 1e5 (DESIGN.md section 4e).
int twi_erode_spec_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zvals, float min_zval, uint32_t num_iters,
                           const tw_erosion_params *p, unsigned long long *d_steps, unsigned *d_fail, bool host_rounds) {
	volatile unsigned *h_done = nullptr;
	if (host_rounds) {int const rc = tw_reserve_pinned(ctx, 64); if (rc) return rc; h_done = (volatile unsigned *)ctx->h_pinned;}
	cudaStream_t const st = ctx->stream;
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	SpecArgs S;
	float *d_pad = nullptr;
	size_t ntile = 0;
	twi_carve c{(char *)scratch}; spec_layout(c, xsize, ysize, S, d_pad, ntile);
	DArgs A;
	memset(&A, 0, sizeof(A));
	A.E = make_eparams(p);
	A.xsize = xsize; A.ysize = ysize; A.num_iters = num_iters; A.dir_table = ctx->d_dir_table;
	A.padded = d_pad; A.slot0 = 0; A.jw = ctx->in_job ? ctx->d_job_words : nullptr; // the graph's round kernel reads them (tw_erode's host rounds never do)
	pad_kernel<<<dim3((NX + 255)/256, NY, 1), 256, 0, st>>>(d_map, d_pad, xsize, ysize, NX, NY, A.E.wpz_minus_half_dxy, nullptr, nullptr);
	TW_LAUNCH_CHECK(ctx);
	size_t const init_n = std::max(ntile, (size_t)S.B);
	spec_init_kernel<<<(unsigned)((init_n + 255)/256), 256, 0, st>>>(S, num_iters, ntile);
	TW_LAUNCH_CHECK(ctx);
	TW_CUDA(ctx, cudaMemsetAsync(d_fail, 0, sizeof(unsigned), st));
	DArgs W = A; // the speculative walkers: one warp per slot, a private 32 x 32 view + 32 words of dirty bits each
	W.nslots = S.B; W.steps_out = nullptr; W.S = S;
	W.WX = std::min(32, NX); W.WY = std::min(32, NY); W.P = whole_pitch(W.WX, W.WY); W.win_elems = (unsigned)(W.P*W.WY + 32);
	unsigned const max_rounds = 2*num_iters + 64;
	if (host_rounds) {
		unsigned const min_rounds = (num_iters + S.B - 1)/S.B;
		for (unsigned round = 0;; ++round) {
			if (round > max_rounds) return tw_set_error(ctx, TW_ERR_STATE, "speculative erosion made no progress (%u rounds)", round);
			launch_droplets<32, M_SPEC>(st, W, 4, (size_t)W.win_elems*sizeof(float));
			spec_round_kernel<<<SPEC_CLUSTER, 1024, 0, st>>>(S, num_iters, d_pad, NX, d_steps, 0xffffffffu, d_fail, 0, false, nullptr);
			TW_LAUNCH_CHECK(ctx);
			if (round + 1 >= min_rounds && (round & 7u) == 7u) { // poll "done" every 8 rounds (not before the window can have covered all droplets): the rounds in between are queued back to back
				TW_CUDA(ctx, cudaMemcpyAsync((void *)h_done, S.ctl + 3, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
				TW_CUDA(ctx, cudaStreamSynchronize(st));
				if (*h_done) break;
			}
		}
	}
	else {
		int const rc = spec_loop_graph(ctx, st, W, num_iters, d_pad, NX, d_steps, max_rounds, d_fail);
		if (rc) return rc;
		TW_CUDA(ctx, cudaGraphLaunch(ctx->spec_graph, st));
		ctx->launches++;
	}
	unpad_kernel<<<dim3((xsize + 255)/256, ysize, 1), 256, 0, st>>>(d_pad, d_map, xsize, ysize, NX, NY, d_min_zvals, min_zval, nullptr);
	TW_LAUNCH_CHECK(ctx);
	if (getenv("TW_SPEC_STATS")) {
		unsigned h[SP_CTL_ROUND + 1];
		TW_CUDA(ctx, cudaMemcpyAsync(h, S.ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
		TW_CUDA(ctx, cudaStreamSynchronize(st));
		unsigned const spec_rounds = std::max(1u, h[SP_CTL_ROUND]);
		fprintf(stderr, "tw spec: %u droplets, window %u: %u rounds (%.1f commits per round), %u walks (%.2f per droplet), %u outgrew their log (log %u, views %u, tiles %u, outside view %u, non-finite at the corner %u), %u walked in place; longest walk %u moves\n",
		        num_iters, S.B, spec_rounds, (double)num_iters/spec_rounds, h[6], (double)h[6]/num_iters, h[7], h[8], h[9], h[10], h[11], h[12], h[5], h[13]);
	}
	return TW_OK;
}

int twi_erode(tw_ctx *ctx, float *d_maps, uint32_t ntiles, int xsize, int ysize, const float *d_min_zvals, float min_zval_all,
              uint32_t num_iters, const tw_erosion_params *p)
{
	ctx->last_erosion_steps = 0;
	if (num_iters == 0 || p->erode_amount <= 0.0) return TW_OK; // erosion disabled, src/erosion.cpp:16
	if (xsize <= 0 || ysize <= 0 || ntiles == 0) return tw_set_error(ctx, TW_ERR_ARG, "tw_erode: empty heightmap");
	if (!ctx->d_dir_table) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	int rc = tw_reserve(ctx, 2, sizeof(twi_slot2_words));
	if (rc) return rc;
	unsigned long long *d_steps = &twi_slot2(ctx)->steps;
	TW_CUDA(ctx, cudaMemsetAsync(d_steps, 0, sizeof(unsigned long long), ctx->stream));
	if (spec_eligible(ntiles, xsize, ysize, num_iters)) { // one big map: the serial order, walked speculatively in parallel and committed in order (M_SPEC)
		rc = tw_reserve(ctx, 1, twi_erode_spec_scratch_bytes(xsize, ysize));
		if (rc) return rc;
		unsigned *d_fail = &twi_slot2(ctx)->fail;
		rc = twi_erode_spec_enqueue(ctx, ctx->d_scratch[1], d_maps, xsize, ysize, d_min_zvals, min_zval_all, num_iters, p, d_steps, d_fail, true);
		if (rc) return rc;
		unsigned long long h_steps = 0;
		TW_CUDA(ctx, cudaMemcpyAsync(&h_steps, d_steps, sizeof(h_steps), cudaMemcpyDeviceToHost, ctx->stream));
		TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		ctx->last_erosion_steps = h_steps;
		return TW_OK;
	}
	// process heightmaps in chunks so that the padded scratch stays within a third of the free device memory (each chunk has its own
	// heaviest-first schedule and its own tail, so fewer, larger chunks are better)
	size_t free_b = 0, total_b = 0;
	TW_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
	size_t budget = (free_b + ctx->scratch_bytes[1])/3;
	if (budget < ((size_t)1 << 30)) budget = (size_t)1 << 30;
	uint32_t const chunk = twi_erode_chunk_for(budget, ntiles, xsize, ysize);
	rc = tw_reserve(ctx, 1, twi_erode_scratch_bytes(ctx, chunk, xsize, ysize));
	if (rc) return rc;
	for (uint32_t t0 = 0; t0 < ntiles; t0 += chunk) {
		uint32_t const nt = (ntiles - t0 < chunk) ? (ntiles - t0) : chunk;
		rc = twi_erode_enqueue(ctx, ctx->stream, 0, ctx->d_scratch[1], chunk, d_maps + (size_t)t0*xsize*ysize, nt, xsize, ysize,
		                       d_min_zvals ? d_min_zvals + t0 : nullptr, min_zval_all, num_iters, p, d_steps);
		if (rc) return rc;
	}
	unsigned long long h_steps = 0;
	TW_CUDA(ctx, cudaMemcpyAsync(&h_steps, d_steps, sizeof(h_steps), cudaMemcpyDeviceToHost, ctx->stream));
	TW_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	ctx->last_erosion_steps = h_steps;
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ coherent batched erosion (tw_erode_sweeps*)
// Building blocks of the sweep algorithm (M_FROZEN above) for one device's band of the padded map; everything is enqueued on ctx->stream.
namespace {
// P[Y - E0][X] = U[clamp(Y - PAD) - u0][clamp(X - PAD)]: the clamped PAD border of src/erosion.cpp:31-37 for the stored rows [E0, E0 + rows)
__global__ void sweep_pad_kernel(const float *__restrict__ U, int u0, int xsize, int ysize, int E0, int rows, int NX, float *__restrict__ P) {
	int const X = blockIdx.x*blockDim.x + threadIdx.x, r = blockIdx.y;
	if (X >= NX || r >= rows) return;
	int const sy = clampi(E0 + r - PAD, ysize - 1), sx = clampi(X - PAD, xsize - 1);
	P[(size_t)r*NX + X] = __ldg(U + (size_t)(sy - u0)*xsize + sx);
}
__global__ void sweep_add_kernel(long long *__restrict__ D, const long long *__restrict__ R, size_t n) { // deltas received from a neighbour: integer sum, exact
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) {D[i] += R[i];}
}
__global__ void sweep_apply_kernel(float *__restrict__ P, long long *__restrict__ D, size_t n) { // map += deltas (one conversion, one fp32 add per cell), deltas = 0
	size_t const i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) {
		long long const d = D[i];
		if (d) {P[i] = P[i] + (float)((double)d*(1.0/FIXED_ONE)); D[i] = 0;}
		else   {P[i] = P[i] + 0.0f;} // the oracle adds unconditionally: -0.0 + 0.0 = +0.0
	}
}
// out[y - y0][x] = max(min_zval, P[(y + PAD) - E0][x + PAD]) for the owned un-padded rows [y0, y1) (src/erosion.cpp:158-162)
__global__ void sweep_unpad_kernel(const float *__restrict__ P, int E0, int NX, int xsize, int y0, int y1, float min_zval, float *__restrict__ out) {
	int const x = blockIdx.x*blockDim.x + threadIdx.x, y = y0 + blockIdx.y;
	if (x >= xsize || y >= y1) return;
	out[(size_t)(y - y0)*xsize + x] = smax(min_zval, P[(size_t)(y + PAD - E0)*NX + x + PAD]);
}
} // namespace

int twi_sweep_pad(tw_ctx *ctx, const float *U, int u0, int xsize, int ysize, int E0, int rows, float *P) {
	int const NX = xsize + 2*PAD;
	sweep_pad_kernel<<<dim3((NX + 255)/256, rows), 256, 0, ctx->stream>>>(U, u0, xsize, ysize, E0, rows, NX, P);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_sweep_view() {return TW_SWEEP_VIEW;}
int twi_sweep_walk(tw_ctx *ctx, float *P, long long *D, int xsize, int ysize, int E0, int own0, int own1, int halo_rule, unsigned it0, unsigned it1,
                   const tw_erosion_params *p, unsigned long long *d_steps)
{
	if (!ctx->d_dir_table) return tw_set_error(ctx, TW_ERR_STATE, "tw_set_sin_table() has not been called");
	DArgs A;
	memset(&A, 0, sizeof(A));
	A.E = make_eparams(p);
	A.padded = P; A.delta = D; A.row0 = E0; A.own0 = own0; A.own1 = own1; A.halo_rule = halo_rule; A.it0 = it0; A.it1 = it1;
	A.xsize = xsize; A.ysize = ysize; A.dir_table = ctx->d_dir_table; A.steps_out = d_steps;
	constexpr unsigned G = 8;
	unsigned const per_sweep = it1 - it0;
	unsigned groups = std::min(per_sweep, ctx->num_sms*12u*(32u/G)); // one droplet per group at a time; a few waves' worth of 8-lane groups
	A.slot0 = 0; A.nslots = groups;
	A.WX = std::min(TW_SWEEP_VIEW, xsize + 2*PAD); A.WY = std::min(TW_SWEEP_VIEW, ysize + 2*PAD);
	A.P = whole_pitch(A.WX, A.WY); A.win_elems = (unsigned)A.P*A.WY;
	launch_droplets<G, M_FROZEN>(ctx->stream, A, 2, (size_t)A.win_elems*sizeof(float));
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_sweep_add(tw_ctx *ctx, long long *D, const long long *R, size_t n) {
	sweep_add_kernel<<<(unsigned)((n + 255)/256), 256, 0, ctx->stream>>>(D, R, n);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_sweep_apply(tw_ctx *ctx, float *P, long long *D, size_t n) {
	sweep_apply_kernel<<<(unsigned)((n + 255)/256), 256, 0, ctx->stream>>>(P, D, n);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
int twi_sweep_unpad(tw_ctx *ctx, const float *P, int E0, int xsize, int y0, int y1, float min_zval, float *out) {
	sweep_unpad_kernel<<<dim3((xsize + 255)/256, y1 - y0), 256, 0, ctx->stream>>>(P, E0, xsize + 2*PAD, xsize, y0, y1, min_zval, out);
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}

// ------------------------------------------------------------------------------------------------ tw_erode_sweeps of one map as a job
namespace {
// The end of a sweep in the job's loop: the next sweep's first droplet into *it0, or - after the last sweep, or once the job is cancelled (tw_cancel; the
// job is then marked stopped) - the end of the loop. The walk and the apply of the sweep it follows have finished: this is the loop's cancellation point.
__global__ void sweep_advance_kernel(unsigned *it0, unsigned sweep, unsigned num_iters, twi_job_words *jw, cudaGraphConditionalHandle loop) {
	unsigned const a = *it0;
	bool const last = (num_iters - a <= sweep);
	if (!last) {*it0 = a + sweep;}
	bool const cancel = !last && twi_cancelled(jw);
	if (cancel) {twi_mark_stopped(jw);}
	if (last || cancel) {cudaGraphSetConditional(loop, 0u);}
}
// the sweeps job's scratch: the padded map (n cells), its fixed-point deltas and the sweep word
void sweeps_layout(twi_carve &c, size_t n, float *&P, long long *&D, unsigned *&ctl) {P = c.take<float>(n); D = c.take<long long>(n); ctl = c.take<unsigned>(1);}
} // namespace

size_t twi_erode_sweeps_scratch_bytes(int xsize, int ysize) {
	twi_carve c; float *P; long long *D; unsigned *ctl; sweeps_layout(c, (size_t)(xsize + 2*PAD)*(ysize + 2*PAD), P, D, ctl);
	return c.bytes;
}

// The sweeps as one CUDA graph: a conditional WHILE node whose body is the walk of a sweep, the apply and sweep_advance_kernel, which clears the condition.
// Its kernel arguments are fixed, so it is kept in the context and rebuilt only when they change (another map size, scratch address, droplet count, sweep,
// halo or erosion parameters), as spec_loop_graph does.
static int sweep_loop_graph(tw_ctx *ctx, cudaStream_t st, DArgs const &W, long long *D, size_t n, unsigned *ctl) {
	struct Key {DArgs W; long long *D; size_t n; unsigned *ctl;} k;
	memset(&k, 0, sizeof(k));
	k.W = W; k.D = D; k.n = n; k.ctl = ctl;
	if (ctx->sweep_graph && ctx->sweep_key.size() == sizeof(k) && !memcmp(ctx->sweep_key.data(), &k, sizeof(k))) return TW_OK;
	if (ctx->sweep_graph) {cudaGraphExecDestroy(ctx->sweep_graph); ctx->sweep_graph = nullptr; ctx->sweep_key.clear();} // a launch still in flight keeps its copy until it ends
	cudaGraph_t g = nullptr;
	cudaGraphExec_t ex = nullptr;
	cudaGraphConditionalHandle h = 0;
	cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
	cudaError_t e = cudaGraphCreate(&g, 0);
	if (e == cudaSuccess) {e = cudaGraphConditionalHandleCreate(&h, g, 1u, cudaGraphCondAssignDefault);}
	if (e == cudaSuccess) {
		cudaGraphNode_t node;
		np.conditional.handle = h; np.conditional.type = cudaGraphCondTypeWhile; np.conditional.size = 1;
		e = cudaGraphAddNode(&node, g, nullptr, 0, &np);
	}
	if (e == cudaSuccess) {e = cudaStreamBeginCaptureToGraph(st, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed);}
	if (e == cudaSuccess) {
		launch_droplets<8, M_FROZEN>(st, W, 2, (size_t)W.win_elems*sizeof(float));
		sweep_apply_kernel<<<(unsigned)((n + 255)/256), 256, 0, st>>>(W.padded, D, n);
		sweep_advance_kernel<<<1, 1, 0, st>>>(ctl, W.sweep, W.num_iters, W.jw, h);
		cudaError_t const le = cudaGetLastError();
		cudaGraph_t body = nullptr;
		e = cudaStreamEndCapture(st, &body);
		if (e == cudaSuccess) {e = le;}
	}
	if (e == cudaSuccess) {e = cudaGraphInstantiate(&ex, g, 0);}
	if (g) {cudaGraphDestroy(g);}
	if (e != cudaSuccess) {cudaGetLastError(); return tw_set_error(ctx, TW_ERR_CUDA, "erosion sweeps graph: %s", cudaGetErrorString(e));}
	ctx->sweep_graph = ex;
	ctx->sweep_key.assign((const unsigned char *)&k, (const unsigned char *)&k + sizeof(k));
	return TW_OK;
}

// tw_erode_sweeps' one-band path on ctx->stream inside a job, nothing waits and nothing is allocated: pad d_map into `scratch`
// (twi_erode_sweeps_scratch_bytes), zero the deltas and the sweep word, the sweeps as one graph launch that ends on the device, unpad with the lower clamp
// *d_min_zval (nullptr: min_zval). d_steps accumulates the droplet moves (the caller zeroes it). The caller has checked sweep and halo as tw_erode_sweeps does.
int twi_erode_sweeps_enqueue(tw_ctx *ctx, void *scratch, float *d_map, int xsize, int ysize, const float *d_min_zval, float min_zval, uint32_t num_iters,
                             const tw_erosion_params *p, uint32_t sweep, int halo, unsigned long long *d_steps) {
	cudaStream_t const st = ctx->stream;
	int const NX = xsize + 2*PAD, NY = ysize + 2*PAD;
	size_t const n = (size_t)NX*NY;
	twi_carve c{(char *)scratch}; float *P; long long *D; unsigned *ctl; sweeps_layout(c, n, P, D, ctl);
	TW_CUDA(ctx, cudaMemsetAsync(D, 0, n*sizeof(long long), st));
	TW_CUDA(ctx, cudaMemsetAsync(ctl, 0, sizeof(unsigned), st));
	pad_kernel<<<dim3((NX + 255)/256, NY, 1), 256, 0, st>>>(d_map, P, xsize, ysize, NX, NY, 0.0f, nullptr, nullptr); // = sweep_pad_kernel of the one band
	TW_LAUNCH_CHECK(ctx);
	DArgs A; // twi_sweep_walk's arguments for the one band (rows [0, NY) stored and owned), with the sweep's bounds on the device
	memset(&A, 0, sizeof(A));
	A.E = make_eparams(p);
	A.padded = P; A.delta = D; A.row0 = 0; A.own0 = 0; A.own1 = NY; A.halo_rule = halo - TW_SWEEP_VIEW - PAD;
	A.xsize = xsize; A.ysize = ysize; A.num_iters = num_iters; A.dir_table = ctx->d_dir_table; A.steps_out = d_steps;
	A.jw = ctx->d_job_words; A.sweep_it0 = ctl; A.sweep = sweep;
	A.slot0 = 0; A.nslots = std::min(sweep, ctx->num_sms*12u*4u); // twi_sweep_walk's groups of a full sweep; the result does not depend on them
	A.WX = std::min(TW_SWEEP_VIEW, NX); A.WY = std::min(TW_SWEEP_VIEW, NY);
	A.P = whole_pitch(A.WX, A.WY); A.win_elems = (unsigned)A.P*A.WY;
	int const rc = sweep_loop_graph(ctx, st, A, D, n, ctl);
	if (rc) return rc;
	TW_CUDA(ctx, cudaGraphLaunch(ctx->sweep_graph, st));
	ctx->launches++;
	unpad_kernel<<<dim3((xsize + 255)/256, ysize, 1), 256, 0, st>>>(P, d_map, xsize, ysize, NX, NY, d_min_zval, min_zval, nullptr); // = sweep_unpad_kernel of the one band
	TW_LAUNCH_CHECK(ctx);
	return TW_OK;
}
