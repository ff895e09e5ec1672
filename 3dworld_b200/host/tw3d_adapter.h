// tw3d_adapter.h - C++ host adapter: the reference's own call surface for the terrain path, implemented on the C ABI (include/tw3d.h).
//
//   tw3d::mesh_xy_grid_cache_t   <->  mesh_xy_grid_cache_t                    src/mesh.h:22-45, src/mesh_gen.cpp:588-650,754-792
//   tw3d::apply_erosion          <->  apply_erosion(float*,int,int,float,unsigned)   src/function_registry.h:354, src/erosion.cpp:14
//   tw3d::erode_heightmap_async  <->  heightmap_t::run_erosion on the set_heightmap image, without stalling the frame   src/heightmap.cpp:153-187
//   tw3d::noise_gen_3d           <->  noise_gen_3d::{set_rand_seeds,gen_sines}        src/upsurface.h:39-50
//   tw3d::create_procedural      <->  voxel_manager::create_procedural               src/voxels.h:196, src/voxels.cpp:278-346
//   tw3d::voxel_mesh             <->  voxel_model::create_block's welded tri_verts    src/voxels.cpp:495-566,1077-1108
//   tw3d::voxel_model            <->  voxel_model's brush edits + per-block create_block src/voxels.cpp:1077-1108,2139-2245
//   tw3d::create_zvals_batch     <->  the height fill + erosion of tile_t::create_zvals for many tiles   src/tiled_mesh.cpp:467-515
//   tw3d::create_tiles_async     <->  a frame's new tiles launched in tile_draw_t::update and collected on a later frame   src/tiled_mesh.cpp:2367-2417
//   tw3d::create_tiles_async_from_heightmap  <->  the same with heightmap-texture tiles (after tw3d::set_heightmap)   src/tiled_mesh.cpp:498-501
//   tw3d::update_heightmap, tw3d::hmap_tiles_touched  <->  terrain_hmap_manager_t's brush edits and re-applied modmap, and the tiles they change   src/heightmap.cpp:36-58,243-308
//   tw3d::set_deferred_gens, tw3d::tile_job_pool  <->  several of them in flight at once, as tile_draw_t::update keeps up to 8   src/tiled_mesh.cpp:2367-2417
//   tw3d::tile_set               <->  the live tiles' calc_shadows_for_light when the light moves or new tiles appear   src/tiled_mesh.cpp:664-692
//
// The reference reads ~20 globals on this path (SURVEY.md 8b); here they are one explicit struct (scene_globals) set once per scene
// with set_globals(). Same names, argument meaning and error behaviour as the reference: argument errors assert/abort like the
// reference's assert()s (define TW3D_NO_ABORT to get a tw3d::error exception instead). Header-only; link with -l3dworld_b200.
// No CPU fallback: all grid evaluation happens on the GPU through the C ABI; without a device ctx() fails.
#pragma once
#include <tw3d.h>
#include <atomic>
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

namespace tw3d {

struct error : std::runtime_error {
	int status;
	error(int s, std::string const &m) : std::runtime_error(m), status(s) {}
};

// every reference global the path reads, under the reference's own names
struct scene_globals {
	int   mesh_gen_mode = TW_MGEN_SINE, mesh_gen_shape = 0, start_eval_sin = 0, GLACIATE = 1, mesh_seed = 0, mesh_rgen_index = 0;
	float mesh_scale = 1.0f, mesh_scale_z_inv = 1.0f, DX_VAL_INV = 16.0f, DY_VAL_INV = 16.0f, MESH_HEIGHT = 0.4f, mesh_height_scale = 1.0f;
	float zmax_est = 1.0f, custom_glaciate_exp = 0.0f;
	tw_hmap_params hmap_params = {1000.0f, 0, 0, 0, 1000.0f, 0, 0, 0, 0, 0, 0, 0, 0, 0};
	int   MESH_X_SIZE = 128, MESH_Y_SIZE = 128;
	float X_SCENE_SIZE = 4.0f, Y_SCENE_SIZE = 4.0f; // get_exact_zval (src/mesh_gen.cpp:818-819)
	int   xoff2 = 0, yoff2 = 0;                      // current mesh scroll offset (src/mesh_gen.cpp:826-829)
	float mesh_file_scale = 1.0f, mesh_file_tz = 0.0f; // scale_mh_texture_val (src/mesh_gen.cpp:120), heightmap-texture tiles
	// erosion (src/erosion.cpp:11,98; src/Textures.cpp:1284-1287)
	float erode_amount = 1.0f, water_plane_z = 0.0f, HALF_DXY = 0.0625f, zmin = -1.0f, zmax = 1.0f, relh_adj_tex = 0.0f, clip_hd1 = 0.5f;
	float zbottom = 0.0f, ztop = 0.0f;                  // set_zvals (src/mesh_gen.cpp:494-504); gen_mesh leaves them alone on a flat mesh, as the reference does
	// sine-table recurrence of gen_mesh (src/mesh_gen.cpp:34,226-231; config keywords mesh_start_mag / mesh_start_freq / mesh_mag_mult / mesh_freq_mult)
	float MESH_START_MAG = 0.02f, MESH_START_FREQ = 240.0f, MESH_MAG_MULT = 2.0f, MESH_FREQ_MULT = 0.5f;
};

namespace detail {
	inline void fail(int status, const char *what, tw_ctx *c) {
		std::string msg = std::string(what) + ": " + (c ? tw_last_error(c) : "no context");
#ifdef TW3D_NO_ABORT
		throw error(status, msg);
#else
		if (status == TW_ERR_ARG) {fprintf(stderr, "tw3d: assertion failed: %s\n", msg.c_str()); abort();} // the reference asserts
		throw error(status, msg);
#endif
	}
	struct state_t {
		scene_globals g;
		std::vector<float> sin_table, sine_params;
		unsigned generation = 0; // bumped by set_globals WHEN IT IS GIVEN A TABLE, so that thread-local contexts re-upload the tables (scalars are read per call)
		std::atomic<unsigned> deferred_gens{1}; // set_deferred_gens
	};
	inline state_t &state() {static state_t s; return s;}
	struct tls_ctx {
		tw_ctx *c = nullptr; unsigned generation = ~0u;
		std::atomic<uint64_t> tile_jobs{0}; // create_tiles_async launches on c: a job whose number is no longer the latest was completed by the next launch
		int hmap_w = 0, hmap_h = 0;         // size of the image set_heightmap gave c
		std::vector<tw_ctx *> gens;         // shared contexts of c for deferred height generations (set_deferred_gens), destroyed with c
		std::vector<uint64_t> gen_launch;   // launch order on each of them
		uint64_t gen_clock = 0;
		~tls_ctx() {if (c) tw_destroy(c);}
	};
	inline tls_ctx &tls() {static thread_local tls_ctx t; return t;}
}

// thread-local context (a tw_ctx is not re-entrant); device from $TW3D_DEVICE (default 0)
inline tw_ctx *ctx() {
	detail::tls_ctx &t = detail::tls();
	detail::state_t &s = detail::state();
	if (!t.c) {
		const char *dev = getenv("TW3D_DEVICE");
		int const rc = tw_create(dev ? atoi(dev) : 0, &t.c);
		if (rc != TW_OK) {t.c = nullptr; throw error(rc, "tw_create failed: no CUDA device (lib3dworld_b200 has no CPU fallback)");}
	}
	if (t.generation != s.generation) {
		int rc = tw_set_sin_table(t.c, s.sin_table.empty() ? nullptr : s.sin_table.data());
		if (rc == TW_OK && !s.sine_params.empty()) {rc = tw_set_sine_params(t.c, s.sine_params.data());}
		if (rc != TW_OK) {detail::fail(rc, "table upload", t.c);}
		t.generation = s.generation;
	}
	return t.c;
}

// sin_table: the reference's sin_table.data() (2*TSIZE floats) or nullptr to build it; sinTable: &sinTable[0][0] (90*5 floats) or nullptr
inline void set_globals(scene_globals const &g, const float *sin_table = nullptr, const float *sinTable = nullptr) {
	detail::state_t &s = detail::state();
	s.g = g;
	if (sin_table) {s.sin_table.assign(sin_table, sin_table + TW_SIN_TABLE_SIZE);}
	if (sinTable)  {s.sine_params.assign(sinTable, sinTable + TW_F_TABLE_SIZE*5);}
	if (sin_table || sinTable) {++s.generation;}
}
inline scene_globals const &globals() {return detail::state().g;}

// How many asynchronous height generations (mesh_xy_grid_cache_t::build_arrays(..., no_wait=1) + enable_glaciate()) a thread keeps in flight at once;
// tile_draw_t::update keeps up to 8 (src/tiled_mesh.cpp:2367-2417). n > 1: each thread launches them on up to n shared contexts of its ctx()
// (tw_create_shared: the same tables, own streams and scratch), picking one with nothing in flight, else the one launched on longest ago, whose
// generation that launch completes first. n = 1 (the default): every generation goes to ctx(), one in flight at a time. The contexts, once created,
// live as long as the thread's ctx(). The grid is copied into the object's pageable host vector, which the launch waits for: the generations stay
// independent of each other, but only the tile jobs of tile_job_pool (outputs in pinned memory) overlap on the device.
inline void set_deferred_gens(unsigned n) {detail::state().deferred_gens = n ? n : 1;}

namespace detail {
	inline tw_ctx *gen_ctx() { // the context of the next asynchronous height generation
		tw_ctx *c = ctx();
		unsigned const n = state().deferred_gens;
		if (n <= 1) return c;
		tls_ctx &t = tls();
		while (t.gens.size() < n) {
			tw_ctx *s = nullptr;
			int const rc = tw_create_shared(c, &s);
			if (rc != TW_OK) {fail(rc, "set_deferred_gens: tw_create_shared", c);}
			t.gens.push_back(s); t.gen_launch.push_back(0);
		}
		size_t pick = n;
		for (size_t i = 0; i < n && pick == n; ++i) {
			int const rc = tw_heightgen_2d_poll(t.gens[i], 0); // TW_OK: nothing in flight (a finished generation's host copy is already complete)
			if (rc == TW_OK) {pick = i;}
			else if (rc != TW_ERR_NOT_READY) {fail(rc, "build_arrays", t.gens[i]);}
		}
		if (pick == n) {pick = 0; for (size_t i = 1; i < n; ++i) {if (t.gen_launch[i] < t.gen_launch[pick]) pick = i;}}
		t.gen_launch[pick] = ++t.gen_clock;
		return t.gens[pick];
	}
}

inline tw_height_params height_params_from_globals(int gen_mode, int gen_shape) {
	scene_globals const &g = globals();
	tw_height_params p;
	memset(&p, 0, sizeof(p));
	p.gen_mode = gen_mode; p.gen_shape = gen_shape; p.start_eval_sin = g.start_eval_sin; p.glaciate = g.GLACIATE;
	p.mesh_scale = g.mesh_scale; p.mesh_scale_z_inv = g.mesh_scale_z_inv; p.dx_val_inv = g.DX_VAL_INV; p.dy_val_inv = g.DY_VAL_INV;
	p.mesh_height = g.MESH_HEIGHT; p.mesh_height_scale = g.mesh_height_scale; p.zmax_est = g.zmax_est; p.custom_glaciate_exp = g.custom_glaciate_exp;
	tw_gen_rx_ry(g.mesh_seed, g.mesh_rgen_index, gen_mode, &p.rx, &p.ry); // gen_rx_ry(), src/mesh_gen.cpp:581-586
	p.hmap = g.hmap_params;
	return p;
}
inline tw_erosion_params erosion_params_from_globals() {
	scene_globals const &g = globals();
	tw_erosion_params e = {g.erode_amount, g.water_plane_z, g.HALF_DXY, g.zmin, g.zmax, g.relh_adj_tex, g.clip_hd1};
	return e;
}

// ------------------------------------------------------------------------------------------------ mesh_xy_grid_cache_t
// Same interface and call order as the reference (build_arrays, then optionally enable_glaciate, then eval_index per cell). The grid is
// evaluated on the GPU as a whole the first time a value is needed (or asynchronously when no_wait is set, mirroring the GLSL path:
// build_arrays returns 0 while the job is in flight, src/mesh_gen.cpp:597-603) and eval_index reads the host copy.
class mesh_xy_grid_cache_t {
	mutable std::vector<float> vals;
	mutable std::mutex mtx;
	mutable bool have_vals = false, job_running = false;
	mutable tw_ctx *job_ctx = nullptr;      // the context the pending job was launched on: a job launched on the main thread (build_arrays no_wait +
	                                        // enable_glaciate) is collected on THAT context even when eval_index runs on an OpenMP worker, whose own
	                                        // thread-local context has nothing pending and would report TW_OK at once (ADVICE round 1)
	mutable int vals_min_start = 0; mutable bool vals_glaciate = false;
	tw_grid2d grid = {0, 0, 1, 1, 0, 0};
	int gen_mode = TW_MGEN_SINE, gen_shape = 0;
	bool do_glaciate = false, async_requested = false;

	void launch(bool glaciate, int min_start_sin, bool wait) const {
		tw_height_params const p = height_params_from_globals(gen_mode, gen_shape);
		vals.resize((size_t)grid.nx*grid.ny);
		tw_ctx *c = wait ? ctx() : detail::gen_ctx();
		int rc = tw_heightgen_2d_launch(c, &grid, &p, glaciate, min_start_sin, vals.data(), nullptr);
		if (rc != TW_OK) {detail::fail(rc, "build_arrays", c);}
		job_running = true; job_ctx = c; vals_glaciate = glaciate; vals_min_start = min_start_sin;
		if (wait) {collect(true);}
	}
	bool collect(bool wait) const { // always called with mtx held
		tw_ctx *c = job_ctx ? job_ctx : ctx();
		int const rc = tw_heightgen_2d_poll(c, wait ? 1 : 0);
		if (rc == TW_ERR_NOT_READY) return false;
		if (rc != TW_OK) {detail::fail(rc, "eval_index", c);}
		job_running = false; have_vals = true; job_ctx = nullptr;
		return true;
	}
public:
	bool build_arrays(float x0, float y0, float dx, float dy, unsigned nx, unsigned ny, bool cache_values=0, bool force_sine_mode=0, bool no_wait=0) {
		assert(nx > 0 && ny > 0); // src/mesh_gen.cpp:589
		std::lock_guard<std::mutex> lock(mtx);
		scene_globals const &g = globals();
		tw_grid2d const ng = {x0, y0, dx, dy, nx, ny};
		int const mode = (force_sine_mode ? (int)TW_MGEN_SINE : g.mesh_gen_mode), shape = (force_sine_mode ? 0 : g.mesh_gen_shape);
		bool const same = (memcmp(&ng, &grid, sizeof(grid)) == 0 && mode == gen_mode && shape == gen_shape);
		if (job_running && !same) {collect(true);} // a different grid was in flight: drain it
		if (!same) {have_vals = false;}
		grid = ng; gen_mode = mode; gen_shape = shape;
		do_glaciate = 0; // must call enable_glaciate() after this call if needed (src/mesh_gen.cpp:594)
		async_requested = false;
		if (gen_mode >= TW_MGEN_SIMPLEX_GPU && no_wait) { // GPU modes: launch now or report progress (src/mesh_gen.cpp:597-603)
			if (job_running) {return collect(false);}
			if (have_vals && vals_glaciate && vals_min_start == 0) return 1;
			async_requested = true; // launched by enable_glaciate(), which setup_height_gen_async always calls next (src/tiled_mesh.cpp:462)
			return 0;
		}
		// cache_values: the reference fills cached_vals with un-glaciated values here (src/mesh_gen.cpp:627-636); every caller then calls enable_glaciate()
		// and reads through eval_index, which applies the glaciation per cell - so the grid is evaluated once, lazily, in the state eval_index asks for,
		// instead of once un-glaciated now and once more glaciated on the first eval_index
		(void)cache_values;
		return 1;
	}
	void enable_glaciate() {
		std::lock_guard<std::mutex> lock(mtx);
		do_glaciate = 1;
		if (async_requested && !job_running) {have_vals = false; launch(true, 0, false); async_requested = false;}
	}
	float eval_index(unsigned x, unsigned y, int min_start_sin=0, bool use_cache=1) const {
		assert(x < grid.nx && y < grid.ny); // src/mesh_gen.cpp:756
		(void)use_cache;
		int const mss = (gen_mode == TW_MGEN_SINE) ? min_start_sin : 0;
		bool ready;
		{std::lock_guard<std::mutex> lock(mtx); ready = (have_vals && !job_running && vals_glaciate == do_glaciate && vals_min_start == mss);} // flags are only read under the mutex
		if (!ready) {
			std::lock_guard<std::mutex> lock(mtx);
			if (job_running) {collect(true);}
			if (!(have_vals && vals_glaciate == do_glaciate && vals_min_start == mss)) {have_vals = false; launch(do_glaciate, mss, true);}
		}
		return vals[(size_t)y*grid.nx + x];
	}
	// whole-grid accessors (what the OpenMP eval_index loops of the reference's callers produce)
	void get_grid(float *out, int min_start_sin=0) const {
		(void)eval_index(0, 0, min_start_sin);
		memcpy(out, vals.data(), vals.size()*sizeof(float));
	}
	void clear_context() {std::lock_guard<std::mutex> lock(mtx); if (job_running) {collect(true);} have_vals = false; vals.clear();}
	void free_cshader() {}
	~mesh_xy_grid_cache_t() {if (job_running) {try {collect(true);} catch (...) {}}}
};

// apply_erosion(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters), src/function_registry.h:354
inline void apply_erosion(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters) {
	tw_erosion_params const e = erosion_params_from_globals();
	if (num_iters == 0 || e.erode_amount <= 0.0) return; // erosion disabled (src/erosion.cpp:16)
	tw_ctx *c = ctx();
	int const rc = tw_erode(c, heightmap, xsize, ysize, min_zval, num_iters, &e);
	if (rc != TW_OK) {detail::fail(rc, "apply_erosion", c);}
}

// ------------------------------------------------------------------------------------------------ point queries (batched)
// float get_exact_zval(float xval, float yval, bool no_xyoff=0) / eval_mesh_sin_terms(xv, yv) / eval_mesh_sin_terms_scaled(xval, yval, xy_scale)
// (src/function_registry.h:340-341, src/mesh_gen.cpp:797-847) for n points at once: xy = n (x, y) pairs. The single-point forms below cost a
// kernel launch per call - callers that place many objects (buildings, scenery) should collect their points and use the batch forms.
inline void eval_points(int kind, const float *xy, size_t n, float *out, float xy_scale = 1.0f, bool no_xyoff = false) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_point_query q;
	q.kind = kind; q.xy_scale = xy_scale; q.mesh_x_size = g.MESH_X_SIZE; q.mesh_y_size = g.MESH_Y_SIZE;
	q.x_scene_size = g.X_SCENE_SIZE; q.y_scene_size = g.Y_SCENE_SIZE; q.xoff2 = g.xoff2; q.yoff2 = g.yoff2; q.no_xyoff = no_xyoff;
	tw_ctx *c = ctx();
	int const rc = tw_eval_points(c, xy, n, &p, &q, out);
	if (rc != TW_OK) {detail::fail(rc, "eval_points", c);}
}
inline void get_exact_zvals(const float *xy, size_t n, float *zvals_out, bool no_xyoff = false) {eval_points(TW_PQ_EXACT_ZVAL, xy, n, zvals_out, 1.0f, no_xyoff);}
inline float get_exact_zval(float xval, float yval, bool no_xyoff = false) {
	float const xy[2] = {xval, yval}; float z = 0.0f;
	get_exact_zvals(xy, 1, &z, no_xyoff);
	return z;
}
inline float eval_mesh_sin_terms(float xv, float yv) {
	float const xy[2] = {xv, yv}; float z = 0.0f;
	eval_points(TW_PQ_SIN_TERMS, xy, 1, &z);
	return z;
}
inline float eval_mesh_sin_terms_scaled(float xval, float yval, float xy_scale) {
	float const xy[2] = {xval, yval}; float z = 0.0f;
	eval_points(TW_PQ_SIN_TERMS_SCALED, xy, 1, &z, xy_scale);
	return z;
}

// the same with the reference's OpenMP semantics (`#pragma omp parallel for schedule(dynamic,1)`, src/erosion.cpp:66): num_threads droplets in
// flight on the one heightmap, order-dependent result like the reference's; num_threads = 1 equals apply_erosion(), 0 = fill the GPU
inline void apply_erosion_parallel(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters, unsigned num_threads = 0) {
	tw_erosion_params const e = erosion_params_from_globals();
	if (num_iters == 0 || e.erode_amount <= 0.0) return;
	tw_ctx *c = ctx();
	int const rc = tw_erode_parallel(c, heightmap, xsize, ysize, min_zval, num_iters, &e, num_threads);
	if (rc != TW_OK) {detail::fail(rc, "apply_erosion_parallel", c);}
}

// Height fill + per-tile erosion of tile_t::create_zvals for a batch of tiles (origins = tile x1,y1 pairs; zvals_out = ntiles*zvsize^2 floats)
inline void create_zvals_batch(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float *zvals_out, tw_minmax *mm = nullptr) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_erosion_params const e = erosion_params_from_globals();
	tw_ctx *c = ctx();
	// apply_erosion(zvals.data(), zvsize, zvsize, zmin, erosion_iters_tt): min_zval is the global zmin (src/tiled_mesh.cpp:515)
	int const rc = tw_create_zvals_batch(c, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, erosion_iters_tt, &e, g.zmin, zvals_out, mm);
	if (rc != TW_OK) {detail::fail(rc, "create_zvals_batch", c);}
}

// A frame's new tiles without stalling the frame - the per-frame pattern of tile_draw_t::update (src/tiled_mesh.cpp:2367-2417, build_arrays(..., no_wait=1)):
// create_tiles_async() enqueues heights, erosion and the tile tail (tile_bounds, normal map) and returns at once; call ready() on later frames and use the
// outputs once it returns true (wait() blocks instead). The outputs named in `out` (tw_tile_outputs, include/tw3d.h) must stay valid until then; zvals and
// normals_rgba may be device memory, or page-locked host memory for a launch that never blocks. One job per context: any other call on this thread's
// context completes the job first (tile_job_pool, below, keeps several in flight). Not copyable; a handle that is destroyed while its job runs waits for it.
// cancel() asks a job whose outputs are no longer wanted (tiles out of range, a map reloaded, the scene quit) to stop and returns at once (tw_cancel); the job
// is then ready soon, and cancelled() says whether its outputs are unspecified: true when its poll reports that it was cut short, and also when another
// call completed it after cancel() (a later launch on the context, or tile_job_pool's slot scan before it relaunches the slot), since this handle cannot
// tell whether the cancel acted. cancel() on a tile set's job throws (TW_ERR_STATE).
class tiles_job {
	tw_ctx *c = nullptr;
	std::atomic<uint64_t> const *latest = nullptr; // the launch count of c's thread
	uint64_t number = 0;
	bool done = true, was_cancelled = false, cancel_asked = false;
	bool poll(bool wait) {
		if (done) return true;
		if (latest->load() != number) {done = true; was_cancelled = cancel_asked; return true;} // a later launch on the same context completed this job before it started
		int const rc = tw_create_tiles_poll(c, wait ? 1 : 0);
		if (rc == TW_ERR_NOT_READY) return false;
		done = true;
		if (rc == TW_ERR_CANCELED) {was_cancelled = true; return true;}
		if (rc != TW_OK) {detail::fail(rc, "create_tiles_async", c);}
		return true;
	}
public:
	tiles_job() = default;
	tiles_job(tw_ctx *ctx_, std::atomic<uint64_t> const *latest_, uint64_t number_) : c(ctx_), latest(latest_), number(number_), done(false) {}
	tiles_job(tiles_job &&o) noexcept : c(o.c), latest(o.latest), number(o.number), done(o.done), was_cancelled(o.was_cancelled), cancel_asked(o.cancel_asked) {o.done = true;}
	tiles_job &operator=(tiles_job &&o) {if (this != &o) {wait(); c = o.c; latest = o.latest; number = o.number; done = o.done; was_cancelled = o.was_cancelled; cancel_asked = o.cancel_asked; o.done = true;} return *this;}
	tiles_job(tiles_job const &) = delete;
	tiles_job &operator=(tiles_job const &) = delete;
	~tiles_job() {try {wait();} catch (...) {}}
	bool ready() {return poll(false);}
	void wait() {poll(true);}
	void cancel() {
		if (done || latest->load() != number) return; // completed already
		int const rc = tw_cancel(c);
		if (rc != TW_OK) {detail::fail(rc, "tiles_job::cancel", c);}
		cancel_asked = true;
	}
	bool cancelled() const {return was_cancelled;} // once the job is ready
};
// wpz_max / size: the water level and tile size of the bounds (tile_t::create_zvals, src/tiled_mesh.cpp:517-541); dx, dy also scale the normals (get_norm).
// The overload with `shading` (tw_tile_shading, include/tw3d.h) adds the AO map (calc_mesh_ao_lighting) and the terrain weights texture (create_texture's terrain
// part) to the same job; its outputs and device tile_params must stay valid until the job is ready. In the GPU gen modes AO makes the zvals those of create_zvals_with_ao.
// The overload with `shadows` (tw_tile_shadows, include/tw3d.h) also computes every light's mesh shadows of the new tiles in the job, as calc_mesh_shadows (below) would
// on the job's zvals: smask and sh_out_* must stay valid until the job is ready; tile_xy, the lights and host sh_in rows are copied during the launch. Build each
// light's tw_shadow_params with shadow_params().
namespace detail {
	// the launch behind every create_tiles_async(_from_heightmap): on context c, whose launches jobs counts; hs = nullptr: heights from the height function
	inline tiles_job launch_tiles(tw_ctx *c, std::atomic<uint64_t> &jobs, const tw_hmap_sampler *hs, const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy,
	                              unsigned erosion_iters_tt, float wpz_max, unsigned size, tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_shadows const &shadows) {
		scene_globals const &g = globals();
		tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape); // with hs: the weights' jitter noise
		tw_erosion_params const e = erosion_params_from_globals();
		uint64_t const number = ++jobs;
		int const rc = hs ? tw_create_tiles_launch_hmap(c, hs, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, erosion_iters_tt, &e, g.zmin, wpz_max, size, &out,
		                                                &shading, shadows.nlights ? &shadows : nullptr)
		                  : tw_create_tiles_launch_shadows(c, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, erosion_iters_tt, &e, g.zmin, wpz_max, size, &out,
		                                                   &shading, shadows.nlights ? &shadows : nullptr);
		if (rc != TW_OK) {fail(rc, hs ? "create_tiles_async_from_heightmap" : "create_tiles_async", c);}
		return tiles_job(c, &jobs, number);
	}
}
inline tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
                                    tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_shadows const &shadows) {
	tw_ctx *c = ctx();
	return detail::launch_tiles(c, detail::tls().tile_jobs, nullptr, origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, shadows);
}
inline tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
                                    tw_tile_outputs const &out, tw_tile_shading const &shading) {
	tw_tile_shadows const none = {nullptr, 0, nullptr}; // no lights: the job of tw_create_tiles_launch_ex
	return create_tiles_async(origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, none);
}
inline tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
                                    tw_tile_outputs const &out) {
	tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr}; // nothing requested: the job of tw_create_tiles_launch
	return create_tiles_async(origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, none);
}

// heightmap-texture mode of tile_t::create_zvals (src/tiled_mesh.cpp:498-501): zvals[y*zvsize + x] = terrain_hmap_manager.get_clamped_height(x1 + x, y1 + y)
// for a batch of tiles, from the 16-bit image hmap16 (width*height*2 bytes, the layout heightmap_t keeps); TEX_EDGE_MODE 2 = mirror as compiled in the reference
inline tw_hmap_sampler hmap_sampler(int width, int height, int tex_edge_mode) {
	scene_globals const &g = globals();
	tw_hmap_sampler hs;
	hs.width = width; hs.height = height; hs.edge_mode = tex_edge_mode; hs.mesh_scale = g.mesh_scale;
	hs.h_scale = 0.0008f*g.mesh_height_scale; // READ_MESH_H_SCALE*mesh_height_scale (src/mesh_gen.cpp:22,120)
	hs.mesh_file_scale = g.mesh_file_scale; hs.mesh_file_tz = g.mesh_file_tz; hs.mesh_scale_z_inv = g.mesh_scale_z_inv;
	return hs;
}
inline void create_zvals_from_heightmap(const uint8_t *hmap16, int width, int height, const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float *zvals_out, int tex_edge_mode = TW_HMAP_EDGE_MIRROR) {
	tw_hmap_sampler const hs = hmap_sampler(width, height, tex_edge_mode);
	tw_ctx *c = ctx();
	int const rc = tw_heightmap_sample_tiles(c, hmap16, &hs, origins_xy, ntiles, zvsize, zvals_out);
	if (rc != TW_OK) {detail::fail(rc, "create_zvals_from_heightmap", c);}
}
// The same heightmap mode as a frame's asynchronous tile job: set_heightmap() keeps the image on this thread's device once (host or device hmap16, as above;
// call it again when the map changes), and create_tiles_async_from_heightmap() is create_tiles_async() with zvals = create_zvals_from_heightmap()'s.
// erosion_iters_tt: whether heightmap tiles are eroded is the engine's choice (0 = not). shading.ao is refused (tw_create_tiles_launch_hmap in tw3d.h).
inline void set_heightmap(const uint8_t *hmap16, int width, int height) {
	tw_ctx *c = ctx();
	int const rc = tw_set_heightmap(c, hmap16, width, height);
	if (rc != TW_OK) {detail::fail(rc, "set_heightmap", c);}
	detail::tls().hmap_w = hmap16 ? width : 0; detail::tls().hmap_h = hmap16 ? height : 0;
}
// terrain_hmap_manager_t's map edits (src/heightmap.cpp:36-58,243-308): after the engine's brush code has changed its CPU image hmap16 (width x height texels,
// the layout set_heightmap took) inside rects (the brush's bounding rect, or the saved edits re-applied when a map loads), update_heightmap copies those texels
// into this thread's context's image without completing or waiting for a frame in flight (tw_update_heightmap): frames launched before it see the old map,
// frames after it the new one. hmap_tiles_touched names the live tiles (origins x1, y1 of zvsize^2 cells) whose heights the edit changes, for the image
// set_heightmap gave and the scene's mesh_scale; re-create those in one tile-set frame with them put and the tiles tile_set::stale_after names relit.
inline void update_heightmap(const uint8_t *hmap16, int width, int height, const tw_hmap_rect *rects, unsigned n) {
	tw_ctx *c = ctx();
	if (width != detail::tls().hmap_w || height != detail::tls().hmap_h) {detail::fail(TW_ERR_ARG, "update_heightmap: the image size differs from set_heightmap's", nullptr);}
	int const rc = tw_update_heightmap(c, hmap16, 2*(size_t)width, rects, n);
	if (rc != TW_OK) {detail::fail(rc, "update_heightmap", c);}
}
inline void hmap_tiles_touched(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, const tw_hmap_rect *rects, unsigned n, uint8_t *touched,
                               int tex_edge_mode = TW_HMAP_EDGE_MIRROR) {
	tw_hmap_sampler const hs = hmap_sampler(detail::tls().hmap_w, detail::tls().hmap_h, tex_edge_mode);
	int const rc = tw_hmap_tiles_touched(&hs, origins_xy, ntiles, zvsize, rects, n, touched);
	if (rc != TW_OK) {detail::fail(rc, "hmap_tiles_touched: bad argument (no set_heightmap image?)", nullptr);}
}
inline tiles_job create_tiles_async_from_heightmap(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max,
                                                   unsigned size, tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_shadows const &shadows,
                                                   int tex_edge_mode = TW_HMAP_EDGE_MIRROR) {
	tw_ctx *c = ctx();
	tw_hmap_sampler const hs = hmap_sampler(detail::tls().hmap_w, detail::tls().hmap_h, tex_edge_mode);
	return detail::launch_tiles(c, detail::tls().tile_jobs, &hs, origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, shadows);
}

// terrain_hmap_manager_t::proc_gen_heightmap (heightmap_t::proc_gen, src/heightmap.cpp:130-215): the globals' height function on a width x height grid
// (cell size dx, dy), run_erosion with erosion_iters droplets, the z range, the texture scalars (info: get_mh_texture_mult/add, mesh_file_scale / _tz, the
// droplet moves) and the 16-bit image data16 (2*width*height bytes). data16 and vals (optional, width*height floats) are host or device memory.
inline void proc_gen_heightmap(unsigned width, unsigned height, float dx, float dy, unsigned erosion_iters, uint8_t *data16, float *vals, tw_heightmap_info *info) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_erosion_params const e = erosion_params_from_globals();
	tw_ctx *c = ctx();
	int const rc = tw_proc_gen_heightmap(c, width, height, dx, dy, &p, erosion_iters, &e, data16, vals, info);
	if (rc != TW_OK) {detail::fail(rc, "proc_gen_heightmap", c);}
}
// The same as a job that does not stall the frame (tw_proc_gen_heightmap_launch): returns at once; ready() / wait() on the tiles_job say when data16, vals and
// *info are complete. set_image: the image also becomes this thread's set_heightmap() image (data16 may then be nullptr), so the frame's
// create_tiles_async_from_heightmap() samples it once the job is ready - or completes the job first when launched earlier. A pageable host data16 / vals
// makes the launch wait for its copy.
inline tiles_job proc_gen_heightmap_async(unsigned width, unsigned height, float dx, float dy, unsigned erosion_iters, uint8_t *data16, float *vals, tw_heightmap_info *info,
                                          bool set_image = false) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_erosion_params const e = erosion_params_from_globals();
	tw_heightmap_outputs const out = {data16, vals, info, set_image ? 1 : 0};
	tw_ctx *c = ctx();
	std::atomic<uint64_t> &jobs = detail::tls().tile_jobs;
	uint64_t const number = ++jobs;
	int const rc = tw_proc_gen_heightmap_launch(c, width, height, dx, dy, &p, erosion_iters, &e, &out);
	if (rc != TW_OK) {detail::fail(rc, "proc_gen_heightmap_async", c);}
	if (set_image) {detail::tls().hmap_w = (int)width; detail::tls().hmap_h = (int)height;}
	return tiles_job(c, &jobs, number);
}

// apply_erosion / apply_erosion_parallel as jobs that do not stall the frame (tw_erode_launch): they return at once, and ready() / wait() on the tiles_job say
// when heightmap (host or device; pageable host memory makes the launch wait for its copies) holds what the synchronous call would have left there.
namespace detail {
	inline tiles_job erode_async(float *heightmap, int xsize, int ysize, float min_zval, float val_mult, float val_add, unsigned num_iters, int num_threads,
	                             float *vals, const char *what) {
		tw_erosion_params const e = erosion_params_from_globals();
		tw_erosion_job const job = {heightmap, xsize, ysize, min_zval, val_mult, val_add, num_iters, &e, num_threads < 0 ? TW_EROSION_SERIAL : TW_EROSION_OPENMP,
		                            num_threads < 0 ? 0u : (uint32_t)num_threads, vals};
		tw_ctx *c = ctx();
		std::atomic<uint64_t> &jobs = tls().tile_jobs;
		uint64_t const number = ++jobs;
		int const rc = tw_erode_launch(c, &job);
		if (rc != TW_OK) {fail(rc, what, c);}
		return tiles_job(c, &jobs, number);
	}
}
constexpr int serial_order = -1; // erode_heightmap_async: the serial droplet order of apply_erosion instead of apply_erosion_parallel's threads
inline tiles_job apply_erosion_async(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters) {
	return detail::erode_async(heightmap, xsize, ysize, min_zval, 0.0f, 0.0f, num_iters, serial_order, nullptr, "apply_erosion_async");
}
inline tiles_job apply_erosion_parallel_async(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters, unsigned num_threads = 0) {
	return detail::erode_async(heightmap, xsize, ysize, min_zval, 0.0f, 0.0f, num_iters, (int)num_threads, nullptr, "apply_erosion_parallel_async");
}
// heightmap_t::run_erosion (src/heightmap.cpp:153-187) on the image set_heightmap() keeps on this thread's device, as one job: to_floats with val_mult /
// val_add (get_mh_texture_mult / _add), erosion with min_zval = the map's minimum, from_floats back into the image. num_threads: serial_order, or the threads
// of apply_erosion_parallel (0 = fill the GPU). vals (optional, width*height floats, host or device) receives the eroded floats. The frame's
// create_tiles_async_from_heightmap() samples the eroded image once the job is ready, or completes the job first when launched earlier.
inline tiles_job erode_heightmap_async(float val_mult, float val_add, unsigned num_iters, int num_threads = serial_order, float *vals = nullptr) {
	return detail::erode_async(nullptr, 0, 0, 0.0f, val_mult, val_add, num_iters, num_threads, vals, "erode_heightmap_async");
}

// The coherent batched sweeps of tw_erode_sweeps (tw3d.h) on one map of this thread's context: reproducible like apply_erosion, and far faster on a big map
// with many droplets. apply_erosion_sweeps blocks and returns the droplet moves; the _async forms are the jobs of tw_erode_launch_ex's TW_EROSION_SWEEPS mode
// and leave what apply_erosion_sweeps would have left (tw_last_erosion_steps = the moves) once the tiles_job is ready. erode_heightmap_sweeps_async is
// erode_heightmap_async with the sweeps in place of the serial order.
inline uint64_t apply_erosion_sweeps(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters, unsigned sweep, int halo) {
	tw_erosion_params const e = erosion_params_from_globals();
	tw_ctx *c = ctx();
	uint64_t moves = 0;
	int const rc = tw_erode_sweeps(c, heightmap, xsize, ysize, min_zval, num_iters, &e, sweep, halo, &moves);
	if (rc != TW_OK) {detail::fail(rc, "apply_erosion_sweeps", c);}
	return moves;
}
namespace detail {
	inline tiles_job erode_sweeps_async(float *heightmap, int xsize, int ysize, float min_zval, float val_mult, float val_add, unsigned num_iters, unsigned sweep, int halo,
	                                    float *vals, const char *what) {
		tw_erosion_params const e = erosion_params_from_globals();
		tw_erosion_job const job = {heightmap, xsize, ysize, min_zval, val_mult, val_add, num_iters, &e, TW_EROSION_SWEEPS, 0u, vals};
		tw_sweep_params const sw = {sweep, halo};
		tw_ctx *c = ctx();
		std::atomic<uint64_t> &jobs = tls().tile_jobs;
		uint64_t const number = ++jobs;
		int const rc = tw_erode_launch_ex(c, &job, &sw);
		if (rc != TW_OK) {fail(rc, what, c);}
		return tiles_job(c, &jobs, number);
	}
}
inline tiles_job apply_erosion_sweeps_async(float *heightmap, int xsize, int ysize, float min_zval, unsigned num_iters, unsigned sweep, int halo) {
	return detail::erode_sweeps_async(heightmap, xsize, ysize, min_zval, 0.0f, 0.0f, num_iters, sweep, halo, nullptr, "apply_erosion_sweeps_async");
}
inline tiles_job erode_heightmap_sweeps_async(float val_mult, float val_add, unsigned num_iters, unsigned sweep, int halo, float *vals = nullptr) {
	return detail::erode_sweeps_async(nullptr, 0, 0, 0.0f, val_mult, val_add, num_iters, sweep, halo, vals, "erode_heightmap_sweeps_async");
}

// Several frames' tile jobs in flight at once: a pool of n shared contexts of this thread's ctx() (tw_create_shared - the same tables and heightmap
// image, own streams and scratch). pool.create_tiles_async(...) takes the arguments of the free functions above and launches on a slot with no job in
// flight; when every slot is busy, on the slot launched on longest ago, whose job that launch completes first (its tiles_job then reports ready).
// A launch never waits for another slot's job. Create and use the pool on one thread, let it outlive the jobs it returned, and destroy it before the
// thread ends (its contexts are shared contexts of the thread's context); destroying it completes its jobs.
class tile_job_pool {
	friend class tile_set; // its frame launches take a slot too
	struct slot {tw_ctx *c = nullptr; std::atomic<uint64_t> jobs{0}; uint64_t launched = 0;};
	std::vector<std::unique_ptr<slot>> slots; // stable addresses: a tiles_job keeps a pointer to its slot's launch count
	uint64_t clock = 0;
	slot &next() {
		ctx(); // the thread's context takes new tables first (set_globals), completing the slots' jobs if it does
		slot *pick = nullptr;
		for (auto &s : slots) {
			int const rc = tw_create_tiles_poll(s->c, 0);   // TW_OK: nothing in flight (a finished job is unpacked into its outputs here)
			if (rc == TW_OK || rc == TW_ERR_CANCELED) {pick = s.get(); break;} // a cancelled job's slot is free again
			if (rc != TW_ERR_NOT_READY) {detail::fail(rc, "create_tiles_async", s->c);}
		}
		if (!pick) {pick = slots[0].get(); for (auto &s : slots) {if (s->launched < pick->launched) pick = s.get();}}
		pick->launched = ++clock;
		return *pick;
	}
public:
	explicit tile_job_pool(unsigned n) {
		tw_ctx *c = ctx();
		for (unsigned i = 0; i < (n ? n : 1); ++i) {
			slots.emplace_back(new slot());
			int const rc = tw_create_shared(c, &slots.back()->c);
			if (rc != TW_OK) {slots.pop_back(); for (auto &s : slots) {tw_destroy(s->c);} detail::fail(rc, "tile_job_pool: tw_create_shared", c);}
		}
	}
	~tile_job_pool() {for (auto &s : slots) {tw_destroy(s->c);}}
	tile_job_pool(tile_job_pool const &) = delete;
	tile_job_pool &operator=(tile_job_pool const &) = delete;
	unsigned size() const {return (unsigned)slots.size();}
	tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
	                             tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_shadows const &shadows) {
		slot &s = next();
		return detail::launch_tiles(s.c, s.jobs, nullptr, origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, shadows);
	}
	tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
	                             tw_tile_outputs const &out, tw_tile_shading const &shading) {
		tw_tile_shadows const none = {nullptr, 0, nullptr};
		return create_tiles_async(origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, none);
	}
	tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
	                             tw_tile_outputs const &out) {
		tw_tile_shading const none = {0.0f, nullptr, nullptr, nullptr, nullptr, nullptr};
		return create_tiles_async(origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, none);
	}
	// heightmap-texture tiles from the image set_heightmap() gave this thread's context
	tiles_job create_tiles_async_from_heightmap(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float wpz_max,
	                                            unsigned size, tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_shadows const &shadows,
	                                            int tex_edge_mode = TW_HMAP_EDGE_MIRROR) {
		slot &s = next();
		tw_hmap_sampler const hs = hmap_sampler(detail::tls().hmap_w, detail::tls().hmap_h, tex_edge_mode);
		return detail::launch_tiles(s.c, s.jobs, &hs, origins_xy, ntiles, zvsize, dx, dy, erosion_iters_tt, wpz_max, size, out, shading, shadows);
	}
};

// tile_t::upload_normal_texture (src/tiled_mesh.cpp:865-880, minus the GL upload) and tile_t::calc_mesh_ao_lighting (:586-662) for a batch of
// finished tiles: normal_data = ntiles*stride^2*4 bytes (RGBA, alpha 0), ao_lighting = ntiles*stride^2 bytes, stride = zvsize-1
inline void tile_normals(const float *zvals, unsigned ntiles, unsigned zvsize, float dx_val, float dy_val, unsigned char *normal_data, float *min_normal_z = nullptr) {
	tw_ctx *c = ctx();
	int const rc = tw_tile_normals_batch(c, zvals, ntiles, zvsize, dx_val, dy_val, normal_data, min_normal_z);
	if (rc != TW_OK) {detail::fail(rc, "tile_normals", c);}
}
// tile_t::create_zvals + calc_mesh_ao_lighting with enable_tiled_mesh_ao for a batch: in the GPU gen modes the (stride+72)^2 context is generated once, zvals are
// its interior (src/tiled_mesh.cpp:479-487,505) and the AO rays test the un-eroded context (:604)
inline void create_zvals_with_ao(const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned erosion_iters_tt, float *zvals_out, unsigned char *ao_lighting, tw_minmax *mm = nullptr) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_erosion_params const e = erosion_params_from_globals();
	tw_ctx *c = ctx();
	int const rc = tw_create_zvals_ao_batch(c, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, erosion_iters_tt, &e, g.zmin, g.HALF_DXY, zvals_out, ao_lighting, mm);
	if (rc != TW_OK) {detail::fail(rc, "create_zvals_with_ao", c);}
}
inline void tile_ao_lighting(const float *zvals, const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx, float dy, unsigned char *ao_lighting) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_ctx *c = ctx();
	int const rc = tw_tile_ao_batch(c, zvals, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, g.HALF_DXY, ao_lighting);
	if (rc != TW_OK) {detail::fail(rc, "tile_ao_lighting", c);}
}

// calc_mesh_shadows(l, lpos, mh, smask, xsize, ysize, sh_in_x, sh_in_y, sh_out_x, sh_out_y) (src/visibility.cpp:508-517) for ALL tiles a light change dirties, in
// one call: tile_t::calc_shadows_for_light's chain (src/tiled_mesh.cpp:664-692: each tile starts from the sh_out of its neighbours toward the light) becomes dependency
// waves on the device. tile_xy = (x1/size, y1/size) per tile; smask = ntiles*zvsize^2 bytes (0 / MESH_SHADOW); sh_out_* optional (ntiles*zvsize floats each).
// no_shadow = (l == LIGHT_MOON && combined_gu). Globals read (shadow_params): X/Y_SCENE_SIZE, DX/DY_VAL(+_INV), XY_SUM_SIZE = MESH_X_SIZE + MESH_Y_SIZE, zmin, zmax.
inline tw_shadow_params shadow_params(const float lpos[3], float dx_val, float dy_val, bool no_shadow = false) {
	scene_globals const &g = globals();
	tw_shadow_params sp;
	for (int d = 0; d < 3; ++d) {sp.lpos[d] = lpos[d];}
	sp.x_scene_size = g.X_SCENE_SIZE; sp.y_scene_size = g.Y_SCENE_SIZE;
	sp.dx_val = dx_val; sp.dy_val = dy_val; sp.dx_val_inv = 1.0f/dx_val; sp.dy_val_inv = 1.0f/dy_val; // set_scene_constants: DX_VAL_INV = 1.0/DX_VAL
	sp.xy_sum_size = g.MESH_X_SIZE + g.MESH_Y_SIZE;
	sp.zmin = g.zmin; sp.zmax = g.zmax; sp.no_shadow = no_shadow ? 1 : 0;
	return sp;
}
inline void calc_mesh_shadows(const float lpos[3], const float *zvals, const int32_t *tile_xy, unsigned ntiles, unsigned zvsize, float dx_val, float dy_val,
                              unsigned char *smask, float *sh_out_x = nullptr, float *sh_out_y = nullptr, bool no_shadow = false) {
	tw_shadow_params const sp = shadow_params(lpos, dx_val, dy_val, no_shadow);
	tw_ctx *c = ctx();
	int const rc = tw_tile_shadows_batch(c, zvals, tile_xy, ntiles, zvsize, &sp, smask, sh_out_x, sh_out_y);
	if (rc != TW_OK) {detail::fail(rc, "calc_mesh_shadows", c);}
}
// The same for new tiles next to existing ones (tw_tile_shadows_batch_ex): sh_in_x / sh_in_y (ntiles*zvsize floats each, either may be null) hold, per tile, the sh_out
// of its neighbour toward the light where that neighbour is an existing tile outside the batch (what calc_shadows_for_light reads from the tile map); rows of tiles
// whose neighbour is in the batch are ignored. Also the way to re-shadow existing tiles once new tiles appear on their light side: pass the new tiles' sh_out.
inline void calc_mesh_shadows(const float lpos[3], const float *zvals, const int32_t *tile_xy, unsigned ntiles, unsigned zvsize, float dx_val, float dy_val,
                              const float *sh_in_x, const float *sh_in_y, unsigned char *smask, float *sh_out_x = nullptr, float *sh_out_y = nullptr, bool no_shadow = false) {
	tw_shadow_params const sp = shadow_params(lpos, dx_val, dy_val, no_shadow);
	tw_ctx *c = ctx();
	int const rc = tw_tile_shadows_batch_ex(c, zvals, tile_xy, ntiles, zvsize, &sp, sh_in_x, sh_in_y, smask, sh_out_x, sh_out_y);
	if (rc != TW_OK) {detail::fail(rc, "calc_mesh_shadows", c);}
}

// The live tiles of tile_draw_t on the device (tw_tile_set, include/tw3d.h), for the two relights of calc_shadows_for_light the engine otherwise does itself
// (src/tiled_mesh.cpp:664-692): when the light moves, relight_async() every live tile; when new tiles appear, put() them (a tile job's device zvals cost one
// copy on the device), ask stale() which shadow textures change, and relight_async() those. Each relight equals calc_mesh_shadows over all resident tiles, bit
// for bit, and recomputes only the tiles whose result can have changed. relight_async returns the tiles_job of create_tiles_async: outputs (smask, sh_out_*
// of every tw_tile_set_light, in request order) are complete once it is ready. Lives on this thread's ctx(); destroy it before the thread ends.
class tile_set {
	tw_ctx *c = nullptr;
	tw_tile_set *s = nullptr;
public:
	tile_set(unsigned zvsize, unsigned nlights) : c(ctx()) {
		int const rc = tw_tile_set_create(c, zvsize, nlights, &s);
		if (rc != TW_OK) {s = nullptr; detail::fail(rc, "tile_set", c);}
	}
	~tile_set() {if (s) tw_tile_set_destroy(s);}
	tile_set(tile_set const &) = delete;
	tile_set &operator=(tile_set const &) = delete;
	tw_tile_set *handle() const {return s;}
	void put(const int32_t *tile_xy, unsigned n, const float *zvals) {
		int const rc = tw_tile_set_put(s, tile_xy, n, zvals);
		if (rc != TW_OK) {detail::fail(rc, "tile_set::put", c);}
	}
	void remove(const int32_t *tile_xy, unsigned n) {
		int const rc = tw_tile_set_remove(s, tile_xy, n);
		if (rc != TW_OK) {detail::fail(rc, "tile_set::remove", c);}
	}
	// (x, y) pairs of the tiles a relight of every resident tile with these lights recomputes
	std::vector<int32_t> stale(const tw_shadow_params *sps, unsigned nlights) const {
		uint32_t k = 0;
		int rc = tw_tile_set_stale(s, sps, nlights, nullptr, 0, &k);
		std::vector<int32_t> out(2*(size_t)k);
		if (rc == TW_OK && k) {rc = tw_tile_set_stale(s, sps, nlights, out.data(), k, &k);}
		if (rc != TW_OK) {detail::fail(rc, "tile_set::stale", c);}
		return out;
	}
	tiles_job relight_async(const int32_t *tile_xy, unsigned n, const tw_tile_set_light *lights, unsigned nlights, uint8_t *recomputed = nullptr) {
		std::atomic<uint64_t> &jobs = detail::tls().tile_jobs;
		uint64_t const number = ++jobs;
		tw_tile_set_request const req = {tile_xy, n, nlights, lights, recomputed};
		int const rc = tw_tile_set_shadows_launch(s, &req);
		if (rc != TW_OK) {detail::fail(rc, "tile_set::relight_async", c);}
		return tiles_job(c, &jobs, number);
	}
	// stale() as it would be after remove(remove_xy) and put(put_xy), without changing the set: the tiles a frame's relight should name
	std::vector<int32_t> stale_after(const tw_shadow_params *sps, unsigned nlights, const int32_t *remove_xy, unsigned nremove, const int32_t *put_xy, unsigned nput) const {
		uint32_t k = 0;
		int rc = tw_tile_set_stale_after(s, sps, nlights, remove_xy, nremove, put_xy, nput, nullptr, 0, &k);
		std::vector<int32_t> out(2*(size_t)k);
		if (rc == TW_OK && k) {rc = tw_tile_set_stale_after(s, sps, nlights, remove_xy, nremove, put_xy, nput, out.data(), k, &k);}
		if (rc != TW_OK) {detail::fail(rc, "tile_set::stale_after", c);}
		return out;
	}
	// A frame in one job (tw_tile_set_create_tiles_launch): frame.remove_xy removed, the new tiles created as create_tiles_async() would (frame.hs: from the
	// heightmap, as create_tiles_async_from_heightmap()) and put into the set at frame.tile_xy, and frame.relight relit - with no blocking put in between.
	// out.zvals may be null (the zvals then stay in the set). Launched on this set's context, or on a slot of `pool` (shared contexts of the same thread's
	// context) so that several frames are in flight at once; only their set-touching tails are ordered on the device. The returned job is ready once every
	// output of the tile job and of the relight is complete.
	tiles_job create_tiles_async(const int32_t *origins_xy, unsigned ntiles, float dx, float dy, unsigned erosion_iters_tt, float wpz_max, unsigned size,
	                             tw_tile_outputs const &out, tw_tile_shading const &shading, tw_tile_set_frame const &frame, tile_job_pool *pool = nullptr) {
		scene_globals const &g = globals();
		tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
		tw_erosion_params const e = erosion_params_from_globals();
		tw_ctx *lc = c;
		std::atomic<uint64_t> *jobs = &detail::tls().tile_jobs;
		if (pool) {tile_job_pool::slot &sl = pool->next(); lc = sl.c; jobs = &sl.jobs;}
		uint64_t const number = ++*jobs;
		int const rc = tw_tile_set_create_tiles_launch(lc, s, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, &p, erosion_iters_tt, &e, g.zmin, wpz_max, size,
		                                               &out, &shading, &frame);
		if (rc != TW_OK) {detail::fail(rc, "tile_set::create_tiles_async", lc);}
		return tiles_job(lc, jobs, number);
	}
};

// tile_t::create_texture's terrain part (src/tiled_mesh.cpp:1071-1248) for a batch of tiles: mesh_weight_data (RGBA = {sand, dirt, grass, rock}, stride^2 texels per
// tile) and has_any_grass. The caller passes what the reference reads from engine tables: h_dirt[] and lttex_dirt[].id (as TW_TEX_* classes), sthresh, the biome corners
// params[y][x].{grass, dirt} of every tile (grass[4] then dirt[4]), get_water_z_height(), vegetation, relh_adj_tex, mesh_gen_shape / mesh_scale_z (noise_scale),
// water_is_lava || DISABLE_WATER == 2. Texels inside cities / over tunnels / under buildings and the tree pass stay with the caller (it overwrites them afterwards).
// (h_dirt / tex_class: the engine's own tables, or tw_gen_tex_height_tables(water_h_off_rel, temperature, glaciate_exp, ...) = init_terrain_mesh + gen_tex_height_tables)
struct weight_tables {float h_dirt[5]; int tex_class[5]; float sthresh[2][2]; float water_level, vegetation; bool snow_to_rock; int mesh_gen_shape; float mesh_scale_z;};
// weight_params: the tw_weight_params of these tables (also what tw_tile_shading::wp of create_tiles_async points to)
inline tw_weight_params weight_params(weight_tables const &wt, unsigned zvsize, float dx_val, float dy_val) {
	scene_globals const &g = globals();
	tw_weight_params W;
	memset(&W, 0, sizeof(W));
	for (int i = 0; i < 5; ++i) {W.h_dirt[i] = wt.h_dirt[i]; W.tex_class[i] = wt.tex_class[i];}
	for (int a = 0; a < 2; ++a) {for (int b = 0; b < 2; ++b) {W.sthresh[a][b] = wt.sthresh[a][b];}}
	W.zmin = g.zmin; W.zmax = g.zmax; W.relh_adj_tex = g.relh_adj_tex; W.water_level = wt.water_level;
	float const MESH_NOISE_SCALE = 0.003;
	W.noise_scale = ((wt.mesh_gen_shape == 2) ? 2.0 : 1.0)*MESH_NOISE_SCALE*wt.mesh_scale_z;          // src/tiled_mesh.cpp:1085-1088, same types
	float const SQRT2 = sqrt(2.0);                                                                     // src/3DWorld.h:132
	W.vnz_scale = (g.mesh_gen_mode == TW_MGEN_DWARP_GPU) ? SQRT2 : 1.0;
	W.vegetation = wt.vegetation; W.snow_to_rock = wt.snow_to_rock ? 1 : 0;
	W.dx_val = dx_val; W.dy_val = dy_val; W.dxdy = dx_val*dy_val;
	W.xy_mult = 1.0/float(zvsize - 2);                                                                 // size = zvsize - 2
	return W;
}
inline void create_texture_weights(const float *zvals, const int32_t *origins_xy, unsigned ntiles, unsigned zvsize, float dx_val, float dy_val, weight_tables const &wt,
                                   const float *tile_params, unsigned char *mesh_weight_data, unsigned char *has_any_grass = nullptr) {
	scene_globals const &g = globals();
	tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_weight_params const W = weight_params(wt, zvsize, dx_val, dy_val);
	tw_ctx *c = ctx();
	int const rc = tw_tile_weights_batch(c, zvals, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx_val, dy_val, zvsize, &p, &W, tile_params, mesh_weight_data, has_any_grass);
	if (rc != TW_OK) {detail::fail(rc, "create_texture_weights", c);}
}

// ------------------------------------------------------------------------------------------------ gen_mesh (ground mode)
// gen_mesh(surface_type=0, keep_sin_table=0, update_zvals=1) for WMODE_GROUND (src/mesh_gen.cpp:257-355): regenerates the sine table from
// the function-static generator state (pass the same tw_rng across calls), fills mesh_height, estimates zmax_est from a 128x128 probe of the
// equation (estimate_zminmax, :447-485), sets the z globals (set_zvals, :494-504), glaciates (:388-404) and erodes (:443).
// The derived globals are written back into scene_globals (zmax_est, zmin, zmax, water_plane_z) exactly as the reference leaves them.
struct gen_mesh_result {float zmin, zmax, zmax_est, zbottom, ztop, water_plane_z;};

inline gen_mesh_result gen_mesh(float *mesh_height /* MESH_Y_SIZE x MESH_X_SIZE, row-major */, tw_rng &sine_rng, float x_scene_size, float y_scene_size,
	unsigned erosion_iters, int xoff2 = 0, int yoff2 = 0, float dx_val = 0.0f, float dy_val = 0.0f, float water_h_off = 0.0f, float water_h_off_rel = 0.0f)
{
	scene_globals g = globals();
	int const MX = g.MESH_X_SIZE, MY = g.MESH_Y_SIZE;
	if (dx_val == 0.0f) {dx_val = 1.0f/g.DX_VAL_INV;}
	if (dy_val == 0.0f) {dy_val = 1.0f/g.DY_VAL_INV;}
	std::vector<float> sinTable(TW_F_TABLE_SIZE*5);
	tw_gen_sine_params(&sine_rng, g.MESH_HEIGHT*g.mesh_height_scale, MX, MY, x_scene_size, y_scene_size, g.mesh_seed, g.mesh_rgen_index, g.mesh_gen_mode,
	                   g.MESH_START_MAG, g.MESH_START_FREQ, g.MESH_MAG_MULT, g.MESH_FREQ_MULT, sinTable.data());
	set_globals(g, nullptr, sinTable.data());
	tw_ctx *c = ctx();
	tw_height_params p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
	tw_grid2d const grid = {(float)(xoff2 - MX/2), (float)(yoff2 - MY/2), dx_val, dy_val, (uint32_t)MX, (uint32_t)MY}; // gen_mesh_sine_table, :201-210
	tw_minmax mm;
	int rc = tw_heightgen_2d(c, &grid, &p, 0, 0, mesh_height, &mm);
	if (rc != TW_OK) {detail::fail(rc, "gen_mesh", c);}
	float zmin = mm.zmin, zmax = mm.zmax;                        // calc_zminmax
	float zmax_est = (zmax < -zmin) ? -zmin : zmax;              // set_zmax_est(max(zmax, -zmin))
	gen_mesh_result r;
	if (zmax == zmin) { // flat mesh: estimate_zminmax returns BEFORE set_zvals (src/mesh_gen.cpp:463-466): zmin/zmax stay the measured pair, zbottom/ztop/water_plane_z keep their old values
		zmax_est = zmax_est + 1.0E-6;
		r.zbottom = g.zbottom; r.ztop = g.ztop; r.zmin = zmin; r.zmax = zmax; r.zmax_est = zmax_est; r.water_plane_z = g.water_plane_z;
	}
	else {
		float const XY_SCENE_SIZE(0.5f*(x_scene_size + y_scene_size));
		float const rm_scale(1000.0*XY_SCENE_SIZE/g.mesh_scale);
		tw_grid2d const probe = {0.0f, 0.0f, rm_scale, rm_scale, 128, 128};   // EST_RAND_PARAM
		std::vector<float> h(128*128);
		rc = tw_heightgen_2d(c, &probe, &p, 0, 0, h.data(), nullptr);
		if (rc != TW_OK) {detail::fail(rc, "estimate_zminmax", c);}
		for (float v : h) {float const a(std::fabs(v)); zmax_est = (zmax_est < a) ? a : zmax_est;}
		if (g.mesh_gen_mode != TW_MGEN_SINE) {zmax_est *= 1.2;}
		zmax_est = 1.1*zmax_est;
		r.zbottom = zmin; r.ztop = zmax;                              // set_zvals
		r.zmin = -zmax_est; r.zmax = zmax_est; r.zmax_est = zmax_est;
		r.water_plane_z = tw_water_z_height(zmax_est, g.GLACIATE, g.custom_glaciate_exp, water_h_off, water_h_off_rel);
	}
	g.zmax_est = zmax_est; g.zmin = r.zmin; g.zmax = r.zmax; g.water_plane_z = r.water_plane_z; g.zbottom = r.zbottom; g.ztop = r.ztop;
	set_globals(g);
	p.zmax_est = zmax_est;
	if (g.GLACIATE) { // gen_terrain_map -> glaciate()
		rc = tw_glaciate_mesh(c, mesh_height, MX, MY, xoff2, yoff2, MX, MY, &p, &mm);
		if (rc != TW_OK) {detail::fail(rc, "glaciate", c);}
		r.zbottom = mm.zmin; r.ztop = mm.zmax;                    // glaciate() recomputes them (calc_zminmax + the zbottom/ztop update, :399-403)
		g.zbottom = r.zbottom; g.ztop = r.ztop; set_globals(g);
	}
	apply_erosion(mesh_height, MX, MY, r.zbottom, erosion_iters);
	return r;
}

// tail of tile_t::create_zvals for a batch of finished tiles (sub_zmin/sub_zmax, mzmin/mzmax, mesh_dz, radius, water bbox), src/tiled_mesh.cpp:517-541
inline void tile_bounds(const float *zvals, unsigned ntiles, unsigned zvsize, float wpz_max, float dx_val, float dy_val, unsigned size, tw_tile_bounds *out) {
	tw_ctx *c = ctx();
	int const rc = tw_tile_bounds_batch(c, zvals, ntiles, zvsize, wpz_max, dx_val, dy_val, size, out);
	if (rc != TW_OK) {detail::fail(rc, "tile_bounds", c);}
}

// noise_gen_3d: the table-generation half of the reference class (src/upsurface.h:39-50); grid evaluation goes through create_procedural
class noise_gen_3d {
	int rs1 = 1, rs2 = 1;
public:
	unsigned num_sines = 0;
	float rdata[TW_N3D_RDATA] = {0};
	void set_rand_seeds(int rs1_, int rs2_) {rs1 = rs1_; rs2 = rs2_;}
	void gen_sines(float mag, float freq) {
		assert(mag > 0.0 && freq > 0.0); // src/upsurface.cpp:19
		tw_noise3d_gen_sines(rs1, rs2, mag, freq, rdata);
		num_sines = TW_N3D_SINES;
	}
};

// the part of voxel_grid<float> that create_procedural touches (src/voxels.h:100-160)
struct voxel_grid_view {
	unsigned nx, ny, nz;
	float vsz[3], lo_pos[3];
	std::vector<float> *data; // resized to nx*ny*nz, index z + (x + y*nx)*nz
};

// the fill of voxel_manager::create_procedural(mag, freq, offset, normalize_to_1, rseed1, rseed2, gen_mode, verbose) (src/voxels.cpp:278) on grid v;
// zscale = (params.invert ? -1.0 : 1.0)*params.z_gradient/(nz-1), mesh_freq_filter from the scene
inline tw_voxel_params procedural_params(voxel_grid_view const &v, float mag, float freq, const float offset[3], bool normalize_to_1, int rseed1, int rseed2,
	int gen_mode, float zscale, int mesh_freq_filter)
{
	scene_globals const &g = globals();
	tw_voxel_params vp;
	memset(&vp, 0, sizeof(vp));
	vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
	for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d]; vp.offset[d] = offset[d];}
	vp.mag = mag; vp.freq = freq; vp.gen_mode = gen_mode; vp.normalize_to_1 = normalize_to_1; vp.rseed1 = rseed1; vp.rseed2 = rseed2;
	vp.octaves = (5 - mesh_freq_filter > 1) ? (5 - mesh_freq_filter) : 1; // max(1, MAX_FREQ_BINS - mesh_freq_filter), src/voxels.cpp:333
	if (gen_mode != TW_MGEN_SINE) {tw_gen_rx_ry(g.mesh_seed, g.mesh_rgen_index, gen_mode, &vp.rx, &vp.ry);}
	vp.zscale = zscale;
	return vp;
}

// voxel_manager::create_procedural (src/voxels.cpp:278) with the parameters of procedural_params
inline void create_procedural(voxel_grid_view const &v, float mag, float freq, const float offset[3], bool normalize_to_1, int rseed1, int rseed2,
	int gen_mode, float zscale, int mesh_freq_filter)
{
	tw_voxel_params const vp = procedural_params(v, mag, freq, offset, normalize_to_1, rseed1, rseed2, gen_mode, zscale, mesh_freq_filter);
	v.data->resize((size_t)v.nx*v.ny*v.nz);
	tw_ctx *c = ctx();
	int const rc = tw_voxel_fill(c, &vp, nullptr, v.data->data());
	if (rc != TW_OK) {detail::fail(rc, "create_procedural", c);}
}

// voxel_model::build after the fill (src/voxels.cpp:1523-1530 + create_block :1077-1108): determine_voxels_outside, remove_unconnected_outside
// (+ remove_interior_holes for remove_unconnected > 2) and the marching-cubes triangles of the whole grid, on the device. `outside` gets the
// reference's flag bytes; zix_xy (optional) = the per-column under-mesh index the reference derives from z_min_matrix (:596-600); the case tables are
// voxel_detail::edge_table / tri_table / edge_to_vals of src/marching_cubes.h. Returns the unwelded triangle soup (9 floats per triangle).
inline std::vector<float> voxel_build(voxel_grid_view const &v, std::vector<unsigned char> &outside, float isolevel, bool invert, bool make_closed_surface,
	unsigned remove_unconnected, bool keep_at_edge, bool sphere_mode_or_no_mesh, bool skip_under_mesh, const uint32_t *zix_xy,
	const unsigned *edge_table, const int *tri_table, const unsigned *edge_to_vals)
{
	tw_voxel_post_params vp;
	memset(&vp, 0, sizeof(vp));
	vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
	for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d];}
	vp.isolevel = isolevel; vp.invert = invert; vp.make_closed_surface = make_closed_surface; vp.remove_unconnected = (int)remove_unconnected;
	vp.keep_at_edge = keep_at_edge; vp.centre_seed = sphere_mode_or_no_mesh; vp.skip_under_mesh = skip_under_mesh;
	outside.resize(v.data->size());
	tw_ctx *c = ctx();
	int rc = tw_voxel_outside(c, v.data->data(), &vp, zix_xy, outside.data());
	if (rc == TW_OK) {rc = tw_voxel_remove_unconnected(c, v.data->data(), outside.data(), &vp, nullptr);}
	uint64_t n = 0;
	if (rc == TW_OK) {rc = tw_voxel_triangles(c, v.data->data(), outside.data(), &vp, edge_table, tri_table, edge_to_vals, nullptr, 0, &n);}
	std::vector<float> tris((size_t)n*9);
	if (rc == TW_OK && n) {rc = tw_voxel_triangles(c, v.data->data(), outside.data(), &vp, edge_table, tri_table, edge_to_vals, tris.data(), n, &n);}
	if (rc != TW_OK) {detail::fail(rc, "voxel_build", c);}
	return tris;
}

// The indexed mesh of create_block (its tri_verts: vertex positions, then three vertex indices per triangle), welded as the reference's vertex cache
// welds it (tw_voxel_mesh_welded), for the field and flags voxel_build leaves behind.
struct voxel_mesh_t {std::vector<float> verts; std::vector<uint32_t> indices;}; // 3 floats per vertex, 3 indices per triangle
inline voxel_mesh_t voxel_mesh(voxel_grid_view const &v, std::vector<unsigned char> const &outside, float isolevel, bool invert, bool make_closed_surface,
	bool skip_under_mesh, const unsigned *edge_table, const int *tri_table, const unsigned *edge_to_vals)
{
	tw_voxel_post_params vp;
	memset(&vp, 0, sizeof(vp));
	vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
	for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d];}
	vp.isolevel = isolevel; vp.invert = invert; vp.make_closed_surface = make_closed_surface; vp.skip_under_mesh = skip_under_mesh;
	voxel_mesh_t m;
	uint64_t nv = 0, nt = 0;
	tw_voxel_mesh out = {nullptr, 0, nullptr, 0, &nv, &nt};
	tw_ctx *c = ctx();
	int rc = tw_voxel_mesh_welded(c, v.data->data(), outside.data(), &vp, edge_table, tri_table, edge_to_vals, &out);
	if (rc == TW_OK && (nv || nt)) {
		m.verts.resize((size_t)nv*3); m.indices.resize((size_t)nt*3);
		out.verts = m.verts.data(); out.vcapacity = nv; out.indices = m.indices.data(); out.tcapacity = nt;
		rc = tw_voxel_mesh_welded(c, v.data->data(), outside.data(), &vp, edge_table, tri_table, edge_to_vals, &out);
	}
	if (rc != TW_OK) {detail::fail(rc, "voxel_mesh", c);}
	return m;
}

// create_procedural + voxel_build as one job that does not stall the frame (tw_voxel_build_launch): returns at once, and ready() / wait() on the returned
// tiles_job say when the outputs are complete, as for create_tiles_async. fill (optional, from procedural_params): fill the grid first; v.data is then an
// optional output (nullptr: only triangles come out), without fill it is the input field. outside (optional, n bytes) receives the flags. tris: capacity*9
// floats owned by the caller, in device or page-locked host memory; ntris = the triangles the grid produces (may exceed capacity: nothing is written beyond
// it). Everything equals create_procedural + voxel_build byte for byte once the job is ready. The tables and a host zix_xy are copied during the launch; a
// host v.data or outside in pageable memory (a std::vector) makes the launch wait for its copies.
inline tiles_job voxel_build_async(voxel_grid_view const &v, tw_voxel_params const *fill, unsigned char *outside, float isolevel, bool invert, bool make_closed_surface,
	unsigned remove_unconnected, bool keep_at_edge, bool sphere_mode_or_no_mesh, bool skip_under_mesh, const uint32_t *zix_xy,
	const unsigned *edge_table, const int *tri_table, const unsigned *edge_to_vals, float *tris, uint64_t capacity, uint64_t &ntris)
{
	tw_voxel_post_params vp;
	memset(&vp, 0, sizeof(vp));
	vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
	for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d];}
	vp.isolevel = isolevel; vp.invert = invert; vp.make_closed_surface = make_closed_surface; vp.remove_unconnected = (int)remove_unconnected;
	vp.keep_at_edge = keep_at_edge; vp.centre_seed = sphere_mode_or_no_mesh; vp.skip_under_mesh = skip_under_mesh;
	if (fill && v.data) {v.data->resize((size_t)v.nx*v.ny*v.nz);}
	tw_voxel_build b;
	memset(&b, 0, sizeof(b));
	b.fill = fill; b.post = &vp; b.zix_xy = zix_xy;
	b.edge_table256 = edge_table; b.tri_table256x16 = tri_table; b.edge_to_vals12x2 = edge_to_vals;
	b.vals = v.data ? v.data->data() : nullptr; b.outside = outside; b.tris = tris; b.capacity = capacity; b.ntris = &ntris;
	tw_ctx *c = ctx();
	std::atomic<uint64_t> &jobs = detail::tls().tile_jobs;
	uint64_t const number = ++jobs;
	int const rc = tw_voxel_build_launch(c, &b);
	if (rc != TW_OK) {detail::fail(rc, "voxel_build_async", c);}
	return tiles_job(c, &jobs, number);
}
// the same job with the welded mesh of voxel_mesh as well (tw_voxel_build_launch_ex), or instead of the soup when tris == nullptr: verts (vcapacity*3
// floats) and indices (tcapacity*3) in device or page-locked host memory, owned by the caller; nverts / ntris_mesh = the mesh's counts once the job is ready
// (may exceed the capacities: nothing is written beyond them).
inline tiles_job voxel_build_async(voxel_grid_view const &v, tw_voxel_params const *fill, unsigned char *outside, float isolevel, bool invert, bool make_closed_surface,
	unsigned remove_unconnected, bool keep_at_edge, bool sphere_mode_or_no_mesh, bool skip_under_mesh, const uint32_t *zix_xy,
	const unsigned *edge_table, const int *tri_table, const unsigned *edge_to_vals, float *tris, uint64_t capacity, uint64_t *ntris,
	float *verts, uint64_t vcapacity, uint32_t *indices, uint64_t tcapacity, uint64_t &nverts, uint64_t &ntris_mesh)
{
	tw_voxel_post_params vp;
	memset(&vp, 0, sizeof(vp));
	vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
	for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d];}
	vp.isolevel = isolevel; vp.invert = invert; vp.make_closed_surface = make_closed_surface; vp.remove_unconnected = (int)remove_unconnected;
	vp.keep_at_edge = keep_at_edge; vp.centre_seed = sphere_mode_or_no_mesh; vp.skip_under_mesh = skip_under_mesh;
	if (fill && v.data) {v.data->resize((size_t)v.nx*v.ny*v.nz);}
	tw_voxel_build b;
	memset(&b, 0, sizeof(b));
	b.fill = fill; b.post = &vp; b.zix_xy = zix_xy;
	b.edge_table256 = edge_table; b.tri_table256x16 = tri_table; b.edge_to_vals12x2 = edge_to_vals;
	b.vals = v.data ? v.data->data() : nullptr; b.outside = outside; b.tris = tris; b.capacity = capacity; b.ntris = ntris;
	tw_voxel_mesh const m = {verts, vcapacity, indices, tcapacity, &nverts, &ntris_mesh};
	tw_ctx *c = ctx();
	std::atomic<uint64_t> &jobs = detail::tls().tile_jobs;
	uint64_t const number = ++jobs;
	int const rc = tw_voxel_build_launch_ex(c, &b, &m);
	if (rc != TW_OK) {detail::fail(rc, "voxel_build_async", c);}
	return tiles_job(c, &jobs, number);
}

// A voxel model edited with brushes (src/voxels.cpp:2139-2245) and meshed per block, as create_block keeps one mesh and vertex cache per block (:1077-1108),
// kept on the device by the thread's context (tw_voxel_model_*). build_async takes the field from fill or from vals (v.data is not read) and meshes every
// block; edit_async writes boxes of new raw values (one box after another, each z fastest, then x, then y) and re-meshes only the blocks whose cubes read a
// voxel that changed. Both return a tiles_job of the context; out (verts / indices in device or page-locked memory, the host block table and counts) is
// complete once it is ready. The jobs cannot be cancelled. read() completes the pending job and copies the raw field, the field after remove_unconnected
// and its flags. Not copyable; destroyed with the context's pending job completed.
class voxel_model {
	tw_voxel_model *m = nullptr;
	tw_ctx *c = nullptr;
	size_t n = 0;
	tiles_job job_of(int rc, const char *what) {
		std::atomic<uint64_t> &jobs = detail::tls().tile_jobs;
		uint64_t const number = ++jobs;
		if (rc != TW_OK) {--jobs; detail::fail(rc, what, c);}
		return tiles_job(c, &jobs, number);
	}
public:
	voxel_model(voxel_grid_view const &v, float isolevel, bool invert, bool make_closed_surface, unsigned remove_unconnected, bool keep_at_edge,
	            bool sphere_mode_or_no_mesh, bool skip_under_mesh, const uint32_t *zix_xy, const unsigned *edge_table, const int *tri_table,
	            const unsigned *edge_to_vals, unsigned bx, unsigned by)
	{
		tw_voxel_post_params vp;
		memset(&vp, 0, sizeof(vp));
		vp.nx = v.nx; vp.ny = v.ny; vp.nz = v.nz;
		for (int d = 0; d < 3; ++d) {vp.lo_pos[d] = v.lo_pos[d]; vp.vsz[d] = v.vsz[d];}
		vp.isolevel = isolevel; vp.invert = invert; vp.make_closed_surface = make_closed_surface; vp.remove_unconnected = (int)remove_unconnected;
		vp.keep_at_edge = keep_at_edge; vp.centre_seed = sphere_mode_or_no_mesh; vp.skip_under_mesh = skip_under_mesh;
		c = ctx();
		n = (size_t)v.nx*v.ny*v.nz;
		int const rc = tw_voxel_model_create(c, &vp, edge_table, tri_table, edge_to_vals, zix_xy, bx, by, &m);
		if (rc != TW_OK) {detail::fail(rc, "voxel_model", c);}
	}
	~voxel_model() {tw_voxel_model_destroy(m);}
	voxel_model(voxel_model const &) = delete;
	voxel_model &operator=(voxel_model const &) = delete;
	tiles_job build_async(tw_voxel_params const *fill, const float *vals, tw_voxel_blocks_out const &out) {
		return job_of(tw_voxel_model_build_launch(m, fill, nullptr, vals, &out), "voxel_model::build_async");
	}
	tiles_job edit_async(std::vector<tw_voxel_box> const &boxes, const float *values, tw_voxel_blocks_out const &out) {
		return job_of(tw_voxel_model_edit_launch(m, boxes.data(), (uint32_t)boxes.size(), values, &out), "voxel_model::edit_async");
	}
	void read(std::vector<float> *raw, std::vector<float> *vals, std::vector<unsigned char> *outside) {
		if (raw) raw->resize(n);
		if (vals) vals->resize(n);
		if (outside) outside->resize(n);
		int const rc = tw_voxel_model_read(m, raw ? raw->data() : nullptr, vals ? vals->data() : nullptr, outside ? outside->data() : nullptr);
		if (rc != TW_OK) {detail::fail(rc, "voxel_model::read", c);}
	}
};

// ------------------------------------------------------------------------------------------------ all GPUs of the box (include/tw3d.h "Multi-GPU")
// One object per process: per-device contexts with the current tables, NUMA-local pinned output bands, the tile loop of tile_draw_t::update
// (src/tiled_mesh.cpp:2367-2417) dealt out over the devices, and the global z range (get_heightmap_z_range, src/map_view.cpp:399-407) reduced with NCCL.
class multi_gpu {
	tw_multi *m = nullptr;
	std::vector<void *> host_bands;
	void check(int rc, const char *what) {if (rc != TW_OK) {throw error(rc, std::string(what) + ": " + (m ? tw_multi_last_error(m) : "tw_multi_create failed"));}}
public:
	explicit multi_gpu(int ndev, const int *devices = nullptr) {
		check(tw_multi_create(devices, ndev, &m), "tw_multi_create");
		detail::state_t &s = detail::state();
		if (!s.sine_params.empty()) {check(tw_multi_set_sine_params(m, s.sine_params.data()), "tw_multi_set_sine_params");}
	}
	~multi_gpu() {for (void *p : host_bands) {tw_multi_free_host(m, p);} tw_multi_destroy(m);}
	multi_gpu(multi_gpu const &) = delete;
	multi_gpu &operator=(multi_gpu const &) = delete;
	int size() const {return tw_multi_size(m);}
	tw_multi *handle() {return m;}
	// pinned host memory on device i's NUMA node for its band of `ntiles` tiles of zvsize^2 floats (owned by this object)
	float *alloc_band(int i, uint32_t ntiles, uint32_t zvsize) {
		uint32_t a, b;
		tw_multi_range(ntiles, size(), i, &a, &b);
		void *p = nullptr;
		check(tw_multi_alloc_host(m, i, (size_t)(b - a)*zvsize*zvsize*sizeof(float), &p), "tw_multi_alloc_host");
		host_bands.push_back(p);
		return (float *)p;
	}
	// tile_t::create_zvals for all tiles, every device on its band; returns the global z range
	tw_minmax create_zvals(const int32_t *origins_xy, uint32_t ntiles, uint32_t zvsize, float dx, float dy, unsigned erosion_iters_tt, float *const *bands, tw_minmax *mm = nullptr) {
		scene_globals const &g = globals();
		tw_height_params const p = height_params_from_globals(g.mesh_gen_mode, g.mesh_gen_shape);
		tw_erosion_params const e = erosion_params_from_globals();
		tw_minmax zr = {0, 0};
		check(tw_create_zvals_sharded(m, origins_xy, ntiles, g.MESH_X_SIZE, g.MESH_Y_SIZE, dx, dy, zvsize, &p, erosion_iters_tt, &e, g.zmin, bands, mm, &zr), "tw_create_zvals_sharded");
		return zr;
	}
	// heightmap_t::run_erosion on a map held as row bands, coherent across the devices (the batched variant, see tw_erode_sweeps in tw3d.h)
	uint64_t erode_sweeps(float *const *bands, int xsize, int ysize, float min_zval, unsigned num_iters, unsigned sweep = 8192, int halo = 64) {
		tw_erosion_params const e = erosion_params_from_globals();
		uint64_t moves = 0;
		check(tw_erode_sweeps_sharded(m, bands, xsize, ysize, min_zval, num_iters, &e, sweep, halo, &moves), "tw_erode_sweeps_sharded");
		return moves;
	}
};

} // namespace tw3d
