// tw_host.cpp - host-side parameter/table generation of the terrain path (tiny, runs once per scene; bit-exact restatements).
//   rand_gen_t               src/rand_gen.h:22-26,66-70,86,90; src/gen_object.cpp:377-381
//   create_sin_table         src/mesh_gen.cpp:72-81
//   compute_scale            src/mesh_gen.cpp:544-548
//   gen_rand_sine_table_entries / apply_mesh_rand_seed   src/mesh_gen.cpp:213-254
//   gen_rx_ry                src/mesh_gen.cpp:581-586
//   noise_gen_3d::gen_sines  src/upsurface.cpp:16-38
//   get_water_z_height       src/mesh_gen.cpp:362,507-512
// Compiled without FMA contraction (-ffp-contract=off) like the reference build (makefile:11, no -march).
#include "../../include/tw3d.h"
#include <cmath>

namespace {

constexpr float PI_F = 3.141592654f;                 // src/3DWorld.h:43
constexpr float TWO_PI_F = (float)(2.0*PI_F);        // src/3DWorld.h:129
constexpr unsigned TSIZE = 32768;                    // src/sinf.h:8
constexpr float SSCALE = (float)TSIZE/TWO_PI_F;      // src/sinf.h:9

struct rand_gen {
	long s1, s2; // 64-bit long (LP64), as rgen_core_t::rseed1/2
	explicit rand_gen(tw_rng const &r) : s1((long)r.rseed1), s2((long)r.rseed2) {}
	rand_gen() : s1(1), s2(1) {}
	void set_state(long a, long b) {s1 = a; s2 = b;}
	void step() {
		if ((s1 = 40014*(s1%53668) - 12211*(s1/53668)) < 0) s1 += 2147483563;
		if ((s2 = 40692*(s2%52774) - 3791 *(s2/52774)) < 0) s2 += 2147483399;
	}
	int rand() {step(); int r = (int)s1 - (int)s2; if (r < 1) r += 2147483562; return r;}
	double randd() {step(); double r = (double)s1 - (double)s2; if (r < 1) r += 2147483562; return r/2147483563.;}
	float rand_float() {return 0.000001*(rand()%1000000);}
	float rand_uniform(float a, float b) {return a + (b - a)*float(randd());}
	void store(tw_rng &r) const {r.rseed1 = s1; r.rseed2 = s2;}
};

void apply_mesh_rand_seed(rand_gen &rgen, int mesh_seed, int mesh_rgen_index, int mode) {
	if (mesh_seed != 0) {rgen.set_state(mesh_seed, 12345);}
	else if (mode != TW_MGEN_SINE) {rgen.set_state(mesh_rgen_index+1, 12345);}
}

} // namespace

// the part of get_water_z_height that does not depend on zmax_est (tw_internal.h)
float twi_water_rel(int glaciate, float custom_glaciate_exp, float water_h_off_rel) {
	float const t(0.42f + water_h_off_rel); // W_PLANE_Z
	float const lo((t < 1.0f) ? t : 1.0f);
	float wpz((0.0f < lo) ? lo : 0.0f);       // CLIP_TO_01
	if (glaciate) {wpz = ((custom_glaciate_exp == 0.0f) ? wpz*wpz*wpz : std::pow(wpz, custom_glaciate_exp));}
	return wpz;
}

extern "C" {

void tw_build_sin_table(float *tab) {
	for (unsigned i = 0; i < TSIZE; ++i) {
		tab[i]       = sinf(i/SSCALE);
		tab[i+TSIZE] = cosf(i/SSCALE);
	}
}

int tw_compute_scale(float mesh_scale, int mesh_freq_filter) {
	int const iscale = int(std::log2(mesh_scale));
	int v = iscale + mesh_freq_filter;
	v = (v < 9-3) ? v : 9-3; // min(NUM_FREQ_COMP-MIN_FREQS, .)
	v = (v > 0) ? v : 0;
	return 10*v;
}

void tw_gen_sine_params(tw_rng *state, float scaled_height, int MX, int MY, float XSS, float YSS, int mesh_seed, int mesh_rgen_index,
	int mode, float start_mag, float start_freq, float mag_mult, float freq_mult, float *T)
{
	float xf_scale((float)MY/(float)MX), yf_scale(1.0/xf_scale);
	if (XSS > YSS) yf_scale *= (float)YSS/(float)XSS;
	if (YSS > XSS) xf_scale *= (float)XSS/(float)YSS;
	float mags[9] = {}, freqs[9] = {};
	freqs[0] = start_freq; mags[0] = start_mag;
	for (int i = 1; i < 9; ++i) {freqs[i] = freqs[i-1]*freq_mult; mags[i] = mags[i-1]*mag_mult;}
	float const mesh_h(scaled_height/std::sqrt(0.1*10));
	rand_gen rgen(*state);
	apply_mesh_rand_seed(rgen, mesh_seed, mesh_rgen_index, mode);
	for (int l = 0; l < 9; ++l) {
		float const x_freq(freqs[l]/((float)MX)), y_freq(freqs[l]/((float)MY));
		float const mheight(mags[l]*mesh_h);
		for (int i = 0; i < 10; ++i) {
			float *e = T + 5*(l*10 + i);
			e[0] = rgen.rand_uniform(0.2, 1.0)*mheight;          // magnitude
			e[1] = rgen.rand_float()*TWO_PI_F;                   // y phase
			e[2] = rgen.rand_float()*TWO_PI_F;                   // x phase
			e[3] = rgen.rand_uniform(0.1, 1.0)*x_freq*yf_scale;  // y frequency
			e[4] = rgen.rand_uniform(0.1, 1.0)*y_freq*xf_scale;  // x frequency
		}
	}
	rgen.store(*state);
}

void tw_gen_rx_ry(int mesh_seed, int mesh_rgen_index, int mode, float *rx, float *ry) {
	rand_gen rgen;
	apply_mesh_rand_seed(rgen, mesh_seed, mesh_rgen_index, mode);
	*rx = rgen.rand_float() + 1.0;
	*ry = rgen.rand_float() + 1.0;
}

void tw_noise3d_gen_sines(int rs1, int rs2, float mag, float freq, float *rdata) {
	rand_gen rgen; rgen.set_state(rs1, rs2);
	for (unsigned i = 0; i < 5; ++i) {          // MAX_FREQ_BINS, low frequencies first
		for (unsigned j = 0; j < 12; ++j) {     // SINES_PER_FREQ
			float *e = rdata + 7*(12*i + j);
			e[0] = rgen.rand_uniform(0.2, 1.0)*mag;
			e[1] = rgen.rand_uniform(0.1, 1.0)*freq;
			e[2] = rgen.randd()*TWO_PI_F;
			e[3] = rgen.rand_uniform(0.1, 1.0)*freq;
			e[4] = rgen.randd()*TWO_PI_F;
			e[5] = rgen.rand_uniform(0.1, 1.0)*freq;
			e[6] = rgen.randd()*TWO_PI_F;
		}
		mag  *= 0.5f;   // M_ATTEN_FACTOR
		freq /= 0.4f;   // F_ATTEN_FACTOR
	}
}

float tw_water_z_height(float zmax_est, int glaciate, float custom_glaciate_exp, float water_h_off, float water_h_off_rel) {
	float const wpz = twi_water_rel(glaciate, custom_glaciate_exp, water_h_off_rel);
	float const zmax_est2(2.0*zmax_est);
	return wpz*zmax_est2 - zmax_est + water_h_off;
}

// init_terrain_mesh() + gen_tex_height_tables() (src/mesh_gen.cpp:407-431, src/Textures.cpp:1757-1761): the relative-height thresholds of the five ground textures
// (mesh_tids_dirt / mesh_rh_dirt, :42-43) moved with the water level, h_dirt[i] = pow(zval, glaciate_exp), clip_hd1 = 0.90*h_dirt[1] + 0.10*h_dirt[0]
void tw_gen_tex_height_tables(float water_h_off_rel, float temperature, float glaciate_exp, float h_dirt[5], int tex_class[5], float *clip_hd1) {
	float const W_PLANE_Z = 0.42;                                                   // src/mesh_gen.cpp:19
	float const mesh_rh_dirt[5] = {0.40, 0.44, 0.60, 0.75, 1.0};                    // :43
	int   const mesh_tids_dirt[5] = {TW_TEX_SAND, TW_TEX_DIRT, TW_TEX_GROUND, TW_TEX_ROCK, TW_TEX_SNOW}; // :42
	float const t(W_PLANE_Z + water_h_off_rel);
	float const lo((t < 1.0f) ? t : 1.0f);
	float const rel_wpz((0.0f < lo) ? lo : 0.0f);                                   // get_rel_wpz(): CLIP_TO_01(W_PLANE_Z + water_h_off_rel), :362
	for (unsigned i = 0; i < 5; ++i) {
		float const def_h(mesh_rh_dirt[i]);
		float h;
		if (mesh_rh_dirt[i] < W_PLANE_Z) {h = def_h*rel_wpz/W_PLANE_Z;}             // below water
		else { // above water
			float const rel_h((def_h - W_PLANE_Z)/(1.0f - W_PLANE_Z));
			h = rel_wpz + rel_h*(1.0 - rel_wpz);
			if (mesh_tids_dirt[i] == TW_TEX_SNOW) {
				h = (def_h < h) ? def_h : h;                                        // min(h, def_h): snow can't get lower when water lowers
				if (temperature > 40.0) h += 0.01*(temperature - 40.0);             // less snow with increasing temperature
			}
		}
		if (tex_class) {tex_class[i] = mesh_tids_dirt[i];}
		h_dirt[i] = std::pow(h, glaciate_exp);                                      // pow(float, float) -> float
	}
	if (clip_hd1) {*clip_hd1 = (0.90*h_dirt[1] + 0.10*h_dirt[0]);}
}

// 1e6-entry direction table for the erosion random-direction fallback (src/erosion.cpp:84-87):
// a = rgen.rand_float()*TWO_PI with rand_float() = 0.000001*(rand()%1000000); dx=cosf(a); dz=sinf(a)
void twi_build_dir_table(float *cs2x1e6) {
	for (int k = 0; k < 1000000; ++k) {
		float const rf(0.000001*k);
		float const a(rf*TWO_PI_F);
		cs2x1e6[2*k] = cosf(a); cs2x1e6[2*k+1] = sinf(a);
	}
}

} // extern "C"
