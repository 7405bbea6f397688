// od_mix.cuh -- vertical turbulent mixing of one particle (Visser random walk), all inner iterations fused.
//
// Restates OceanDrift.vertical_mixing (opendrift/models/oceandrift.py:397-571) for diffusivity taken from the
// environment profiles, with the profile block exactly as Environment.get_environment hands it over
// (opendrift/models/basemodel/environment.py:697-724): per block layer the float32 horizontal interpolation of
// ReaderBlock (interpolation/structured.py:148-163), time-interpolated in float64 (basereader/structured.py:366-383),
// then written back through a float32 cast for every layer but the last.  The reference materialises (nz, N)
// profile arrays (1 GB per variable at 5 M particles x 50 layers) and loops dt/dt_mix times over N-sized NumPy
// expressions; here each thread evaluates the levels of its K column it actually visits (a sliding 8-level window)
// and runs the whole inner loop.
//   gradK = -np.gradient(K, z)  thresholded at 1e-10            (:500-502)
//   zi = round(interp1d(-z_levels -> index)(-z))  as uint16     (:513)
//   z -= moving * (dKdz*dt_mix - R*sqrt(K*|dt_mix|*2/r)), R = 2*U(0,1)-1, r = 1/3   (:524-528)
//   reflect at the surface (:531-533) and at the sea floor (:537-540), buoyancy w*dt_mix (:543),
//   surface pinning (:548-549), surface_stick (:370-374).
// Random numbers: either the caller's array (NumPy's legacy generator, for bit parity with the reference) or
// Philox4x32-10 keyed by (seed, element ID, step, iteration) -- independent of the order of the particle arrays.
#pragma once
#include "od_interp.cuh"

namespace od {

// Philox4x32-10 (Salmon et al., SC'11), counter-based; philox_uniform2 returns two uniform doubles in [0, 1)
OD_HD void philox_round(unsigned& c0, unsigned& c1, unsigned& c2, unsigned& c3, unsigned k0, unsigned k1) {
        const unsigned long long p0 = 0xD2511F53ull * c0, p1 = 0xCD9E8D57ull * c2;
        const unsigned n0 = (unsigned)(p1 >> 32) ^ c1 ^ k0, n1 = (unsigned)p1;
        const unsigned n2 = (unsigned)(p0 >> 32) ^ c3 ^ k1, n3 = (unsigned)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}
OD_HD void philox_uniform2(unsigned long long seed, unsigned id, unsigned step, unsigned iter, double& u0, double& u1) {
        unsigned c0 = id, c1 = step, c2 = iter, c3 = 0x6f647274u;
        unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
        for (int r = 0; r < 10; ++r) {
            philox_round(c0, c1, c2, c3, k0, k1);
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        // 53-bit doubles like NumPy's random(): (a >> 5, b >> 6)
        u0 = ((double)(c0 >> 5) * 67108864.0 + (double)(c1 >> 6)) * (1.0 / 9007199254740992.0);
        u1 = ((double)(c2 >> 5) * 67108864.0 + (double)(c3 >> 6)) * (1.0 / 9007199254740992.0);
}

struct MixParams {
    GroupGeom g;                 // 1-component 3-D group: ocean_vertical_diffusivity
    PairRef pr;
    int64_t n;
    const double* lon;           // positions at the START of the step (where the environment profiles are sampled)
    const double* lat;
    const void* z_in;            // float32 or float64 (z_in_f64)
    double* z_out;               // always float64: the reference's z becomes float64 here (:527)
    const int32_t* moving;       // NULL = all moving
    const void* terminal_velocity;   // NULL = 0; float32 or float64 (tv_f64)
    const int32_t* ids;          // element IDs (Philox key); NULL = array index
    const double* rand;          // [ntimes][n] uniform draws of the legacy generator, or NULL -> Philox
    double dt_mix;               // signed like the time step
    double zmin_const;           // -(sea_floor_depth + sea_surface_height) when no per-particle array is given
    const float* sea_floor;      // optional per-particle sea_floor_depth_below_sea_level (float32)
    unsigned long long seed;
    int32_t ntimes, z_in_f64, tv_f64, mix_at_surface, pos_f32, step_index;
    const double* zl;            // [nz] block level depths as the reader gives them (mixing_z)
    const double* xs;            // [nz] -mixing_z sorted increasing
    const double* xy;            // [nz] index of each xs entry
    int32_t uniform_dz;
    // Analytical diffusivity (vertical_mixing:diffusivitymodel other than a usable ocean-model field, oceandrift.py:429-453):
    // 1 m levels mixing_z = -arange(nlev), nlev = int(ceil(max(MLD) + 2)); K from the wind speed and the mixed layer depth.
    int32_t model;               // 0 environment profile, 1 windspeed_Large1994, 2 windspeed_Sundby1983, 3 constant
    double dz0;                  // np.diff(mixing_z)[0] when the spacing is uniform
    const float* wind_speed;     // [n] float32 sqrt(x_wind^2 + y_wind^2) at the start of the step
    const float* mld;            // [n] float32 ocean_mixed_layer_thickness, or NULL -> mld_const
    float mld_const, pad2_;
    double background;           // vertical_mixing:background_diffusivity
    double k_const;              // model 3
    // 'Let particles stick to bottom' (oceandrift.py:559-564 -> interact_with_seafloor, basemodel/__init__.py:748-783)
    int32_t seafloor_action;     // 0 none, 1 lift_to_seafloor, 2 deactivate
    int32_t seafloor_code;
    int32_t iter0;               // first inner iteration of this launch within the step (per-iteration launches for hook overrides)
    int32_t skip_surface_stick;
    int32_t* status;
    int32_t* moving_out;
    unsigned* counter;
};

// physics_methods.py:217-249 (Large et al. 1994) and :203-215 (Sundby 1983) for one level (depth d metres) of one
// particle, in NumPy's dtype flow: float32 wind stress and MLD factors, float64 depth ratio.
OD_HD double k_analytic(const MixParams& p, float ws, float m, int l) {
    const double d = (double)l, bg = p.background;
    if (p.model == 3) return p.k_const;
    if (p.model == 2) {
        double K = OD_DADD(76.1e-4, (double)OD_FMUL(OD_FMUL((float)2.26e-4, ws), ws));
        if (d > (double)OD_FADD(m, -1.0f)) K = OD_DADD(K, bg) / 2.0;
        if (d >= (double)m) K = bg;
        return K;
    }
    const float stress = OD_FMUL(OD_FMUL(OD_FMUL(ws, ws), (float)1.25e-3), (float)1.22);
    const double sigma = d / (double)m;
    double G = OD_DADD(OD_DADD(sigma, OD_DMUL(-2.0, OD_DMUL(sigma, sigma))), pow(sigma, 3.0));
    if (G >= 1.0) G = OD_DMUL(G, 0.0);
    const float c = OD_FMUL(OD_FMUL(m, (float)0.2), (float)0.4);
    double K = OD_DADD(OD_DMUL(OD_DMUL((double)c, G), (double)stress), OD_DMUL(sigma, bg));
    if (d >= (double)m) K = bg;
    return K;
}

// One level of the particle's diffusivity column (environment profile), on demand.
OD_HD double k_level_raw(const MixParams& p, const HorizW& h, int l) {
    double v = NAN;
    if (h.valid && p.pr.mode != 3) {
        const long long layer = (long long)p.g.nx * p.g.ny;
        const float* t = p.pr.tex + ((long long)l * layer) * 2;
        const Tex2 a00 = ld_tex2(t + 2ll * h.i00), a01 = ld_tex2(t + 2ll * h.i01);
        const Tex2 a10 = ld_tex2(t + 2ll * h.i10), a11 = ld_tex2(t + 2ll * h.i11);
        const double hA = (double)bilin(h, a00.x, a01.x, a10.x, a11.x);
        if (p.pr.mode == 1) v = hA;
        else {
            const double hB = (double)bilin(h, a00.y, a01.y, a10.y, a11.y);
            v = p.pr.mode == 2 ? hB : OD_DADD(OD_DMUL(hA, OD_DSUB(1.0, p.pr.w)), OD_DMUL(hB, p.pr.w));
        }
    }
    if (l < p.g.nz - 1) v = (double)(float)v;      // environment.py:706-713 (float32 write-back, all but the last layer)
    return v;
}

OD_HD double k_level(const MixParams& p, const HorizW& h, int l) {
    double v = k_level_raw(p, h, l);
    if (l == p.g.nz - 1 && p.g.nz > 1 && v != v) v = k_level_raw(p, h, l - 1);       // environment.py:715-724
    if (!(fabs(v) <= 1.7976931348623157e308)) v = (double)p.g.fallback[0];          // masked -> fallback (:803-806)
    return v;
}

// A window of OD_MIX_WINDOW consecutive levels of the column, recentred (and recomputed) when the particle
// leaves it: a random-walk step is a fraction of a level, so one window serves a whole time step almost always.
#define OD_MIX_WINDOW 8
struct KWindow {
    double v[OD_MIX_WINDOW];
    int lo;
    float ws, mld;               // analytical models: this particle's wind speed and mixed layer depth
};

OD_HD void k_window_fill(const MixParams& p, const HorizW& h, KWindow& w, int centre) {
    const int nz = p.g.nz;
    int lo = centre - OD_MIX_WINDOW / 2;
    if (lo > nz - OD_MIX_WINDOW) lo = nz - OD_MIX_WINDOW;
    if (lo < 0) lo = 0;
    w.lo = lo;
    for (int k = 0; k < OD_MIX_WINDOW; ++k)
        w.v[k] = (lo + k < nz) ? (p.model ? k_analytic(p, w.ws, w.mld, lo + k) : k_level(p, h, lo + k)) : 0.0;
}

OD_HD double k_get(const MixParams& p, const HorizW& h, KWindow& w, int l) {
    if (l < w.lo || l >= w.lo + OD_MIX_WINDOW) k_window_fill(p, h, w, l);
    return w.v[l - w.lo];            // dynamically indexed: 64 bytes of (L1-resident) local memory per thread
}

// -np.gradient(K, mixing_z)[l] with numpy's edge_order=1 formulas, |g| < 1e-10 -> 0
OD_HD double neg_gradient(const MixParams& p, const HorizW& h, KWindow& w, int l) {
    const int nz = p.g.nz;
    double gr;
    if (l == 0) {
        gr = OD_DSUB(k_get(p, h, w, 1), k_get(p, h, w, 0)) / (p.uniform_dz ? p.dz0 : OD_DSUB(p.zl[1], p.zl[0]));
    } else if (l == nz - 1) {
        gr = OD_DSUB(k_get(p, h, w, nz - 1), k_get(p, h, w, nz - 2)) / (p.uniform_dz ? p.dz0 : OD_DSUB(p.zl[nz - 1], p.zl[nz - 2]));
    } else if (p.uniform_dz) {
        gr = OD_DSUB(k_get(p, h, w, l + 1), k_get(p, h, w, l - 1)) / OD_DMUL(2.0, p.dz0);
    } else {
        const double dx1 = OD_DSUB(p.zl[l], p.zl[l - 1]), dx2 = OD_DSUB(p.zl[l + 1], p.zl[l]);
        const double a = -(dx2) / OD_DMUL(dx1, OD_DADD(dx1, dx2));
        const double b = OD_DSUB(dx2, dx1) / OD_DMUL(dx1, dx2);
        const double c = dx1 / OD_DMUL(dx2, OD_DADD(dx1, dx2));
        gr = OD_DADD(OD_DADD(OD_DMUL(a, k_get(p, h, w, l - 1)), OD_DMUL(b, k_get(p, h, w, l))), OD_DMUL(c, k_get(p, h, w, l + 1)));
    }
    gr = -gr;
    return fabs(gr) < 1e-10 ? 0.0 : gr;
}

// index of the nearest profile level: np.round(interp1d(-mixing_z, range(nz), fill_value=(0, nz-1))(-z))
OD_HD int nearest_level(const MixParams& p, const double* xs, const double* xy, double x_new) {
    const int nz = p.g.nz;
    double y;
    const double x_first = p.model ? 0.0 : xs[0], x_last = p.model ? (double)(nz - 1) : xs[nz - 1];
    if (x_new < x_first) y = 0.0;
    else if (x_new > x_last) y = (double)(nz - 1);
    else if (p.model) {                      // levels 0, 1, 2, ...: the table is its own index
        const int lo = (int)ceil(x_new);      // searchsorted(side='left')
        const int idx = lo < 1 ? 1 : (lo > nz - 1 ? nz - 1 : lo);
        const double x0 = (double)(idx - 1);
        const double slope = OD_DSUB((double)idx, x0) / OD_DSUB((double)idx, x0);
        y = OD_DADD(OD_DMUL(slope, OD_DSUB(x_new, x0)), x0);
    } else {
        int lo = 0, hi = nz;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (xs[mid] < x_new) lo = mid + 1; else hi = mid;
        }
        const int idx = lo < 1 ? 1 : (lo > nz - 1 ? nz - 1 : lo);
        const double slope = OD_DSUB(xy[idx], xy[idx - 1]) / OD_DSUB(xs[idx], xs[idx - 1]);
        y = OD_DADD(OD_DMUL(slope, OD_DSUB(x_new, xs[idx - 1])), xy[idx - 1]);
    }
    int zi = (int)rint(y);
    return zi < 0 ? 0 : (zi > nz - 1 ? nz - 1 : zi);
}

// SedimentDrift.bottom_interaction (sedimentdrift.py:108-116) inside the loop, kept apart from MixParams: with settling the input
// moving / status are only read, and every element's values after the loop go to the outputs here.
struct SettleParams {
    int32_t* moving_out;         // [n]
    int32_t* status_out;         // [n], or NULL when seafloor_action != 2
    unsigned* undecided;         // elements whose settling depended on the others (see mix_particle)
};

OD_HD void count_one(unsigned* c) {
#if defined(__CUDA_ARCH__)
    atomicAdd(c, 1u);
#else
    *c += 1u;
#endif
}

// SETTLE: after the sea floor, an element at or below Zmin that still moves settles (moving = 0 from there on).  The reference
// calls bottom_interaction only in iterations where SOME element is below Zmin before the lift; an element that was below itself
// decides that alone.  One that ends the iteration exactly at Zmin, moving, without having been below is left moving and counted
// in *s->undecided: its result is only valid if no other element was below, which the caller cannot know from here.
template <bool PROJ = false, bool SETTLE = false>
OD_HD void mix_particle(const MixParams& p, int64_t i, const double* xs, const double* xy, const SettleParams* s = nullptr) {
    const GroupGeom& g = p.g;
    // the particle's diffusivity column (environment profile) is evaluated lazily, a window of levels at a time
    HorizW h;
    KWindow kw;
    kw.lo = -(1 << 20);
    kw.ws = kw.mld = 0.0f;
    if (p.model) {
        h.valid = false;
        kw.ws = p.wind_speed ? p.wind_speed[i] : 0.0f;
        kw.mld = p.mld ? p.mld[i] : p.mld_const;
    } else {
        h = PROJ ? horiz_weights_h(g, p.lon[i], p.lat[i], p.pos_f32 != 0) : horiz_weights(g, p.lon[i], p.lat[i], p.pos_f32 != 0);
    }

    // ---- inner loop ---------------------------------------------------------------------------------------------
    double z = p.z_in_f64 ? ((const double*)p.z_in)[i] : (double)((const float*)p.z_in)[i];
    double mv = p.moving ? (double)p.moving[i] : 1.0;
    bool deactivated = false;
    const double w = p.terminal_velocity ? (p.tv_f64 ? ((const double*)p.terminal_velocity)[i]
                                                      : (double)((const float*)p.terminal_velocity)[i]) : 0.0;
    const double zmin = p.sea_floor ? -(double)p.sea_floor[i] : p.zmin_const;
    const double adt = fabs(p.dt_mix);
    const double r = 1.0 / 3;
    const unsigned id = p.ids ? (unsigned)p.ids[i] : (unsigned)i;
    double spare = 0.0;
    bool settled = false, undecided = false;
    for (int it = 0; it < p.ntimes; ++it) {
        const bool surface = z == 0.0;
        const int zi = nearest_level(p, xs, xy, -z);
        const double Kz = k_get(p, h, kw, zi);
        const double dKdz = neg_gradient(p, h, kw, zi);
        double U;
        if (p.rand) {
            U = p.rand[(int64_t)it * p.n + i];
        } else {
            // one Philox block serves two iterations; a launch that starts on an odd iteration regenerates its block
            const int git = p.iter0 + it;
            if ((git & 1) == 0 || it == 0) {
                double a, b;
                philox_uniform2(p.seed, id, (unsigned)p.step_index, (unsigned)(git >> 1), a, b);
                U = (git & 1) ? b : a;
                spare = b;
            } else {
                U = spare;
            }
        }
        const double R = OD_DSUB(OD_DMUL(2.0, U), 1.0);
        const double walk = OD_DMUL(R, sqrt(OD_DMUL(OD_DMUL(Kz, adt), 2.0) / r));
        z = OD_DSUB(z, OD_DMUL(mv, OD_DSUB(OD_DMUL(dKdz, p.dt_mix), walk)));
        if (z >= 0.0) z = -z;                                         // reflect from the surface
        if (z < zmin && mv == 1.0) z = OD_DSUB(OD_DMUL(2.0, zmin), z);    // reflect from the sea floor
        z = OD_DADD(z, OD_DMUL(OD_DMUL(w, p.dt_mix), mv));           // buoyancy
        if (!p.mix_at_surface && surface) z = 0.0;
        if (z > 0.0 && !p.skip_surface_stick) z = 0.0;                 // surface_stick
        [[maybe_unused]] const bool below = z < zmin;            // before the lift
        if (p.seafloor_action && z < zmin) {                           // stick to the bottom
            z = zmin;
            if (p.seafloor_action == 2) {                              // deactivate_elements: moving = 0 from here on
                mv = 0.0;
                deactivated = true;
            }
        }
        if constexpr (SETTLE) {
            if (z <= zmin && mv == 1.0) {
                if (below) {
                    mv = 0.0;
                    settled = true;
                } else {
                    undecided = true;
                }
            }
        }
    }
    p.z_out[i] = z;
    if constexpr (SETTLE) {
        const int32_t st = s->status_out ? p.status[i] : 0;
        s->moving_out[i] = (settled || deactivated) ? 0 : (p.moving ? p.moving[i] : 1);
        if (s->status_out) s->status_out[i] = (deactivated && st == 0) ? p.seafloor_code : st;
        if (deactivated && p.counter) count_one(p.counter);
        if (undecided) count_one(s->undecided);
    } else if (deactivated) {
        if (p.status[i] == 0) p.status[i] = p.seafloor_code;
        p.moving_out[i] = 0;
#if defined(__CUDA_ARCH__)
        if (p.counter) atomicAdd(p.counter, 1u);
#else
        if (p.counter) *p.counter += 1u;
#endif
    }
}

// SedimentDrift.resuspension (sedimentdrift.py:118-126) for one element: current_speed() squares the float32 environment components
// and takes a float32 root (sqrtf is correctly rounded, as NumPy's), compared with the threshold as a float32 (NEP 50: a Python
// float is weak); where it fires moving = 1 and z += 0.01 in z's own dtype.
OD_HD void resuspend_one(int64_t i, const float* u, const float* v, float threshold, int32_t* moving, void* z, int z_f64) {
    const float speed = sqrtf(OD_FADD(OD_FMUL(u[i], u[i]), OD_FMUL(v[i], v[i])));
    if (!(speed > threshold && moving[i] == 0)) return;
    moving[i] = 1;
    if (z_f64) ((double*)z)[i] = OD_DADD(((double*)z)[i], 0.01);
    else ((float*)z)[i] = OD_FADD(((float*)z)[i], 0.01f);
}

}  // namespace od
