// od_sealevel.cuh -- a varying sea surface height in OceanDrift.
//
//   store_prev_gather_one   update_previous_state (opendrift/models/basemodel/__init__.py:642-657) for an environment variable
//   store_prev_scatter_one  (sea_surface_height, required with store_previous_if drift:vertical_advection, oceandrift.py:73-74).
//                           The store is the reference's `_environment_previous[var]`: float32, one slot per trajectory (keyed by
//                           ID - id_base like the previous positions of od_bookkeep.cuh), NaN at the start of the run.  The
//                           reference, on a step that released elements, first writes the present value of the newly seeded
//                           elements (age_seconds == time_step) at their POSITIONS in the active arrays
//                               store[newly_seeded_rel_indices] = present[newly_seeded_rel_indices]
//                           then gathers previous = store[ID] and stores store[ID] = present.  Positions and IDs differ once
//                           elements were removed before a later release, so an element can gather NaN or another element's
//                           value; that is reproduced.  One gather covers both writes:
//                               prev[i] = (k_i < n && newly[k_i]) ? present[k_i] : store[k_i],   k_i = ID_i - id_base
//                           and the positional writes go to slots the gather does not read; the scatter store[k_i] = present[i]
//                           is a second launch (it overwrites slots the gather reads).
//   vadv_corrected_one      OceanDrift.vertical_advection with drift:vertical_advection_correction (oceandrift.py:325-350):
//                               w -= (delta_zeta / dt) * (z + H) / H,   delta_zeta = ssh - ssh_prev,   H = ssh + floor
//                               z = np.minimum(0, z + moving * w * dt)   for z < 0 (z <= 0 with vertical_advection_at_surface)
//                           in NumPy's dtypes (NEP 50: Python floats are weak): delta_zeta, w_surface and H are float32; the
//                           rest is float32 or float64 as z is; moving (int32) * w is float64.  Every operation is rounded on
//                           its own: no fused multiply-add.  np.minimum propagates NaN.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define OD_SL_HD __host__ __device__ __forceinline__
#else
#define OD_SL_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define OD_SL_MUL_F(a, b) __fmul_rn((a), (b))
#define OD_SL_ADD_F(a, b) __fadd_rn((a), (b))
#define OD_SL_SUB_F(a, b) __fsub_rn((a), (b))
#define OD_SL_DIV_F(a, b) __fdiv_rn((a), (b))
#define OD_SL_MUL_D(a, b) __dmul_rn((a), (b))
#define OD_SL_ADD_D(a, b) __dadd_rn((a), (b))
#define OD_SL_SUB_D(a, b) __dsub_rn((a), (b))
#define OD_SL_DIV_D(a, b) __ddiv_rn((a), (b))
#else
#define OD_SL_MUL_F(a, b) ((a) * (b))
#define OD_SL_ADD_F(a, b) ((a) + (b))
#define OD_SL_SUB_F(a, b) ((a) - (b))
#define OD_SL_DIV_F(a, b) ((a) / (b))
#define OD_SL_MUL_D(a, b) ((a) * (b))
#define OD_SL_ADD_D(a, b) ((a) + (b))
#define OD_SL_SUB_D(a, b) ((a) - (b))
#define OD_SL_DIV_D(a, b) ((a) / (b))
#endif

namespace od {

struct StorePrevParams {
    int64_t n;                   // active elements
    const float* present;        // [n] present value (start-of-step environment)
    const int32_t* ids;          // [n]
    const void* age;             // [n] age_seconds float32 / float64 (age_f64), after increase_age_and_retire; NULL: no release this step
    float* store;                // [n_total] keyed by ID - id_base
    float* prev;                 // [n] out: the previous value of each active element
    int64_t n_total;
    int32_t id_base;
    int32_t age_f64;
    double dt;                   // time_step.total_seconds() (signed)
};

// newly_seeded_rel_indices: age_seconds == time_step.total_seconds() (a float32 array against a weak Python float: float32 compare)
OD_SL_HD bool sl_newly(const StorePrevParams& p, int64_t j) {
    if (!p.age) return false;
    return p.age_f64 ? ((const double*)p.age)[j] == p.dt : ((const float*)p.age)[j] == (float)p.dt;
}

OD_SL_HD void store_prev_gather_one(const StorePrevParams& p, int64_t i) {
    const int64_t k = (int64_t)p.ids[i] - p.id_base;
    float v = NAN;
    if (k >= 0 && k < p.n && sl_newly(p, k)) v = p.present[k];
    else if (k >= 0 && k < p.n_total) v = p.store[k];
    p.prev[i] = v;
    // the positional write of the reference (kept where no active element's ID owns the slot; the scatter overwrites the others)
    if (i < p.n_total && sl_newly(p, i)) p.store[i] = p.present[i];
}

OD_SL_HD void store_prev_scatter_one(const StorePrevParams& p, int64_t i) {
    const int64_t k = (int64_t)p.ids[i] - p.id_base;
    if (k >= 0 && k < p.n_total) p.store[k] = p.present[i];
}

struct VadvCorrParams {
    int64_t n;
    void* z;                     // float32 / float64 (z_f64), updated in place
    const float* w;              // upward_sea_water_velocity
    const float* ssh;            // sea_surface_height
    const float* ssh_prev;       // previous sea_surface_height
    const float* floor;          // sea_floor_depth_below_sea_level, or NULL: floor_const
    const int32_t* moving;
    float floor_const;
    int32_t z_f64;
    int32_t at_surface;          // drift:vertical_advection_at_surface
    double dt;
};

OD_SL_HD double sl_min0(double v) { return v != v ? v : (v < 0.0 ? v : 0.0); }      // np.minimum(0, v): NaN propagates

OD_SL_HD void vadv_corrected_one(const VadvCorrParams& p, int64_t i) {
    const float fl = p.floor ? p.floor[i] : p.floor_const;
    const float s = p.ssh[i];
    const float ws = OD_SL_DIV_F(OD_SL_SUB_F(s, p.ssh_prev[i]), (float)p.dt);     // w_surface, float32
    const float H = OD_SL_ADD_F(s, fl);                                              // total_depth, float32
    const double mv = (double)p.moving[i];
    if (p.z_f64) {
        double* zp = (double*)p.z;
        const double z = zp[i];
        if (!(p.at_surface ? z <= 0.0 : z < 0.0)) return;
        const double we = OD_SL_DIV_D(OD_SL_MUL_D((double)ws, OD_SL_ADD_D(z, (double)H)), (double)H);
        const double w = OD_SL_SUB_D((double)p.w[i], we);
        zp[i] = sl_min0(OD_SL_ADD_D(z, OD_SL_MUL_D(OD_SL_MUL_D(mv, w), p.dt)));
    } else {
        float* zp = (float*)p.z;
        const float z = zp[i];
        if (!(p.at_surface ? z <= 0.0f : z < 0.0f)) return;
        const float we = OD_SL_DIV_F(OD_SL_MUL_F(ws, OD_SL_ADD_F(z, H)), H);
        const float w = OD_SL_SUB_F(p.w[i], we);
        zp[i] = (float)sl_min0(OD_SL_ADD_D((double)z, OD_SL_MUL_D(OD_SL_MUL_D(mv, (double)w), p.dt)));
    }
}

}  // namespace od
