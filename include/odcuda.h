/* odcuda.h -- C-ABI of libodcuda.so: the H100 (sm_90a) particle-advection hot path behind
 * OpenDrift's Python interface.
 *
 * The reference (OpenDrift 1.14.10, pure Python) has no FFI for this path; its extension API is
 * Python subclassing.  Each entry point below replaces the *body* of a reference Python method and
 * is bound from Python with ctypes (opendrift_b200/_lib.py).  Reference interface replaced, per call:
 *
 *   od_geod_fwd           pyproj.Geod(ellps='WGS84').fwd as called at
 *                         opendrift/models/basemodel/__init__.py:4651-4657, physics_methods.py:632-635
 *   od_update_positions   OpenDriftSimulation.update_positions   basemodel/__init__.py:4630-4669
 *   od_field_* / od_interp  StructuredReader._get_variables_interpolated_ + ReaderBlock.interpolate
 *                         readers/basereader/structured.py:202-400, readers/interpolation/structured.py:107-163,
 *                         readers/interpolation/interpolators.py:105-139, 174-197; the float32 cast and
 *                         fallback fill of Environment.get_environment  basemodel/environment.py:695-696, 782-791
 *   od_advect_current     PhysicsMethods.advect_ocean_current    models/physics_methods.py:611-691
 *   od_step_oceandrift    OceanDrift.update + horizontal_diffusion  models/oceandrift.py:185-211,
 *                         basemodel/__init__.py:1746-1772 (current -> wind -> vertical advection -> diffusion)
 *   od_sort_* / od_permute LagrangianArray element order (elements/elements.py:197-228) -- locality only
 *
 * Conventions: every pointer named d_* is a CUDA device pointer owned by the caller (PyTorch tensors are
 * used only as allocators); h_* are host pointers.  All calls enqueue work on the context's stream and
 * return immediately, except where stated.  Return value: 0 on success, negative od_status otherwise;
 * od_last_error() gives the text.  Nothing throws or aborts.  A context is not thread-safe.
 */
#ifndef ODCUDA_H
#define ODCUDA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct od_ctx od_ctx;

enum od_status {
    OD_OK = 0,
    OD_ERR_CUDA = -1,
    OD_ERR_ARG = -2,
    OD_ERR_STATE = -3,
    OD_ERR_NOMEM = -4
};

enum od_scheme { OD_EULER = 0, OD_RK2 = 1, OD_RK4 = 2 };

/* how a time sample combines the two slabs of a pair */
enum od_time_mode {
    OD_T_LERP = 0,     /* slab_a*(1-w) + slab_b*w                        (structured.py:353-364) */
    OD_T_FIRST = 1,    /* slab_a only: time == time_before               (structured.py:224-229, 339) */
    OD_T_SECOND = 2,   /* slab_b only */
    OD_T_MISSING = 3   /* reader does not cover this time: every particle gets the fallback value
                          (OutsideTemporalCoverageError -> NaN -> fallback, environment.py:642-654, 782-791) */
};

enum od_lon_mode { OD_LON_0_360 = 0, OD_LON_PM180 = 1 };

enum od_interp_flags { OD_INTERP_POS_F32 = 1, OD_INTERP_NO_FALLBACK = 2, OD_INTERP_Z_F64 = 4,
                       OD_INTERP_NO_ROTATE = 8 /* projected vector pairs stay along the grid's axes (rotate_to_proj=None) */,
                       OD_INTERP_OUT_F64 = 16 /* d_out are float64 arrays holding what the READER returns: the unrounded float64 vertical /
                                                 time lerp of a 3-D block (interpolation/structured.py:139-140), the float32 value of a 2-D one */,
                       OD_INTERP_NEAREST = 32 /* nearest grid point, as the reference samples land_binary_mask (Nearest2DInterpolator,
                                                 interpolators.py:26-40); 2-D one-component geographic groups */ };

#define OD_MAX_LEVELS 128
#define OD_ABI_VERSION 1

int od_abi_version(void);

/* ---- context ---------------------------------------------------------------------------- */
int od_create(int device, od_ctx** out);
void od_destroy(od_ctx* ctx);
const char* od_last_error(od_ctx* ctx);
/* use an existing CUDA stream (cudaStream_t passed as void*; NULL = legacy default stream) */
int od_set_stream(od_ctx* ctx, void* cuda_stream);
int od_sync(od_ctx* ctx);                        /* blocks until the stream is idle */
/* OD_OPT_TILE: od_advect_current (RK schemes) stages a box of pair texels per thread block in shared memory with one
 * TMA load (cp.async.bulk.tensor.4d) and serves the bilinear corners of all stages from it; pays off for cell-sorted
 * particle arrays, results are bit-identical either way.
 * OD_OPT_SPEC (default 1): RK4 launches of the default arithmetic on a geographic, non-periodic 3-D current group between
 * two reader times take the specialised step kernel (csrc/od_spec.cuh); 0 keeps the general kernel.  Results are
 * bit-identical either way (tests/test_zz_gpu_spec.py). */
enum od_option { OD_OPT_TILE = 1, OD_OPT_SPEC = 2 };
int od_set_option(od_ctx* ctx, int option, int value);
int od_device_sm_count(od_ctx* ctx);

/* ---- forcing fields ---------------------------------------------------------------------
 * A field *group* is one reader block geometry carrying 1 or 2 components that are always
 * sampled together (e.g. x/y_sea_water_velocity; upward_sea_water_velocity; x/y_wind).
 * x0/xspan/y0/yspan follow Linear2DInterpolator: xi = (x - x0) / xspan * (nx - 1) with
 * x0 = (double)xgrid[0], xspan = (double)(float)(xgrid[nx-1] - xgrid[0]) for float32 grids.
 * xmin..ymax is the reader's coverage box (covers_positions_xy).  h_z_levels: nz level depths
 * as the reader returns them (increasing or decreasing), ignored when nz == 1.
 * fallback[c]: value used where the sample is not finite / not covered; NaN = none.
 * wrap_x: the grid covers the globe east-west (reference: Variables.global_coverage, readers/basereader/variables.py:289-301)
 * and is periodic: the block the sampler sees is the nx stored columns plus one virtual column that repeats column 0 at
 * xgrid[nx-1] + dx (what a reference reader hands to ReaderBlock(wrap_x=True) so that the seam cell is covered,
 * readers/interpolation/structured.py:35-48, reader_netCDF_CF_generic.py:452-463).  Then xspan = (double)(float)(xgrid[nx-1] + dx -
 * xgrid[0]), the index scale is nx instead of nx - 1, and the east-west coverage test is skipped (variables.py:239-242).
 * proj: a reader whose grid lies on a projected plane (proj.kind != 0; its x / y axes, x0 .. ymax, are metres in that plane):
 * positions are projected before the index arithmetic (Variables.lonlat2xy, readers/basereader/variables.py:129-143; the
 * longitude is modulated first as lon_mode says, :259-280) and, with rotate_vectors, the two components of the group are
 * rotated from the plane's axes to east / north after the interpolation (rotate_vectors, :59-109, :799-837).  Sampled by the
 * general kernels (od_interp, the reader-chain family of step kernels, mixing, Leeway); kind 0 = geographic (+proj=latlong).
 * OD_PROJ_OB_TRAN, a rotated pole (+proj=ob_tran +o_proj=longlat +o_lat_p +o_lon_p +lon_0): the axes are rotated longitude /
 * latitude in degrees.  Its parameters travel in the fields of the other kinds: lon_0 = +lon_0, lat_1 = +o_lat_p,
 * lat_2 = +o_lon_p, a = +R (the angles do not use it; it must be > 0), k_0 = 1, everything else 0.  As in the reference, the
 * coverage test takes the rotated x modulated as lon_mode says (covers_positions_xy, variables.py:244-247) and the index
 * takes np.mod(x, 360) when xmin > 0, the unmodulated x otherwise (basereader/structured.py:213-215); vector pairs are
 * rotated with a y-axis line of 0.1 degrees. */
#define OD_PROJ_STERE_SPHERE 1
#define OD_PROJ_MERC 2
#define OD_PROJ_LCC 3
#define OD_PROJ_STERE_ELLPS 4
#define OD_PROJ_OB_TRAN 5
typedef struct od_proj_desc {
    int32_t kind;                 /* OD_PROJ_STERE_SPHERE: +proj=stere on a sphere (+R, or +a with +e=0 / +es=0);
                                     OD_PROJ_MERC: +proj=merc; OD_PROJ_LCC: +proj=lcc (+lat_1 [+lat_2]); sphere or ellipsoid (es);
                                     OD_PROJ_STERE_ELLPS: +proj=stere on an ellipsoid (es > 0), all four aspects;
                                     OD_PROJ_OB_TRAN: +proj=ob_tran +o_proj=longlat (fields: see above) */
    int32_t has_lat_ts;           /* +lat_ts given (stere: polar aspects only; merc: the latitude of true scale replaces k_0) */
    double a;                     /* sphere radius / semi-major axis, m */
    double lat_0, lon_0, lat_ts;  /* degrees */
    double k_0, x_0, y_0;
    double es;                    /* squared eccentricity of the ellipsoid, 0 = sphere (merc, lcc) */
    double lat_1, lat_2;          /* standard parallels of the cone, degrees (lat_2 = lat_1: one parallel) */
} od_proj_desc;

typedef struct od_group_desc {
    int32_t ncomp;            /* 1 or 2 */
    int32_t nx, ny, nz;
    int32_t lon_mode;         /* od_lon_mode */
    int32_t n_slots;          /* ring of time slabs kept on the device (>= 2) */
    int32_t wrap_x;           /* 0 / 1, see above */
    int32_t global_x;         /* 0 / 1: east-west global coverage by the reference's rule (variables.py:289-301), periodic or not: the
                                 coverage test is north-south only (variables.py:239-242); points in the east-west gap of a global grid
                                 that is not periodic get the edge value (the NaN loop of Linear2DInterpolator) */
    double x0, xspan, y0, yspan;
    double xmin, xmax, ymin, ymax;
    float fallback[2];
    od_proj_desc proj;        /* kind 0: geographic */
    int32_t rotate_vectors;   /* the group's two components are an x / y vector pair to be rotated to east / north */
    int32_t pad_;
} od_group_desc;

#define OD_MAX_GROUPS 64
int od_group_define(od_ctx* ctx, int group, const od_group_desc* desc, const double* h_z_levels);
/* release the device memory of a group (its id can be defined again) */
int od_group_free(od_ctx* ctx, int group);
/* copy one time slab of one component ([nz][ny][nx] float32, C order) into ring slot `slot`;
 * src may be host (pinned or pageable) or device memory */
int od_group_upload(od_ctx* ctx, int group, int slot, int comp, const float* src, int src_is_device);
/* Fill non-finite cells of an uploaded slab from their finite 3x3 neighbours (maximum), layer by layer, up to
 * max_iterations passes: the NaN handling of Linear2DInterpolator (readers/interpolation/interpolators.py:9-20,
 * 121-139; the reference uses at most 10, the library accepts up to 16).  Enqueued without a host round trip: a slab
 * without holes costs one read pass.  h_remaining may be NULL; if given it receives the number of cells still missing
 * (and the call synchronises). */
int od_group_fill_nan(od_ctx* ctx, int group, int slot, int comp, int max_iterations, int64_t* h_remaining);
/* raw device pointer of a ring slot component, e.g. as the target of an NCCL broadcast */
int od_group_slot_ptr(od_ctx* ctx, int group, int slot, int comp, float** d_out);
/* tell the library a slot's contents changed behind its back (after a broadcast into od_group_slot_ptr) */
int od_group_touch(od_ctx* ctx, int group, int slot);
/* Build the pair texels of the slabs in slots (slot_a, slot_b) now, on the current stream, ahead of the first launch that
 * samples between them (e.g. on the copy stream right after the later slab was put into its slot).  The cache entry the
 * launches used last is never overwritten; a launch that samples the pair orders its stream behind the build.  No-op when
 * the pair is cached already. */
int od_group_prepare_pair(od_ctx* ctx, int group, int slot_a, int slot_b);
/* Sub-block readers: the blocks a reader hands out cover the elements plus a buffer (StructuredReader block cache,
 * readers/basereader/structured.py:243-318; block supplier readers/reader_netCDF_CF_generic.py:404-626).  The group keeps the slots
 * it was defined with (capacity = its full grid); this call replaces nx, ny and the block-relative index geometry (the block's own
 * float32 axes, as ReaderBlock's interpolator sees them: interpolation/interpolators.py:110-111) by those of a window of the
 * grid and invalidates the ring; slabs are then uploaded densely for the window.  ncomp, nz, n_slots must be unchanged. */
int od_group_set_window(od_ctx* ctx, int group, const od_group_desc* window);
/* bounding box of the elements (what the block request is made for): h_out4 = lon min, lon max, lat min, lat max; NaNs ignored;
 * synchronises */
int od_bbox(od_ctx* ctx, int64_t n, const double* d_lon, const double* d_lat, double* h_out4);
/* environment:fallback:* of the group's variables (Environment.get_environment, models/basemodel/environment.py:782-801): the
 * values are read at every launch, so that a reader bound once serves models / runs with different fallbacks. NaN = none. */
int od_group_set_fallback(od_ctx* ctx, int group, float fallback0, float fallback1);

/* one time sample of a group: which two ring slots bracket it and how they combine */
typedef struct od_time_sample {
    int32_t slot_a, slot_b;
    int32_t mode;             /* od_time_mode */
    int32_t pad_;
    double w;                 /* weight of slot_b for OD_T_LERP */
} od_time_sample;

/* get_variables_interpolated fast path: d_out[c] (float32[n]) for c < ncomp; d_out entries may be NULL.
 * z may be NULL for nz == 1.  lon/lat float64.  flags: OD_INTERP_POS_F32 | OD_INTERP_NO_FALLBACK.
 * OD_INTERP_NO_FALLBACK returns NaN where the reader has no data (what Reader.get_variables_interpolated
 * hands to Environment, which applies the fallback itself).  OD_INTERP_POS_F32: the positions hold float32 values (the
 * reference's element arrays are float32 from seeding until the first update_positions,
 * elements/elements.py:156-158) and NumPy then does the index arithmetic of interpolators.py:110-111 in
 * float32; the kernel reproduces that. */
int od_interp(od_ctx* ctx, int group, const od_time_sample* ts, int64_t n,
              const double* d_lon, const double* d_lat, const void* d_z, int flags,
              void* d_out0, void* d_out1);     /* float32[n], or float64[n] with OD_INTERP_OUT_F64 */

/* ---- geodesic --------------------------------------------------------------------------- */
/* in place: (lon, lat) <- WGS84 direct(lon, lat, az_deg, dist_m); lon normalised to [-180, 180] */
int od_geod_fwd(od_ctx* ctx, int64_t n, double* d_lon, double* d_lat,
                const double* d_az_deg, const double* d_dist_m);

/* update_positions: velocities float32 (vel_f64 = 0) or float64 (vel_f64 = 1) -- the reference's
 * arithmetic follows the dtype of its inputs; moving may be NULL (all 1). */
int od_update_positions(od_ctx* ctx, int64_t n, double* d_lon, double* d_lat,
                        const void* d_xvel, const void* d_yvel, int vel_f64,
                        const int32_t* d_moving, double dt);

/* ---- fused advection -------------------------------------------------------------------- */
#define OD_MATH_EXACT 0
#define OD_MATH_FAST 1
#define OD_MATH_SERIES 2

typedef struct od_advect_args {
    int32_t scheme;               /* od_scheme */
    int32_t group_uv;             /* 2-component current group */
    od_time_sample t_start;       /* time t        (stage 1; ignored when d_k1_u given) */
    od_time_sample t_mid;         /* time t + dt/2 (stages 2, 3) */
    od_time_sample t_end;         /* time t + dt   (stage 4) */
    double dt;                    /* seconds, may be negative */
    int64_t n;
    double* d_lon;                /* in/out float64 */
    double* d_lat;
    const void* d_z;              /* float32 (or float64 when z_f64) or NULL (2-D group) */
    const void* d_factor;         /* factor * current_drift_factor per particle; NULL = 1 */
    int32_t factor_f64;           /* dtype of d_factor: 0 float32, 1 float64 (reference promotes scalars
                                     to float64 arrays, elements/elements.py:213-216) */
    int32_t pos_f32;              /* lon/lat hold float32 values (first step after seeding), see od_interp */
    const int32_t* d_moving;      /* elements.moving (0 = frozen); NULL = all moving */
    const float* d_k1_u;          /* optional start-of-step environment (already sampled) */
    const float* d_k1_v;
    double truncate_below;        /* drift:truncate_ocean_model_below_m, <= 0 disables */
    /* optional outputs: start-of-step sampled current (float32[n]) */
    float* d_env_u;
    float* d_env_v;
    int32_t z_f64;                /* dtype of d_z (and d_z_inout): the reference's z is float32 until vertical mixing
                                     makes it float64 (oceandrift.py:527) */
    int32_t pad3_;
    const double* d_noise_cur;    /* drift:current_uncertainty[_uniform] (environment.py:869-885): scaled float64 draws
                                     [stage 0..3][kind 0 normal, 1 uniform][component u, v][n], added to the float32
                                     current of every stage as the reference does per get_environment call; NULL = none */
    int32_t noise_kinds;          /* bit 0: normal draws present, bit 1: uniform draws present */
    int32_t fast;                 /* arithmetic mode (OD_MATH_*):
                                     0 EXACT : restatement of the reference arithmetic, operation by operation
                                               (bit-exact field sampling, float32 mid-point azimuths, full Karney geodesic);
                                     2 SERIES: the same bit-exact sampling; every move by the fifth-order short-arc
                                               series of the direct geodesic (<= 1e-13 deg from the full solution, which
                                               it falls back to for long steps and near the poles); mid-points skip the
                                               float32 azimuth rounding (od_advect.cuh SeriesMath).  ~1e-9 deg from
                                               EXACT per step, the size of the reference's own float32 arctan2 noise;
                                     1 FAST  : float32 sampling and mid-latitude moves on float64 positions
                                               (~1e-7 deg from the reference after 100 steps; od_advect.cuh FastMath) */
    /* Reader priority list for the current (Environment.get_environment loops over the readers of a variable on the
     * still-missing elements, environment.py:613-780 -- e.g. a nested model inside a coarser one): up to OD_MAX_CHAIN further
     * two-component groups, sampled in order wherever the groups before them return NaN; the fallback values of
     * group_uv apply after the last one. */
    int32_t n_chain;
    int32_t chain_group[2];
    int32_t pad4_;
    od_time_sample chain_t[2][3]; /* per chained group: time t, t + dt/2, t + dt */
} od_advect_args;
#define OD_MAX_CHAIN 2

int od_advect_current(od_ctx* ctx, const od_advect_args* a);

/* The same step for particle arrays that live in HOST memory -- what a caller that keeps the reference's NumPy element
 * arrays (opendrift/elements/elements.py) hands over: a->n particles at h_lon / h_lat / h_z, results to h_out_lon /
 * h_out_lat (may alias the inputs).  a->d_lon, d_lat, d_z are ignored; d_factor / d_moving (device, optional) are
 * indexed like the host arrays; k1 / env / noise arrays are not supported here.  The range is cut into `chunks` pieces
 * (0 = default 12; first and last half size) whose host->device copies, kernel and device->host copies are pipelined
 * on three internal streams behind the work already enqueued on the context's stream.  Host memory should be pinned
 * (cudaHostAlloc / cudaHostRegister) for the copies to overlap.  Returns after the results have landed. */
typedef struct od_host_io {
    const double* h_lon;
    const double* h_lat;
    const void* h_z;              /* float32, or float64 when a->z_f64; NULL for a 2-D group */
    double* h_out_lon;
    double* h_out_lat;
    int32_t chunks;
    int32_t pad_;
    void* h_out_z;                /* od_step_oceandrift_host with vertical advection: updated depths (dtype as h_z; may alias h_z) */
} od_host_io;

int od_advect_current_host(od_ctx* ctx, const od_advect_args* a, const od_host_io* io);

typedef struct od_step_args {
    od_advect_args cur;           /* current advection */
    /* wind drift (advect_wind): group_wind < 0 disables */
    int32_t group_wind;
    int32_t wdf_f64;              /* dtype of d_wdf */
    od_time_sample t_wind;        /* sampled at time t, start-of-step positions */
    const void* d_wdf;            /* wind_drift_factor per particle */
    double wind_drift_depth;      /* drift:wind_drift_depth (0 = surface only) */
    /* vertical advection: group_w < 0 disables; z updated in place */
    int32_t group_w;
    int32_t w_at_surface;         /* drift:vertical_advection_at_surface */
    od_time_sample t_w;
    void* d_z_inout;              /* depth to update (dtype per cur.z_f64); may differ from cur.d_z */
    /* horizontal diffusion: d_rand_x NULL disables; standard normal draws (float64[n]) */
    const double* d_rand_x;
    const double* d_rand_y;
    const float* d_diffusivity;   /* per particle float32, or NULL -> diffusivity_const */
    float diffusivity_const;
    int32_t z_inout_f64;          /* dtype of d_z_inout: 0 float32, 1 float64 */
    const double* d_noise_wind;   /* drift:wind_uncertainty: [component][n] scaled normal draws, or NULL */
} od_step_args;

int od_step_oceandrift(od_ctx* ctx, const od_step_args* a);
/* the fused step for HOST particle arrays (od_host_io above): a->cur.d_lon / d_lat / d_z and a->d_z_inout are ignored; the
 * per-particle device arrays (d_factor, d_moving, d_wdf, d_diffusivity, d_rand_x / y) are indexed like the host arrays;
 * the wind-noise array is not supported here. */
int od_step_oceandrift_host(od_ctx* ctx, const od_step_args* a, const od_host_io* io);

/* ---- Leeway ------------------------------------------------------------------------------------------
 * Leeway.update (models/leeway.py:430-494): optional capsizing, leeway move + current move + jibing in one launch.
 * Wind and current are 2-D two-component groups sampled at the start-of-step position.  Elements with a missing
 * sample get status = missing_code (report_missing_variables) and do not move. */
typedef struct od_leeway_args {
    int32_t group_wind, group_cur;
    od_time_sample t_wind, t_cur;
    int64_t n;
    double* d_lon;
    double* d_lat;
    const float* d_dw_slope;
    const float* d_dw_offset;
    const float* d_dw_eps;
    float* d_cw_slope;            /* in/out: sign flips when an element jibes */
    const float* d_cw_offset;
    const float* d_cw_eps;
    uint8_t* d_orientation;       /* in/out */
    uint8_t* d_capsized;          /* NULL = none; in/out when capsize_on */
    const void* d_jibe_probability;   /* float32, or float64 when jp_f64 */
    const int32_t* d_moving;
    int32_t* d_status;            /* NULL = do not flag missing data */
    const int32_t* d_ids;
    const double* d_rand;         /* np.random.random(n) of this step (parity), or NULL: Philox keyed by (seed, ID, step) */
    double dt;
    uint64_t seed;
    float capsize_fraction;       /* capsizing:leeway_fraction */
    int32_t jp_f64, pos_f32, step_index, missing_code, pad_;
    /* processes:capsizing (leeway.py:438-454): elements with capsized == capsize_from (0 in forward, 1 in backward runs) flip
     * with probability (0.5 + 0.5 tanh((wind - wind_threshold) / wind_sigma)) |dt| / 3600 */
    int32_t capsize_on, capsize_from;
    float wind_threshold, wind_sigma;      /* capsizing:wind_threshold, capsizing:wind_threshold_sigma */
    const double* d_rand_capsize; /* [n] the reference's np.random.rand(len(eligible)) draws scattered to the eligible elements (parity),
                                     or NULL: Philox keyed by (seed, ID, step) */
    /* drift:current_uncertainty[_uniform] / drift:wind_uncertainty (environment.py:869-891): the step's draws, added to the float32
     * samples as the reference adds them (float32(float64(value) + draw), normal first, then uniform) */
    const double* d_noise_cur;    /* [kind 0 normal, 1 uniform][component][n] for the kinds flagged in noise_kinds, or NULL */
    const double* d_noise_wind;   /* [component][n], or NULL */
    int32_t noise_kinds, pad2_;
} od_leeway_args;

int od_leeway_step(od_ctx* ctx, const od_leeway_args* a);

/* ---- Stokes drift and reductions -----------------------------------------------------------------
 * od_minmax_f32: min / max of a[i] (or a[i] + b[i] when d_b is given) with NaNs ignored, returned to the host
 * (synchronises).  These are the collective decisions the reference takes with .max() / .min() on environment
 * arrays (physics_methods.py:799-812, 899, 771-775; basemodel/__init__.py:1754). */
int od_minmax_f32(od_ctx* ctx, int64_t n, const float* d_a, const float* d_b, float* h_min, float* h_max);

/* PhysicsMethods.stokes_drift (models/physics_methods.py:793-848): depth-profiled Stokes velocity from the
 * float32 environment samples and the geodesic move, in place. */
typedef struct od_stokes_args {
    int64_t n;
    double* d_lon;
    double* d_lat;
    const void* d_z;              /* float32, or float64 when z_f64 */
    const float* d_us;            /* sea_surface_wave_stokes_drift_x/y_velocity sampled at the start of the step */
    const float* d_vs;
    const float* d_hs;            /* sea_surface_wave_significant_height (hs_mode 0) */
    const float* d_xwind;         /* wind (wave period, and Hs for hs_mode 1); NULL = no wind */
    const float* d_ywind;
    const int32_t* d_moving;
    double dt;
    int32_t z_f64;
    int32_t hs_mode;              /* 0: Hs from d_hs; 1: 0.0246 |wind|^2; 2: Hs = 1 (no Hs and no wind anywhere) */
    int32_t profile;              /* 0 monochromatic, 1 exponential, 2 Phillips, 3 windsea_swell (models/physics_methods.py:418-455) */
    int32_t pad_;
    double factor;                /* stokes_drift(factor): the velocities are multiplied by it (models/physics_methods.py:843) ... */
    const void* d_factor;         /* ... or by this per-element array (float32, or float64 when factor_f64); NULL = the scalar */
    int32_t factor_f64, pad2_;
    /* profile 3: swell and wind-sea direction ('to', degrees), period and significant height at the elements (float32) */
    const float* d_swell_dir;
    const float* d_swell_period;
    const float* d_swell_hs;
    const float* d_windsea_dir;
    const float* d_windsea_period;
    const float* d_windsea_hs;
} od_stokes_args;

int od_stokes_drift(od_ctx* ctx, const od_stokes_args* a);

/* drift:use_tabularised_stokes_drift (basemodel/environment.py:844-863, physics_methods.py:488-568): Stokes drift and significant
 * wave height from the float32 wind, in place.  ws = sqrt(x^2 + y^2) (float64, capped at 30); d_us / d_vs = float32(wind * wf) with
 * wf = np.polyval(h_wf, ws) in float64; d_hs = float32(np.polyval(h_hs, ws)).  h_wf / h_hs are host arrays of 1..8 coefficients,
 * highest power first.  d_us and d_vs (both or neither) and d_hs may be NULL: that output is not written. */
int od_stokes_parameterised(od_ctx* ctx, int64_t n, const float* d_xwind, const float* d_ywind, const double* h_wf, int32_t n_wf,
                            const double* h_hs, int32_t n_hs, float* d_us, float* d_vs, float* d_hs);

/* ---- vertical turbulent mixing ----------------------------------------------------------------
 * OceanDrift.vertical_mixing (models/oceandrift.py:397-571) with diffusivity from the environment profiles of
 * a 3-D one-component group: all int(dt/dt_mix) inner random-walk iterations in one launch.  Positions are
 * the START-of-step positions (where the reference samples environment_profiles); z_out is float64 (the
 * reference's z becomes float64 here) and may not alias z_in. */
typedef struct od_mix_args {
    int32_t group_k;              /* ocean_vertical_diffusivity group (1 component, nz > 1) */
    int32_t ntimes;               /* abs(int(time_step / dt_mix)) */
    od_time_sample t_k;
    int64_t n;
    const double* d_lon;
    const double* d_lat;
    const void* d_z_in;           /* float32, or float64 when z_in_f64 */
    double* d_z_out;
    const int32_t* d_moving;      /* NULL = all moving */
    const void* d_terminal_velocity;   /* NULL = 0; float32, or float64 when tv_f64 */
    const int32_t* d_ids;         /* element IDs keying the device generator; NULL = array index */
    const double* d_rand;         /* [ntimes][n] draws of np.random.random (parity with the reference), or NULL:
                                     Philox4x32-10 keyed by (seed, ID, step_index, iteration) */
    const float* d_sea_floor;     /* per-particle sea_floor_depth_below_sea_level, or NULL -> sea_floor_const */
    double dt_mix;                /* vertical_mixing:timestep with the sign of the time step */
    double sea_floor_const;
    uint64_t seed;
    int32_t step_index;
    int32_t z_in_f64, tv_f64;
    int32_t mix_at_surface;       /* drift:vertical_mixing_at_surface */
    int32_t pos_f32;              /* see od_interp */
    int32_t model;                /* vertical_mixing:diffusivitymodel as the reference resolves it (oceandrift.py:429-453):
                                     0 OD_MIX_ENVIRONMENT: the profile of group_k;  otherwise group_k is ignored and the
                                     column is analytical on 1 m levels mixing_z = -arange(nlev):
                                     1 OD_MIX_LARGE1994, 2 OD_MIX_SUNDBY1983 (physics_methods.py:203-249), 3 OD_MIX_CONSTANT */
    int32_t nlev;                 /* analytical models: len(-arange(0, max(MLD) + 2)) */
    int32_t seafloor_action;      /* what 'Let particles stick to bottom' (oceandrift.py:559-564) does at the end of an iteration to an
                                     element below the sea floor: 0 nothing (no reader provides the depth: interact_with_seafloor
                                     returns at once, basemodel/__init__.py:752-753), 1 lift_to_seafloor, 2 deactivate (lifted,
                                     status = seafloor_code unless already set, moving = 0 for the remaining iterations) */
    const float* d_wind_speed;    /* [n] float32 sqrt(x_wind^2 + y_wind^2) at the start of the step (models 1, 2) */
    const float* d_mld;           /* [n] float32 ocean_mixed_layer_thickness, or NULL -> mld_const */
    double mld_const;
    double background;            /* vertical_mixing:background_diffusivity */
    double k_const;               /* model 3: the constant diffusivity */
    int32_t* d_status;            /* seafloor_action 2 */
    int32_t* d_moving_out;        /* seafloor_action 2: the array d_moving points to, writable */
    int32_t seafloor_code;
    int32_t iter0;                /* index of this call's first inner iteration within the time step: a subclass that overrides the
                                     per-iteration hooks of the loop (surface_stick, surface_wave_mixing, bottom_interaction,
                                     update_terminal_velocity: oceandrift.py:369-379, 553-564) gets one launch per iteration (ntimes = 1)
                                     with the device generator continuing where the fused loop would be */
    int64_t* h_n_deactivated;     /* seafloor_action 2, optional: elements deactivated by this call (synchronises) */
    int32_t skip_surface_stick;   /* the model overrides surface_stick(): the launch leaves elements above the surface alone */
    int32_t pad3_;
} od_mix_args;
#define OD_MIX_ENVIRONMENT 0
#define OD_MIX_LARGE1994 1
#define OD_MIX_SUNDBY1983 2
#define OD_MIX_CONSTANT 3

int od_vertical_mixing(od_ctx* ctx, const od_mix_args* a);

/* SedimentDrift (models/sedimentdrift.py): od_vertical_mixing with bottom_interaction (:108-116) in every inner iteration.  After
 * the sea floor, an element at or below Zmin whose moving is 1 settles: moving = 0 for the remaining iterations.  Here a->d_moving
 * and a->d_status are only read (a->d_moving_out is not used) and nothing of the elements is modified in place: every element's
 * moving goes to d_moving_out and, with seafloor_action 2, its status to d_status_out.  The reference settles elements only in
 * iterations where some element of the whole array is below Zmin before the lift; an element that ends an iteration exactly at
 * Zmin, moving, without having been below itself cannot be decided here.  It is left moving and counted in *h_undecided; a
 * non-zero count means the result is to be discarded and the step's mixing redone with the decision taken over all elements.
 * h_undecided (required) and a->h_n_deactivated are read back together (synchronises). */
int od_vertical_mixing_settle(od_ctx* ctx, const od_mix_args* a, int32_t* d_moving_out, int32_t* d_status_out, int64_t* h_undecided);

/* SedimentDrift.resuspension (models/sedimentdrift.py:118-126): where float32 sqrt(u*u + v*v) > threshold (a float32 comparison) and
 * moving == 0, moving = 1 and z += 0.01 in z's dtype (float64 when z_f64, else float32).  u, v: the step's float32 current. */
int od_resuspend(od_ctx* ctx, int64_t n, const float* d_u, const float* d_v, float threshold, int32_t* d_moving, void* d_z, int32_t z_f64);

/* ---- ShipDrift ---------------------------------------------------------------------------------
 * ShipDrift.update (models/shipdrift.py:216-343) for n ships in one launch, from the float32 start-of-step environment: the current
 * move, then the move with the velocity of the wind / wave / form-drag force balance, then the stranding flag.
 *   d_el: the six float32 element arrays length, height, draft, beam, wind_drag_coeff, water_drag_coeff (a host array of 6 device
 *         pointers); d_orientation: uint8.
 *   d_env: float32 x_sea_water_velocity, y_sea_water_velocity, x_wind, y_wind, Hs, period, Stokes x, Stokes y, land_binary_mask
 *         (a host array of 9 device pointers; Stokes NULL: the wave direction is the wind's; mask NULL: no stranding).
 *   hs_wind: Hs = 0.0246 ws^2, written into the Hs array; tm_wind: the period from the wind (float64 arithmetic), written into the
 *   period array as float32; tm_fill_on: period values of exactly 0 are replaced by tm_fill.
 *   d_wtab / d_wbox: the wforce.dat table and its Delaunay tetrahedra per grid box (layout in csrc/od_ship.cuh).
 *   Where land_binary_mask == 1: status = strand_code (when 0) and moving = 0; *h_stranded = 1 if that happened (synchronises). */
int od_ship_step(od_ctx* ctx, int64_t n, double* d_lon, double* d_lat, int32_t* d_moving, int32_t* d_status, const float* const* d_el,
                 const uint8_t* d_orientation, float* const* d_env, const double* d_wtab, const int32_t* d_wbox, int32_t nomega,
                 int32_t nbeam, int32_t ndraft, int32_t hs_wind, int32_t tm_wind, int32_t tm_fill_on, float tm_fill, int32_t strand_code,
                 double dt, int32_t* h_stranded);

/* ---- PlastDrift ---------------------------------------------------------------------------------
 * PlastDrift.update after the current move (models/plastdrift.py:80-107) for n elements in one launch, each element in turn:
 *   (a) with d_z_out: z = -(double(K / tv) * E) written to d_z_out (float64), for every element whatever `moving`.
 *       K: float32 ocean_vertical_diffusivity; tv: terminal_velocity, float32 or float64 (tv_f64), the quotient in tv's dtype.
 *       E: d_rand (float64 standard exponential draws) or, with d_rand NULL, -log(1 - u) with u from Philox keyed by
 *       (seed, d_ids[i], step_index, a tag of its own).
 *       *h_negative = 1 if some scale is negative and not NaN (synchronises); without d_z_out the depth is d_z_in (z_f64).
 *   (b) with d_stokes (a host array of 11 device pointers: Stokes x, y, Hs, x_wind, y_wind, then the six windsea_swell arrays,
 *       as in od_stokes_args): the Stokes move at the element's depth (hs_mode, profile as in od_stokes_args).
 *   (c) with d_wdf (wind_drift_factor, float32 or float64: wdf_f64): the wind move at the element's depth, with
 *       drift:wind_drift_depth = wind_drift_depth.
 * (b) and (c) move only where d_moving != 0 (NULL: everywhere). */
int od_plast_step(od_ctx* ctx, int64_t n, double* d_lon, double* d_lat, const int32_t* d_moving, const void* d_z_in, int32_t z_f64,
                  double* d_z_out, const float* d_k, const void* d_tv, int32_t tv_f64, const double* d_rand, const int32_t* d_ids,
                  unsigned long long seed, int32_t step_index, const float* const* d_stokes, int32_t hs_mode, int32_t profile,
                  const float* d_xwind, const float* d_ywind, const void* d_wdf, int32_t wdf_f64, double wind_drift_depth, double dt,
                  int32_t* h_negative);

/* ---- LarvalFish ----------------------------------------------------------------------------------------
 * od_larval_develop: LarvalFish.update_fish_larvae and update_terminal_velocity (models/larvalfish.py) for n elements in one
 * launch (csrc/od_larval.cuh).  d_t, d_s: float32 sea_water_temperature and sea_water_salinity.  Each element array is float32 or
 * float64 by its *_f64 flag; hatched is uint8 or float64.
 *   develop != 0: hatching (stage_fraction, hatched), growth (weight) and length, in place.
 *   d_w_out != NULL: the terminal velocity of every element, float64 if diameter_f64 || nbs_f64, else float32.
 *   h_flags != NULL: OR of LARVAL_STAGED (1: some element is an egg or a larva), LARVAL_HOT (2: some T > 100) and
 *   LARVAL_NAN_T (4: some T is NaN) (synchronises); NULL: no read-back.
 * od_larval_migrate: larvae_vertical_migration: every element with hatched == 1 gets
 *   z = min(0, z + direction * fraction * swim(length) * dt), z float32 or float64 (z_f64). */
int od_larval_develop(od_ctx* ctx, int64_t n, const float* d_t, const float* d_s, void* d_hatched, int32_t hatched_f64,
                      void* d_stage, int32_t stage_f64, void* d_weight, int32_t weight_f64, void* d_length, int32_t length_f64,
                      const void* d_diameter, int32_t diameter_f64, const void* d_nbs, int32_t nbs_f64, int32_t develop,
                      void* d_w_out, double dt, int32_t* h_flags);
int od_larval_migrate(od_ctx* ctx, int64_t n, const void* d_hatched, int32_t hatched_f64, const void* d_length, int32_t length_f64,
                      void* d_z, int32_t z_f64, double fraction, double direction, double dt);

/* ---- analytical readers on a projected plane ---------------------------------------------------------
 * BASELINE configs[0]: opendrift/readers/reader_double_gyre.py (a ContinuousReader, basereader/continuous.py:9-48) on the
 * spherical stereographic plane its constructor asks pyproj for (reader_double_gyre.py:27-31).  The reader chain of
 * Variables.get_variables_interpolated (basereader/variables.py:860-920: modulate_longitude, Proj forward, coverage,
 * get_variables, rotate_vectors :59-109, NaN for uncovered) is evaluated per particle on the device. */

#define OD_ANALYTIC_DOUBLE_GYRE 1
typedef struct od_analytic_desc {
    int32_t kind;                 /* OD_ANALYTIC_DOUBLE_GYRE */
    int32_t lon_mode;             /* modulate_longitude: 0 np.mod(lon, 360), 1 np.mod(lon + 180, 360) - 180 */
    od_proj_desc proj;
    double xmin, xmax, ymin, ymax;   /* coverage in the reader's plane (reader attributes of the same names) */
    double par[4];                /* double gyre: A, epsilon, omega (reader_double_gyre.py:27-28), unused */
    double rot_delta;             /* length of the y-axis line of rotate_vectors: 10 (m) for a projected plane */
    float fallback[2];            /* environment:fallback:x/y_sea_water_velocity, NaN = none */
} od_analytic_desc;

/* Reader.get_variables_interpolated(['x_sea_water_velocity', 'y_sea_water_velocity'], time, lon, lat): float32 east /
 * north velocity, NaN where the reader does not cover the position (no fallback).  t_seconds = (time - initial_time)
 * .total_seconds().  flags: OD_INTERP_POS_F32. */
int od_analytic_interp(od_ctx* ctx, const od_analytic_desc* r, double t_seconds, int64_t n, const double* d_lon,
                       const double* d_lat, int flags, float* d_u, float* d_v);

/* PhysicsMethods.advect_ocean_current (models/physics_methods.py:611-691) with the analytical reader as the current:
 * Euler / RK2 / RK4 stage loop + WGS84 moves in one launch.  Times are seconds since the reader's initial_time. */
typedef struct od_analytic_advect_args {
    int32_t scheme;               /* od_scheme */
    int32_t math;                 /* OD_MATH_* */
    int32_t factor_f64, pos_f32;
    double t_start, t_mid, t_end; /* t, t + dt/2, t + dt */
    double dt;
    int64_t n;
    double* d_lon;                /* in/out float64 */
    double* d_lat;
    const void* d_factor;         /* factor * current_drift_factor per particle, or NULL */
    const int32_t* d_moving;      /* or NULL */
    const float* d_k1_u;          /* optional start-of-step environment */
    const float* d_k1_v;
    float* d_env_u;               /* optional outputs: start-of-step sampled current */
    float* d_env_v;
} od_analytic_advect_args;

int od_analytic_advect(od_ctx* ctx, const od_analytic_desc* r, const od_analytic_advect_args* a);

/* ---- output buffer ------------------------------------------------------------------------------------------
 * OpenDriftSimulation.state_to_buffer (models/basemodel/__init__.py:2384-2499): lon / lat / z / status of the active
 * elements into column `col` of device-resident [n_total][ncols] arrays addressed by element ID (float32 positions and
 * depth, as the reference's result arrays; rows of elements that are not active keep their fill value). */
typedef struct od_history_args {
    int64_t n;                    /* active elements */
    int64_t n_total;              /* rows of the buffers (all seeded elements) */
    int32_t col, ncols;
    int32_t z_f64, pad_;
    const int32_t* d_ids;         /* [n] element IDs = row indices */
    const double* d_lon;
    const double* d_lat;
    const void* d_z;              /* float32, or float64 when z_f64 */
    const int32_t* d_status;
    float* d_buf_lon;             /* [n_total][ncols] */
    float* d_buf_lat;
    float* d_buf_z;
    int32_t* d_buf_status;
} od_history_args;

int od_history_scatter(od_ctx* ctx, const od_history_args* a);

/* ---- per-element housekeeping (csrc/od_bookkeep.cuh) ----------------------------------------------------
 * od_vertical_buoyancy replaces OceanDrift.vertical_buoyancy (models/oceandrift.py:352-367): the buoyancy move of the
 * depth, z[z < 0] = min(0, z + terminal_velocity * dt), and -- when d_sea_floor is given -- the sea-floor interaction it
 * ends with (OpenDriftSimulation.interact_with_seafloor, models/basemodel/__init__.py:748-783: 'lift_to_seafloor', or
 * 'deactivate' when seafloor_code != 0).  Out of place (d_z_out may alias d_z_in); NumPy's dtype rules. */
typedef struct od_buoyancy_args {
    int64_t n;
    const void* d_z_in;           /* float32, or float64 when z_f64 */
    void* d_z_out;                /* same dtype */
    const void* d_terminal_velocity;   /* float32 / float64 (tv_f64); NULL: sea-floor interaction only */
    const float* d_sea_floor;     /* sea_floor_depth_below_sea_level sampled at the elements; NULL: no sea-floor interaction */
    int32_t* d_status;            /* updated for seafloor_code != 0 */
    int32_t* d_moving;
    double dt;
    float sea_surface_height;
    int32_t z_f64, tv_f64;
    int32_t seafloor_code;        /* status number of 'seafloor' for general:seafloor_action = deactivate, else 0 */
    int64_t* h_n_deactivated;     /* optional: number of elements deactivated by this call (synchronises) */
} od_buoyancy_args;

int od_vertical_buoyancy(od_ctx* ctx, const od_buoyancy_args* a);

/* od_bookkeeping replaces, in one pass over the active elements, what OpenDriftSimulation.run does between
 * get_environment and update() (models/basemodel/__init__.py:2249-2270): deactivate_outside (:2358-2386),
 * state_to_buffer (:2384-2403, into column `col` of the device output block of od_history_scatter; d_buf_lon NULL = nothing
 * is written) and increase_age_and_retire (:2345-2356), with deactivate_elements' rule (:1774-1795: an already deactivated
 * element keeps its status, moving = 0).  h_counts[0..2] = elements newly 'outside', newly 'retired', with status != 0
 * after the pass (synchronises when h_counts is given). */
typedef struct od_bookkeep_args {
    int64_t n;
    const double* d_lon;
    const double* d_lat;
    const void* d_z;              /* float32 / float64 (z_f64): only for the output block */
    void* d_age;                  /* age_seconds, float32 / float64 (age_f64), updated in place */
    int32_t* d_status;
    int32_t* d_moving;
    const int32_t* d_ids;
    double dt_age;                /* time_step.total_seconds() */
    double max_age;               /* drift:max_age_seconds; NaN = none */
    double west, east, south, north;   /* drift:deactivate_*_of; NaN = none */
    int32_t outside_code, retired_code;
    int32_t z_f64, age_f64;
    int32_t pos_f32;
    int32_t only_deactivated;     /* sub-step between output times: write only the elements with status != 0 (into the next output column) */
    int64_t n_total;
    int32_t col, ncols;
    float* d_buf_lon;
    float* d_buf_lat;
    float* d_buf_z;
    int32_t* d_buf_status;
    int64_t* h_counts;            /* [3] or NULL */
} od_bookkeep_args;

int od_bookkeeping(od_ctx* ctx, const od_bookkeep_args* a);

/* OpenDriftSimulation.interact_with_coastline (basemodel/__init__.py:671-746) for a land_binary_mask that a gridded reader
 * provides (sampled with od_interp + OD_INTERP_NEAREST), general:coastline_approximation_precision = None: 'stranding'
 * deactivates the elements on land that are not in the air; 'previous' deactivates elements released on land
 * ('seeded_on_land') and moves every element on land back to its position of the previous step.  Elements the mask does not
 * cover (NaN) become 'missing_data' (report_missing_variables, :2501-2515) when missing_code != 0.  The previous positions
 * are float32 arrays keyed by ID - id_base, as the reference holds them (a copy of its float32 result block, :2164-2165);
 * od_store_previous is update_previous_state (:642-669) for lon / lat.  h_counts[4]: newly stranded, seeded_on_land,
 * missing_data, moved back (synchronises). */
typedef struct od_coast_args {
    int64_t n;
    const float* d_mask;
    double* d_lon;
    double* d_lat;
    const void* d_z;              /* float32 / float64 (z_f64), NULL = 0 */
    const void* d_age;            /* age_seconds, float32 / float64 (age_f64) */
    int32_t* d_status;
    int32_t* d_moving;
    const int32_t* d_ids;
    float* d_prev_lon;
    float* d_prev_lat;
    int64_t n_total;
    int32_t id_base;
    int32_t action;               /* 1 stranding, 2 previous; 3: general:seafloor_action = 'previous' (interact_with_seafloor :775-783):
                                     d_mask holds sea_floor_depth_below_sea_level, elements below the floor go back to their previous position */
    float ssh;                    /* action 3: sea_surface_height */
    int32_t stranded_code, seeded_code, missing_code;
    int32_t check_seeded;
    int32_t z_f64, age_f64;
    int64_t* h_counts;            /* [4] or NULL */
} od_coast_args;
int od_coastline(od_ctx* ctx, const od_coast_args* a);
int od_store_previous(od_ctx* ctx, int64_t n, const double* d_lon, const double* d_lat, const int32_t* d_ids, int32_t id_base,
                      int64_t n_total, float* d_prev_lon, float* d_prev_lat);

/* ---- a varying sea surface height (csrc/od_sealevel.cuh) ------------------------------------------------------
 * od_store_previous_env is update_previous_state (basemodel/__init__.py:642-657) for one float32 environment variable
 * (sea_surface_height): d_prev[i] = the stored value of element i -- the present one for an element released this step --
 * then d_store[ID - id_base] = d_present.  d_store is [n_total], NaN at the start of the run.  d_age (age_seconds after
 * increase_age_and_retire, float32 / float64 by age_f64) is given on steps that released elements, else NULL; elements of
 * age == dt are the newly seeded ones, whose present values the reference also writes at their POSITIONS in the store --
 * reproduced.  Two launches.
 * od_vertical_advection_corrected is OceanDrift.vertical_advection with drift:vertical_advection_correction
 * (oceandrift.py:325-350), in place on d_z (float32 / float64 by z_f64): w -= (delta_zeta / dt) * (z + H) / H with
 * delta_zeta = ssh - ssh_prev, H = ssh + sea floor depth (d_floor, or floor_const when NULL), then z = min(0, z + moving*w*dt)
 * for z < 0 (z <= 0 when at_surface); NumPy's dtypes and operation order. */
int od_store_previous_env(od_ctx* ctx, int64_t n, const float* d_present, const int32_t* d_ids, const void* d_age, int32_t age_f64,
                          double dt, int32_t id_base, int64_t n_total, float* d_store, float* d_prev);
int od_vertical_advection_corrected(od_ctx* ctx, int64_t n, void* d_z, int32_t z_f64, const float* d_w, const float* d_ssh,
                                    const float* d_ssh_prev, const float* d_floor, float floor_const, const int32_t* d_moving,
                                    int32_t at_surface, double dt);

/* ---- particle exchange of the spatial-tile mode --------------------------------------------------------------
 * BASELINE configs[2]: every rank owns one longitude strip of the domain (and holds only that part of the forcing, plus a halo);
 * after a step the elements that left their strip travel to the new owner in ONE all-to-all.  od_pack_by_owner groups the
 * elements by the strip their longitude falls in (h_bounds[0..world]: strip r = [bounds[r], bounds[r+1]), the edge strips
 * open-ended) -- stable, elements of one owner keep their order -- and packs them as fixed-size records: the given SoA columns
 * side by side, column c at byte offset sum(col_bytes[:c]).  h_counts[r] = elements for rank r (synchronises): the split sizes of
 * the all_to_all_single over d_records.  od_unpack_records is the inverse on the receiving side.  (There is no reference
 * counterpart: the reference is a single process.) */
#define OD_PACK_MAX_COLS 16
#define OD_PACK_MAX_WORLD 64
typedef struct od_pack_args {
    int64_t n;
    const double* d_lon;                       /* decides the owner */
    const double* h_bounds;                    /* [world + 1] strip edges (host) */
    int32_t world, ncols;
    const void* d_cols[OD_PACK_MAX_COLS];      /* SoA columns, n elements each */
    int32_t col_bytes[OD_PACK_MAX_COLS];       /* bytes per element of each column */
    int32_t rec_bytes, pad_;                   /* = sum(col_bytes) */
    void* d_records;                           /* out: [n][rec_bytes] */
    int32_t* d_perm;                           /* out, optional: perm[row] = index of the element packed into that row */
    int64_t* h_counts;                         /* out: [world] (host) */
} od_pack_args;

int od_pack_by_owner(od_ctx* ctx, const od_pack_args* a);
int od_unpack_records(od_ctx* ctx, int64_t n, const void* d_records, int32_t ncols, void* const* d_cols, const int32_t* col_bytes,
                      int32_t rec_bytes);

/* ---- particle order (locality) ---------------------------------------------------------- */
/* d_perm_out[k] = index of the particle that should sit at position k when particles are ordered by
 * the grid cell (and level) of `group` they are in.  Stable counting sort. */
int od_sort_by_cell(od_ctx* ctx, int group, int64_t n, const double* d_lon, const double* d_lat,
                    const float* d_z, int32_t* d_perm_out);
/* dst[k] = src[perm[k]] for an array of elem_size-byte elements (1, 2, 4 or 8) */
int od_permute(od_ctx* ctx, int64_t n, const int32_t* d_perm, const void* d_src, void* d_dst, int elem_size);
/* dst[perm[k]] = src[k] */
int od_unpermute(od_ctx* ctx, int64_t n, const int32_t* d_perm, const void* d_src, void* d_dst, int elem_size);

/* Stable partition for remove_deactivated_elements (basemodel/__init__.py:1797-1826, elements.py:197-228):
 * perm_out = [indices with status == 0, in order | indices with status != 0, in order]; *h_n_keep = number kept
 * (synchronises).  Apply with od_permute to every element column. */
int od_partition_active(od_ctx* ctx, int64_t n, const int32_t* d_status, int32_t* d_perm_out, int64_t* h_n_keep);

/* counters of the library's own kernel launches since creation (for bench.py's gpu_launches) */
int64_t od_launch_count(od_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* ODCUDA_H */
