// od_interp.cuh -- regular-grid sampling of a forcing field group at one particle position.
//
// Restates, per particle, what the reference does per array:
//   Variables.get_variables_interpolated[_xy]   opendrift/readers/basereader/variables.py:860-920, 709-858
//     (longitude modulation :259-280, coverage test :229-257, NaN for uncovered :841-853)
//   Linear2DInterpolator                        opendrift/readers/interpolation/interpolators.py:105-139
//     (fractional index :110-111; scipy.ndimage.map_coordinates(order=1, cval=nan) :122)
//   Linear1DInterpolator                        interpolators.py:174-197
//   ReaderBlock._interpolate_horizontal_layers  opendrift/readers/interpolation/structured.py:148-163
//     (float32 layer results stored into a float64 array, then the vertical lerp in float64)
//   time interpolation                          opendrift/readers/basereader/structured.py:353-364
//   float32 cast + fallback                     opendrift/models/basemodel/environment.py:695-696, 782-791
//
// Rounding points are reproduced exactly (no FMA contraction where NumPy/SciPy round twice).
//
// Device layout of a group ("pair texels"): for the two time slabs A, B that bracket a sample the library
// keeps one interleaved array  tex[z][y][x][c0A, c1A, c0B, c1B]  (ncomp = 2, one 16-byte load per corner)
// or tex[z][y][x][c0A, c0B] (ncomp = 1, one 8-byte load), so that one bilinear corner of both components
// and both times is a single vector load.
#pragma once
#include "od_geod.cuh"
#include "od_proj.cuh"

namespace od {

#if defined(__CUDA_ARCH__)
#define OD_DMUL(a, b) __dmul_rn((a), (b))
#define OD_DADD(a, b) __dadd_rn((a), (b))
#define OD_DSUB(a, b) __dsub_rn((a), (b))
#define OD_FMUL(a, b) __fmul_rn((a), (b))
#define OD_FADD(a, b) __fadd_rn((a), (b))
#else
#define OD_DMUL(a, b) ((a) * (b))
#define OD_DADD(a, b) ((a) + (b))
#define OD_DSUB(a, b) ((a) - (b))
#define OD_FMUL(a, b) ((a) * (b))
#define OD_FADD(a, b) ((a) + (b))
#endif

struct GroupGeom {
    int nx, ny, nz, ncomp;
    int lon_mode;            // 0: np.mod(lon, 360); 1: np.mod(lon + 180, 360) - 180
    int wrap;                // 1: periodic east-west; one virtual column (= column 0) follows the nx stored ones
    int glob;                // 1: east-west global coverage (periodic or not): no east-west coverage test
    double x0, xspan, y0, yspan;
    double xmin, xmax, ymin, ymax;
    double nxm1, nym1;
    double inv_dx, inv_dy;   // (nx-1)/xspan, (ny-1)/yspan (fast sampler only)
    double rxspan, ryspan;   // RN(1/xspan), RN(1/yspan), or 0 when div_rn() must use a true division
    double zmin, zmax;       // min / max of the level depths
    float fallback[2];
    const double* zs;        // [nz] level depths in increasing order
    const double* zy;        // [nz] layer index of zs[i] (as float64), what interp1d maps to
    // Readers on a projected plane (x0 .. ymax are then metres in that plane): positions are projected before the index
    // arithmetic (Variables.lonlat2xy, variables.py:129-143) and the components of a vector pair are rotated from the plane's
    // axes to east / north (rotate_vectors, :59-109).  Only the general kernels (reader chain family, od_interp, mixing,
    // Leeway, sorting) look at these; the default step kernels are launched for geographic groups only.
    int proj_kind;           // 0 geographic, else OD_PROJ_*
    int rotate;              // 2-component group whose components are an x / y vector pair
    double rot_delta;        // length of the line along the plane's y axis that defines the rotation (10 m)
    ProjStere proj;
};

struct PairRef {
    const float* tex;        // pair texels
    int mode;                // od_time_mode (3 = reader does not cover the time: fallback)
    int pad_;
    double w;                // weight of B
};

struct VertW {
    int ia, ib;
    double wa;
};

// numpy's np.mod(x, 360.0)
OD_HD double np_mod360(double x) {
    if (x >= 0.0 && x < 360.0) return x;          // fmod(x, 360) == x exactly
    double r = fmod(x, 360.0);
    if (r != 0.0) {
        if (r < 0.0) r += 360.0;
    } else {
        r = 0.0;
    }
    return r;
}

// Linear1DInterpolator.__init__ for one particle.  z is the particle depth; z_f32 tells whether the reference's
// z array is float32 (element default) or float64 (after vertical mixing has touched it, oceandrift.py:527).
template <typename ZPtr>
OD_HD VertW vert_weights(const GroupGeom& g, ZPtr zs, ZPtr zy, double z, bool z_f32 = true) {
    VertW v;
    if (g.nz <= 1) {
        v.ia = v.ib = 0;
        v.wa = 1.0;
        return v;
    }
    // z[z < zgrid.min()] = zgrid.min()  (float64 comparison; the store rounds to the dtype of z)
    double xn = z;
    if (xn < g.zmin) xn = z_f32 ? (double)(float)g.zmin : g.zmin;
    if (xn > g.zmax) xn = z_f32 ? (double)(float)g.zmax : g.zmax;
    // np.searchsorted(zs, xn) (side='left'), clipped to [1, nz-1]
    int lo = 0, hi = g.nz;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (zs[mid] < xn) lo = mid + 1; else hi = mid;
    }
    int idx = lo < 1 ? 1 : (lo > g.nz - 1 ? g.nz - 1 : lo);
    const double x_lo = zs[idx - 1], x_hi = zs[idx], y_lo = zy[idx - 1], y_hi = zy[idx];
    // SciPy's interp1d(kind='linear') hands 1-D float64 tables to np.interp, which returns the table value itself at a
    // knot (and at the last point) and the slope form slope * (x - xp[j]) + fp[j] in between -- at a knot the slope form
    // can be off by an ulp, which would put 1e-16 of the neighbouring layer into a particle that sits exactly on a level
    // (every surface particle when the first level is z = 0).
    double yn;
    if (xn == x_hi) yn = y_hi;
    else if (xn == x_lo) yn = y_lo;
    else {
        const double slope = (y_hi - y_lo) / (x_hi - x_lo);
        yn = OD_DADD(OD_DMUL(slope, OD_DSUB(xn, x_lo)), y_lo);
    }
    double fl = floor(yn);
    int ia = (int)fl;
    if (!(fl >= 0.0)) ia = 0;                        // also NaN
    if (ia > g.nz - 1) ia = g.nz - 1;
    v.ia = ia;
    v.ib = ia + 1 < g.nz - 1 ? ia + 1 : g.nz - 1;
    v.wa = OD_DSUB(1.0, OD_DSUB(yn, (double)ia));
    return v;
}

// bilinear weights of scipy's order-1 spline: w0 = 1 - frac, w1 = 1 - w0
struct HorizW {
    int i00, i01, i10, i11;     // texel offsets (in texels) of the four corners within one layer
    int ix, iy, ix1, iy1;       // cell indices of the corners
    double wy0, wy1, wx0, wx1;
    bool valid;
};

// numpy's np.mod for float32 operands
OD_HD float np_mod360f(float x) {
    if (x >= 0.0f && x < 360.0f) return x;
    float r = fmodf(x, 360.0f);
    if (r != 0.0f) {
        if (r < 0.0f) r += 360.0f;
    } else {
        r = 0.0f;
    }
    return r;
}

// pos_f32: lon/lat carry float32 values (the reference's element arrays are float32 until the first
// update_positions, opendrift/elements/elements.py:156-158), so NumPy does the longitude modulation and
// the fractional-index arithmetic of interpolators.py:110-111 in float32.
// Correctly rounded d / s from the correctly rounded reciprocal r = RN(1/s) (Markstein 1990: q0 = RN(d r),
// e = d - q0 s exactly (FMA), q = RN(q0 + e r) equals RN(d/s) whenever the significand of s is not all ones --
// make_geom() passes r = 0 in that case and for spans outside the normal range, which selects the true division).
// NaN stays NaN; an infinite d gives NaN instead of infinity, and both fail the coverage test that follows.
OD_HD double div_rn(double d, double s, double r) {
#if defined(__CUDA_ARCH__)
    if (r == 0.0 || (fabs(d) < 1e-250 && d != 0.0)) return d / s;      // tiny numerators: the residual would underflow
    const double q0 = __dmul_rn(d, r);
    const double e = __fma_rn(-q0, s, d);
    return __fma_rn(e, r, q0);
#else
    (void)r;
    return d / s;
#endif
}

// r for div_rn: RN(1/s) if the shortcut is valid for this divisor, else 0
static inline double div_rn_reciprocal(double s) {
    union { double d; unsigned long long u; } c;
    c.d = s;
    const unsigned long long mant = c.u & 0xFFFFFFFFFFFFFull;
    const int ex = (int)((c.u >> 52) & 0x7FF);
    if (!(s == s) || ex < 100 || ex > 1900 || mant == 0xFFFFFFFFFFFFFull) return 0.0;
    return 1.0 / s;
}

OD_HD HorizW horiz_weights(const GroupGeom& g, double lon, double lat, bool pos_f32) {
    HorizW h;
    double x, xi, yi;
    const double y = lat;
    if (pos_f32) {
        const float xf = (g.lon_mode == 0) ? np_mod360f((float)lon) : OD_FADD(np_mod360f(OD_FADD((float)lon, 180.0f)), -180.0f);
        x = (double)xf;
        xi = (double)OD_FMUL(OD_FADD(xf, -(float)g.x0) / (float)g.xspan, (float)g.nxm1);
        yi = (double)OD_FMUL(OD_FADD((float)lat, -(float)g.y0) / (float)g.yspan, (float)g.nym1);
    } else {
        x = (g.lon_mode == 0) ? np_mod360(lon) : OD_DSUB(np_mod360(OD_DADD(lon, 180.0)), 180.0);
        xi = OD_DMUL(div_rn(OD_DSUB(x, g.x0), g.xspan, g.rxspan), g.nxm1);
        yi = OD_DMUL(div_rn(OD_DSUB(y, g.y0), g.yspan, g.ryspan), g.nym1);
    }
    // global readers are tested north-south only (variables.py:239-242)
    const bool covered = (g.glob != 0 || ((x >= g.xmin) && (x <= g.xmax))) && (y >= g.ymin) && (y <= g.ymax) &&
                         (xi == xi) && (yi == yi);          // (a NaN position is not covered)
    // A covered point whose fractional index falls outside [0, n-1] -- the float32 span of the block makes that happen
    // by up to 1e-7 of the grid length on the last row / column -- first comes back NaN from map_coordinates
    // (mode='constant', cval=nan) and is then re-interpolated by the NaN loop of Linear2DInterpolator with
    // mode='nearest' (interpolators.py:121-139): the edge value.  Clamping the index gives the same number.
    if (covered) {
        xi = xi < 0.0 ? 0.0 : (xi > g.nxm1 ? g.nxm1 : xi);
        yi = yi < 0.0 ? 0.0 : (yi > g.nym1 ? g.nym1 : yi);
    }
    h.valid = covered;
    if (!covered) {
        h.i00 = h.i01 = h.i10 = h.i11 = 0;
        h.ix = h.iy = h.ix1 = h.iy1 = 0;
        h.wy0 = h.wy1 = h.wx0 = h.wx1 = 0.0;
        return h;
    }
    const double fx = floor(xi), fy = floor(yi);
    int ix = (int)fx;
    const int iy = (int)fy;
    const int nxv = g.nx + g.wrap;                       // columns of the block incl. the virtual one
    int ix1 = ix + 1 < nxv ? ix + 1 : nxv - 1;
    if (ix >= g.nx) ix -= g.nx;                          // the virtual column is column 0
    if (ix1 >= g.nx) ix1 -= g.nx;
    const int iy1 = iy + 1 < g.ny ? iy + 1 : g.ny - 1;
    h.wx0 = OD_DSUB(1.0, OD_DSUB(xi, fx));
    h.wx1 = OD_DSUB(1.0, h.wx0);
    h.wy0 = OD_DSUB(1.0, OD_DSUB(yi, fy));
    h.wy1 = OD_DSUB(1.0, h.wy0);
    h.ix = ix; h.iy = iy; h.ix1 = ix1; h.iy1 = iy1;
    h.i00 = iy * g.nx + ix;
    h.i01 = iy * g.nx + ix1;
    h.i10 = iy1 * g.nx + ix;
    h.i11 = iy1 * g.nx + ix1;
    return h;
}

// map_coordinates(order=1) accumulation order: (y0,x0), (y0,x1), (y1,x0), (y1,x1); result cast to float32
OD_HD float bilin(const HorizW& h, float a00, float a01, float a10, float a11) {
    double t = OD_DMUL(OD_DMUL((double)a00, h.wy0), h.wx0);
    t = OD_DADD(t, OD_DMUL(OD_DMUL((double)a01, h.wy0), h.wx1));
    t = OD_DADD(t, OD_DMUL(OD_DMUL((double)a10, h.wy1), h.wx0));
    t = OD_DADD(t, OD_DMUL(OD_DMUL((double)a11, h.wy1), h.wx1));
    return (float)t;
}

struct alignas(16) Tex4 { float x, y, z, w; };
struct alignas(8) Tex2 { float x, y; };

OD_HD Tex4 ld_tex4(const float* p) {
#if defined(__CUDA_ARCH__)
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    Tex4 r = {t.x, t.y, t.z, t.w};
#else
    Tex4 r = {p[0], p[1], p[2], p[3]};
#endif
    return r;
}

OD_HD Tex2 ld_tex2(const float* p) {
#if defined(__CUDA_ARCH__)
    const float2 t = __ldg(reinterpret_cast<const float2*>(p));
    Tex2 r = {t.x, t.y};
#else
    Tex2 r = {p[0], p[1]};
#endif
    return r;
}

// A box of pair texels staged in shared memory by TMA (cp.async.bulk.tensor) for the particles of one thread
// block; texels outside the box (or of another pair buffer) are fetched from global memory.
struct TileView {
    const float* smem;        // [bz][by][bx][4] floats, or nullptr when the block has no tile
    const float* tex;         // the pair-texel buffer the tile mirrors
    int x0, y0, z0;           // box origin (cell indices, layer)
    int bx, by, bz;           // box extents
};

// Where the eight corners of one sample live: either all inside the staged box (shared memory, box strides) or in
// the global pair-texel buffer.  One test per sample; the loads then go through a generic pointer.
struct TexelSource {
    const float* base;        // such that texel (layer, iy, ix) is at base + 4 * ((layer * ly + iy) * lx + ix)
    int lx;                   // row stride in texels
    long long plane;          // layer stride in floats (4 * lx * ly)
};

OD_HD TexelSource texel_source(const float* tex, const TileView& tv, int nx, int ny, int ix, int ix1, int iy, int iy1,
                               int ia, int ib) {
    TexelSource t;
#if defined(__CUDA_ARCH__)
    if (tv.smem && tex == tv.tex && ix1 >= ix && ix >= tv.x0 && ix1 < tv.x0 + tv.bx && iy >= tv.y0 && iy1 < tv.y0 + tv.by &&
        ia >= tv.z0 && ib < tv.z0 + tv.bz) {
        t.base = tv.smem - 4 * ((tv.z0 * tv.by + tv.y0) * tv.bx + tv.x0);
        t.lx = tv.bx;
        t.plane = 4ll * tv.bx * tv.by;
        return t;
    }
#endif
    t.base = tex;
    t.lx = nx;
    t.plane = 4ll * nx * ny;
    return t;
}

// first texel of a layer; corners are then addressed with 32-bit offsets 4 * (iy * lx + ix) (a layer holds fewer
// than 2^29 texels: od_group_define checks)
OD_HD const float* layer_ptr(const TexelSource& t, int layer) { return t.base + (long long)layer * t.plane; }

OD_HD Tex4 fetch4(const float* layer, int off) {
    const float* p = layer + off;
#if defined(__CUDA_ARCH__)
    const float4 v = *reinterpret_cast<const float4*>(p);
    Tex4 r = {v.x, v.y, v.z, v.w};
    return r;
#else
    Tex4 r = {p[0], p[1], p[2], p[3]};
    return r;
#endif
}

OD_HD bool finite_f(float v) { return fabsf(v) <= 3.4028234663852886e38f; }   // false for NaN / inf

// vertical + time combination of the four horizontal results (layer a/b x time A/B) of one component
OD_HD float combine(const GroupGeom& g, const PairRef& pr, const VertW& vw,
                    float haA, float hbA, float haB, float hbB) {
    if (g.nz > 1) {
        // horiz[ia]*wa + horiz[ib]*(1-wa) in float64 (interpolators.py:195-197)
        const double omw = OD_DSUB(1.0, vw.wa);
        const double vA = OD_DADD(OD_DMUL((double)haA, vw.wa), OD_DMUL((double)hbA, omw));
        if (pr.mode == 1) return (float)vA;
        const double vB = OD_DADD(OD_DMUL((double)haB, vw.wa), OD_DMUL((double)hbB, omw));
        if (pr.mode == 2) return (float)vB;
        // env_before*(1-w) + env_after*w in float64 (structured.py:353-364), then float32 (environment.py:695)
        return (float)OD_DADD(OD_DMUL(vA, OD_DSUB(1.0, pr.w)), OD_DMUL(vB, pr.w));
    }
    if (pr.mode == 1) return haA;
    if (pr.mode == 2) return haB;
    // 2-D variables stay float32: float32 array * Python float -> float32 (NumPy weak scalars)
    const float w1 = (float)pr.w, w0 = (float)OD_DSUB(1.0, pr.w);
    return OD_FADD(OD_FMUL(haA, w0), OD_FMUL(haB, w1));
}

// Sample a 2-component group (e.g. x/y_sea_water_velocity) -> float32 u, v with fallback applied.
// (the part after the horizontal index / weight arithmetic, so that groups on the same grid can share it)
// the four horizontal results (component u, v x time A, B) of one layer: four corner texels, four bilinears
struct LayerVals { float uA, vA, uB, vB; };

OD_HD LayerVals layer_bilin(const HorizW& h, const float* lp, int o00, int o01, int o10, int o11, int mode) {
    const Tex4 a00 = fetch4(lp, o00), a01 = fetch4(lp, o01), a10 = fetch4(lp, o10), a11 = fetch4(lp, o11);
    LayerVals r = {0.f, 0.f, 0.f, 0.f};
    if (mode != 2) {
        r.uA = bilin(h, a00.x, a01.x, a10.x, a11.x);
        r.vA = bilin(h, a00.y, a01.y, a10.y, a11.y);
    }
    if (mode != 1) {
        r.uB = bilin(h, a00.z, a01.z, a10.z, a11.z);
        r.vB = bilin(h, a00.w, a01.w, a10.w, a11.w);
    }
    return r;
}

OD_HD void sample2_h(const GroupGeom& g, const PairRef& pr, const VertW& vw, const HorizW& h,
                     float& u, float& v, const TileView& tv = TileView()) {
    float ru = NAN, rv = NAN;
    if (h.valid && pr.mode != 3) {
        const TexelSource ts = texel_source(pr.tex, tv, g.nx, g.ny, h.ix, h.ix1, h.iy, h.iy1, vw.ia, vw.ib);
        const int r0 = 4 * h.iy * ts.lx, r1 = 4 * h.iy1 * ts.lx;
        const int o00 = r0 + 4 * h.ix, o01 = r0 + 4 * h.ix1, o10 = r1 + 4 * h.ix, o11 = r1 + 4 * h.ix1;
        // one layer at a time: four texels live instead of eight (the kernel runs at 64 registers per thread)
        const LayerVals A = layer_bilin(h, layer_ptr(ts, vw.ia), o00, o01, o10, o11, pr.mode);
        LayerVals B = A;
        if (g.nz > 1) {
#if defined(__CUDA_ARCH__) && defined(OD_LAYER_FENCE)
            asm volatile("" ::: "memory");
#endif
            B = layer_bilin(h, layer_ptr(ts, vw.ib), o00, o01, o10, o11, pr.mode);
        }
        ru = combine(g, pr, vw, A.uA, B.uA, A.uB, B.uB);
        rv = combine(g, pr, vw, A.vA, B.vA, A.vB, B.vB);
    }
    // masked_invalid -> fallback (environment.py:782-791); fallback NaN = keep missing
    if (!finite_f(ru)) ru = g.fallback[0];
    if (!finite_f(rv)) rv = g.fallback[1];
    u = ru;
    v = rv;
}

OD_HD void sample2(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat,
                   float& u, float& v, bool pos_f32 = false, const TileView& tv = TileView()) {
    const HorizW h = horiz_weights(g, lon, lat, pos_f32);
    sample2_h(g, pr, vw, h, u, v, tv);
}

// Sample a 1-component group (e.g. upward_sea_water_velocity).
OD_HD float sample1_h(const GroupGeom& g, const PairRef& pr, const VertW& vw, const HorizW& h) {
    float r = NAN;
    if (h.valid && pr.mode != 3) {
        const long long layer = (long long)g.nx * g.ny;
        const float* ta = pr.tex + ((long long)vw.ia * layer) * 2;
        const Tex2 a00 = ld_tex2(ta + 2ll * h.i00), a01 = ld_tex2(ta + 2ll * h.i01);
        const Tex2 a10 = ld_tex2(ta + 2ll * h.i10), a11 = ld_tex2(ta + 2ll * h.i11);
        Tex2 b00 = a00, b01 = a01, b10 = a10, b11 = a11;
        if (g.nz > 1) {
            const float* tb = pr.tex + ((long long)vw.ib * layer) * 2;
            b00 = ld_tex2(tb + 2ll * h.i00); b01 = ld_tex2(tb + 2ll * h.i01);
            b10 = ld_tex2(tb + 2ll * h.i10); b11 = ld_tex2(tb + 2ll * h.i11);
        }
        float aA = 0.f, bA = 0.f, aB = 0.f, bB = 0.f;
        if (pr.mode != 2) {
            aA = bilin(h, a00.x, a01.x, a10.x, a11.x);
            if (g.nz > 1) bA = bilin(h, b00.x, b01.x, b10.x, b11.x);
        }
        if (pr.mode != 1) {
            aB = bilin(h, a00.y, a01.y, a10.y, a11.y);
            if (g.nz > 1) bB = bilin(h, b00.y, b01.y, b10.y, b11.y);
        }
        r = combine(g, pr, vw, aA, bA, aB, bB);
    }
    if (!finite_f(r)) r = g.fallback[0];
    return r;
}

OD_HD float sample1(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat,
                     bool pos_f32 = false) {
    const HorizW h = horiz_weights(g, lon, lat, pos_f32);
    return sample1_h(g, pr, vw, h);
}

// ---- groups on a projected plane ------------------------------------------------------------------------------------------------
struct HorizWP {
    HorizW h;
    double px, py;           // position in the reader's plane (for the rotation of vector components)
};

// horiz_weights for any group: geographic groups as above; projected groups project first, then the same index arithmetic in
// float64 on the plane coordinates (pyproj returns float64 whatever the dtype of the positions; the longitude is modulated
// first -- in float32 while the element arrays are float32 -- as Variables.get_variables_interpolated does, :912-913)
OD_HD HorizWP horiz_weights_any(const GroupGeom& g, double lon, double lat, bool pos_f32) {
    HorizWP r;
    r.px = r.py = 0.0;
    if (!g.proj_kind) {
        r.h = horiz_weights(g, lon, lat, pos_f32);
        return r;
    }
    HorizW& h = r.h;
    h.valid = false;
    h.i00 = h.i01 = h.i10 = h.i11 = 0;
    h.ix = h.iy = h.ix1 = h.iy1 = 0;
    h.wy0 = h.wy1 = h.wx0 = h.wx1 = 0.0;
    double xl;
    if (pos_f32) {
        const float xf = (g.lon_mode == 0) ? np_mod360f((float)lon) : OD_FADD(np_mod360f(OD_FADD((float)lon, 180.0f)), -180.0f);
        xl = (double)xf;
    } else {
        xl = (g.lon_mode == 0) ? np_mod360(lon) : OD_DSUB(np_mod360(OD_DADD(lon, 180.0)), 180.0);
    }
    double px, py;
    if (!stere_forward(g.proj, xl, lat, px, py)) return r;
    r.px = px;
    r.py = py;
    double xc = px;          // x of the coverage test
    double xx = px;          // x of the index
    if (g.proj_kind == OD_PROJ_OB_TRAN) {
        // rotated degrees, which the reference treats as geographic: the coverage test modulates them with the convention of the
        // reader's TRUE corner longitudes (covers_positions_xy / modulate_longitude, variables.py:244-247, 259-280), the index
        // takes them mod 360 only when xmin > 0 (basereader/structured.py:213-215) -- the two can disagree, as they do there
        xc = (g.lon_mode == 0) ? np_mod360(px) : OD_DSUB(np_mod360(OD_DADD(px, 180.0)), 180.0);
        if (g.xmin > 0.0) xx = np_mod360(px);
    }
    if (!(xc >= g.xmin && xc <= g.xmax && py >= g.ymin && py <= g.ymax)) return r;
    double xi = OD_DMUL(div_rn(OD_DSUB(xx, g.x0), g.xspan, g.rxspan), g.nxm1);
    double yi = OD_DMUL(div_rn(OD_DSUB(py, g.y0), g.yspan, g.ryspan), g.nym1);
    if (!(xi == xi) || !(yi == yi)) return r;
    xi = xi < 0.0 ? 0.0 : (xi > g.nxm1 ? g.nxm1 : xi);
    yi = yi < 0.0 ? 0.0 : (yi > g.nym1 ? g.nym1 : yi);
    const double fx = floor(xi), fy = floor(yi);
    const int ix = (int)fx, iy = (int)fy;
    const int ix1 = ix + 1 < g.nx ? ix + 1 : g.nx - 1;
    const int iy1 = iy + 1 < g.ny ? iy + 1 : g.ny - 1;
    h.wx0 = OD_DSUB(1.0, OD_DSUB(xi, fx));
    h.wx1 = OD_DSUB(1.0, h.wx0);
    h.wy0 = OD_DSUB(1.0, OD_DSUB(yi, fy));
    h.wy1 = OD_DSUB(1.0, h.wy0);
    h.ix = ix; h.iy = iy; h.ix1 = ix1; h.iy1 = iy1;
    h.i00 = iy * g.nx + ix;
    h.i01 = iy * g.nx + ix1;
    h.i10 = iy1 * g.nx + ix;
    h.i11 = iy1 * g.nx + ix1;
    h.valid = true;
    return r;
}

// vertical + time combination without the final float32 rounding: what the reader hands to rotate_vectors (float64 for 3-D
// blocks, float32 values for 2-D ones)
OD_HD double combine_d(const GroupGeom& g, const PairRef& pr, const VertW& vw, float haA, float hbA, float haB, float hbB) {
    if (g.nz > 1) {
        const double omw = OD_DSUB(1.0, vw.wa);
        const double vA = OD_DADD(OD_DMUL((double)haA, vw.wa), OD_DMUL((double)hbA, omw));
        if (pr.mode == 1) return vA;
        const double vB = OD_DADD(OD_DMUL((double)haB, vw.wa), OD_DMUL((double)hbB, omw));
        if (pr.mode == 2) return vB;
        return OD_DADD(OD_DMUL(vA, OD_DSUB(1.0, pr.w)), OD_DMUL(vB, pr.w));
    }
    return (double)combine(g, pr, vw, haA, hbA, haB, hbB);
}

// sample2 for any group: a projected vector pair is rotated to east / north in float64 and then becomes float32.
// (Kernels that may meet projected groups are compiled twice -- template parameter PROJ -- because the projection / rotation code
// raises their register count, 72 -> 106 for Leeway, also when the groups they serve are geographic.)
OD_HD void sample2_any(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat, float& u, float& v, bool pos_f32) {
    if (!g.proj_kind) {
        sample2(g, pr, vw, lon, lat, u, v, pos_f32);
        return;
    }
    const HorizWP hp = horiz_weights_any(g, lon, lat, pos_f32);
    const HorizW& h = hp.h;
    float ru = NAN, rv = NAN;
    if (h.valid && pr.mode != 3) {
        const TexelSource ts = texel_source(pr.tex, TileView(), g.nx, g.ny, h.ix, h.ix1, h.iy, h.iy1, vw.ia, vw.ib);
        const int r0 = 4 * h.iy * ts.lx, r1 = 4 * h.iy1 * ts.lx;
        const int o00 = r0 + 4 * h.ix, o01 = r0 + 4 * h.ix1, o10 = r1 + 4 * h.ix, o11 = r1 + 4 * h.ix1;
        const LayerVals A = layer_bilin(h, layer_ptr(ts, vw.ia), o00, o01, o10, o11, pr.mode);
        LayerVals B = A;
        if (g.nz > 1) B = layer_bilin(h, layer_ptr(ts, vw.ib), o00, o01, o10, o11, pr.mode);
        const double du = combine_d(g, pr, vw, A.uA, B.uA, A.uB, B.uB);
        const double dv = combine_d(g, pr, vw, A.vA, B.vA, A.vB, B.vB);
        if (g.rotate) {
            double sr, cr;
            sincos(rotation_to_geographic(g.proj, hp.px, hp.py, g.rot_delta), &sr, &cr);
            ru = (float)OD_DSUB(OD_DMUL(du, cr), OD_DMUL(dv, sr));
            rv = (float)OD_DADD(OD_DMUL(du, sr), OD_DMUL(dv, cr));
        } else {
            ru = (float)du;
            rv = (float)dv;
        }
    }
    if (!finite_f(ru)) ru = g.fallback[0];
    if (!finite_f(rv)) rv = g.fallback[1];
    u = ru;
    v = rv;
}

// ---- the reader's own output precision (Reader.get_variables_interpolated, variables.py:860-920) ----------------------------------
// What a reader hands back before Environment casts it to float32: float64 for 3-D blocks (the vertical lerp and the time
// lerp run in float64, interpolation/structured.py:139-140, basereader/structured.py:353-364), the float32 value for 2-D
// blocks; a projected vector pair rotated in float64.  NaN where the reader has no data (the caller applies no fallback).
OD_HD void sample2_any_d(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat, double& u, double& v, bool pos_f32) {
    const HorizWP hp = horiz_weights_any(g, lon, lat, pos_f32);
    const HorizW& h = hp.h;
    double ru = NAN, rv = NAN;
    if (h.valid && pr.mode != 3) {
        const TexelSource ts = texel_source(pr.tex, TileView(), g.nx, g.ny, h.ix, h.ix1, h.iy, h.iy1, vw.ia, vw.ib);
        const int r0 = 4 * h.iy * ts.lx, r1 = 4 * h.iy1 * ts.lx;
        const int o00 = r0 + 4 * h.ix, o01 = r0 + 4 * h.ix1, o10 = r1 + 4 * h.ix, o11 = r1 + 4 * h.ix1;
        const LayerVals A = layer_bilin(h, layer_ptr(ts, vw.ia), o00, o01, o10, o11, pr.mode);
        LayerVals B = A;
        if (g.nz > 1) B = layer_bilin(h, layer_ptr(ts, vw.ib), o00, o01, o10, o11, pr.mode);
        const double du = combine_d(g, pr, vw, A.uA, B.uA, A.uB, B.uB);
        const double dv = combine_d(g, pr, vw, A.vA, B.vA, A.vB, B.vB);
        if (g.proj_kind && g.rotate) {
            double sr, cr;
            sincos(rotation_to_geographic(g.proj, hp.px, hp.py, g.rot_delta), &sr, &cr);
            ru = OD_DSUB(OD_DMUL(du, cr), OD_DMUL(dv, sr));
            rv = OD_DADD(OD_DMUL(du, sr), OD_DMUL(dv, cr));
        } else {
            ru = du;
            rv = dv;
        }
    }
    u = ru;
    v = rv;
}

OD_HD double sample1_any_d(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat, bool pos_f32) {
    const HorizW h = horiz_weights_any(g, lon, lat, pos_f32).h;
    double r = NAN;
    if (h.valid && pr.mode != 3) {
        const long long layer = (long long)g.nx * g.ny;
        const float* ta = pr.tex + ((long long)vw.ia * layer) * 2;
        const Tex2 a00 = ld_tex2(ta + 2ll * h.i00), a01 = ld_tex2(ta + 2ll * h.i01);
        const Tex2 a10 = ld_tex2(ta + 2ll * h.i10), a11 = ld_tex2(ta + 2ll * h.i11);
        Tex2 b00 = a00, b01 = a01, b10 = a10, b11 = a11;
        if (g.nz > 1) {
            const float* tb = pr.tex + ((long long)vw.ib * layer) * 2;
            b00 = ld_tex2(tb + 2ll * h.i00); b01 = ld_tex2(tb + 2ll * h.i01);
            b10 = ld_tex2(tb + 2ll * h.i10); b11 = ld_tex2(tb + 2ll * h.i11);
        }
        float aA = 0.f, bA = 0.f, aB = 0.f, bB = 0.f;
        if (pr.mode != 2) {
            aA = bilin(h, a00.x, a01.x, a10.x, a11.x);
            if (g.nz > 1) bA = bilin(h, b00.x, b01.x, b10.x, b11.x);
        }
        if (pr.mode != 1) {
            aB = bilin(h, a00.y, a01.y, a10.y, a11.y);
            if (g.nz > 1) bB = bilin(h, b00.y, b01.y, b10.y, b11.y);
        }
        r = combine_d(g, pr, vw, aA, bA, aB, bB);
    }
    return r;
}

// ---- nearest grid point (land_binary_mask) ------------------------------------------------------------------------------------
// Nearest2DInterpolator (readers/interpolation/interpolators.py:26-40), which ReaderBlock.interpolate uses for land_binary_mask
// (interpolation/structured.py:117-119): index = np.round((x - xgrid.min()) / (xgrid.max() - xgrid.min()) * len(xgrid)) -- scaled
// by the NUMBER of grid points, not by the number of intervals, as the reference writes it --, rounded half to even, cast to
// uint32 (a negative value wraps and lands on the last point) and clamped to len - 1; in float32 while the positions are
// float32.  2-D one-component groups on increasing geographic axes without a virtual column (the library refuses others).
OD_HD int nearest_index(double d, double span, double rspan, int n, bool f32) {
    double r;
    if (f32) r = (double)rintf(OD_FMUL((float)d / (float)span, (float)n));       // (d is the float32 difference here)
    else r = rint(OD_DMUL(div_rn(d, span, rspan), (double)n));
    if (!(r >= 0.0) || r >= (double)n) return n - 1;
    return (int)r;
}

OD_HD float sample1_nearest(const GroupGeom& g, const PairRef& pr, double lon, double lat, bool pos_f32) {
    float r = NAN;
    double x, dx, dy;
    if (pos_f32) {
        const float xf = (g.lon_mode == 0) ? np_mod360f((float)lon) : OD_FADD(np_mod360f(OD_FADD((float)lon, 180.0f)), -180.0f);
        x = (double)xf;
        dx = (double)OD_FADD(xf, -(float)g.x0);
        dy = (double)OD_FADD((float)lat, -(float)g.y0);
    } else {
        x = (g.lon_mode == 0) ? np_mod360(lon) : OD_DSUB(np_mod360(OD_DADD(lon, 180.0)), 180.0);
        dx = OD_DSUB(x, g.x0);
        dy = OD_DSUB(lat, g.y0);
    }
    const bool covered = (g.glob != 0 || ((x >= g.xmin) && (x <= g.xmax))) && (lat >= g.ymin) && (lat <= g.ymax) && (dx == dx) && (dy == dy);
    if (covered && pr.mode != 3) {
        const int ix = nearest_index(dx, g.xspan, g.rxspan, g.nx, pos_f32);
        const int iy = nearest_index(dy, g.yspan, g.ryspan, g.ny, pos_f32);
        const Tex2 a = ld_tex2(pr.tex + 2ll * ((long long)iy * g.nx + ix));
        if (pr.mode == 1) r = a.x;
        else if (pr.mode == 2) r = a.y;
        else {                       // (a mask the reader does not serve as a static variable: the float32 time lerp of 2-D variables)
            const float w1 = (float)pr.w, w0 = (float)OD_DSUB(1.0, pr.w);
            r = OD_FADD(OD_FMUL(a.x, w0), OD_FMUL(a.y, w1));
        }
    }
    if (!finite_f(r)) r = g.fallback[0];
    return r;
}

// horizontal weights only (scalar groups: the mixing column, the sort key, vertical velocity)
OD_HD HorizW horiz_weights_h(const GroupGeom& g, double lon, double lat, bool pos_f32) {
    return horiz_weights_any(g, lon, lat, pos_f32).h;
}

OD_HD float sample1_any(const GroupGeom& g, const PairRef& pr, const VertW& vw, double lon, double lat, bool pos_f32) {
    if (!g.proj_kind) return sample1(g, pr, vw, lon, lat, pos_f32);
    return sample1_h(g, pr, vw, horiz_weights_h(g, lon, lat, pos_f32));
}

}  // namespace od
