// od_step.cu -- the step kernels of libodcuda.so (current advection, the fused OceanDrift step, the analytical reader) and
// their launchers.  Their instantiations are most of the library's device code, so the build compiles this file once per
// arithmetic mode and step variant (-DOD_STEP_MATH=FastMath|SeriesMath|ExactMath -DOD_STEP_EXTRAS=0|1|2) and the nine
// objects compile in parallel.  Each kernel instantiation lives in exactly one object.
#include <type_traits>

#include "od_ctx.cuh"
#include "od_spec.cuh"

#if !defined(OD_STEP_MATH) || !defined(OD_STEP_EXTRAS)
#error "od_step.cu is compiled once per arithmetic mode and step variant: -DOD_STEP_MATH=... -DOD_STEP_EXTRAS=0|1|2"
#endif

// Calls f(std::integral_constant<int, SCHEME>, std::bool_constant<F64>) for the advection scheme (OD_EULER, OD_RK2, else
// OD_RK4) and the factor dtype: every launcher instantiates its kernel for all six combinations through this.
template <class F>
static void dispatch_scheme(int scheme, bool f64, F&& f) {
    auto by_dtype = [&](auto s) {
        if (f64) f(s, std::bool_constant<true>{});
        else f(s, std::bool_constant<false>{});
    };
    if (scheme == OD_EULER) by_dtype(std::integral_constant<int, 0>{});
    else if (scheme == OD_RK2) by_dtype(std::integral_constant<int, 1>{});
    else by_dtype(std::integral_constant<int, 2>{});
}

template <int SCHEME, bool F64, int EXTRAS, class MATH>
__global__ void __launch_bounds__(OD_BLOCK, OD_STEP_MINB) step_kernel(const __grid_constant__ StepParams p) {
    __shared__ LevelsSmem lv;
    __shared__ LevelsSmem lvw;
    if (p.cs.g.nz > 1) load_levels(lv, p.cs.g);
    if (EXTRAS && p.w_on && p.gw.nz > 1) load_levels(lvw, p.gw);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    step_particle_full<SCHEME, F64, EXTRAS, MATH>(p, i, lv.zs, lv.zy, lvw.zs, lvw.zy);
}

// The step specialised for the common launch (od_spec.cuh): straight-line sampler, rare cases flagged and redone by the
// general step.  Same results as step_kernel<SCHEME, F64, EXTRAS, SeriesMath>, bit for bit.
template <int SCHEME, bool F64, int EXTRAS, bool LERP>
__global__ void __launch_bounds__(OD_BLOCK, OD_SPEC_MINB) step_spec_kernel(const __grid_constant__ StepParams p) {
    __shared__ LevelsSmem lv;
    __shared__ LevelsSmem lvw;
    load_levels(lv, p.cs.g);
    if (EXTRAS && p.w_on && p.gw.nz > 1) load_levels(lvw, p.gw);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int rc = step_particle_spec<SCHEME, F64, EXTRAS, LERP>(p, i, lv.zs, lv.zy, lvw.zs, lvw.zy);
    if (rc) step_particle_redo<SCHEME, F64, EXTRAS, SeriesMath, false>(&p, i, lv.zs, lv.zy, lvw.zs, lvw.zy, rc == 2);
}

// The same step with a reader priority list for the current (StepParams::cg): a separate kernel so that the default one is
// not touched by it.  EXTRAS is 0 or 1 here (1 also serves vertical advection only).
template <int SCHEME, bool F64, int EXTRAS, class MATH>
__global__ void __launch_bounds__(OD_BLOCK) step_chain_kernel(const __grid_constant__ StepParams p) {
    __shared__ LevelsSmem lv;
    __shared__ LevelsSmem lvw;
    if (p.cs.g.nz > 1) load_levels(lv, p.cs.g);
    if (EXTRAS && p.w_on && p.gw.nz > 1) load_levels(lvw, p.gw);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    step_particle_full<SCHEME, F64, EXTRAS, MATH, true>(p, i, lv.zs, lv.zy, lvw.zs, lvw.zy);
}

// ---- TMA-staged variant -----------------------------------------------------------------------------------
// One elected thread computes nothing itself: the block first reduces the bounding box of its particles' stage-1
// cells; if the box (plus halo) fits the tensor map's box, thread 0 issues ONE cp.async.bulk.tensor.4d load of
// {4 floats, BX, BY, BZ} pair texels into shared memory and the block waits on the mbarrier; all bilinear
// corners of all RK stages that fall inside the box are then served from shared memory (fetch4), the rest and
// blocks whose particles are too spread out (unsorted input, tile-row wrap) go to global memory as before.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int SCHEME, bool F64, int EXTRAS, class MATH>
__global__ void __launch_bounds__(OD_BLOCK, OD_STEP_MINB) step_tiled_kernel(const __grid_constant__ StepParams p, const __grid_constant__ CUtensorMap tmap,
                                                                            const float* tile_tex) {
    __shared__ LevelsSmem lv;
    __shared__ LevelsSmem lvw;
    __shared__ alignas(128) float tile[OD_TILE_BZ * OD_TILE_BY * OD_TILE_BX * 4];
    __shared__ alignas(8) unsigned long long mbar;
    __shared__ int bbox[6 * (OD_BLOCK / 32)];
    __shared__ int tile_org[4];                 // x0, y0, z0, ok
    const GroupGeom& g = p.cs.g;
    if (g.nz > 1) load_levels(lv, g);
    if (EXTRAS && p.w_on && p.gw.nz > 1) load_levels(lvw, p.gw);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < p.n;
    // bounding box of the stage-1 corners of this block's particles
    int mnx = 1 << 30, mxx = -1, mny = 1 << 30, mxy = -1, mnz = 1 << 30, mxz = -1;
    if (active) {
        const HorizW h = horiz_weights(g, p.lon[i], p.lat[i], p.pos_f32 != 0);
        if (h.valid) {
            const bool zf32 = p.z_f64 == 0;
            double z0 = p.z ? (zf32 ? (double)((const float*)p.z)[i] : ((const double*)p.z)[i]) : 0.0;
            if (p.truncate_below > 0.0 && z0 < -p.truncate_below) z0 = zf32 ? (double)(float)(-p.truncate_below) : -p.truncate_below;
            const VertW vw = vert_weights(g, (const double*)lv.zs, (const double*)lv.zy, z0, zf32);
            mnx = h.ix; mxx = h.ix1; mny = h.iy; mxy = h.iy1; mnz = vw.ia; mxz = vw.ib;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        mnx = min(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mxx = max(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
        mny = min(mny, __shfl_xor_sync(0xffffffffu, mny, o)); mxy = max(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
        mnz = min(mnz, __shfl_xor_sync(0xffffffffu, mnz, o)); mxz = max(mxz, __shfl_xor_sync(0xffffffffu, mxz, o));
    }
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        bbox[warp * 6 + 0] = mnx; bbox[warp * 6 + 1] = mxx; bbox[warp * 6 + 2] = mny;
        bbox[warp * 6 + 3] = mxy; bbox[warp * 6 + 4] = mnz; bbox[warp * 6 + 5] = mxz;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < OD_BLOCK / 32; ++w) {
            mnx = min(mnx, bbox[w * 6 + 0]); mxx = max(mxx, bbox[w * 6 + 1]); mny = min(mny, bbox[w * 6 + 2]);
            mxy = max(mxy, bbox[w * 6 + 3]); mnz = min(mnz, bbox[w * 6 + 4]); mxz = max(mxz, bbox[w * 6 + 5]);
        }
        const int bz = g.nz < OD_TILE_BZ ? g.nz : OD_TILE_BZ;
        const int x0 = max(0, mnx - OD_TILE_HALO), y0 = max(0, mny - OD_TILE_HALO);
        const bool ok = mxx >= 0 && (mxx + OD_TILE_HALO - x0) < OD_TILE_BX && (mxy + OD_TILE_HALO - y0) < OD_TILE_BY &&
                        (mxz - mnz) < bz;
        tile_org[0] = x0; tile_org[1] = y0; tile_org[2] = ok ? mnz : 0; tile_org[3] = ok ? 1 : 0;
        if (ok) {
            const unsigned bytes = (unsigned)(bz * OD_TILE_BY * OD_TILE_BX * 16);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(bytes) : "memory");
            asm volatile(
                "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                ::"r"(smem_u32(tile)), "l"(reinterpret_cast<unsigned long long>(&tmap)), "r"(smem_u32(&mbar)),
                  "r"(0), "r"(x0), "r"(y0), "r"(mnz) : "memory");
        }
    }
    __syncthreads();
    TileView tv;
    tv.smem = nullptr; tv.tex = tile_tex;
    tv.x0 = tile_org[0]; tv.y0 = tile_org[1]; tv.z0 = tile_org[2];
    tv.bx = OD_TILE_BX; tv.by = OD_TILE_BY; tv.bz = g.nz < OD_TILE_BZ ? g.nz : OD_TILE_BZ;
    if (tile_org[3]) {
        unsigned done = 0;
        while (!done) {
            asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                         : "=r"(done) : "r"(smem_u32(&mbar)), "r"(0) : "memory");
        }
        tv.smem = tile;
    }
    if (!active) return;
    step_particle_full<SCHEME, F64, EXTRAS, MATH>(p, i, lv.zs, lv.zy, lvw.zs, lvw.zy, tv);
}

template <int EXTRAS, class MATH>
int launch_step_tiled(od_ctx* ctx, int scheme, bool f64, const StepParams& p, const PairEntry* pe) {
    const int grid = grid_for(p.n);
    cudaStream_t s = ctx->stream;
    dispatch_scheme(scheme, f64, [&](auto S, auto F) {
        step_tiled_kernel<decltype(S)::value, decltype(F)::value, EXTRAS, MATH><<<grid, OD_BLOCK, 0, s>>>(p, pe->tmap, pe->tex);
    });
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

template <int E, class MATH>
int launch_step_chain(od_ctx* ctx, int scheme, bool f64, const StepParams& p) {
    const int grid = grid_for(p.n);
    cudaStream_t s = ctx->stream;
    dispatch_scheme(scheme, f64, [&](auto S, auto F) {
        step_chain_kernel<decltype(S)::value, decltype(F)::value, E, MATH><<<grid, OD_BLOCK, 0, s>>>(p);
    });
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}
#if OD_STEP_EXTRAS == 2
extern template int launch_step_chain<1, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);   // (in the EXTRAS = 1 object)
#endif

template <int EXTRAS, class MATH>
int launch_step(od_ctx* ctx, int scheme, bool f64, const StepParams& p) {
    const int grid = grid_for(p.n);
    cudaStream_t s = ctx->stream;
    if constexpr (std::is_same<MATH, SeriesMath>::value) {
        if (ctx->spec && f64 && spec_eligible(p, scheme) &&
            !(EXTRAS != 0 && ((p.wind_on && p.gwind.proj_kind != 0) || (p.w_on && p.gw.proj_kind != 0)))) {
            if (spec_all_lerp(p)) step_spec_kernel<2, true, EXTRAS, true><<<grid, OD_BLOCK, 0, s>>>(p);
            else step_spec_kernel<2, true, EXTRAS, false><<<grid, OD_BLOCK, 0, s>>>(p);
            CK(cudaGetLastError());
            ctx->launches++;
            return OD_OK;
        }
    }
    const bool general = p.n_chain > 0 || p.cs.g.proj_kind != 0 || (EXTRAS != 0 && ((p.wind_on && p.gwind.proj_kind != 0) || (p.w_on && p.gw.proj_kind != 0)));
    if (general) return launch_step_chain<EXTRAS == 0 ? 0 : 1, MATH>(ctx, scheme, f64, p);
    dispatch_scheme(scheme, f64, [&](auto S, auto F) {
        step_kernel<decltype(S)::value, decltype(F)::value, EXTRAS, MATH><<<grid, OD_BLOCK, 0, s>>>(p);
    });
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

// ---- analytical reader on a projected plane (od_analytic.cuh) ---------------------------------------------
template <int SCHEME, bool F64, class MATH>
__global__ void __launch_bounds__(OD_BLOCK) analytic_step_kernel(const __grid_constant__ AnalyticStepParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    analytic_step_particle<SCHEME, F64, MATH>(p, i);
}

template <class MATH>
int launch_analytic(od_ctx* ctx, int scheme, bool f64, const AnalyticStepParams& p) {
    const int grid = grid_for(p.n);
    cudaStream_t s = ctx->stream;
    dispatch_scheme(scheme, f64, [&](auto S, auto F) {
        analytic_step_kernel<decltype(S)::value, decltype(F)::value, MATH><<<grid, OD_BLOCK, 0, s>>>(p);
    });
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

#if OD_STEP_EXTRAS == 0
template int launch_step<0, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);
template int launch_step_chain<0, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);
template int launch_step_tiled<0, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&, const PairEntry*);
template int launch_analytic<OD_STEP_MATH>(od_ctx*, int, bool, const AnalyticStepParams&);
#elif OD_STEP_EXTRAS == 1
template int launch_step<1, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);
template int launch_step_chain<1, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);
#elif OD_STEP_EXTRAS == 2
template int launch_step<2, OD_STEP_MATH>(od_ctx*, int, bool, const StepParams&);
#endif
