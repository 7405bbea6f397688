// od_kernels.cu -- libodcuda.so: CUDA kernels (sm_90a) and the C-ABI of include/odcuda.h; the step kernels are in od_step.cu.
//
// One thread per particle; particle state is SoA in HBM (float64 lon/lat, float32 z, per-particle
// factors); forcing lives in "pair texel" arrays (see od_interp.cuh) so that a bilinear corner of both
// velocity components and both bracketing time slabs is one 16-byte load.  The whole RK4 stage loop,
// the four WGS84 geodesic moves and (in od_step_oceandrift) wind drift, vertical advection and the
// horizontal random walk run in a single kernel launch per time step.
#include <cuda.h>            // CUtensorMap types only; the encoder is fetched with cudaGetDriverEntryPoint
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#include "../../include/odcuda.h"
#include "od_advect.cuh"
#include "od_mix.cuh"
#include "od_stokes.cuh"
#include "od_leeway.cuh"
#include "od_ship.cuh"
#include "od_plast.cuh"
#include "od_larval.cuh"
#include "od_analytic.cuh"
#include "od_history.cuh"
#include "od_bookkeep.cuh"
#include "od_sealevel.cuh"
#include "od_ctx.cuh"

extern "C" int od_abi_version(void) { return OD_ABI_VERSION; }

extern "C" int od_create(int device, od_ctx** out) {
    if (!out) return OD_ERR_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return OD_ERR_CUDA;
    if (cudaSetDevice(device) != cudaSuccess) return OD_ERR_CUDA;
    od_ctx* c = new od_ctx();
    c->device = device;
    cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
    *out = c;
    return OD_OK;
}

static void free_group(Group& g) {
    for (float* p : g.slots) if (p) cudaFree(p);
    g.slots.clear();
    g.version.clear();
    if (g.d_zs) cudaFree(g.d_zs);
    if (g.d_zy) cudaFree(g.d_zy);
    if (g.d_zl) cudaFree(g.d_zl);
    if (g.d_mxs) cudaFree(g.d_mxs);
    if (g.d_mxy) cudaFree(g.d_mxy);
    g.d_zs = g.d_zy = g.d_zl = g.d_mxs = g.d_mxy = nullptr;
    g.h_levels.clear();
    for (auto& p : g.pairs) {
        if (p.tex) cudaFree(p.tex);
        if (p.ready) cudaEventDestroy(p.ready);
        p = PairEntry();
    }
    g.defined = false;
}

extern "C" void od_destroy(od_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (auto& g : ctx->groups) free_group(g);
    if (ctx->d_keys) cudaFree(ctx->d_keys);
    if (ctx->d_bins) cudaFree(ctx->d_bins);
    if (ctx->d_red) cudaFree(ctx->d_red);
    if (ctx->d_bbox) cudaFree(ctx->d_bbox);
    if (ctx->d_cnt) cudaFree(ctx->d_cnt);
    if (ctx->d_fill) cudaFree(ctx->d_fill);
    if (ctx->d_fillcnt) cudaFree(ctx->d_fillcnt);
    if (ctx->d_tilesums) cudaFree(ctx->d_tilesums);
    if (ctx->hbuf) cudaFree(ctx->hbuf);
    for (int k = 0; k < 3; ++k)
        if (ctx->hstream[k]) cudaStreamDestroy(ctx->hstream[k]);
    if (ctx->hready) cudaEventDestroy(ctx->hready);
    delete ctx;
}

extern "C" const char* od_last_error(od_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

extern "C" int od_set_stream(od_ctx* ctx, void* s) {
    if (!ctx) return OD_ERR_ARG;
    ctx->stream = (cudaStream_t)s;
    return OD_OK;
}

extern "C" int od_set_option(od_ctx* ctx, int option, int value) {
    if (!ctx) return OD_ERR_ARG;
    if (option == OD_OPT_TILE) { ctx->tile = value ? 1 : 0; return OD_OK; }
    if (option == OD_OPT_SPEC) { ctx->spec = value ? 1 : 0; return OD_OK; }
    return fail(ctx, OD_ERR_ARG, "od_set_option: unknown option");
}

extern "C" int od_sync(od_ctx* ctx) {
    if (!ctx) return OD_ERR_ARG;
    CK(cudaStreamSynchronize(ctx->stream));
    return OD_OK;
}

extern "C" int od_device_sm_count(od_ctx* ctx) { return ctx ? ctx->sm_count : 0; }
extern "C" int64_t od_launch_count(od_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------------------------------------
// field groups
// ------------------------------------------------------------------------------------------------
extern "C" int od_group_define(od_ctx* ctx, int group, const od_group_desc* d, const double* h_z) {
    if (!ctx || !d || group < 0 || group >= OD_MAX_GROUPS) return fail(ctx, OD_ERR_ARG, "od_group_define: bad group");
    if (d->ncomp < 1 || d->ncomp > 2 || d->nx < 2 || d->ny < 2 || d->nz < 1 || d->nz > OD_MAX_LEVELS ||
        d->n_slots < 2 || d->n_slots > 64)
        return fail(ctx, OD_ERR_ARG, "od_group_define: bad shape");
    if (d->nz > 1 && !h_z) return fail(ctx, OD_ERR_ARG, "od_group_define: z levels missing");
    if (d->proj.kind != 0) {
        ProjStere tmp;
        if (proj_from_desc(&d->proj, &tmp) != 0) return fail(ctx, OD_ERR_ARG, "od_group_define: unsupported projection (spherical +proj=stere, +proj=merc, +proj=lcc) or bad projection parameters");
        if (d->wrap_x || d->global_x) return fail(ctx, OD_ERR_ARG, "od_group_define: a projected group cannot be periodic / global in x");
    }
    if ((size_t)d->nx * d->ny * d->nz >= (1ull << 31)) return fail(ctx, OD_ERR_ARG, "od_group_define: block too large");
    if ((size_t)d->nx * d->ny >= (1ull << 28)) return fail(ctx, OD_ERR_ARG, "od_group_define: layer too large (32-bit corner offsets)");
    CK(cudaSetDevice(ctx->device));
    Group& g = ctx->groups[group];
    free_group(g);
    g.desc = *d;
    g.slots.assign((size_t)d->n_slots * d->ncomp, nullptr);
    g.version.assign(d->n_slots, 0);
    g.capacity = g.cells();
    for (auto& p : g.slots) CK(cudaMalloc(&p, g.cells() * sizeof(float)));
    if (d->nz > 1) {
        std::vector<double> zs(d->nz), zy(d->nz);
        bool inc = h_z[1] > h_z[0];
        for (int i = 0; i < d->nz; ++i) {
            int src = inc ? i : d->nz - 1 - i;
            zs[i] = h_z[src];
            zy[i] = (double)src;
        }
        for (int i = 1; i < d->nz; ++i)
            if (!(zs[i] > zs[i - 1])) return fail(ctx, OD_ERR_ARG, "od_group_define: z levels not monotonic");
        g.zmin = zs[0];
        g.zmax = zs[d->nz - 1];
        CK(cudaMalloc(&g.d_zs, d->nz * sizeof(double)));
        CK(cudaMalloc(&g.d_zy, d->nz * sizeof(double)));
        CK(cudaMemcpyAsync(g.d_zs, zs.data(), d->nz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(g.d_zy, zy.data(), d->nz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        // tables of the vertical-mixing index search: interp1d(-levels -> layer index), x sorted increasing
        g.h_levels.assign(h_z, h_z + d->nz);
        std::vector<double> mxs(d->nz), mxy(d->nz);
        for (int i = 0; i < d->nz; ++i) {
            int src = inc ? d->nz - 1 - i : i;          // -levels increasing <=> levels decreasing
            mxs[i] = -h_z[src];
            mxy[i] = (double)src;
        }
        CK(cudaMalloc(&g.d_zl, d->nz * sizeof(double)));
        CK(cudaMalloc(&g.d_mxs, d->nz * sizeof(double)));
        CK(cudaMalloc(&g.d_mxy, d->nz * sizeof(double)));
        CK(cudaMemcpyAsync(g.d_zl, h_z, d->nz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(g.d_mxs, mxs.data(), d->nz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(g.d_mxy, mxy.data(), d->nz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    g.defined = true;
    return OD_OK;
}

extern "C" int od_group_free(od_ctx* ctx, int group) {
    if (!ctx || group < 0 || group >= OD_MAX_GROUPS) return fail(ctx, OD_ERR_ARG, "od_group_free: bad group");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    free_group(ctx->groups[group]);
    return OD_OK;
}

static int check_slot(od_ctx* ctx, int group, int slot, int comp) {
    if (!ctx || group < 0 || group >= OD_MAX_GROUPS || !ctx->groups[group].defined)
        return fail(ctx, OD_ERR_STATE, "group not defined");
    const Group& g = ctx->groups[group];
    if (slot < 0 || slot >= g.desc.n_slots || comp < 0 || comp >= g.desc.ncomp)
        return fail(ctx, OD_ERR_ARG, "bad slot/component");
    return OD_OK;
}

extern "C" int od_group_upload(od_ctx* ctx, int group, int slot, int comp, const float* src, int on_device) {
    int rc = check_slot(ctx, group, slot, comp);
    if (rc) return rc;
    if (!src) return fail(ctx, OD_ERR_ARG, "od_group_upload: null source");
    Group& g = ctx->groups[group];
    CK(cudaMemcpyAsync(g.slots[(size_t)slot * g.desc.ncomp + comp], src, g.cells() * sizeof(float),
                       on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
    g.version[slot] = ++ctx->tick;
    return OD_OK;
}

// Grow-only scratch: *p holds at least `need` elements of `elem` bytes afterwards; a buffer that is large enough is kept.
// A failed allocation leaves *p null and *cap 0, so that the next call allocates again.
static int grow(od_ctx* ctx, void** p, int64_t* cap, int64_t need, size_t elem) {
    if (*cap >= need) return OD_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    CK(cudaMalloc(p, (size_t)need * elem));
    *cap = need;
    return OD_OK;
}

#define OD_FILL_MAX_IT 16
__global__ void fill_nan_coop_kernel(float* a, float* tmp, int nx, int ny, int64_t cells, int max_iterations, unsigned* cnt);

extern "C" int od_group_fill_nan(od_ctx* ctx, int group, int slot, int comp, int max_iterations, int64_t* h_remaining) {
    int rc = check_slot(ctx, group, slot, comp);
    if (rc) return rc;
    if (max_iterations < 0 || max_iterations > OD_FILL_MAX_IT) return fail(ctx, OD_ERR_ARG, "od_group_fill_nan: bad iteration count");
    Group& g = ctx->groups[group];
    CK(cudaSetDevice(ctx->device));
    if (ctx->coop_fill_blocks < 0) {                 // once: how many blocks of the fill can be co-resident (cooperative launch)?
        int per_sm = 0, coop = 0;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device);
        if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fill_nan_coop_kernel, 256, 0) == cudaSuccess && per_sm > 0)
            // (not the whole device: a cooperative grid starts only when ALL its blocks fit at once, and a collective's kernel may
            //  be resident on the copy stream, spinning on a peer that is itself waiting to start this launch -- seen as stalls of
            //  2-10 ms at slab changes on 2 and 4 GPUs; the grid is sized as if 16 SMs were taken: it then fits beside any
            //  collective kernel -- NCCL uses at most 32 thread blocks -- and still fills the rest of the device)
            ctx->coop_fill_blocks = per_sm * (ctx->sm_count > 32 ? ctx->sm_count - 16 : (ctx->sm_count > 1 ? ctx->sm_count / 2 : 1));
        else
            ctx->coop_fill_blocks = 0;
        cudaGetLastError();
    }
    if (ctx->coop_fill_blocks == 0)
        return fail(ctx, OD_ERR_CUDA, "od_group_fill_nan: the device cannot launch fill_nan_coop_kernel cooperatively");
    float* a = g.slots[(size_t)slot * g.desc.ncomp + comp];
    int64_t cells = (int64_t)g.cells();
    if (!ctx->d_fillcnt) CK(cudaMalloc(&ctx->d_fillcnt, (OD_FILL_MAX_IT + 2) * sizeof(unsigned)));
    rc = grow(ctx, (void**)&ctx->d_fill, &ctx->fill_cap, cells, sizeof(float));
    if (rc) return rc;
    // Everything below is enqueued without a host round trip: cnt[it] = cells still missing before pass `it`;
    // the passes stop once it is zero, so a slab without holes costs one read pass.
    unsigned* cnt = ctx->d_fillcnt;
    CK(cudaMemsetAsync(cnt, 0, (OD_FILL_MAX_IT + 2) * sizeof(unsigned), ctx->stream));
    const int blocks = (int)((cells + 255) / 256);
    const int gridc = blocks < ctx->coop_fill_blocks ? blocks : ctx->coop_fill_blocks;
    float* tmp = ctx->d_fill;
    int nx = g.desc.nx, ny = g.desc.ny;
    void* args[] = {&a, &tmp, &nx, &ny, &cells, &max_iterations, &cnt};
    CK(cudaLaunchCooperativeKernel((const void*)fill_nan_coop_kernel, dim3(gridc), dim3(256), args, 0, ctx->stream));
    ctx->launches++;
    g.version[slot] = ++ctx->tick;
    if (h_remaining) {                               // optional: the caller asks how many cells stayed missing (synchronises)
        unsigned res = 0;
        CK(cudaMemcpyAsync(&res, cnt + max_iterations, sizeof(res), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *h_remaining = res;
    }
    return OD_OK;
}

extern "C" int od_group_slot_ptr(od_ctx* ctx, int group, int slot, int comp, float** out) {
    int rc = check_slot(ctx, group, slot, comp);
    if (rc) return rc;
    if (!out) return fail(ctx, OD_ERR_ARG, "od_group_slot_ptr: null out");
    Group& g = ctx->groups[group];
    *out = g.slots[(size_t)slot * g.desc.ncomp + comp];
    return OD_OK;
}

extern "C" int od_group_touch(od_ctx* ctx, int group, int slot) {
    int rc = check_slot(ctx, group, slot, 0);
    if (rc) return rc;
    ctx->groups[group].version[slot] = ++ctx->tick;
    return OD_OK;
}

// Sub-block readers (readers/basereader/structured.py:243-318, reader_netCDF_CF_generic.py:404-626): the blocks a reader hands
// out cover the elements plus a buffer, not its whole grid.  The group keeps the slots it was defined with (capacity = the full
// grid) and the blocks in them share ONE window of it: nx, ny and the block-relative index geometry (x0, xspan, ... of the block's
// own float32 axes, as ReaderBlock's interpolator sees them) are replaced here, the ring is invalidated, and the caller uploads
// the window's slabs densely ([nz][ny][nx] of the window).
extern "C" int od_group_set_window(od_ctx* ctx, int group, const od_group_desc* d) {
    int rc = check_slot(ctx, group, 0, 0);
    if (rc) return rc;
    if (!d) return fail(ctx, OD_ERR_ARG, "od_group_set_window: null descriptor");
    Group& g = ctx->groups[group];
    if (d->ncomp != g.desc.ncomp || d->nz != g.desc.nz || d->n_slots != g.desc.n_slots || d->nx < 2 || d->ny < 2 ||
        (size_t)d->nx * d->ny * d->nz > g.capacity)
        return fail(ctx, OD_ERR_ARG, "od_group_set_window: the window must keep ncomp / nz / n_slots and fit the group's slots");
    float fb0 = g.desc.fallback[0], fb1 = g.desc.fallback[1];
    g.desc = *d;
    g.desc.fallback[0] = fb0; g.desc.fallback[1] = fb1;
    CK(cudaStreamSynchronize(ctx->stream));          // launches that still read the old window's texels
    for (auto& v : g.version) v = ++ctx->tick;       // every slot's contents are stale now
    for (auto& p : g.pairs) {                        // and so are the pair texels (their tensor maps encode the old shape)
        p.slot_a = p.slot_b = -1;
        p.tmap_ok = false;
    }
    return OD_OK;
}

// bounding box (xmin, xmax, ymin, ymax) of the elements' positions, NaNs ignored; longitudes as they are stored
__global__ void __launch_bounds__(256) bbox_kernel(int64_t n, const double* __restrict__ lon, const double* __restrict__ lat,
                                                   unsigned long long* __restrict__ out) {
    // order-preserving map of a double onto an unsigned integer
    auto enc = [](double v) { unsigned long long u = (unsigned long long)__double_as_longlong(v);
                              return (u >> 63) ? ~u : (u | 0x8000000000000000ull); };
    unsigned long long lo_x = ~0ull, hi_x = 0, lo_y = ~0ull, hi_y = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = lon[i], y = lat[i];
        if (x == x) { const unsigned long long e = enc(x); lo_x = min(lo_x, e); hi_x = max(hi_x, e); }
        if (y == y) { const unsigned long long e = enc(y); lo_y = min(lo_y, e); hi_y = max(hi_y, e); }
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo_x = min(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o)); hi_x = max(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
        lo_y = min(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o)); hi_y = max(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&out[0], lo_x); atomicMax(&out[1], hi_x); atomicMin(&out[2], lo_y); atomicMax(&out[3], hi_y);
    }
}

extern "C" int od_bbox(od_ctx* ctx, int64_t n, const double* d_lon, const double* d_lat, double* h_out4) {
    if (!ctx || !h_out4 || n < 0 || (n > 0 && (!d_lon || !d_lat))) return fail(ctx, OD_ERR_ARG, "od_bbox: bad arguments");
    for (int k = 0; k < 4; ++k) h_out4[k] = NAN;
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    if (!ctx->d_bbox) CK(cudaMalloc(&ctx->d_bbox, 4 * sizeof(unsigned long long)));
    unsigned long long* d = ctx->d_bbox;
    const unsigned long long init[4] = {~0ull, 0ull, ~0ull, 0ull};
    CK(cudaMemcpyAsync(d, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    const int blocks = (int)((n + 255) / 256 < (int64_t)ctx->sm_count * 8 ? (n + 255) / 256 : (int64_t)ctx->sm_count * 8);
    bbox_kernel<<<blocks, 256, 0, ctx->stream>>>(n, d_lon, d_lat, d);
    CK(cudaGetLastError());
    ctx->launches++;
    unsigned long long r[4];
    CK(cudaMemcpyAsync(r, d, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 4; ++k) {
        const bool empty = (k & 1) ? r[k] == 0ull : r[k] == ~0ull;
        if (empty) continue;
        const unsigned long long u = (r[k] >> 63) ? (r[k] & 0x7fffffffffffffffull) : ~r[k];
        long long bits = (long long)u;
        double v;
        memcpy(&v, &bits, sizeof(v));
        h_out4[k] = v;
    }
    return OD_OK;
}

extern "C" int od_group_set_fallback(od_ctx* ctx, int group, float fallback0, float fallback1) {
    int rc = check_slot(ctx, group, 0, 0);
    if (rc) return rc;
    ctx->groups[group].desc.fallback[0] = fallback0;
    ctx->groups[group].desc.fallback[1] = fallback1;
    return OD_OK;
}

// ---- NaN holes (land) ---------------------------------------------------------------------------------
// Linear2DInterpolator fills missing values by repeatedly replacing every non-finite cell with the maximum of
// its finite 3x3 neighbours (expand_numpy_array: scipy grey_dilation(size=3), interpolators.py:9-20), as often
// as some particle still interpolates to NaN, at most 10 times (:121-139); the mutation persists in the cached
// block.  A filled cell never changes again and finite cells are never touched, so filling a block 10 times
// when it is uploaded gives every particle inside the block the value the reference's lazy loop would give.
//
// All passes of the fill in one cooperative launch: count, then (dilate, commit) until nothing is missing or
// max_iterations passes ran.  A slab without holes costs one read pass and one grid barrier.
__global__ void __launch_bounds__(256) fill_nan_coop_kernel(float* a, float* tmp, int nx, int ny,
                                                            int64_t cells, int max_iterations, unsigned* cnt) {
    cooperative_groups::grid_group grid = cooperative_groups::this_grid();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, first = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t layer = (int64_t)nx * ny;
    unsigned c = 0;
    for (int64_t i = first; i < cells; i += stride) c += !(fabsf(a[i]) <= 3.4028234663852886e38f);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&cnt[0], c);
    grid.sync();
    for (int it = 0; it < max_iterations; ++it) {
        if (*((volatile unsigned*)&cnt[it]) == 0) break;          // uniform across the grid (read after the barrier)
        unsigned still = 0;
        for (int64_t i = first; i < cells; i += stride) {
            const float v = a[i];
            if (fabsf(v) <= 3.4028234663852886e38f) {
                tmp[i] = v;
                continue;
            }
            const int64_t base = (i / layer) * layer;
            const int r = (int)((i - base) / nx), cc0 = (int)((i - base) % nx);
            float best = -INFINITY;
            bool found = false;
            for (int dr = -1; dr <= 1; ++dr) {
                const int rr = min(max(r + dr, 0), ny - 1);
                for (int dc = -1; dc <= 1; ++dc) {
                    const int cc = min(max(cc0 + dc, 0), nx - 1);
                    const float w = a[base + (int64_t)rr * nx + cc];
                    if (fabsf(w) <= 3.4028234663852886e38f) {
                        best = fmaxf(best, w);
                        found = true;
                    }
                }
            }
            tmp[i] = found ? best : NAN;
            still += found ? 0u : 1u;
        }
        if (still) atomicAdd(&cnt[it + 1], still);
        grid.sync();
        for (int64_t i = first; i < cells; i += stride) a[i] = tmp[i];
        grid.sync();
    }
}

// interleave two time slabs (and two components) into pair texels
__global__ void __launch_bounds__(OD_BLOCK) pack_pair2_kernel(const float* __restrict__ a0, const float* __restrict__ a1,
                                                               const float* __restrict__ b0, const float* __restrict__ b1,
                                                               float4* __restrict__ tex, int64_t cells) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < cells; i += stride) tex[i] = make_float4(a0[i], a1[i], b0[i], b1[i]);
}

__global__ void __launch_bounds__(OD_BLOCK) pack_pair1_kernel(const float* __restrict__ a0, const float* __restrict__ b0,
                                                               float2* __restrict__ tex, int64_t cells) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < cells; i += stride) tex[i] = make_float2(a0[i], b0[i]);
}

typedef CUresult (*od_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                       const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static od_encode_tiled_fn tensor_map_encoder() {
    static od_encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (od_encode_tiled_fn)f;
    }
    return fn;
}

// tensor map of a two-component pair-texel buffer: dims {4, nx, ny, nz} float32, box {4, BX, BY, min(BZ, nz)}
static bool make_tensor_map(const Group& g, float* tex, CUtensorMap* out) {
    od_encode_tiled_fn enc = tensor_map_encoder();
    if (!enc || g.desc.ncomp != 2) return false;
    const cuuint64_t dims[4] = {4, (cuuint64_t)g.desc.nx, (cuuint64_t)g.desc.ny, (cuuint64_t)g.desc.nz};
    const cuuint64_t strides[3] = {16, (cuuint64_t)g.desc.nx * 16, (cuuint64_t)g.desc.nx * g.desc.ny * 16};
    const cuuint32_t box[4] = {4, OD_TILE_BX, OD_TILE_BY, (cuuint32_t)(g.desc.nz < OD_TILE_BZ ? g.desc.nz : OD_TILE_BZ)};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (g.desc.nx < OD_TILE_BX || g.desc.ny < OD_TILE_BY) return false;
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, tex, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// A cached pair is about to be read or overwritten on ctx->stream: order the stream behind its build when that ran ahead on
// another stream (od_group_prepare_pair) and may not have finished.
static int order_after_build(od_ctx* ctx, PairEntry& p) {
    if (!p.pending) return OD_OK;
    if (cudaEventQuery(p.ready) == cudaSuccess) {
        p.pending = false;
        return OD_OK;
    }
    cudaGetLastError();                              // (cudaErrorNotReady is not an error)
    CK(cudaStreamWaitEvent(ctx->stream, p.ready, 0));
    return OD_OK;
}

// Pack slabs sa, sb of group g into the cache entry `victim` on ctx->stream, with at most `max_blocks` thread blocks.
static int build_pair(od_ctx* ctx, Group& g, int sa, int sb, PairEntry* victim, int max_blocks) {
    const int nc = g.desc.ncomp;
    if (!victim->tex) {
        // first pair of this group: allocate the whole cache now, so that no later step pays for a cudaMalloc
        // (tens of milliseconds for a 200 MB block on a cold device, and an implicit device synchronisation)
        // (sized for the group's full grid: a sub-block reader's windows vary in size, od_group_set_window)
        CK(cudaMalloc(&victim->tex, g.capacity * sizeof(float) * 2 * nc));
        victim->tmap_ok = make_tensor_map(g, victim->tex, &victim->tmap);
        for (auto& p : g.pairs) {
            if (p.tex) continue;
            if (cudaMalloc(&p.tex, g.capacity * sizeof(float) * 2 * nc) != cudaSuccess) {   // best effort: a smaller cache still works
                p.tex = nullptr;
                cudaGetLastError();
                break;
            }
            p.tmap_ok = make_tensor_map(g, p.tex, &p.tmap);
        }
    }
    int rc = order_after_build(ctx, *victim);
    if (rc) return rc;
    victim->pending = false;
    const int64_t cells = (int64_t)g.cells();
    int blocks = (int)((cells + OD_BLOCK - 1) / OD_BLOCK);
    if (blocks > max_blocks) blocks = max_blocks;
    if (nc == 2)
        pack_pair2_kernel<<<blocks, OD_BLOCK, 0, ctx->stream>>>(g.slots[(size_t)sa * 2], g.slots[(size_t)sa * 2 + 1],
                                                                g.slots[(size_t)sb * 2], g.slots[(size_t)sb * 2 + 1],
                                                                (float4*)victim->tex, cells);
    else
        pack_pair1_kernel<<<blocks, OD_BLOCK, 0, ctx->stream>>>(g.slots[sa], g.slots[sb], (float2*)victim->tex, cells);
    CK(cudaGetLastError());
    ctx->launches++;
    victim->slot_a = sa;
    victim->slot_b = sb;
    victim->ver_a = g.version[sa];
    victim->ver_b = g.version[sb];
    victim->last_use = ++ctx->tick;
    return OD_OK;
}

// Build the pair texels of slots (slot_a, slot_b) ahead of their first use, on the current stream (the copy stream that has
// just put one of the two slabs into its slot).  The entry the launches use most recently is never overwritten; the build
// records an event that resolve_pair orders the using stream behind.  A pair that is cached already costs nothing.
extern "C" int od_group_prepare_pair(od_ctx* ctx, int group, int slot_a, int slot_b) {
    int rc = check_slot(ctx, group, slot_a, 0);
    if (rc) return rc;
    rc = check_slot(ctx, group, slot_b, 0);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    Group& g = ctx->groups[group];
    PairEntry* newest = nullptr;
    for (auto& p : g.pairs) {
        if (p.tex && p.slot_a == slot_a && p.slot_b == slot_b && p.ver_a == g.version[slot_a] && p.ver_b == g.version[slot_b])
            return OD_OK;
        if (p.tex && (!newest || p.last_use > newest->last_use)) newest = &p;
    }
    PairEntry* victim = nullptr;
    for (auto& p : g.pairs) {
        if (&p == newest) continue;
        if (!p.tex) { victim = &p; break; }
        if (!victim || p.last_use < victim->last_use) victim = &p;
    }
    if (!victim) return OD_OK;                       // a one-entry cache: the pair is built when it is first needed
    // One thread block per SM: the build fits beside the step kernel's blocks and has a reader hour to finish, so it takes
    // memory bandwidth the issue-bound step leaves over rather than SM slots from it.
    rc = build_pair(ctx, g, slot_a, slot_b, victim, ctx->sm_count);
    if (rc) return rc;
    if (!victim->ready) CK(cudaEventCreateWithFlags(&victim->ready, cudaEventDisableTiming));
    CK(cudaEventRecord(victim->ready, ctx->stream));
    victim->pending = true;
    return OD_OK;
}

// Resolve a time sample to pair texels (building / reusing a cached pair).
static int resolve_pair(od_ctx* ctx, int group, const od_time_sample& ts, PairRef* out) {
    Group& g = ctx->groups[group];
    if (ts.mode == OD_T_MISSING) {
        out->tex = nullptr; out->mode = OD_T_MISSING; out->pad_ = 0; out->w = 0.0;
        return OD_OK;
    }
    int sa = ts.slot_a, sb = ts.slot_b;
    if (ts.mode == OD_T_FIRST) sb = (sb < 0 || sb >= g.desc.n_slots) ? sa : sb;
    if (ts.mode == OD_T_SECOND) sa = (sa < 0 || sa >= g.desc.n_slots) ? sb : sa;
    if (sa < 0 || sa >= g.desc.n_slots || sb < 0 || sb >= g.desc.n_slots || ts.mode < 0 || ts.mode > 2)
        return fail(ctx, OD_ERR_ARG, "bad time sample");
    out->w = ts.w;
    out->pad_ = 0;
    // a single-slab sample can be served by any cached pair that contains the slab; one whose build ahead is still running is
    // taken only when no other pair has the slab
    if (ts.mode != OD_T_LERP) {
        const int need = ts.mode == OD_T_FIRST ? sa : sb;
        for (int pass = 0; pass < 2; ++pass) {
            for (auto& p : g.pairs) {
                if (!p.tex) continue;
                if (pass == 0 && p.pending && cudaEventQuery(p.ready) != cudaSuccess) { cudaGetLastError(); continue; }
                int mode = -1;
                if (p.slot_a == need && p.ver_a == g.version[need]) mode = OD_T_FIRST;
                else if (p.slot_b == need && p.ver_b == g.version[need]) mode = OD_T_SECOND;
                if (mode < 0) continue;
                const int rc = order_after_build(ctx, p);
                if (rc) return rc;
                out->tex = p.tex; out->mode = mode; p.last_use = ++ctx->tick;
                return OD_OK;
            }
        }
    }
    for (auto& p : g.pairs) {
        if (p.tex && p.slot_a == sa && p.slot_b == sb && p.ver_a == g.version[sa] && p.ver_b == g.version[sb]) {
            const int rc = order_after_build(ctx, p);
            if (rc) return rc;
            out->tex = p.tex;
            out->mode = ts.mode;
            p.last_use = ++ctx->tick;
            return OD_OK;
        }
    }
    // build into the least recently used entry
    PairEntry* victim = &g.pairs[0];
    for (auto& p : g.pairs) {
        if (!p.tex) { victim = &p; break; }
        if (p.last_use < victim->last_use) victim = &p;
    }
    const int rc = build_pair(ctx, g, sa, sb, victim, ctx->sm_count * 8);
    if (rc) return rc;
    out->tex = victim->tex;
    out->mode = ts.mode;
    return OD_OK;
}

static GroupGeom make_geom(const Group& g) {
    GroupGeom q;
    memset(&q, 0, sizeof(q));
    q.nx = g.desc.nx; q.ny = g.desc.ny; q.nz = g.desc.nz; q.ncomp = g.desc.ncomp;
    q.lon_mode = g.desc.lon_mode;
    q.wrap = g.desc.wrap_x ? 1 : 0;
    q.glob = (g.desc.global_x || g.desc.wrap_x) ? 1 : 0;
    q.x0 = g.desc.x0; q.xspan = g.desc.xspan; q.y0 = g.desc.y0; q.yspan = g.desc.yspan;
    q.xmin = g.desc.xmin; q.xmax = g.desc.xmax; q.ymin = g.desc.ymin; q.ymax = g.desc.ymax;
    q.nxm1 = (double)(g.desc.nx - 1 + q.wrap); q.nym1 = (double)(g.desc.ny - 1);
    q.inv_dx = q.nxm1 / q.xspan; q.inv_dy = q.nym1 / q.yspan;
    q.rxspan = div_rn_reciprocal(q.xspan); q.ryspan = div_rn_reciprocal(q.yspan);
    q.zmin = g.zmin; q.zmax = g.zmax;
    q.fallback[0] = g.desc.fallback[0]; q.fallback[1] = g.desc.fallback[1];
    q.zs = g.d_zs; q.zy = g.d_zy;
    if (g.desc.proj.kind != 0 && proj_from_desc(&g.desc.proj, &q.proj) == 0) {
        q.proj_kind = g.desc.proj.kind;
        q.rotate = g.desc.rotate_vectors ? 1 : 0;
        // rotate_vectors: 10 m along the y axis of a projected plane, 0.1 degrees on a rotated-pole one (variables.py:79-82)
        q.rot_delta = q.proj_kind == OD_PROJ_OB_TRAN ? kObTranRotDelta : 10.0;
    }
    return q;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
struct InterpParams {
    GroupGeom g;
    PairRef pr;
    int64_t n;
    const double* lon;
    const double* lat;
    const void* z;
    void* out0;                  // float32, or float64 with out_f64
    void* out1;
    int pos_f32, z_f64;
    int out_f64, nearest;
};

template <bool PROJ>
__global__ void __launch_bounds__(OD_BLOCK) interp_kernel(const InterpParams p) {
    __shared__ LevelsSmem lv;
    if (p.g.nz > 1) load_levels(lv, p.g);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const double z = (p.z && p.g.nz > 1) ? (p.z_f64 ? ((const double*)p.z)[i] : (double)((const float*)p.z)[i]) : 0.0;
    const VertW vw = vert_weights(p.g, (const double*)lv.zs, (const double*)lv.zy, z, p.z_f64 == 0);
    if (p.nearest) {             // land_binary_mask (2-D, one component, geographic: od_interp checks)
        const float r = sample1_nearest(p.g, p.pr, p.lon[i], p.lat[i], p.pos_f32 != 0);
        if (p.out0) { if (p.out_f64) ((double*)p.out0)[i] = (double)r; else ((float*)p.out0)[i] = r; }
        return;
    }
    if (p.out_f64) {             // the reader's own precision (no fallback: od_interp requires OD_INTERP_NO_FALLBACK with it)
        if (p.g.ncomp == 2) {
            double u, v;
            sample2_any_d(p.g, p.pr, vw, p.lon[i], p.lat[i], u, v, p.pos_f32 != 0);
            if (p.out0) ((double*)p.out0)[i] = u;
            if (p.out1) ((double*)p.out1)[i] = v;
        } else if (p.out0) {
            ((double*)p.out0)[i] = sample1_any_d(p.g, p.pr, vw, p.lon[i], p.lat[i], p.pos_f32 != 0);
        }
        return;
    }
    if (p.g.ncomp == 2) {
        float u, v;
        if (PROJ) sample2_any(p.g, p.pr, vw, p.lon[i], p.lat[i], u, v, p.pos_f32 != 0);
        else sample2(p.g, p.pr, vw, p.lon[i], p.lat[i], u, v, p.pos_f32 != 0);
        if (p.out0) ((float*)p.out0)[i] = u;
        if (p.out1) ((float*)p.out1)[i] = v;
    } else {
        const float r = PROJ ? sample1_any(p.g, p.pr, vw, p.lon[i], p.lat[i], p.pos_f32 != 0) : sample1(p.g, p.pr, vw, p.lon[i], p.lat[i], p.pos_f32 != 0);
        if (p.out0) ((float*)p.out0)[i] = r;
    }
}

// counters[b] += the lanes of this warp whose flags have bit b set, for b < K: one atomic per warp and non-zero count.
// Every lane of the warp calls it.
template <int K>
__device__ __forceinline__ void tally_flags(unsigned* counters, int flags) {
#pragma unroll
    for (int b = 0; b < K; ++b) {
        const unsigned m = __ballot_sync(0xffffffffu, (flags >> b) & 1);
        if (m && (threadIdx.x & 31) == 0) atomicAdd(counters + b, (unsigned)__popc(m));
    }
}

__global__ void __launch_bounds__(256) coast_kernel(const CoastParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    tally_flags<4>(p.counters, i < p.n ? coast_one(p, i) : 0);
}

__global__ void __launch_bounds__(256) store_previous_kernel(int64_t n, const double* __restrict__ lon, const double* __restrict__ lat,
                                                             const int32_t* __restrict__ ids, int32_t id_base, int64_t n_total,
                                                             float* __restrict__ prev_lon, float* __restrict__ prev_lat) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) store_previous_one(i, lon, lat, ids, id_base, n_total, prev_lon, prev_lat);
}

__global__ void __launch_bounds__(256) store_prev_gather_kernel(const StorePrevParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) store_prev_gather_one(p, i);
}

__global__ void __launch_bounds__(256) store_prev_scatter_kernel(const StorePrevParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) store_prev_scatter_one(p, i);
}

__global__ void __launch_bounds__(256) vadv_corrected_kernel(const VadvCorrParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) vadv_corrected_one(p, i);
}

__global__ void __launch_bounds__(OD_BLOCK) geod_fwd_kernel(int64_t n, double* __restrict__ lon, double* __restrict__ lat,
                                                             const double* __restrict__ az, const double* __restrict__ dist) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double lo, la;
    geod_direct(lon[i], lat[i], az[i], dist[i], lo, la);
    lon[i] = lo;
    lat[i] = la;
}

template <bool F64>
__global__ void __launch_bounds__(OD_BLOCK) update_positions_kernel(int64_t n, double* __restrict__ lon, double* __restrict__ lat,
                                                                     const void* __restrict__ xv, const void* __restrict__ yv,
                                                                     const int32_t* __restrict__ moving, double dt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double lon0 = lon[i], lat0 = lat[i];
    const double mv = moving ? (double)moving[i] : 1.0;
    const GeodStart gs = geod_start(lat0);
    double lo, la;
    if (F64) final_move_f64(gs, lon0, ((const double*)xv)[i], ((const double*)yv)[i], mv, dt, lo, la);
    else     final_move_f32(gs, lon0, ((const float*)xv)[i], ((const float*)yv)[i], mv, dt, lo, la);
    lon[i] = lo;
    lat[i] = la;
}

// ---- vertical mixing -----------------------------------------------------------------------------
template <bool PROJ>
__global__ void __launch_bounds__(OD_BLOCK) mix_kernel(const MixParams p) {
    __shared__ double xs[OD_MAX_LEVELS];
    __shared__ double xy[OD_MAX_LEVELS];
    for (int i = threadIdx.x; p.model == 0 && i < p.g.nz; i += blockDim.x) {
        xs[i] = p.xs[i];
        xy[i] = p.xy[i];
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    mix_particle<PROJ>(p, i, xs, xy);
}

template <bool PROJ>
__global__ void __launch_bounds__(OD_BLOCK) mix_settle_kernel(const MixParams p, const SettleParams st) {
    __shared__ double xs[OD_MAX_LEVELS];
    __shared__ double xy[OD_MAX_LEVELS];
    for (int i = threadIdx.x; p.model == 0 && i < p.g.nz; i += blockDim.x) {
        xs[i] = p.xs[i];
        xy[i] = p.xy[i];
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    mix_particle<PROJ, true>(p, i, xs, xy, &st);
}

__global__ void __launch_bounds__(256) resuspend_kernel(int64_t n, const float* __restrict__ u, const float* __restrict__ v,
                                                        float threshold, int32_t* __restrict__ moving, void* __restrict__ z, int32_t z_f64) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        resuspend_one(i, u, v, threshold, moving, z, z_f64);
}

// ---- ShipDrift -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ship_kernel(const ShipParams p) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
        ship_particle(p, i);
}

// ---- PlastDrift ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OD_BLOCK) plast_kernel(const PlastParams p) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
        plast_particle(p, i);
}

// ---- LarvalFish ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OD_BLOCK) larval_develop_kernel(const LarvalParams p, unsigned* flags) {
    unsigned acc = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
        acc |= larval_develop_one(p, i);
    if (flags) {
        acc = __reduce_or_sync(0xffffffffu, acc);
        if (acc && (threadIdx.x & 31) == 0) atomicOr(flags, acc);
    }
}

__global__ void __launch_bounds__(OD_BLOCK) larval_migrate_kernel(const LarvalParams p) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
        larval_migrate_one(p, i);
}

// ---- Leeway -------------------------------------------------------------------------------------------
template <bool PROJ>
__global__ void __launch_bounds__(OD_BLOCK) leeway_kernel(const LeewayParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) leeway_particle<PROJ>(p, i);
}

// ---- Stokes drift and reductions --------------------------------------------------------------------
__global__ void __launch_bounds__(OD_BLOCK) stokes_kernel(const StokesParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) stokes_particle(p, i);
}

// order-preserving map float -> unsigned so that atomicMin/atomicMax work on floats
__device__ __forceinline__ unsigned f2ord(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
static float ord2f(unsigned u) {
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// min and max of a[i] (+ b[i]) over all i, NaNs ignored; grid-stride, warp shuffle, one atomic pair per warp
__global__ void __launch_bounds__(256) minmax_kernel(int64_t n, const float* __restrict__ a, const float* __restrict__ b,
                                                     unsigned* __restrict__ out) {
    unsigned lo = 0xffffffffu, hi = 0u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = b ? __fadd_rn(a[i], b[i]) : a[i];
        if (v == v) {
            const unsigned o = f2ord(v);
            lo = min(lo, o);
            hi = max(hi, o);
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&out[0], lo);
        atomicMax(&out[1], hi);
    }
}

__global__ void __launch_bounds__(256) stokes_tab_kernel(const StokesTabParams p) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
        stokes_tab_one(p, i);
}

// ---- particle ordering ---------------------------------------------------------------------------
struct SortParams {
    GroupGeom g;
    int64_t n;
    const double* lon;
    const double* lat;
    const float* z;
    int tile, ntx, nty;
};

template <bool PROJ>
__global__ void __launch_bounds__(OD_BLOCK) cell_key_kernel(const SortParams p, int32_t* __restrict__ keys,
                                                             int32_t* __restrict__ bins) {
    __shared__ LevelsSmem lv;
    if (p.g.nz > 1) load_levels(lv, p.g);
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int key = -1;                                    // (lanes past the end: a group of their own, no count)
    if (i < p.n) {
        const HorizW h = PROJ ? horiz_weights_h(p.g, p.lon[i], p.lat[i], false) : horiz_weights(p.g, p.lon[i], p.lat[i], false);
        key = 0;
        if (h.valid) {
            const int iy = h.i00 / p.g.nx, ix = h.i00 - iy * p.g.nx;
            const VertW vw = vert_weights(p.g, (const double*)lv.zs, (const double*)lv.zy, (p.z && p.g.nz > 1) ? (double)p.z[i] : 0.0);
            key = 1 + (vw.ia * p.nty + iy / p.tile) * p.ntx + ix / p.tile;
        }
        keys[i] = key;
    }
    // cell-sorted particles: the lanes of a warp mostly share one to three bins; one atomic per bin and warp
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&bins[key], __popc(peers));
}

// exclusive scan of the bin counts, one block (bins <= a few hundred thousand)
__global__ void __launch_bounds__(1024) scan_bins_kernel(int32_t* __restrict__ bins, int nbins) {
    __shared__ int32_t warp_sums[32];
    __shared__ int32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nbins; base += 1024) {
        const int i = base + threadIdx.x;
        int v = i < nbins ? bins[i] : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(0xffffffffu, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int s = warp_sums[threadIdx.x];
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(0xffffffffu, s, o);
                if (threadIdx.x >= o) s += y;
            }
            warp_sums[threadIdx.x] = s;
        }
        __syncthreads();
        const int warp_off = (threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
        const int incl = x + warp_off + carry;
        if (i < nbins) bins[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = incl;
        __syncthreads();
    }
}

// Large bin tables: exclusive scan of 4096-entry tiles (in place, tile totals to tile_sums), scan of the tile totals with
// the one-block kernel above, then the tile offsets are added back.  Three short launches instead of one block walking
// the whole table (0.7 ms for the 819 201 bins of a 512 x 512 x 50 grid).
#define OD_SCAN_TILE 4096
__global__ void __launch_bounds__(1024) scan_tiles_kernel(int32_t* __restrict__ bins, int nbins, int32_t* __restrict__ tile_sums) {
    __shared__ int32_t warp_sums[32];
    const int base = blockIdx.x * OD_SCAN_TILE + threadIdx.x * 4;
    int v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = base + k < nbins ? bins[base + k] : 0;
    const int mine = v[0] + v[1] + v[2] + v[3];
    int x = mine;
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, x, o);
        if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        int t = warp_sums[threadIdx.x];
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(0xffffffffu, t, o);
            if (threadIdx.x >= o) t += y;
        }
        warp_sums[threadIdx.x] = t;
    }
    __syncthreads();
    int run = x - mine + ((threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0);      // exclusive prefix of this thread
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (base + k < nbins) bins[base + k] = run;
        run += v[k];
    }
    if (threadIdx.x == 1023) tile_sums[blockIdx.x] = run;
}

__global__ void __launch_bounds__(1024) add_tile_offsets_kernel(int32_t* __restrict__ bins, int nbins, const int32_t* __restrict__ tile_sums) {
    const int off = tile_sums[blockIdx.x];
    const int base = blockIdx.x * OD_SCAN_TILE + threadIdx.x * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (base + k < nbins) bins[base + k] += off;
}

static int scan_exclusive(od_ctx* ctx, int32_t* bins, int nbins) {
    if (nbins <= 2 * OD_SCAN_TILE) {
        scan_bins_kernel<<<1, 1024, 0, ctx->stream>>>(bins, nbins);
        ctx->launches++;
        return OD_OK;
    }
    const int ntiles = (nbins + OD_SCAN_TILE - 1) / OD_SCAN_TILE;
    const int rc = grow(ctx, (void**)&ctx->d_tilesums, &ctx->tiles_cap, ntiles, sizeof(int32_t));
    if (rc) return rc;
    scan_tiles_kernel<<<ntiles, 1024, 0, ctx->stream>>>(bins, nbins, ctx->d_tilesums);
    scan_bins_kernel<<<1, 1024, 0, ctx->stream>>>(ctx->d_tilesums, ntiles);
    add_tile_offsets_kernel<<<ntiles, 1024, 0, ctx->stream>>>(bins, nbins, ctx->d_tilesums);
    ctx->launches += 3;
    return OD_OK;
}

__global__ void __launch_bounds__(OD_BLOCK) scatter_perm_kernel(int64_t n, const int32_t* __restrict__ keys,
                                                                 int32_t* __restrict__ bins, int32_t* __restrict__ perm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int key = i < n ? keys[i] : -1;
    // the lanes of a warp that share a bin take consecutive places of it: the first of them reserves the group's range
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
    int base = 0;
    if (key >= 0 && lane == leader) base = atomicAdd(&bins[key], __popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (key >= 0) perm[base + __popc(peers & ((1u << lane) - 1u))] = (int32_t)i;
}

// ---- stable partition (deactivated-element compaction) ---------------------------------------------------
// LagrangianArray.move_elements keeps the relative order of both the kept and the moved elements
// (elements/elements.py:223-228).  Pass 1 counts the kept elements per block, a single-block scan turns the
// counts into offsets, pass 2 writes perm = [kept indices in order | removed indices in order].
#define OD_PART_BLOCK 256
__global__ void __launch_bounds__(OD_PART_BLOCK) partition_count_kernel(int64_t n, const int32_t* __restrict__ status,
                                                                        int32_t* __restrict__ block_keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int keep = (i < n && status[i] == 0) ? 1 : 0;
    const int c = __syncthreads_count(keep);
    if (threadIdx.x == 0) block_keep[blockIdx.x] = c;
}

__global__ void __launch_bounds__(OD_PART_BLOCK) partition_scatter_kernel(int64_t n, const int32_t* __restrict__ status,
                                                                          const int32_t* __restrict__ block_keep_excl,
                                                                          int64_t n_keep, int32_t* __restrict__ perm) {
    __shared__ int warp_keep[OD_PART_BLOCK / 32];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < n;
    const int keep = (valid && status[i] == 0) ? 1 : 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int rank_in_warp = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) warp_keep[warp] = __popc(ballot);
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; ++w) before += warp_keep[w];
    const int64_t keep_base = block_keep_excl[blockIdx.x];
    const int64_t first = (int64_t)blockIdx.x * blockDim.x;
    if (!valid) return;
    const int local_keep_rank = before + rank_in_warp;              // kept elements before me in this block
    const int local_index = (int)(i - first);
    if (keep) perm[keep_base + local_keep_rank] = (int32_t)i;
    else perm[n_keep + (first - keep_base) + (local_index - local_keep_rank)] = (int32_t)i;
}

template <typename T>
__global__ void __launch_bounds__(OD_BLOCK) permute_kernel(int64_t n, const int32_t* __restrict__ perm,
                                                            const T* __restrict__ src, T* __restrict__ dst, int inverse) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (inverse) dst[perm[k]] = src[k];
    else dst[k] = src[perm[k]];
}

// ---- particle exchange of the spatial-tile mode (BASELINE configs[2]: "halo particles that cross tile boundaries are
// exchanged with a single all-to-all") -------------------------------------------------------------------------------------
// Every rank owns one longitude strip.  After a step the elements are grouped by the rank that owns their new position and
// packed as fixed-size records (one row per element, the SoA columns side by side) so that ONE all_to_all_single moves them:
//   pass 1  owner of every element (search in the strip bounds) + per-block histogram, written owner-major [owner][block]
//   scan    exclusive scan of that table = first output row of every (owner, block) pair (stable: blocks in order)
//   pass 2  rank of the element among its block's elements with the same owner (warp match + per-warp counts) -> row;
//           the element's columns are copied into its record
// The receiving side scatters the records back into SoA columns (unpack_records_kernel).
#define OD_PACK_BLOCK 256

struct PackParams {
    int64_t n;
    const double* lon;
    int world, ncols, rec_bytes, nblocks;
    double bounds[OD_PACK_MAX_WORLD + 1];
    const unsigned char* cols[OD_PACK_MAX_COLS];
    int col_bytes[OD_PACK_MAX_COLS];
    int col_off[OD_PACK_MAX_COLS];
};

__device__ __forceinline__ int strip_of(const PackParams& p, double x) {
    // torch.bucketize(lon, inner_bounds, right=True) clamped: number of inner bounds <= x  (NaN -> last strip, like bucketize)
    int o = 0;
    for (int k = 1; k < p.world; ++k) o += (x >= p.bounds[k]) ? 1 : 0;
    if (!(x == x)) o = p.world - 1;
    return o;
}

// one field of a record, column -> record or back: b bytes at byte offset off of records of rec_bytes; a 4- or 8-byte
// field that every record keeps aligned moves as one word
__device__ __forceinline__ void copy_field(unsigned char* dst, const unsigned char* src, int b, int off, int rec_bytes) {
    if (b == 8 && ((off | rec_bytes) & 7) == 0) *reinterpret_cast<uint64_t*>(dst) = *reinterpret_cast<const uint64_t*>(src);
    else if (b == 4 && ((off | rec_bytes) & 3) == 0) *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<const uint32_t*>(src);
    else for (int k = 0; k < b; ++k) dst[k] = src[k];
}

__global__ void __launch_bounds__(OD_PACK_BLOCK) owner_count_kernel(const __grid_constant__ PackParams p, int32_t* __restrict__ table) {
    __shared__ int hist[OD_PACK_MAX_WORLD];
    for (int k = threadIdx.x; k < p.world; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n) atomicAdd(&hist[strip_of(p, p.lon[i])], 1);
    __syncthreads();
    for (int k = threadIdx.x; k < p.world; k += blockDim.x) table[(int64_t)k * p.nblocks + blockIdx.x] = hist[k];
}

__global__ void __launch_bounds__(OD_PACK_BLOCK) owner_pack_kernel(const __grid_constant__ PackParams p, const int32_t* __restrict__ table,
                                                                   unsigned char* __restrict__ records, int32_t* __restrict__ perm) {
    __shared__ int warp_cnt[OD_PACK_BLOCK / 32][OD_PACK_MAX_WORLD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < (OD_PACK_BLOCK / 32) * OD_PACK_MAX_WORLD; k += blockDim.x) (&warp_cnt[0][0])[k] = 0;
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < p.n;
    const int owner = valid ? strip_of(p, p.lon[i]) : -1;
    const unsigned same = __match_any_sync(0xffffffffu, owner);
    const int rank_in_warp = __popc(same & ((1u << lane) - 1u));
    if (valid && rank_in_warp == 0) warp_cnt[warp][owner] = __popc(same);
    __syncthreads();
    if (!valid) return;
    int before = 0;
    for (int w = 0; w < warp; ++w) before += warp_cnt[w][owner];
    const int64_t row = (int64_t)table[(int64_t)owner * p.nblocks + blockIdx.x] + before + rank_in_warp;
    if (perm) perm[row] = (int32_t)i;
    unsigned char* rec = records + row * p.rec_bytes;
    for (int c = 0; c < p.ncols; ++c)
        copy_field(rec + p.col_off[c], p.cols[c] + i * p.col_bytes[c], p.col_bytes[c], p.col_off[c], p.rec_bytes);
}

struct UnpackParams {
    int64_t n;
    int ncols, rec_bytes;
    unsigned char* cols[OD_PACK_MAX_COLS];
    int col_bytes[OD_PACK_MAX_COLS];
    int col_off[OD_PACK_MAX_COLS];
};

__global__ void __launch_bounds__(OD_PACK_BLOCK) unpack_records_kernel(const __grid_constant__ UnpackParams p, const unsigned char* __restrict__ records) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const unsigned char* rec = records + i * p.rec_bytes;
    for (int c = 0; c < p.ncols; ++c)
        copy_field(p.cols[c] + i * p.col_bytes[c], rec + p.col_off[c], p.col_bytes[c], p.col_off[c], p.rec_bytes);
}

// ------------------------------------------------------------------------------------------------
// C-ABI entry points
// ------------------------------------------------------------------------------------------------
static int need_group(od_ctx* ctx, int group, int ncomp) {
    if (!ctx) return OD_ERR_ARG;
    if (group < 0 || group >= OD_MAX_GROUPS || !ctx->groups[group].defined) return fail(ctx, OD_ERR_STATE, "group not defined");
    if (ncomp && ctx->groups[group].desc.ncomp != ncomp) return fail(ctx, OD_ERR_ARG, "group has wrong component count");
    return OD_OK;
}

extern "C" int od_interp(od_ctx* ctx, int group, const od_time_sample* ts, int64_t n, const double* lon, const double* lat,
                         const void* z, int flags, void* out0, void* out1) {
    int rc = need_group(ctx, group, 0);
    if (rc) return rc;
    if (!ts || n < 0 || (n > 0 && (!lon || !lat))) return fail(ctx, OD_ERR_ARG, "od_interp: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    InterpParams p;
    p.g = make_geom(ctx->groups[group]);
    rc = resolve_pair(ctx, group, *ts, &p.pr);
    if (rc) return rc;
    p.n = n; p.lon = lon; p.lat = lat; p.z = z; p.out0 = out0; p.out1 = out1; p.pos_f32 = flags & OD_INTERP_POS_F32;
    p.z_f64 = (flags & OD_INTERP_Z_F64) ? 1 : 0;
    p.out_f64 = (flags & OD_INTERP_OUT_F64) ? 1 : 0;
    p.nearest = (flags & OD_INTERP_NEAREST) ? 1 : 0;
    if (p.out_f64 && !p.nearest && !(flags & OD_INTERP_NO_FALLBACK))
        return fail(ctx, OD_ERR_ARG, "od_interp: OD_INTERP_OUT_F64 is the reader's output (use it with OD_INTERP_NO_FALLBACK)");
    if (p.nearest && (p.g.ncomp != 1 || p.g.nz > 1 || p.g.proj_kind != 0 || p.g.wrap != 0 || !(p.g.xspan > 0.0) || !(p.g.yspan > 0.0)))
        return fail(ctx, OD_ERR_ARG, "od_interp: OD_INTERP_NEAREST serves 2-D one-component geographic groups on increasing, non-periodic axes");
    if (flags & OD_INTERP_NO_FALLBACK) p.g.fallback[0] = p.g.fallback[1] = NAN;
    if (flags & OD_INTERP_NO_ROTATE) p.g.rotate = 0;
    if (p.g.proj_kind) interp_kernel<true><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(p);
    else interp_kernel<false><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_geod_fwd(od_ctx* ctx, int64_t n, double* lon, double* lat, const double* az, const double* dist) {
    if (!ctx || n < 0 || (n > 0 && (!lon || !lat || !az || !dist))) return fail(ctx, OD_ERR_ARG, "od_geod_fwd: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    geod_fwd_kernel<<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, lon, lat, az, dist);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_update_positions(od_ctx* ctx, int64_t n, double* lon, double* lat, const void* xv, const void* yv,
                                   int vel_f64, const int32_t* moving, double dt) {
    if (!ctx || n < 0 || (n > 0 && (!lon || !lat || !xv || !yv))) return fail(ctx, OD_ERR_ARG, "od_update_positions: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    if (vel_f64) update_positions_kernel<true><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, lon, lat, xv, yv, moving, dt);
    else         update_positions_kernel<false><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, lon, lat, xv, yv, moving, dt);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

static int fill_current(od_ctx* ctx, const od_advect_args* a, StepParams* p) {
    int rc = need_group(ctx, a->group_uv, 2);
    if (rc) return rc;
    if (a->scheme < 0 || a->scheme > 2) return fail(ctx, OD_ERR_ARG, "unknown advection scheme");
    if (a->n < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat))) return fail(ctx, OD_ERR_ARG, "null particle arrays");
    const Group& g = ctx->groups[a->group_uv];
    if (g.desc.nz > 1 && !a->d_z) return fail(ctx, OD_ERR_ARG, "3-D current group needs z");
    if ((a->d_k1_u == nullptr) != (a->d_k1_v == nullptr)) return fail(ctx, OD_ERR_ARG, "k1 needs both components");
    memset(p, 0, sizeof(*p));
    p->cs.g = make_geom(g);
    p->has_k1 = a->d_k1_u != nullptr;
    if (!p->has_k1) {
        rc = resolve_pair(ctx, a->group_uv, a->t_start, &p->cs.t_start);
        if (rc) return rc;
    }
    if (a->scheme != OD_EULER) {
        rc = resolve_pair(ctx, a->group_uv, a->t_mid, &p->cs.t_mid);
        if (rc) return rc;
    }
    if (a->scheme == OD_RK4) {
        rc = resolve_pair(ctx, a->group_uv, a->t_end, &p->cs.t_end);
        if (rc) return rc;
    }
    if (a->n_chain < 0 || a->n_chain > OD_MAX_CHAIN) return fail(ctx, OD_ERR_ARG, "reader chain longer than OD_MAX_CHAIN");
    p->n_chain = a->n_chain;
    for (int k = 0; k < a->n_chain; ++k) {
        rc = need_group(ctx, a->chain_group[k], 2);
        if (rc) return rc;
        const Group& gk = ctx->groups[a->chain_group[k]];
        if (gk.desc.nz > 1 && !a->d_z) return fail(ctx, OD_ERR_ARG, "3-D current group needs z");
        p->cg[k] = make_geom(gk);
        p->cg[k].fallback[0] = p->cg[k].fallback[1] = NAN;
        if (!p->has_k1) {
            rc = resolve_pair(ctx, a->chain_group[k], a->chain_t[k][0], &p->ct[k][0]);
            if (rc) return rc;
        }
        if (a->scheme != OD_EULER) {
            rc = resolve_pair(ctx, a->chain_group[k], a->chain_t[k][1], &p->ct[k][1]);
            if (rc) return rc;
        }
        if (a->scheme == OD_RK4) {
            rc = resolve_pair(ctx, a->chain_group[k], a->chain_t[k][2], &p->ct[k][2]);
            if (rc) return rc;
        }
    }
    if (a->n_chain > 0) {          // the environment fallback applies after the last reader of the list
        p->chain_fallback[0] = p->cs.g.fallback[0];
        p->chain_fallback[1] = p->cs.g.fallback[1];
        p->cs.g.fallback[0] = p->cs.g.fallback[1] = NAN;
    }
    p->dt = a->dt;
    p->dt32 = (float)a->dt;
    p->adt32 = (float)fabs(a->dt);
    p->n = a->n;
    p->lon = a->d_lon; p->lat = a->d_lat; p->z = a->d_z;
    p->factor = a->d_factor; p->moving = a->d_moving;
    p->k1u = a->d_k1_u; p->k1v = a->d_k1_v;
    p->env_u = a->d_env_u; p->env_v = a->d_env_v;
    p->truncate_below = a->truncate_below;
    p->pos_f32 = a->pos_f32;
    p->z_f64 = a->z_f64;
    p->noise_cur = a->noise_kinds ? a->d_noise_cur : nullptr;
    p->noise_kinds = a->noise_kinds;
    if (a->noise_kinds && !a->d_noise_cur) return fail(ctx, OD_ERR_ARG, "noise_kinds set without d_noise_cur");
    return OD_OK;
}

static const PairEntry* find_tmap(const Group& g, const float* tex) {
    for (const auto& pe : g.pairs)
        if (pe.tex == tex && pe.tmap_ok) return &pe;
    return nullptr;
}

template <int EXTRAS>
static int launch_step_mode(od_ctx* ctx, int mode, int scheme, bool f64, const StepParams& p) {
    if (mode == OD_MATH_FAST) return launch_step<EXTRAS, FastMath>(ctx, scheme, f64, p);
    if (mode == OD_MATH_SERIES) return launch_step<EXTRAS, SeriesMath>(ctx, scheme, f64, p);
    return launch_step<EXTRAS, ExactMath>(ctx, scheme, f64, p);
}

extern "C" int od_advect_current(od_ctx* ctx, const od_advect_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_advect_current: null argument");
    CK(cudaSetDevice(ctx->device));
    StepParams p;
    int rc = fill_current(ctx, a, &p);
    if (rc) return rc;
    if (a->n == 0) return OD_OK;
    const PairEntry* pe = nullptr;
    if (ctx->tile && a->scheme != OD_EULER && a->n_chain == 0)          // tile the pair the RK stages sample (t_mid)
        pe = find_tmap(ctx->groups[a->group_uv], p.cs.t_mid.tex);
    if (a->fast < 0 || a->fast > OD_MATH_SERIES) return fail(ctx, OD_ERR_ARG, "od_advect_current: unknown arithmetic mode");
    if (pe) {
        if (a->fast == OD_MATH_FAST) return launch_step_tiled<0, FastMath>(ctx, a->scheme, a->factor_f64 != 0, p, pe);
        if (a->fast == OD_MATH_SERIES) return launch_step_tiled<0, SeriesMath>(ctx, a->scheme, a->factor_f64 != 0, p, pe);
        return launch_step_tiled<0, ExactMath>(ctx, a->scheme, a->factor_f64 != 0, p, pe);
    }
    return launch_step_mode<0>(ctx, a->fast, a->scheme, a->factor_f64 != 0, p);
}

// advect_ocean_current on HOST arrays: the particle range is cut into chunks; each chunk's host->device copies, kernel
// and device->host copies go to one of three streams (and staging buffers), so the PCIe transfers of neighbouring
// chunks overlap each other (both directions) and the kernel.  The first and last chunks are half size: the pipeline
// fills and drains faster.  Pinned host memory is needed for the copies to overlap.  Returns when the results are in
// h_out_lon / h_out_lat.
static int fill_step(od_ctx* ctx, const od_step_args* a, StepParams* pp);

static int host_pipeline(od_ctx* ctx, const od_advect_args* a, const od_step_args* step, const od_host_io* io) {
    const int64_t n = a->n;
    if (n < 0 || (n > 0 && (!io->h_lon || !io->h_lat || !io->h_out_lon || !io->h_out_lat)))
        return fail(ctx, OD_ERR_ARG, "od_advect_current_host: null host arrays");
    if (a->d_k1_u || a->d_k1_v || a->d_env_u || a->d_env_v || a->d_noise_cur)
        return fail(ctx, OD_ERR_ARG, "od_advect_current_host: k1 / env / noise arrays are not supported on the host path");
    CK(cudaSetDevice(ctx->device));
    const Group* gp = (a->group_uv >= 0 && a->group_uv < OD_MAX_GROUPS) ? &ctx->groups[a->group_uv] : nullptr;
    const bool has_z = io->h_z != nullptr;
    if (gp && gp->defined && gp->desc.nz > 1 && !has_z) return fail(ctx, OD_ERR_ARG, "3-D current group needs z");
    // resolve the pairs once, on the caller's stream (uploads / pair packing were enqueued there)
    StepParams p;
    double dummy = 0.0;
    int rc;
    if (step) {
        od_step_args b = *step;
        b.cur.n = 0;
        b.cur.d_lon = b.cur.d_lat = &dummy;
        b.cur.d_z = has_z ? (const void*)&dummy : nullptr;
        if (b.group_w >= 0) b.d_z_inout = &dummy;
        rc = fill_step(ctx, &b, &p);
    } else {
        od_advect_args b = *a;
        b.n = 0;
        b.d_lon = b.d_lat = &dummy;
        b.d_z = has_z ? (const void*)&dummy : nullptr;
        rc = fill_current(ctx, &b, &p);
    }
    if (rc) return rc;
    if (n == 0) return OD_OK;
    if (a->fast < 0 || a->fast > OD_MATH_SERIES) return fail(ctx, OD_ERR_ARG, "od_advect_current_host: unknown arithmetic mode");
    if (!ctx->hready) {
        CK(cudaEventCreateWithFlags(&ctx->hready, cudaEventDisableTiming));
        for (int k = 0; k < 3; ++k) CK(cudaStreamCreateWithFlags(&ctx->hstream[k], cudaStreamNonBlocking));
    }
    int chunks = io->chunks > 0 ? io->chunks : 12;
    if (chunks > n) chunks = (int)n;
    // chunk boundaries: weights 1/2, 1, ..., 1, 1/2
    const double unit = chunks > 2 ? (double)n / (chunks - 1) : (double)n / chunks;
    const int64_t cap = (int64_t)unit + 2;
    const size_t zsz = a->z_f64 ? 8 : 4;
    rc = grow(ctx, (void**)&ctx->hbuf, &ctx->hbuf_cap, cap, 3 * 24);        // three buffers of lon, lat (float64), z (<= 8 B)
    if (rc) return rc;
    CK(cudaEventRecord(ctx->hready, ctx->stream));
    static const bool trace = getenv("OD_HOST_TRACE") != nullptr;       // debugging aid: per-chunk timeline on stderr
    std::vector<cudaEvent_t> tev;
    cudaEvent_t t0 = nullptr;
    if (trace) {
        cudaEventCreate(&t0);
        cudaEventRecord(t0, ctx->stream);
    }
    auto mark = [&](cudaStream_t st) {
        if (!trace) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, st);
        tev.push_back(e);
    };
    const size_t fsz = a->factor_f64 ? 8 : 4;
    cudaStream_t caller = ctx->stream;
    int64_t lo = 0;
    rc = OD_OK;
    for (int c = 0; c < chunks && rc == OD_OK; ++c) {
        int64_t hi;
        if (c == chunks - 1) hi = n;
        else if (chunks > 2) hi = (int64_t)(unit * (c + 0.5));
        else hi = (int64_t)(unit * (c + 1));
        if (hi > n) hi = n;
        const int64_t m = hi - lo;
        if (m <= 0) continue;
        const int k = c % 3;
        cudaStream_t st = ctx->hstream[k];
        double* d_lon = (double*)(ctx->hbuf + k * ctx->hbuf_cap * 24);
        double* d_lat = d_lon + ctx->hbuf_cap;
        char* d_z = (char*)(d_lat + ctx->hbuf_cap);
        if (c < 3) CK(cudaStreamWaitEvent(st, ctx->hready, 0));
        mark(st);
        CK(cudaMemcpyAsync(d_lon, io->h_lon + lo, m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_lat, io->h_lat + lo, m * 8, cudaMemcpyHostToDevice, st));
        if (has_z) CK(cudaMemcpyAsync(d_z, (const char*)io->h_z + lo * zsz, m * zsz, cudaMemcpyHostToDevice, st));
        mark(st);
        StepParams q = p;
        q.n = m;
        q.lon = d_lon; q.lat = d_lat; q.z = has_z ? (const void*)d_z : nullptr;
        q.factor = a->d_factor ? (const void*)((const char*)a->d_factor + lo * fsz) : nullptr;
        q.moving = a->d_moving ? a->d_moving + lo : nullptr;
        if (step) {
            if (q.wind_on) q.wdf = (const char*)step->d_wdf + lo * (step->wdf_f64 ? 8 : 4);
            if (q.w_on) { q.z_inout = d_z; q.zio_f64 = a->z_f64; }
            if (q.diff_on) {
                q.rand_x = step->d_rand_x + lo; q.rand_y = step->d_rand_y + lo;
                if (step->d_diffusivity) q.diffusivity = step->d_diffusivity + lo;
            }
        }
        ctx->stream = st;
        rc = !step ? launch_step_mode<0>(ctx, a->fast, a->scheme, a->factor_f64 != 0, q)
                   : (!q.wind_on && !q.diff_on) ? launch_step_mode<2>(ctx, a->fast, a->scheme, a->factor_f64 != 0, q)
                                                : launch_step_mode<1>(ctx, a->fast, a->scheme, a->factor_f64 != 0, q);
        ctx->stream = caller;
        if (rc) break;
        mark(st);
        CK(cudaMemcpyAsync(io->h_out_lon + lo, d_lon, m * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(io->h_out_lat + lo, d_lat, m * 8, cudaMemcpyDeviceToHost, st));
        if (step && q.w_on) CK(cudaMemcpyAsync((char*)io->h_out_z + lo * zsz, d_z, m * zsz, cudaMemcpyDeviceToHost, st));
        mark(st);
        lo = hi;
    }
    for (int k = 0; k < 3; ++k) {
        cudaError_t e = cudaStreamSynchronize(ctx->hstream[k]);
        if (e != cudaSuccess && rc == OD_OK) rc = fail(ctx, OD_ERR_CUDA, "od_advect_current_host", e);
    }
    if (trace) {
        fprintf(stderr, "od_advect_current_host timeline (ms after the caller's stream reached the call): chunk: h2d-start h2d-end kernel-end d2h-end\n");
        for (size_t k = 0; k + 3 < tev.size() + 0; k += 4) {
            float t[4];
            for (int j = 0; j < 4; ++j) cudaEventElapsedTime(&t[j], t0, tev[k + j]);
            fprintf(stderr, "  %2zu: %7.3f %7.3f %7.3f %7.3f\n", k / 4, t[0], t[1], t[2], t[3]);
        }
        for (auto e : tev) cudaEventDestroy(e);
        cudaEventDestroy(t0);
    }
    return rc;
}

extern "C" int od_advect_current_host(od_ctx* ctx, const od_advect_args* a, const od_host_io* io) {
    if (!ctx || !a || !io) return fail(ctx, OD_ERR_ARG, "od_advect_current_host: null argument");
    return host_pipeline(ctx, a, nullptr, io);
}

// extras of the fused OceanDrift step (wind move, vertical advection, horizontal diffusion) into StepParams
static int fill_step(od_ctx* ctx, const od_step_args* a, StepParams* pp) {
    StepParams& p = *pp;
    int rc = fill_current(ctx, &a->cur, &p);
    if (rc) return rc;
    if (a->group_wind >= 0) {
        rc = need_group(ctx, a->group_wind, 2);
        if (rc) return rc;
        if (!a->d_wdf) return fail(ctx, OD_ERR_ARG, "wind drift needs wind_drift_factor");
        if (ctx->groups[a->group_wind].desc.nz != 1) return fail(ctx, OD_ERR_ARG, "wind group must be 2-D");
        p.wind_on = 1;
        p.wdf_f64 = a->wdf_f64;
        p.gwind = make_geom(ctx->groups[a->group_wind]);
        rc = resolve_pair(ctx, a->group_wind, a->t_wind, &p.pwind);
        if (rc) return rc;
        p.wdf = a->d_wdf;
        p.wind_drift_depth = a->wind_drift_depth;
        p.noise_wind = a->d_noise_wind;
    }
    if (a->group_w >= 0) {
        rc = need_group(ctx, a->group_w, 1);
        if (rc) return rc;
        if (!a->d_z_inout || !a->cur.d_z) return fail(ctx, OD_ERR_ARG, "vertical advection needs z");
        p.w_on = 1;
        p.w_at_surface = a->w_at_surface;
        p.gw = make_geom(ctx->groups[a->group_w]);
        rc = resolve_pair(ctx, a->group_w, a->t_w, &p.pw);
        if (rc) return rc;
        p.z_inout = a->d_z_inout;
        p.zio_f64 = a->z_inout_f64;
        // same reader block as the current (one grid, one level table): the kernel reuses the cell and the weights
        const Group& gu = ctx->groups[a->cur.group_uv];
        const Group& gw = ctx->groups[a->group_w];
        const od_group_desc &du = gu.desc, &dw = gw.desc;
        p.w_same_grid = du.nx == dw.nx && du.ny == dw.ny && du.nz == dw.nz && du.lon_mode == dw.lon_mode && du.wrap_x == dw.wrap_x && du.global_x == dw.global_x &&
                        du.x0 == dw.x0 && du.xspan == dw.xspan && du.y0 == dw.y0 && du.yspan == dw.yspan && du.xmin == dw.xmin &&
                        du.xmax == dw.xmax && du.ymin == dw.ymin && du.ymax == dw.ymax && gu.h_levels == gw.h_levels;
    }
    if (a->d_rand_x) {
        if (!a->d_rand_y) return fail(ctx, OD_ERR_ARG, "diffusion needs both random arrays");
        p.diff_on = 1;
        p.rand_x = a->d_rand_x; p.rand_y = a->d_rand_y;
        p.diffusivity = a->d_diffusivity;
        p.diffusivity_const = a->diffusivity_const;
    }
    return OD_OK;
}

extern "C" int od_step_oceandrift(od_ctx* ctx, const od_step_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_step_oceandrift: null argument");
    CK(cudaSetDevice(ctx->device));
    StepParams p;
    int rc = fill_step(ctx, a, &p);
    if (rc) return rc;
    if (a->cur.n == 0) return OD_OK;
    if (a->cur.fast < 0 || a->cur.fast > OD_MATH_SERIES) return fail(ctx, OD_ERR_ARG, "od_step_oceandrift: unknown arithmetic mode");
    // vertical advection only: the kernel variant without the wind / diffusion code (smaller instruction footprint)
    if (!p.wind_on && !p.diff_on) return launch_step_mode<2>(ctx, a->cur.fast, a->cur.scheme, a->cur.factor_f64 != 0, p);
    return launch_step_mode<1>(ctx, a->cur.fast, a->cur.scheme, a->cur.factor_f64 != 0, p);
}

// The fused step on HOST arrays (see od_advect_current_host): lon / lat / z in, lon / lat (/ z when vertical advection is
// on) out.  Per-particle device arrays of the step (factor, moving, wdf, diffusivity, random draws) are indexed like
// the host arrays.
extern "C" int od_step_oceandrift_host(od_ctx* ctx, const od_step_args* a, const od_host_io* io) {
    if (!ctx || !a || !io) return fail(ctx, OD_ERR_ARG, "od_step_oceandrift_host: null argument");
    if (a->d_noise_wind) return fail(ctx, OD_ERR_ARG, "od_step_oceandrift_host: noise arrays are not supported on the host path");
    if (a->group_w >= 0 && (!io->h_z || !io->h_out_z)) return fail(ctx, OD_ERR_ARG, "od_step_oceandrift_host: vertical advection needs h_z and h_out_z");
    return host_pipeline(ctx, &a->cur, a, io);
}

// ---- analytical reader on a projected plane (od_analytic.cuh) ---------------------------------------------
__global__ void __launch_bounds__(OD_BLOCK) analytic_interp_kernel(AnalyticReader R, double t, int64_t n, const double* __restrict__ lon,
                                                                  const double* __restrict__ lat, int pos_f32,
                                                                  float* __restrict__ u, float* __restrict__ v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float a, b;
    analytic_sample_raw(R, t, lon[i], lat[i], pos_f32 != 0, a, b);
    if (u) u[i] = a;
    if (v) v[i] = b;
}

static int make_analytic(od_ctx* ctx, const od_analytic_desc* r, AnalyticReader* R) {
    switch (analytic_from_desc(r, R)) {
        case 0: return OD_OK;
        case 1: return fail(ctx, OD_ERR_ARG, "unknown analytical reader kind");
        case 2: return fail(ctx, OD_ERR_ARG, "unknown projection kind");
        default: return fail(ctx, OD_ERR_ARG, "projection needs a > 0 and k_0 > 0");
    }
}

extern "C" int od_analytic_interp(od_ctx* ctx, const od_analytic_desc* r, double t_seconds, int64_t n, const double* lon,
                                  const double* lat, int flags, float* u, float* v) {
    if (!ctx || !r || n < 0 || (n > 0 && (!lon || !lat))) return fail(ctx, OD_ERR_ARG, "od_analytic_interp: bad arguments");
    AnalyticReader R;
    int rc = make_analytic(ctx, r, &R);
    if (rc) return rc;
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    analytic_interp_kernel<<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(R, t_seconds, n, lon, lat, flags & OD_INTERP_POS_F32, u, v);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_analytic_advect(od_ctx* ctx, const od_analytic_desc* r, const od_analytic_advect_args* a) {
    if (!ctx || !r || !a) return fail(ctx, OD_ERR_ARG, "od_analytic_advect: null argument");
    if (a->scheme < 0 || a->scheme > 2) return fail(ctx, OD_ERR_ARG, "unknown advection scheme");
    if (a->math < 0 || a->math > OD_MATH_SERIES) return fail(ctx, OD_ERR_ARG, "od_analytic_advect: unknown arithmetic mode");
    if (a->n < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat))) return fail(ctx, OD_ERR_ARG, "null particle arrays");
    if ((a->d_k1_u == nullptr) != (a->d_k1_v == nullptr)) return fail(ctx, OD_ERR_ARG, "k1 needs both components");
    AnalyticStepParams p;
    memset(&p, 0, sizeof(p));
    int rc = make_analytic(ctx, r, &p.R);
    if (rc) return rc;
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    p.t_start = a->t_start; p.t_mid = a->t_mid; p.t_end = a->t_end;
    p.dt = a->dt;
    p.dt32 = (float)a->dt;
    p.has_k1 = a->d_k1_u != nullptr;
    p.pos_f32 = a->pos_f32;
    p.n = a->n;
    p.lon = a->d_lon; p.lat = a->d_lat;
    p.factor = a->d_factor; p.moving = a->d_moving;
    p.k1u = a->d_k1_u; p.k1v = a->d_k1_v;
    p.env_u = a->d_env_u; p.env_v = a->d_env_v;
    // the analytical sampler has no float32 variant: OD_MATH_FAST keeps its float32 mid-point moves only
    if (a->math == OD_MATH_FAST) return launch_analytic<FastMath>(ctx, a->scheme, a->factor_f64 != 0, p);
    if (a->math == OD_MATH_SERIES) return launch_analytic<SeriesMath>(ctx, a->scheme, a->factor_f64 != 0, p);
    return launch_analytic<ExactMath>(ctx, a->scheme, a->factor_f64 != 0, p);
}

// ---- output buffer on the device (od_history.cuh) -----------------------------------------------------------
__global__ void __launch_bounds__(OD_BLOCK) history_scatter_kernel(const HistoryParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    history_scatter_one(p, i);
}

extern "C" int od_history_scatter(od_ctx* ctx, const od_history_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_history_scatter: null argument");
    if (a->n < 0 || a->n_total < 0 || a->ncols <= 0 || a->col < 0 || a->col >= a->ncols)
        return fail(ctx, OD_ERR_ARG, "od_history_scatter: bad sizes");
    if (a->n > 0 && (!a->d_ids || !a->d_lon || !a->d_lat || !a->d_z || !a->d_status || !a->d_buf_lon || !a->d_buf_lat ||
                     !a->d_buf_z || !a->d_buf_status))
        return fail(ctx, OD_ERR_ARG, "od_history_scatter: null arrays");
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    HistoryParams p;
    p.n = a->n; p.n_total = a->n_total; p.col = a->col; p.ncols = a->ncols; p.z_f64 = a->z_f64; p.pad_ = 0;
    p.ids = a->d_ids; p.lon = a->d_lon; p.lat = a->d_lat; p.z = a->d_z; p.status = a->d_status;
    p.blon = a->d_buf_lon; p.blat = a->d_buf_lat; p.bz = a->d_buf_z; p.bstatus = a->d_buf_status;
    history_scatter_kernel<<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

// ---- housekeeping (od_bookkeep.cuh) --------------------------------------------------------------------------
__global__ void __launch_bounds__(256) buoyancy_kernel(const BuoyancyParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool d = i < p.n && buoyancy_one(p, i);
    if (p.counter) tally_flags<1>(p.counter, d);
}

__global__ void __launch_bounds__(256) bookkeep_kernel(const BookkeepParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    tally_flags<3>(p.counters, i < p.n ? bookkeep_one(p, i) : 0);
}

static int counters(od_ctx* ctx) {
    if (!ctx->d_cnt) CK(cudaMalloc(&ctx->d_cnt, 4 * sizeof(unsigned)));
    CK(cudaMemsetAsync(ctx->d_cnt, 0, 4 * sizeof(unsigned), ctx->stream));
    return OD_OK;
}

// out[0..k) = the first k counters of the last housekeeping launch (synchronises)
static int read_counters(od_ctx* ctx, int k, int64_t* out) {
    unsigned c[4];
    CK(cudaMemcpyAsync(c, ctx->d_cnt, k * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int j = 0; j < k; ++j) out[j] = c[j];
    return OD_OK;
}

extern "C" int od_vertical_buoyancy(od_ctx* ctx, const od_buoyancy_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_vertical_buoyancy: null argument");
    if (a->n < 0 || (a->n > 0 && (!a->d_z_in || !a->d_z_out))) return fail(ctx, OD_ERR_ARG, "od_vertical_buoyancy: bad arguments");
    if (a->seafloor_code != 0 && (!a->d_status || !a->d_moving)) return fail(ctx, OD_ERR_ARG, "od_vertical_buoyancy: deactivation needs status and moving");
    if (a->h_n_deactivated) *a->h_n_deactivated = 0;
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    int rc = counters(ctx);
    if (rc) return rc;
    BuoyancyParams p;
    p.n = a->n; p.z_in = a->d_z_in; p.z_out = a->d_z_out; p.tv = a->d_terminal_velocity; p.sea_floor = a->d_sea_floor;
    p.status = a->d_status; p.moving = a->d_moving; p.counter = ctx->d_cnt; p.dt = a->dt; p.ssh = a->sea_surface_height;
    p.z_f64 = a->z_f64; p.tv_f64 = a->tv_f64; p.seafloor_code = a->seafloor_code;
    buoyancy_kernel<<<(unsigned)((a->n + 255) / 256), 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return a->h_n_deactivated ? read_counters(ctx, 1, a->h_n_deactivated) : OD_OK;
}

extern "C" int od_bookkeeping(od_ctx* ctx, const od_bookkeep_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_bookkeeping: null argument");
    if (a->n < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat || !a->d_age || !a->d_status || !a->d_moving)))
        return fail(ctx, OD_ERR_ARG, "od_bookkeeping: bad arguments");
    if (a->d_buf_lon && (!a->d_buf_lat || !a->d_buf_z || !a->d_buf_status || !a->d_ids || !a->d_z || a->ncols <= 0 || a->col < 0 ||
                         a->col >= a->ncols || a->n_total < 0))
        return fail(ctx, OD_ERR_ARG, "od_bookkeeping: bad output block");
    if (a->h_counts) a->h_counts[0] = a->h_counts[1] = a->h_counts[2] = 0;
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    int rc = counters(ctx);
    if (rc) return rc;
    BookkeepParams p;
    p.n = a->n; p.lon = a->d_lon; p.lat = a->d_lat; p.z = a->d_z; p.age = a->d_age; p.status = a->d_status; p.moving = a->d_moving;
    p.ids = a->d_ids; p.counters = ctx->d_cnt; p.dt_age = a->dt_age; p.max_age = a->max_age;
    p.west = a->west; p.east = a->east; p.south = a->south; p.north = a->north;
    p.outside_code = a->outside_code; p.retired_code = a->retired_code; p.z_f64 = a->z_f64; p.age_f64 = a->age_f64;
    p.pos_f32 = a->pos_f32; p.only_deactivated = a->only_deactivated;
    p.n_total = a->n_total; p.col = a->col; p.ncols = a->ncols;
    p.blon = a->d_buf_lon; p.blat = a->d_buf_lat; p.bz = a->d_buf_z; p.bstatus = a->d_buf_status;
    bookkeep_kernel<<<(unsigned)((a->n + 255) / 256), 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return a->h_counts ? read_counters(ctx, 3, a->h_counts) : OD_OK;
}

extern "C" int od_coastline(od_ctx* ctx, const od_coast_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_coastline: null argument");
    if (a->n < 0 || (a->n > 0 && (!a->d_mask || !a->d_lon || !a->d_lat || !a->d_status || !a->d_moving)))
        return fail(ctx, OD_ERR_ARG, "od_coastline: bad arguments");
    if (a->action < 1 || a->action > 3) return fail(ctx, OD_ERR_ARG, "od_coastline: action is 1 (stranding), 2 (previous) or 3 (sea floor: previous)");
    if (a->action == 3 && a->n > 0 && !a->d_z) return fail(ctx, OD_ERR_ARG, "od_coastline: the sea-floor action needs the depths");
    if (a->action >= 2 && a->n > 0 && (!a->d_ids || !a->d_prev_lon || !a->d_prev_lat || (a->check_seeded && !a->d_age)))
        return fail(ctx, OD_ERR_ARG, "od_coastline: 'previous' needs IDs, previous positions (and ages while elements are released)");
    if (a->h_counts) a->h_counts[0] = a->h_counts[1] = a->h_counts[2] = a->h_counts[3] = 0;
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    int rc = counters(ctx);
    if (rc) return rc;
    CoastParams p;
    p.n = a->n; p.mask = a->d_mask; p.lon = a->d_lon; p.lat = a->d_lat; p.z = a->d_z; p.age = a->d_age; p.status = a->d_status;
    p.moving = a->d_moving; p.ids = a->d_ids; p.prev_lon = a->d_prev_lon; p.prev_lat = a->d_prev_lat; p.counters = ctx->d_cnt;
    p.n_total = a->n_total; p.id_base = a->id_base; p.action = a->action; p.ssh = a->ssh; p.stranded_code = a->stranded_code;
    p.seeded_code = a->seeded_code; p.missing_code = a->missing_code; p.check_seeded = a->check_seeded; p.z_f64 = a->z_f64; p.age_f64 = a->age_f64;
    coast_kernel<<<(unsigned)((a->n + 255) / 256), 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return a->h_counts ? read_counters(ctx, 4, a->h_counts) : OD_OK;
}

extern "C" int od_store_previous(od_ctx* ctx, int64_t n, const double* lon, const double* lat, const int32_t* ids, int32_t id_base,
                                 int64_t n_total, float* prev_lon, float* prev_lat) {
    if (!ctx || n < 0 || (n > 0 && (!lon || !lat || !ids || !prev_lon || !prev_lat))) return fail(ctx, OD_ERR_ARG, "od_store_previous: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    store_previous_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(n, lon, lat, ids, id_base, n_total, prev_lon, prev_lat);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_store_previous_env(od_ctx* ctx, int64_t n, const float* present, const int32_t* ids, const void* age, int32_t age_f64,
                                     double dt, int32_t id_base, int64_t n_total, float* store, float* prev) {
    if (!ctx || n < 0 || n_total < 0 || (n > 0 && (!present || !ids || !store || !prev)))
        return fail(ctx, OD_ERR_ARG, "od_store_previous_env: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    StorePrevParams p;
    p.n = n; p.present = present; p.ids = ids; p.age = age; p.store = store; p.prev = prev; p.n_total = n_total; p.id_base = id_base;
    p.age_f64 = age_f64; p.dt = dt;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    // gather (and the positional writes) must be complete before the scatter overwrites the slots it reads: two launches
    store_prev_gather_kernel<<<blocks, 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    store_prev_scatter_kernel<<<blocks, 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return OD_OK;
}

extern "C" int od_vertical_advection_corrected(od_ctx* ctx, int64_t n, void* z, int32_t z_f64, const float* w, const float* ssh,
                                               const float* ssh_prev, const float* floor, float floor_const, const int32_t* moving,
                                               int32_t at_surface, double dt) {
    if (!ctx || n < 0 || (n > 0 && (!z || !w || !ssh || !ssh_prev || !moving)))
        return fail(ctx, OD_ERR_ARG, "od_vertical_advection_corrected: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    VadvCorrParams p;
    p.n = n; p.z = z; p.w = w; p.ssh = ssh; p.ssh_prev = ssh_prev; p.floor = floor; p.moving = moving; p.floor_const = floor_const;
    p.z_f64 = z_f64; p.at_surface = at_surface; p.dt = dt;
    vadv_corrected_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_leeway_step(od_ctx* ctx, const od_leeway_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_leeway_step: null argument");
    int rc = need_group(ctx, a->group_wind, 2);
    if (rc) return rc;
    rc = need_group(ctx, a->group_cur, 2);
    if (rc) return rc;
    if (ctx->groups[a->group_wind].desc.nz != 1 || ctx->groups[a->group_cur].desc.nz != 1)
        return fail(ctx, OD_ERR_ARG, "od_leeway_step: wind and surface current groups must be 2-D");
    if (a->n < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat || !a->d_dw_slope || !a->d_dw_offset || !a->d_dw_eps ||
                                  !a->d_cw_slope || !a->d_cw_offset || !a->d_cw_eps || !a->d_orientation || !a->d_jibe_probability)))
        return fail(ctx, OD_ERR_ARG, "od_leeway_step: bad arguments");
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    LeewayParams p;
    memset(&p, 0, sizeof(p));
    p.gwind = make_geom(ctx->groups[a->group_wind]);
    p.gcur = make_geom(ctx->groups[a->group_cur]);
    rc = resolve_pair(ctx, a->group_wind, a->t_wind, &p.pwind);
    if (rc) return rc;
    rc = resolve_pair(ctx, a->group_cur, a->t_cur, &p.pcur);
    if (rc) return rc;
    p.n = a->n; p.lon = a->d_lon; p.lat = a->d_lat;
    p.dw_slope = a->d_dw_slope; p.dw_offset = a->d_dw_offset; p.dw_eps = a->d_dw_eps;
    p.cw_slope = a->d_cw_slope; p.cw_offset = a->d_cw_offset; p.cw_eps = a->d_cw_eps;
    p.orientation = a->d_orientation; p.capsized = a->d_capsized; p.jibe_probability = a->d_jibe_probability;
    p.moving = a->d_moving; p.status = a->d_status; p.ids = a->d_ids; p.rand = a->d_rand; p.dt = a->dt; p.seed = a->seed;
    p.capsize_fraction = a->capsize_fraction; p.jp_f64 = a->jp_f64; p.pos_f32 = a->pos_f32; p.step_index = a->step_index;
    p.capsize_on = a->capsize_on; p.capsize_from = a->capsize_from; p.wind_threshold = a->wind_threshold;
    p.wind_sigma = a->wind_sigma; p.rand_capsize = a->d_rand_capsize;
    p.noise_cur = a->d_noise_cur; p.noise_wind = a->d_noise_wind; p.noise_kinds = a->noise_kinds;
    if (a->capsize_on && !a->d_capsized) return fail(ctx, OD_ERR_ARG, "od_leeway_step: capsizing needs the capsized array");
    p.missing_code = a->missing_code;
    if (p.gwind.proj_kind || p.gcur.proj_kind) leeway_kernel<true><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    else leeway_kernel<false><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_minmax_f32(od_ctx* ctx, int64_t n, const float* d_a, const float* d_b, float* h_min, float* h_max) {
    if (!ctx || n < 0 || (n > 0 && !d_a) || !h_min || !h_max) return fail(ctx, OD_ERR_ARG, "od_minmax_f32: bad arguments");
    *h_min = INFINITY;
    *h_max = -INFINITY;
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    if (!ctx->d_red) CK(cudaMalloc(&ctx->d_red, 2 * sizeof(unsigned)));
    const unsigned init[2] = {0xffffffffu, 0u};
    CK(cudaMemcpyAsync(ctx->d_red, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    int blocks = (int)((n + 255) / 256);
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    minmax_kernel<<<blocks, 256, 0, ctx->stream>>>(n, d_a, d_b, ctx->d_red);
    CK(cudaGetLastError());
    ctx->launches++;
    unsigned res[2];
    CK(cudaMemcpyAsync(res, ctx->d_red, sizeof(res), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (res[0] != 0xffffffffu) {
        *h_min = ord2f(res[0]);
        *h_max = ord2f(res[1]);
    }
    return OD_OK;
}

extern "C" int od_stokes_drift(od_ctx* ctx, const od_stokes_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_stokes_drift: null argument");
    if (a->n < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat || !a->d_z || !a->d_us || !a->d_vs)))
        return fail(ctx, OD_ERR_ARG, "od_stokes_drift: bad arguments");
    if (a->hs_mode < 0 || a->hs_mode > 2 || a->profile < 0 || a->profile > 3 || (a->hs_mode == 0 && !a->d_hs && a->profile != 3))
        return fail(ctx, OD_ERR_ARG, "od_stokes_drift: bad mode");
    if (a->profile == 3 && (!a->d_swell_dir || !a->d_swell_period || !a->d_swell_hs || !a->d_windsea_dir || !a->d_windsea_period ||
                            !a->d_windsea_hs))
        return fail(ctx, OD_ERR_ARG, "od_stokes_drift: the windsea_swell profile needs the six swell / wind-sea arrays");
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    StokesParams p;
    memset(&p, 0, sizeof(p));
    p.n = a->n; p.lon = a->d_lon; p.lat = a->d_lat; p.z = a->d_z; p.us = a->d_us; p.vs = a->d_vs; p.hs = a->d_hs;
    p.xwind = a->d_xwind; p.ywind = a->d_ywind; p.moving = a->d_moving; p.dt = a->dt;
    p.z_f64 = a->z_f64; p.hs_mode = a->hs_mode; p.profile = a->profile;
    p.factor = a->factor; p.factor_arr = a->d_factor; p.factor_f64 = a->factor_f64;
    p.sw_dir = a->d_swell_dir; p.sw_period = a->d_swell_period; p.sw_hs = a->d_swell_hs;
    p.ws_dir = a->d_windsea_dir; p.ws_period = a->d_windsea_period; p.ws_hs = a->d_windsea_hs;
    stokes_kernel<<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_stokes_parameterised(od_ctx* ctx, int64_t n, const float* xwind, const float* ywind, const double* wf_coef,
                                       int32_t n_wf, const double* hs_coef, int32_t n_hs, float* us, float* vs, float* hs) {
    if (!ctx || n < 0 || (!us) != (!vs) || (!us && !hs) || (n > 0 && (!xwind || !ywind)))
        return fail(ctx, OD_ERR_ARG, "od_stokes_parameterised: bad arguments");
    if ((us && (!wf_coef || n_wf < 1 || n_wf > OD_TAB_MAX_COEF)) || (hs && (!hs_coef || n_hs < 1 || n_hs > OD_TAB_MAX_COEF)))
        return fail(ctx, OD_ERR_ARG, "od_stokes_parameterised: 1 to 8 coefficients per polynomial");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    StokesTabParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.xwind = xwind; p.ywind = ywind; p.us = us; p.vs = vs; p.hs = hs;
    if (us) { p.n_wf = n_wf; memcpy(p.wf, wf_coef, sizeof(double) * n_wf); }
    if (hs) { p.n_hs = n_hs; memcpy(p.hsc, hs_coef, sizeof(double) * n_hs); }
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    stokes_tab_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

// od_vertical_mixing, and with st its settling variant (od_vertical_mixing_settle)
static int mix_launch(od_ctx* ctx, const od_mix_args* a, const SettleParams* st, int64_t* h_undecided) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: null argument");
    if (a->n < 0 || a->ntimes < 0 || (a->n > 0 && (!a->d_lon || !a->d_lat || !a->d_z_in || !a->d_z_out)))
        return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: bad arguments");
    if (a->model < OD_MIX_ENVIRONMENT || a->model > OD_MIX_CONSTANT) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: unknown diffusivity model");
    MixParams p;
    memset(&p, 0, sizeof(p));
    if (a->model == OD_MIX_ENVIRONMENT) {
        int rc = need_group(ctx, a->group_k, 1);
        if (rc) return rc;
        const Group& g = ctx->groups[a->group_k];
        if (g.desc.nz < 2) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: the diffusivity group must be 3-D");
        if (a->n == 0) return OD_OK;
        CK(cudaSetDevice(ctx->device));
        p.g = make_geom(g);
        rc = resolve_pair(ctx, a->group_k, a->t_k, &p.pr);
        if (rc) return rc;
        p.zl = g.d_zl; p.xs = g.d_mxs; p.xy = g.d_mxy;
        const std::vector<double>& lv = g.h_levels;
        p.uniform_dz = 1;
        p.dz0 = lv[1] - lv[0];
        for (size_t k = 1; k + 1 < lv.size(); ++k)
            if (lv[k + 1] - lv[k] != p.dz0) p.uniform_dz = 0;
    } else {
        if (a->nlev < 2 || a->nlev > 65535) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: analytical models need 2 <= nlev <= 65535");
        if (a->model != OD_MIX_CONSTANT && !a->d_wind_speed) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: wind speed array missing");
        if (a->n == 0) return OD_OK;
        CK(cudaSetDevice(ctx->device));
        p.g.nz = a->nlev;
        p.uniform_dz = 1;
        p.dz0 = -1.0;                       // mixing_z = -arange(nlev)
        p.wind_speed = a->d_wind_speed; p.mld = a->d_mld; p.mld_const = (float)a->mld_const;
        p.background = a->background; p.k_const = a->k_const;
    }
    p.model = a->model;
    p.n = a->n; p.lon = a->d_lon; p.lat = a->d_lat; p.z_in = a->d_z_in; p.z_out = a->d_z_out;
    p.moving = a->d_moving; p.terminal_velocity = a->d_terminal_velocity; p.ids = a->d_ids; p.rand = a->d_rand;
    p.dt_mix = a->dt_mix; p.zmin_const = -(double)(float)a->sea_floor_const; p.sea_floor = a->d_sea_floor;
    p.seed = a->seed; p.ntimes = a->ntimes; p.z_in_f64 = a->z_in_f64; p.tv_f64 = a->tv_f64;
    p.mix_at_surface = a->mix_at_surface; p.pos_f32 = a->pos_f32; p.step_index = a->step_index;
    p.seafloor_action = a->seafloor_action; p.seafloor_code = a->seafloor_code; p.status = a->d_status; p.moving_out = a->d_moving_out;
    p.iter0 = a->iter0; p.skip_surface_stick = a->skip_surface_stick;
    if (a->h_n_deactivated) *a->h_n_deactivated = 0;
    if (a->seafloor_action < 0 || a->seafloor_action > 2 || (a->seafloor_action == 2 && (!a->d_status || !(st ? st->status_out : a->d_moving_out))))
        return fail(ctx, OD_ERR_ARG, "od_vertical_mixing: bad sea-floor action");
    if (a->seafloor_action == 2 || st) {
        int rc = counters(ctx);
        if (rc) return rc;
        p.counter = ctx->d_cnt;
    }
    if (st) {
        SettleParams s = *st;
        s.undecided = ctx->d_cnt + 1;
        if (p.g.proj_kind) mix_settle_kernel<true><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p, s);
        else mix_settle_kernel<false><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p, s);
    } else if (p.g.proj_kind) {
        mix_kernel<true><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    } else {
        mix_kernel<false><<<grid_for(a->n), OD_BLOCK, 0, ctx->stream>>>(p);
    }
    CK(cudaGetLastError());
    ctx->launches++;
    if (st) {                                        // one read of both counters
        int64_t c[2];
        int rc = read_counters(ctx, 2, c);
        if (rc) return rc;
        if (a->h_n_deactivated) *a->h_n_deactivated = a->seafloor_action == 2 ? c[0] : 0;
        *h_undecided = c[1];
        return OD_OK;
    }
    return a->seafloor_action == 2 && a->h_n_deactivated ? read_counters(ctx, 1, a->h_n_deactivated) : OD_OK;
}

extern "C" int od_vertical_mixing(od_ctx* ctx, const od_mix_args* a) {
    return mix_launch(ctx, a, nullptr, nullptr);
}

extern "C" int od_vertical_mixing_settle(od_ctx* ctx, const od_mix_args* a, int32_t* d_moving_out, int32_t* d_status_out,
                                         int64_t* h_undecided) {
    if (!h_undecided || (a && a->n > 0 && !d_moving_out)) return fail(ctx, OD_ERR_ARG, "od_vertical_mixing_settle: bad arguments");
    *h_undecided = 0;
    SettleParams st;
    st.moving_out = d_moving_out;
    st.status_out = a && a->seafloor_action == 2 ? d_status_out : nullptr;
    st.undecided = nullptr;
    return mix_launch(ctx, a, &st, h_undecided);
}

extern "C" int od_resuspend(od_ctx* ctx, int64_t n, const float* u, const float* v, float threshold, int32_t* moving, void* z,
                            int32_t z_f64) {
    if (!ctx || n < 0 || (n > 0 && (!u || !v || !moving || !z))) return fail(ctx, OD_ERR_ARG, "od_resuspend: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    resuspend_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(n, u, v, threshold, moving, z, z_f64);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_ship_step(od_ctx* ctx, int64_t n, double* lon, double* lat, int32_t* moving, int32_t* status, const float* const* el,
                            const uint8_t* orientation, float* const* env, const double* wtab, const int32_t* wbox, int32_t nomega,
                            int32_t nbeam, int32_t ndraft, int32_t hs_wind, int32_t tm_wind, int32_t tm_fill_on, float tm_fill,
                            int32_t strand_code, double dt, int32_t* h_stranded) {
    if (!ctx || n < 0 || !el || !env || !h_stranded || nomega < 2 || nbeam < 2 || ndraft < 2)
        return fail(ctx, OD_ERR_ARG, "od_ship_step: bad arguments");
    *h_stranded = 0;
    if (n == 0) return OD_OK;
    if (!lon || !lat || !orientation || !wtab || !wbox || !env[0] || !env[1] || !env[2] || !env[3] || !env[4] || !env[5] ||
        (!env[6]) != (!env[7]) || (env[8] && !status))
        return fail(ctx, OD_ERR_ARG, "od_ship_step: bad arguments");
    for (int k = 0; k < 6; ++k)
        if (!el[k]) return fail(ctx, OD_ERR_ARG, "od_ship_step: null element array");
    CK(cudaSetDevice(ctx->device));
    ShipParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.lon = lon; p.lat = lat; p.moving = moving; p.status = status;
    p.length = el[0]; p.height = el[1]; p.draft = el[2]; p.beam = el[3]; p.cf = el[4]; p.cd = el[5];
    p.orientation = orientation;
    p.cu = env[0]; p.cv = env[1]; p.xw = env[2]; p.yw = env[3]; p.hs = env[4]; p.tm = env[5]; p.sx = env[6]; p.sy = env[7];
    p.mask = env[8];
    p.wtab = wtab; p.wbox = wbox; p.nomega = nomega; p.nbeam = nbeam; p.ndraft = ndraft;
    p.hs_wind = hs_wind; p.tm_wind = tm_wind; p.tm_fill_on = tm_fill_on; p.tm_fill = tm_fill; p.strand_code = strand_code;
    p.dt = dt;
    if (p.mask) {
        if (!ctx->d_red) CK(cudaMalloc(&ctx->d_red, 2 * sizeof(unsigned)));
        CK(cudaMemsetAsync(ctx->d_red, 0, sizeof(unsigned), ctx->stream));
        p.stranded = ctx->d_red;
    }
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    ship_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    if (p.mask) {
        unsigned flag = 0;
        CK(cudaMemcpyAsync(&flag, ctx->d_red, sizeof(flag), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *h_stranded = flag ? 1 : 0;
    }
    return OD_OK;
}

extern "C" int od_plast_step(od_ctx* ctx, int64_t n, double* lon, double* lat, const int32_t* moving, const void* z_in, int32_t z_f64,
                             double* z_out, const float* k, const void* tv, int32_t tv_f64, const double* rand, const int32_t* ids,
                             unsigned long long seed, int32_t step_index, const float* const* stokes, int32_t hs_mode, int32_t profile,
                             const float* xwind, const float* ywind, const void* wdf, int32_t wdf_f64, double wind_drift_depth, double dt,
                             int32_t* h_negative) {
    if (!ctx || n < 0 || !h_negative) return fail(ctx, OD_ERR_ARG, "od_plast_step: bad arguments");
    *h_negative = 0;
    if (stokes && (hs_mode < 0 || hs_mode > 2 || profile < 0 || profile > 3))
        return fail(ctx, OD_ERR_ARG, "od_plast_step: bad Stokes mode");
    if (n == 0) return OD_OK;
    if (!lon || !lat || (!z_out && !z_in) || (z_out && (!k || !tv)) || (wdf && (!xwind || !ywind)) ||
        (stokes && (!stokes[0] || !stokes[1] || (hs_mode == 0 && profile != 3 && !stokes[2]))))
        return fail(ctx, OD_ERR_ARG, "od_plast_step: bad arguments");
    if (stokes && profile == 3)
        for (int j = 5; j < 11; ++j)
            if (!stokes[j]) return fail(ctx, OD_ERR_ARG, "od_plast_step: the windsea_swell profile needs the six swell / wind-sea arrays");
    CK(cudaSetDevice(ctx->device));
    PlastParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.lon = lon; p.lat = lat; p.moving = moving; p.z_in = z_in; p.z_f64 = z_f64; p.z_out = z_out;
    p.k = k; p.tv = tv; p.tv_f64 = tv_f64; p.rand = rand; p.ids = ids; p.seed = seed; p.step_index = step_index;
    if (stokes) {
        p.stokes_on = 1;
        p.st.us = stokes[0]; p.st.vs = stokes[1]; p.st.hs = stokes[2]; p.st.xwind = stokes[3]; p.st.ywind = stokes[4];
        p.st.sw_dir = stokes[5]; p.st.sw_period = stokes[6]; p.st.sw_hs = stokes[7];
        p.st.ws_dir = stokes[8]; p.st.ws_period = stokes[9]; p.st.ws_hs = stokes[10];
        p.st.hs_mode = hs_mode; p.st.profile = profile; p.st.factor = 1.0;
    }
    if (wdf) {
        p.wind_on = 1;
        p.xwind = xwind; p.ywind = ywind; p.wdf = wdf; p.wdf_f64 = wdf_f64; p.wdd = fabs(wind_drift_depth);
    }
    p.dt = dt;
    if (z_out) {
        if (!ctx->d_red) CK(cudaMalloc(&ctx->d_red, 2 * sizeof(unsigned)));
        CK(cudaMemsetAsync(ctx->d_red, 0, sizeof(unsigned), ctx->stream));
        p.negative = ctx->d_red;
    }
    int64_t blocks = (n + OD_BLOCK - 1) / OD_BLOCK;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    plast_kernel<<<(unsigned)blocks, OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    if (z_out) {
        unsigned flag = 0;
        CK(cudaMemcpyAsync(&flag, ctx->d_red, sizeof(flag), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *h_negative = flag ? 1 : 0;
    }
    return OD_OK;
}

extern "C" int od_larval_develop(od_ctx* ctx, int64_t n, const float* t, const float* s, void* hatched, int32_t hatched_f64,
                                 void* stage, int32_t stage_f64, void* weight, int32_t weight_f64, void* length, int32_t length_f64,
                                 const void* diameter, int32_t diameter_f64, const void* nbs, int32_t nbs_f64, int32_t develop,
                                 void* w_out, double dt, int32_t* h_flags) {
    if (!ctx || n < 0) return fail(ctx, OD_ERR_ARG, "od_larval_develop: bad arguments");
    if (h_flags) *h_flags = 0;
    if (n == 0) return OD_OK;
    if (!t || (develop && (!hatched || !stage || !weight || !length)) || (w_out && (!s || !diameter || !nbs)))
        return fail(ctx, OD_ERR_ARG, "od_larval_develop: bad arguments");
    CK(cudaSetDevice(ctx->device));
    LarvalParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.t = t; p.s = s; p.hatched = hatched; p.stage = stage; p.weight = weight; p.length = length;
    p.diameter = diameter; p.nbs = nbs; p.w_out = w_out; p.develop = develop; p.dt = dt;
    p.hatched_f64 = hatched_f64; p.stage_f64 = stage_f64; p.weight_f64 = weight_f64; p.length_f64 = length_f64;
    p.diameter_f64 = diameter_f64; p.nbs_f64 = nbs_f64;
    unsigned* flags = nullptr;
    if (h_flags) {
        if (!ctx->d_red) CK(cudaMalloc(&ctx->d_red, 2 * sizeof(unsigned)));
        CK(cudaMemsetAsync(ctx->d_red, 0, sizeof(unsigned), ctx->stream));
        flags = ctx->d_red;
    }
    int64_t blocks = (n + OD_BLOCK - 1) / OD_BLOCK;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    larval_develop_kernel<<<(unsigned)blocks, OD_BLOCK, 0, ctx->stream>>>(p, flags);
    CK(cudaGetLastError());
    ctx->launches++;
    if (h_flags) {
        unsigned f = 0;
        CK(cudaMemcpyAsync(&f, ctx->d_red, sizeof(f), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *h_flags = (int32_t)f;
    }
    return OD_OK;
}

extern "C" int od_larval_migrate(od_ctx* ctx, int64_t n, const void* hatched, int32_t hatched_f64, const void* length,
                                 int32_t length_f64, void* z, int32_t z_f64, double fraction, double direction, double dt) {
    if (!ctx || n < 0 || (n > 0 && (!hatched || !length || !z))) return fail(ctx, OD_ERR_ARG, "od_larval_migrate: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    LarvalParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.hatched = (void*)hatched; p.hatched_f64 = hatched_f64; p.length = (void*)length; p.length_f64 = length_f64;
    p.z = z; p.z_f64 = z_f64; p.swim = fraction; p.dir = direction; p.dt = dt;
    int64_t blocks = (n + OD_BLOCK - 1) / OD_BLOCK;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    larval_migrate_kernel<<<(unsigned)blocks, OD_BLOCK, 0, ctx->stream>>>(p);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_sort_by_cell(od_ctx* ctx, int group, int64_t n, const double* lon, const double* lat, const float* z,
                               int32_t* perm) {
    int rc = need_group(ctx, group, 0);
    if (rc) return rc;
    if (n < 0 || n >= (1ll << 31) || (n > 0 && (!lon || !lat || !perm))) return fail(ctx, OD_ERR_ARG, "od_sort_by_cell: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    const Group& g = ctx->groups[group];
    SortParams p;
    p.g = make_geom(g);
    p.n = n; p.lon = lon; p.lat = lat; p.z = z;
    p.tile = 4;
    p.ntx = (g.desc.nx + p.tile - 1) / p.tile;
    p.nty = (g.desc.ny + p.tile - 1) / p.tile;
    const int64_t nbins = 1 + (int64_t)p.ntx * p.nty * g.desc.nz;
    if (nbins >= (1ll << 30)) return fail(ctx, OD_ERR_ARG, "od_sort_by_cell: too many bins");
    rc = grow(ctx, (void**)&ctx->d_keys, &ctx->keys_cap, n, sizeof(int32_t));
    if (rc) return rc;
    rc = grow(ctx, (void**)&ctx->d_bins, &ctx->bins_cap, nbins, sizeof(int32_t));
    if (rc) return rc;
    CK(cudaMemsetAsync(ctx->d_bins, 0, nbins * sizeof(int32_t), ctx->stream));
    if (p.g.proj_kind) cell_key_kernel<true><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(p, ctx->d_keys, ctx->d_bins);
    else cell_key_kernel<false><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(p, ctx->d_keys, ctx->d_bins);
    rc = scan_exclusive(ctx, ctx->d_bins, (int)nbins);
    if (rc) return rc;
    scatter_perm_kernel<<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, ctx->d_keys, ctx->d_bins, perm);
    CK(cudaGetLastError());
    ctx->launches += 2;
    return OD_OK;
}

extern "C" int od_partition_active(od_ctx* ctx, int64_t n, const int32_t* d_status, int32_t* d_perm, int64_t* h_n_keep) {
    if (!ctx || n < 0 || n >= (1ll << 31) || (n > 0 && (!d_status || !d_perm)) || !h_n_keep)
        return fail(ctx, OD_ERR_ARG, "od_partition_active: bad arguments");
    *h_n_keep = 0;
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    const int nblocks = (int)((n + OD_PART_BLOCK - 1) / OD_PART_BLOCK);
    int rc = grow(ctx, (void**)&ctx->d_bins, &ctx->bins_cap, nblocks + 1, sizeof(int32_t));
    if (rc) return rc;
    CK(cudaMemsetAsync(ctx->d_bins + nblocks, 0, sizeof(int32_t), ctx->stream));
    partition_count_kernel<<<nblocks, OD_PART_BLOCK, 0, ctx->stream>>>(n, d_status, ctx->d_bins);
    rc = scan_exclusive(ctx, ctx->d_bins, nblocks + 1);                            // exclusive; last entry = total
    if (rc) return rc;
    int32_t total = 0;
    CK(cudaMemcpyAsync(&total, ctx->d_bins + nblocks, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    partition_scatter_kernel<<<nblocks, OD_PART_BLOCK, 0, ctx->stream>>>(n, d_status, ctx->d_bins, (int64_t)total, d_perm);
    CK(cudaGetLastError());
    ctx->launches += 2;
    *h_n_keep = total;
    return OD_OK;
}

static int permute_impl(od_ctx* ctx, int64_t n, const int32_t* perm, const void* src, void* dst, int es, int inverse) {
    if (!ctx || n < 0 || (n > 0 && (!perm || !src || !dst)) || src == dst) return fail(ctx, OD_ERR_ARG, "od_permute: bad arguments");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    if (es == 4) permute_kernel<uint32_t><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, perm, (const uint32_t*)src, (uint32_t*)dst, inverse);
    else if (es == 8) permute_kernel<uint64_t><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, perm, (const uint64_t*)src, (uint64_t*)dst, inverse);
    else if (es == 1) permute_kernel<uint8_t><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, perm, (const uint8_t*)src, (uint8_t*)dst, inverse);
    else if (es == 2) permute_kernel<uint16_t><<<grid_for(n), OD_BLOCK, 0, ctx->stream>>>(n, perm, (const uint16_t*)src, (uint16_t*)dst, inverse);
    else return fail(ctx, OD_ERR_ARG, "od_permute: element size must be 1, 2, 4 or 8");
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}

extern "C" int od_permute(od_ctx* ctx, int64_t n, const int32_t* perm, const void* src, void* dst, int es) {
    return permute_impl(ctx, n, perm, src, dst, es, 0);
}

extern "C" int od_unpermute(od_ctx* ctx, int64_t n, const int32_t* perm, const void* src, void* dst, int es) {
    return permute_impl(ctx, n, perm, src, dst, es, 1);
}


// ---- od_pack_by_owner / od_unpack_records --------------------------------------------------------------------------------------
static int pack_layout(int ncols, const int32_t* col_bytes, int* off, int* rec_bytes) {
    int o = 0;
    for (int c = 0; c < ncols; ++c) {
        if (col_bytes[c] < 1 || col_bytes[c] > 64) return -1;
        off[c] = o;
        o += col_bytes[c];
    }
    *rec_bytes = o;
    return 0;
}

extern "C" int od_pack_by_owner(od_ctx* ctx, const od_pack_args* a) {
    if (!ctx || !a) return fail(ctx, OD_ERR_ARG, "od_pack_by_owner: null argument");
    if (a->n < 0 || a->n >= (1ll << 31) || a->world < 1 || a->world > OD_PACK_MAX_WORLD || a->ncols < 1 || a->ncols > OD_PACK_MAX_COLS ||
        !a->h_bounds || !a->h_counts || (a->n > 0 && (!a->d_lon || !a->d_records)))
        return fail(ctx, OD_ERR_ARG, "od_pack_by_owner: bad arguments");
    PackParams p;
    memset(&p, 0, sizeof(p));
    if (pack_layout(a->ncols, a->col_bytes, p.col_off, &p.rec_bytes) || p.rec_bytes != a->rec_bytes)
        return fail(ctx, OD_ERR_ARG, "od_pack_by_owner: record layout does not match the column widths");
    for (int r = 0; r < a->world; ++r) a->h_counts[r] = 0;
    if (a->n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    p.n = a->n; p.lon = a->d_lon; p.world = a->world; p.ncols = a->ncols;
    for (int k = 0; k <= a->world; ++k) p.bounds[k] = a->h_bounds[k];
    for (int c = 0; c < a->ncols; ++c) {
        if (!a->d_cols[c]) return fail(ctx, OD_ERR_ARG, "od_pack_by_owner: null column");
        p.cols[c] = (const unsigned char*)a->d_cols[c];
        p.col_bytes[c] = a->col_bytes[c];
    }
    p.nblocks = (int)((a->n + OD_PACK_BLOCK - 1) / OD_PACK_BLOCK);
    const int64_t nbins = (int64_t)p.nblocks * a->world + 1;           // (+1: the grand total lands behind the table)
    int rc = grow(ctx, (void**)&ctx->d_bins, &ctx->bins_cap, nbins, sizeof(int32_t));
    if (rc) return rc;
    CK(cudaMemsetAsync(ctx->d_bins + (nbins - 1), 0, sizeof(int32_t), ctx->stream));
    owner_count_kernel<<<p.nblocks, OD_PACK_BLOCK, 0, ctx->stream>>>(p, ctx->d_bins);
    ctx->launches++;
    rc = scan_exclusive(ctx, ctx->d_bins, (int)nbins);
    if (rc) return rc;
    owner_pack_kernel<<<p.nblocks, OD_PACK_BLOCK, 0, ctx->stream>>>(p, ctx->d_bins, (unsigned char*)a->d_records, a->d_perm);
    CK(cudaGetLastError());
    ctx->launches++;
    // first row of every owner (+ the total) -> counts
    std::vector<int32_t> first(a->world + 1);
    for (int r = 0; r <= a->world; ++r)
        CK(cudaMemcpyAsync(&first[r], ctx->d_bins + (int64_t)r * p.nblocks, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int r = 0; r < a->world; ++r) a->h_counts[r] = (int64_t)first[r + 1] - first[r];
    return OD_OK;
}

extern "C" int od_unpack_records(od_ctx* ctx, int64_t n, const void* d_records, int32_t ncols, void* const* d_cols, const int32_t* col_bytes,
                                 int32_t rec_bytes) {
    if (!ctx || n < 0 || ncols < 1 || ncols > OD_PACK_MAX_COLS || !d_cols || !col_bytes || (n > 0 && !d_records))
        return fail(ctx, OD_ERR_ARG, "od_unpack_records: bad arguments");
    UnpackParams p;
    memset(&p, 0, sizeof(p));
    if (pack_layout(ncols, col_bytes, p.col_off, &p.rec_bytes) || p.rec_bytes != rec_bytes)
        return fail(ctx, OD_ERR_ARG, "od_unpack_records: record layout does not match the column widths");
    if (n == 0) return OD_OK;
    CK(cudaSetDevice(ctx->device));
    p.n = n; p.ncols = ncols;
    for (int c = 0; c < ncols; ++c) {
        if (!d_cols[c]) return fail(ctx, OD_ERR_ARG, "od_unpack_records: null column");
        p.cols[c] = (unsigned char*)d_cols[c];
        p.col_bytes[c] = col_bytes[c];
    }
    unpack_records_kernel<<<(unsigned)((n + OD_PACK_BLOCK - 1) / OD_PACK_BLOCK), OD_PACK_BLOCK, 0, ctx->stream>>>(p, (const unsigned char*)d_records);
    CK(cudaGetLastError());
    ctx->launches++;
    return OD_OK;
}
