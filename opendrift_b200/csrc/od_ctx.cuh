// od_ctx.cuh -- the library context (od_ctx), its field groups and the launch helpers shared by the translation units of
// libodcuda.so: od_kernels.cu (C-ABI, housekeeping kernels) and od_step.cu (the step kernels, one object per arithmetic mode).
#pragma once
#include <cuda.h>            // CUtensorMap types only; the encoder is fetched with cudaGetDriverEntryPoint
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/odcuda.h"
#include "od_advect.cuh"
#include "od_analytic.cuh"

using namespace od;

#define OD_PAIR_CACHE 4
// Launch shape of the step kernel: 128-thread blocks, at least 8 resident blocks per SM (64 registers, 32 warps/SM).
#ifndef OD_BLOCK
#define OD_BLOCK 128
#endif
#ifndef OD_STEP_MINB
#define OD_STEP_MINB 8
#endif
// The specialised step kernel (od_spec.cuh) at 6 blocks per SM: 80 registers, 24 warps/SM.  At 8 blocks (64 registers) it
// spilled 132-176 B per thread; with the wind move (EXTRAS = 1) it took 20 % longer, and steps that start or end on a reader
// time 3-7 % longer (DESIGN.md §5).
#ifndef OD_SPEC_MINB
#define OD_SPEC_MINB 6
#endif

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
// Box of pair texels one thread block stages in shared memory (TMA).  Particles are sorted by (layer, 4x4-cell
// tile), so the 128 particles of a block typically sit in ~10 neighbouring tiles of one tile row: 48 x 8 cells
// (4-cell tile + 2-cell halo on each side for the RK stage excursions) x 2 layers = 12 KB.
#define OD_TILE_BX 48
#define OD_TILE_BY 8
#define OD_TILE_BZ 2
#define OD_TILE_HALO 2

struct PairEntry {
    CUtensorMap tmap;            // 4-D tiled view {4 floats, nx, ny, nz} of tex (valid when tmap_ok)
    bool tmap_ok = false;
    float* tex = nullptr;
    int slot_a = -1, slot_b = -1;
    uint64_t ver_a = 0, ver_b = 0;
    uint64_t last_use = 0;
    // built ahead on another stream (od_group_prepare_pair): `ready` marks the end of the build, and a launch that reads or
    // rebuilds the entry orders its stream behind it while `pending` is set
    cudaEvent_t ready = nullptr;
    bool pending = false;
};

struct Group {
    bool defined = false;
    od_group_desc desc;
    std::vector<float*> slots;          // [n_slots * ncomp] raw slabs [nz][ny][nx]
    std::vector<uint64_t> version;      // [n_slots]
    double* d_zs = nullptr;             // increasing level depths
    double* d_zy = nullptr;             // their layer indices
    double* d_zl = nullptr;             // levels as the reader gives them (mixing_z)
    double* d_mxs = nullptr;            // -levels sorted increasing (interp1d of vertical mixing)
    double* d_mxy = nullptr;            // their layer indices
    std::vector<double> h_levels;
    double zmin = 0, zmax = 0;
    PairEntry pairs[OD_PAIR_CACHE];
    size_t capacity = 0;                // cells every slot was allocated for (the group's full grid)
    size_t cells() const { return (size_t)desc.nx * desc.ny * desc.nz; }
};

struct od_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    Group groups[OD_MAX_GROUPS];
    int64_t launches = 0;
    uint64_t tick = 0;
    int sm_count = 0;
    // sort scratch
    int32_t* d_keys = nullptr;
    int32_t* d_bins = nullptr;
    int64_t keys_cap = 0, bins_cap = 0;
    int32_t* d_tilesums = nullptr;      // tile totals of the two-level scan
    int64_t tiles_cap = 0;
    unsigned* d_red = nullptr;          // reduction scratch
    unsigned long long* d_bbox = nullptr;   // od_bbox's four extrema
    unsigned* d_cnt = nullptr;          // counters of the housekeeping kernels
    float* d_fill = nullptr;            // scratch slab of the NaN fill
    unsigned* d_fillcnt = nullptr;      // per-pass missing-cell counters
    int coop_fill_blocks = -1;          // co-resident grid of fill_nan_coop_kernel (0: the device cannot launch it)
    int64_t fill_cap = 0;
    int tile = 0;                       // OD_OPT_TILE: stage field boxes in shared memory with TMA
    int spec = 1;                       // OD_OPT_SPEC: launches that qualify take the specialised step kernel (od_spec.cuh)
    // host-array pipeline (od_advect_current_host): three streams, three staging buffers back to back in hbuf
    cudaStream_t hstream[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t hready = nullptr;
    char* hbuf = nullptr;
    int64_t hbuf_cap = 0;               // particles per staging buffer (24 bytes each)
};

static inline int fail(od_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
    if (c) {
        c->err = what;
        if (e != cudaSuccess) {
            c->err += ": ";
            c->err += cudaGetErrorString(e);
        }
    }
    return code;
}

#define CK(call)                                                         \
    do {                                                                 \
        cudaError_t e_ = (call);                                         \
        if (e_ != cudaSuccess) return fail(ctx, OD_ERR_CUDA, #call, e_); \
    } while (0)

static inline int grid_for(int64_t n) { return (int)((n + OD_BLOCK - 1) / OD_BLOCK); }

// Level table of a group staged in shared memory (the vertical search is data dependent).
struct LevelsSmem {
    double zs[OD_MAX_LEVELS];
    double zy[OD_MAX_LEVELS];
};

__device__ __forceinline__ void load_levels(LevelsSmem& s, const GroupGeom& g) {
    for (int i = threadIdx.x; i < g.nz; i += blockDim.x) {
        s.zs[i] = g.zs[i];
        s.zy[i] = g.zy[i];
    }
}

// Launchers of the step kernels, defined in od_step.cu and instantiated there for one arithmetic mode (MATH) per object.
template <int EXTRAS, class MATH>
int launch_step(od_ctx* ctx, int scheme, bool f64, const StepParams& p);
template <int EXTRAS, class MATH>
int launch_step_tiled(od_ctx* ctx, int scheme, bool f64, const StepParams& p, const PairEntry* pe);
template <class MATH>
int launch_analytic(od_ctx* ctx, int scheme, bool f64, const AnalyticStepParams& p);
