// Host build of csrc/od_sealevel.cuh for the CPU tests (tests/sealevel_host.py): the same per-element functions the device
// kernels run, one loop per launch.  Compiled with -ffp-contract=off, as the device build rounds every operation on its own.
#include <stdint.h>
#include "../../opendrift_b200/csrc/od_sealevel.cuh"

using namespace od;

extern "C" {

int hs2_store_previous_env(int64_t n, const float* present, const int32_t* ids, const void* age, int32_t age_f64, double dt,
                           int32_t id_base, int64_t n_total, float* store, float* prev) {
    if (n < 0 || n_total < 0) return -2;
    StorePrevParams p;
    p.n = n; p.present = present; p.ids = ids; p.age = age; p.store = store; p.prev = prev; p.n_total = n_total; p.id_base = id_base;
    p.age_f64 = age_f64; p.dt = dt;
    for (int64_t i = 0; i < n; ++i) store_prev_gather_one(p, i);       // launch 1
    for (int64_t i = 0; i < n; ++i) store_prev_scatter_one(p, i);      // launch 2
    return 0;
}

int hs2_vertical_advection_corrected(int64_t n, void* z, int32_t z_f64, const float* w, const float* ssh, const float* ssh_prev,
                                     const float* floor, float floor_const, const int32_t* moving, int32_t at_surface, double dt) {
    if (n < 0) return -2;
    VadvCorrParams p;
    p.n = n; p.z = z; p.w = w; p.ssh = ssh; p.ssh_prev = ssh_prev; p.floor = floor; p.moving = moving; p.floor_const = floor_const;
    p.z_f64 = z_f64; p.at_surface = at_surface; p.dt = dt;
    for (int64_t i = 0; i < n; ++i) vadv_corrected_one(p, i);
    return 0;
}

}
