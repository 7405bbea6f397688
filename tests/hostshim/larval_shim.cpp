// Host build of LarvalFish's device code for the CPU tests (tests/larval_host.py): larval_develop_one and larval_migrate_one of
// csrc/od_larval.cuh, one loop per launch, with the argument checks and parameter fill of od_larval_develop / od_larval_migrate.
// Compiled with -ffp-contract=off, as the device build rounds every operation on its own.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "../../opendrift_b200/csrc/od_larval.cuh"

using namespace od;

extern "C" {

int hs7_larval_develop(int64_t n, const float* t, const float* s, void* hatched, int32_t hatched_f64, void* stage, int32_t stage_f64,
                       void* weight, int32_t weight_f64, void* length, int32_t length_f64, const void* diameter, int32_t diameter_f64,
                       const void* nbs, int32_t nbs_f64, int32_t develop, void* w_out, double dt, int32_t* h_flags) {
    if (n < 0) return -2;
    if (h_flags) *h_flags = 0;
    if (n == 0) return 0;
    if (!t || (develop && (!hatched || !stage || !weight || !length)) || (w_out && (!s || !diameter || !nbs))) return -2;
    LarvalParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.t = t; p.s = s; p.hatched = hatched; p.stage = stage; p.weight = weight; p.length = length;
    p.diameter = diameter; p.nbs = nbs; p.w_out = w_out; p.develop = develop; p.dt = dt;
    p.hatched_f64 = hatched_f64; p.stage_f64 = stage_f64; p.weight_f64 = weight_f64; p.length_f64 = length_f64;
    p.diameter_f64 = diameter_f64; p.nbs_f64 = nbs_f64;
    unsigned acc = 0;
    for (int64_t i = 0; i < n; ++i) acc |= larval_develop_one(p, i);
    if (h_flags) *h_flags = (int32_t)acc;
    return 0;
}

int hs7_larval_migrate(int64_t n, const void* hatched, int32_t hatched_f64, const void* length, int32_t length_f64, void* z,
                       int32_t z_f64, double fraction, double direction, double dt) {
    if (n < 0 || (n > 0 && (!hatched || !length || !z))) return -2;
    LarvalParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.hatched = (void*)hatched; p.hatched_f64 = hatched_f64; p.length = (void*)length; p.length_f64 = length_f64;
    p.z = z; p.z_f64 = z_f64; p.swim = fraction; p.dir = direction; p.dt = dt;
    for (int64_t i = 0; i < n; ++i) larval_migrate_one(p, i);
    return 0;
}

}
