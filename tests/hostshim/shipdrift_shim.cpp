// Host build of ShipDrift's device code for the CPU tests (tests/shipdrift_host.py): ship_particle of csrc/od_ship.cuh, one loop per
// launch, with the argument checks and parameter fill of od_ship_step.  Compiled with -ffp-contract=off, as the device build rounds
// every operation on its own.
#include <stdint.h>
#include <string.h>
#include "../../opendrift_b200/csrc/od_ship.cuh"

using namespace od;

extern "C" {

int hs5_ship_step(int64_t n, double* lon, double* lat, int32_t* moving, int32_t* status, const float* const* el,
                  const uint8_t* orientation, float* const* env, const double* wtab, const int32_t* wbox, int32_t nomega, int32_t nbeam,
                  int32_t ndraft, int32_t hs_wind, int32_t tm_wind, int32_t tm_fill_on, float tm_fill, int32_t strand_code, double dt,
                  int32_t* h_stranded) {
    if (n < 0 || !el || !env || !h_stranded || nomega < 2 || nbeam < 2 || ndraft < 2) return -2;
    *h_stranded = 0;
    if (n == 0) return 0;
    if (!lon || !lat || !orientation || !wtab || !wbox || !env[0] || !env[1] || !env[2] || !env[3] || !env[4] || !env[5] ||
        (!env[6]) != (!env[7]) || (env[8] && !status))
        return -2;
    for (int k = 0; k < 6; ++k)
        if (!el[k]) return -2;
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
    unsigned flag = 0;
    if (p.mask) p.stranded = &flag;
    for (int64_t i = 0; i < n; ++i) ship_particle(p, i);
    *h_stranded = flag ? 1 : 0;
    return 0;
}

// the table lookup alone (ship_wforce), for the bit-for-bit comparison with scipy: f / d at (omega[k], bl[k], dl[k])
int hs5_ship_wforce(int64_t n, const double* omega, const double* bl, const double* dl, const double* wtab, const int32_t* wbox,
                    int32_t nomega, int32_t nbeam, int32_t ndraft, double* f, double* d) {
    ShipParams p;
    memset(&p, 0, sizeof(p));
    p.wtab = wtab; p.wbox = wbox; p.nomega = nomega; p.nbeam = nbeam; p.ndraft = ndraft;
    for (int64_t k = 0; k < n; ++k) {
        const int bo = ship_cell(wtab, nomega, omega[k]);
        const int bb = ship_cell(wtab + nomega, nbeam, bl[k]);
        const int bd = ship_cell(wtab + nomega + nbeam, ndraft, dl[k]);
        ship_wforce(p, (bo * (nbeam - 1) + bb) * (ndraft - 1) + bd, omega[k], bl[k], dl[k], f[k], d[k]);
    }
    return 0;
}

}
