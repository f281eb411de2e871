// Collective detection (include/gpsb200.h: gpsb200_collective; DESIGN §11.7): a lattice of receiver positions and time
// offsets scored against the power grids of one acquisition search.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace cd {

static_assert(sizeof(gpsb200_collective_config_t) == 72, "gpsb200_collective_config_t layout");
static_assert(sizeof(gpsb200_collective_t) == 96, "gpsb200_collective_t layout");
static_assert(sizeof(gpsb200_cd_score_t) == 8 && sizeof(gpsb200_cd_cell_t) == 8, "score / cell layout");

constexpr int kRow = 6072;   // a normalised row, stored twice over and padded: q[(d + b)] for d < 3000, b < 3072

// The lattice config's part of the contract's checks (cfg not NULL), and the hypothesis count it gives.
std::string check(const gpsb200_collective_config_t *cfg);
int64_t hypotheses(const gpsb200_collective_config_t *cfg);

struct Setup;
struct Scratch {
    DeviceArray<uint64_t> d_rowsum;             // [nprn][nbins][2] 128-bit row sums (lo, hi)
    DeviceArray<uint16_t> d_q;                  // [nprn][nbins][kRow]
    DeviceArray<gpsb200_cd_score_t> d_scores;   // [nhyp]
    DeviceArray<gpsb200_cd_cell_t> d_table;     // [nhyp][nprn], only when the caller wants it
    DeviceArray<gpsb200_ephemeris_t> d_eph;     // [32]
    DeviceArray<Setup> d_setup;                 // [1]
    DeviceArray<gpsb200_collective_t> d_rec;    // [1]
    DeviceArray<gpsb200_acq_result_t> d_seed;   // [32]
};

// Steps 2-8 on the grid [nprn][nbins][3000] and results d_res [nprn] (device) a search with acq and f_lo_prn left, on s;
// waits for seed [nprn], out and, when not NULL, scores [nhyp] and table [nhyp][nprn] (host).
cudaError_t launch(Scratch &sc, const uint64_t *d_grid, const gpsb200_acq_result_t *d_res,
                   const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                   const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                   gpsb200_acq_result_t *seed, gpsb200_collective_t *out, gpsb200_cd_score_t *scores,
                   gpsb200_cd_cell_t *table, cudaStream_t s);

}  // namespace cd
}  // namespace gpsb200
