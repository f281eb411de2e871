// Position, velocity and time from tracked channels (include/gpsb200.h: gpsb200_pvt; DESIGN §11).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace pvt {

constexpr int kWarps = 4;                // fixes per CTA of k_pvt (one warp each)
constexpr int64_t kWeekMs = 604800000;   // ms of a GPS week

static_assert(sizeof(gpsb200_raim_config_t) == 32, "gpsb200_raim_config_t layout");
static_assert(sizeof(gpsb200_raim_t) == 48, "gpsb200_raim_t layout");
static_assert(sizeof(gpsb200_araim_config_t) == 96, "gpsb200_araim_config_t layout");
static_assert(sizeof(gpsb200_araim_t) == 64, "gpsb200_araim_t layout");
static_assert(sizeof(gpsb200_coarse_config_t) == 48, "gpsb200_coarse_config_t layout");
static_assert(sizeof(gpsb200_coarse_t) == 32, "gpsb200_coarse_t layout");
static_assert(sizeof(gpsb200_search_config_t) == 32, "gpsb200_search_config_t layout");
static_assert(sizeof(gpsb200_search_t) == 64, "gpsb200_search_t layout");
static_assert(sizeof(gpsb200_snapshot_config_t) == 16, "gpsb200_snapshot_config_t layout");
static_assert(sizeof(gpsb200_snapshot_t) == 56, "gpsb200_snapshot_t layout");

// What a fix call runs beside the fixes: nothing (gpsb200_pvt), the RAIM or ARAIM stage, coarse-time fixes or searches,
// from tracked epochs or (snapshot, snapshot_search) from snapshot records.
enum class Mode { plain, raim, araim, coarse, search, snapshot, snapshot_search };

// A fix call's stage: at most one of raim, araim, coarse and search is set, each with the records [nfix] it fills.
// ms [nfix][nchan] (coarse, search) and node_rms [nfix][nodes] (search) may stay NULL. meas [nfix][nchan] (coarse or
// search only): the measurements are these snapshot records, and the epochs are neither read nor checked.
struct Stage {
    const gpsb200_raim_config_t *raim = nullptr;
    gpsb200_raim_t *raim_out = nullptr;
    const gpsb200_araim_config_t *araim = nullptr;
    gpsb200_araim_t *araim_out = nullptr;
    const gpsb200_coarse_config_t *coarse = nullptr;
    gpsb200_coarse_t *coarse_out = nullptr;
    const gpsb200_search_config_t *search = nullptr;
    gpsb200_search_t *search_out = nullptr;
    int64_t *ms = nullptr;
    double *node_rms = nullptr;
    const gpsb200_snapshot_t *meas = nullptr;
    Mode mode() const {
        return raim     ? Mode::raim
               : araim  ? Mode::araim
               : coarse ? (meas ? Mode::snapshot : Mode::coarse)
               : search ? (meas ? Mode::snapshot_search : Mode::search)
                        : Mode::plain;
    }
};

// Empty when the call is well-formed (see the header).
std::string check(const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs, const int32_t *nepochs,
                  int max_epochs, const gpsb200_pvt_config_t *cfg, const Stage &st);

// The a-priori config's part of check (gpsb200_pvt_coarse), also collective detection's.
std::string check_coarse(const gpsb200_coarse_config_t &c);

// The RAIM tables of gpsb200_raim_thresholds (raim_thresholds.cpp); false when p_fa or p_md is outside 1e-12..0.5.
bool raim_thresholds(double p_fa, double p_md, double *T, double *lambda);
// The ARAIM test multipliers of gpsb200_araim_kfa (raim_thresholds.cpp); false when a probability is outside 1e-12..0.5.
bool araim_kfa(double p_fa_vert, double p_fa_horz, double *kh, double *kv);

// Device scratch of the fix calls of one context, grown as needed, and what gpsb200_pvt_replay re-runs.
struct Scratch {
    DeviceArray<gpsb200_track_epoch_t> d_epochs;  // [nchan][max_epochs]
    DeviceArray<gpsb200_pvt_chan_t> d_chans;     // [GPSB200_TRK_MAX_CHAN]
    DeviceArray<int32_t> d_n;                    // [GPSB200_TRK_MAX_CHAN]
    DeviceArray<gpsb200_fix_t> d_fixes;          // [nfix]
    DeviceArray<double> d_res;                   // [nfix][nchan]
    bool have_last = false;                      // the arguments of the previous call, for replay
    int nchan = 0, max_epochs = 0, ref = -1;
    int64_t ref_sample = 0, ref_ms = 0;
    gpsb200_pvt_config_t cfg{};
    bool want_res = false;
    Mode mode = Mode::plain;
    // the RAIM stage of the previous call (gpsb200_pvt_raim), and the tables of the last p_fa / p_md seen
    gpsb200_raim_config_t raim_cfg{};
    DeviceArray<gpsb200_raim_t> d_raim;          // [nfix]
    double tab_p_fa = 0.0, tab_p_md = 0.0;       // 0: no tables yet
    double tab_T[GPSB200_RAIM_MAX_DOF] = {}, tab_lambda[GPSB200_RAIM_MAX_DOF] = {};
    // the ARAIM stage of the previous call (gpsb200_pvt_araim)
    gpsb200_araim_config_t araim_cfg{};
    DeviceArray<gpsb200_araim_t> d_araim;        // [nfix]
    double kfa_h[GPSB200_RAIM_MAX_DOF] = {}, kfa_v[GPSB200_RAIM_MAX_DOF] = {};
    // the coarse-time call of the previous call (gpsb200_pvt_coarse)
    bool want_ms = false;
    gpsb200_coarse_config_t coarse_cfg{};
    DeviceArray<gpsb200_coarse_t> d_coarse;      // [nfix]
    DeviceArray<int64_t> d_ms;                   // [nfix][nchan]
    // the search of the previous call (gpsb200_pvt_search): records, and the per-instant scratch of pvt.cu's kernels
    bool want_node_rms = false;
    gpsb200_search_config_t search_cfg{};
    DeviceArray<gpsb200_search_t> d_search;      // [nfix]
    DeviceArray<double> d_sat;                   // [nfix][32][3]
    DeviceArray<uint32_t> d_used;                // [nfix]
    DeviceArray<int32_t> d_searched, d_nok;      // [nfix]
    DeviceArray<double> d_hits;                  // one pass's OK-node lists (pvt.cu: SearchHit, search_pass)
    DeviceArray<double> d_node_rms;              // [nfix][nodes], only when the caller asks for it
    DeviceArray<gpsb200_snapshot_t> d_meas;      // [nfix][nchan]: the snapshot records of a snapshot call
};

// Upload, run the kernels of st's stage on s and download the fixes [nfix], the residuals [nfix][nchan] (when not NULL)
// and the stage's outputs; waits for the results.
cudaError_t run(Scratch &sc, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg, gpsb200_fix_t *fixes,
                double *residuals, const Stage &st, cudaStream_t s);
// Enqueue the previous call's kernels again on its device-resident inputs.
cudaError_t replay(Scratch &sc, cudaStream_t s);
// gpsb200_search_nodes: xyz [n][3], the ECEF positions of the n-node search grid.
void search_nodes(int n, double *xyz);

}  // namespace pvt
}  // namespace gpsb200
