// GPS L1 C/A acquisition search at 3 Msps (include/gpsb200.h: gpsb200_acquire): C/A code delay x Doppler grid over K
// coherent 1 ms periods, non-coherently summed, reduced per PRN. Exact integer arithmetic (DESIGN §9, tests/acq_model.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace acq {

constexpr int kCode = 3000;                    // samples per C/A period at 3 Msps
constexpr int kThreads = 256;                  // threads of k_acq_grid
constexpr int kCtasPerSm = 3;                  // its launch bound: CTAs per SM
constexpr int kTausPerThread = 12;             // delays per thread: 256 x 12 = 3072 >= 3000 (the last 72 are discarded)
constexpr int kTaus = kThreads * kTausPerThread;
constexpr int kPrefix = 6144;                  // prefix sums S[0..6144] of one window (needs 3072 + 3000 - 1 <= 6143)
constexpr int kMaxEdges = 1024;                // sign changes of a sampled C/A replica (<= 1022), padded to a multiple of 8
constexpr int kExclude = 3;                    // P2 excludes delays within +-3 samples (one chip) of the peak

// Device scratch of the searches of one context, grown as needed.
struct Scratch {
    DeviceArray<int16_t> d_edges;      // [33][kMaxEdges] sign-change positions of every PRN's replica, row 0 unused
    DeviceArray<int32_t> d_nedges;     // [33]
    DeviceArray<uint64_t> d_grid;      // [nprn][nbins][3000] when the caller wants the grid or the search is split
    DeviceArray<uint64_t> d_rows;      // [nprn][nbins][3]: P1, P2, tau1 of every row
    DeviceArray<gpsb200_acq_result_t> d_res;   // [32]
    PinnedArray<gpsb200_acq_result_t> h_res;   // [32]
    DeviceArray<uint32_t> d_u;         // [nbins] phase steps; with per-PRN windows [nprn][nbins]
    DeviceArray<int32_t> d_prn;        // [32]
    DeviceArray<double> d_flo;         // [32] first bin of each PRN's window (gpsb200_acquire_windows)
    DeviceArray<int64_t> d_boff;       // batches (gpsb200_snapshot_batch): [nwin] window offsets in samples,
    DeviceArray<int32_t> d_bprn;       // [nwin][nprn] PRN,
    DeviceArray<double> d_bflo;        // [nwin][nprn] first bin
    DeviceArray<gpsb200_acq_result_t> d_bres;   // and [nwin][nprn] results of every (window, PRN) pair
    bool ready = false;                // d_edges / d_nedges uploaded, kernel attributes set, sms read
    int sms = 0;                       // SM count of the device (the split rule)
    int force_split = 0;               // 0: the split rule; else the split of every search (a test hook)
};

// Empty when the search is well-formed: PRNs 1..32, 1 <= K <= 100, 1 <= nbins <= GPSB200_ACQ_MAX_BINS, every bin within
// +-1.5 MHz, sample size SC08/SC16, a window [s0, s0 + 3000 K + 2999) inside a buffer of nsamples samples. With
// windows, the bins are f_lo_prn[p] + j step_hz (f_lo_prn not NULL) and cfg->f_lo_hz is not looked at.
std::string check(const gpsb200_acq_config_t *cfg, int64_t nsamples, int sample_size, bool windows = false,
                  const double *f_lo_prn = nullptr);
// The CTAs per row of a search of `rows` = nprn x nbins rows on `sms` SMs: of 1, 2, 3, 4, 6 the one with the least
// per-SM work when the CTAs spread evenly, ceil(rows split / sms) / split, the smallest on ties; split_of applies a
// forced split instead when one is set. split_allowed: whether a split is one of those.
int split_for(int rows, int sms);
int split_of(const Scratch &sc, int nprn, int nbins);
bool split_allowed(int split);
// The split of a batch pass of npair (window, PRN) pairs: split_of while its rows npair x nbins are fewer than a full
// wave (kCtasPerSm CTAs on every SM) or a split is forced, else 1: a split only pays while SMs would idle.
int batch_split(const Scratch &sc, int npair, int nbins);
// Samples the search reads from s0 on: 3000 K + 2999.
int64_t window_samples(const gpsb200_acq_config_t *cfg);
// Phase step of bin j: (uint32) llround(f_j * 2^32 / 3e6).
uint32_t phase_step(double f_hz);

cudaError_t scratch_reserve(Scratch &sc, const gpsb200_acq_config_t *cfg, bool windows, bool want_grid);
// Scratch of a batch pass of nwin windows (launch_batch).
cudaError_t batch_reserve(Scratch &sc, const gpsb200_acq_config_t *cfg, int nwin);
// Enqueue the search of the samples at `window` (the first sample is s0) on s; results land in sc.h_res after a
// synchronize of s, the grid (want_grid) in sc.d_grid. f_lo_prn (NULL: cfg->f_lo_hz for every PRN): per-PRN windows.
cudaError_t launch(Scratch &sc, const void *window, int sample_size, const gpsb200_acq_config_t *cfg,
                   const double *f_lo_prn, bool want_grid, cudaStream_t s);

// Enqueue the per-PRN window search of nwin windows on s and wait for it: window w starts win_off[w] samples from src,
// pair (w, q) searches PRN cfg->prn[q] from first bin f_lo[w nprn + q]; res [nwin][nprn] (host) as gpsb200_acquire_windows
// run on each window gives it (with f_lo[..] = cfg->f_lo_hz, as gpsb200_acquire gives it). nwin nprn <= 65535.
cudaError_t launch_batch(Scratch &sc, const void *src, int sample_size, const gpsb200_acq_config_t *cfg, int nwin,
                         const int64_t *win_off, const double *f_lo, gpsb200_acq_result_t *res, cudaStream_t s);

}  // namespace acq
}  // namespace gpsb200
