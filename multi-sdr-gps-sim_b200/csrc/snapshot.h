// Snapshot measurement (include/gpsb200.h: gpsb200_snapshot_measure; DESIGN §11.5): each acquired peak refined, over
// the searched window, to a code phase in 2^-32 chips and a carrier step in 3e6/2^32 Hz, in exact integer arithmetic.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace snap {

constexpr int kChunk = 3000;                   // samples per chunk (one nominal C/A period)
constexpr int kThreads = 256;                  // threads of k_snapshot
constexpr int kPerThread = (kChunk + kThreads - 1) / kThreads;   // 12 samples per thread and chunk

// Empty when the call is well-formed: the search config as gpsb200_acquire checks it, res [nprn] in its PRN order with
// delays 0..2999 and |doppler_hz| <= 10 kHz, and the snapshot config in range.
std::string check(const gpsb200_acq_config_t *acq, int64_t nsamples, int sample_size, const gpsb200_acq_result_t *res,
                  const gpsb200_snapshot_config_t *cfg);
// The snapshot config's part of check (cfg not NULL).
std::string check_config(const gpsb200_snapshot_config_t *cfg);
// Header step 1 and the WEAK rule, on the host: the records the kernel starts from (and leaves as they are when WEAK).
void seed(const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res, const gpsb200_snapshot_config_t *cfg,
          gpsb200_snapshot_t *out);

struct Scratch {
    DeviceArray<gpsb200_snapshot_t> d_rec;    // [32]
    DeviceArray<gpsb200_snapshot_t> d_brec;   // [nwin][nprn] of a batch pass
};
// Enqueue the refinement of rec [nprn] (seeded) over the window at `window` (stream sample s0 first) on s and wait for
// the records. chips: [33][1023] chips as +-1 (trk::chips_upload).
cudaError_t launch(Scratch &sc, const void *window, int sample_size, int K, int nprn, const int8_t *chips, int iterations,
                   gpsb200_snapshot_t *rec, cudaStream_t s);

// A batch (gpsb200_snapshot_batch): the device scratch one window of acq's search and measurement may take, and the
// windows of a pass of nwin, as the header states them. The row cap keeps a pass's (window, PRN) pairs, grid y of the
// search, far below the grid's limit of 65535.
int64_t batch_window_bytes(const gpsb200_acq_config_t *acq, int sample_size);
int batch_pass(const gpsb200_acq_config_t *acq, int sample_size, int nwin);
static_assert(GPSB200_SNAP_BATCH_SCRATCH / (3000 * 8) < 65535, "a pass of two windows or more stays under grid y's limit");
// Enqueue the refinement of rec [nwin][nprn] (seeded) on s and wait for the records: window w's samples start
// d_win_off[w] (device) samples from src.
cudaError_t launch_batch(Scratch &sc, const void *src, int sample_size, int K, int nwin, int nprn,
                         const int64_t *d_win_off, const int8_t *chips, int iterations, gpsb200_snapshot_t *rec,
                         cudaStream_t s);

}  // namespace snap
}  // namespace gpsb200
