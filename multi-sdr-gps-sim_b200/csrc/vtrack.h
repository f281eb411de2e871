// Vector tracking (include/gpsb200.h: gpsb200_vtrack; DESIGN §10.1): the channels' periods of track.cu with NCOs
// commanded by one FP64 navigation filter per update interval.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace vtk {

constexpr int kMaxCluster = 16;

// Empty when the call is well-formed (see the header).
std::string check(const gpsb200_vtrack_state_t *st, const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg,
                  int max_updates, bool epochs, int max_epochs, int64_t nsamples, int64_t base, int sample_size);
std::string check_config(const gpsb200_vtrack_config_t *cfg);

// Device scratch of the vector-tracking calls of one context, grown as needed.
struct Scratch {
    DeviceArray<gpsb200_vtrack_state_t> d_state;   // [1]
    DeviceArray<gpsb200_pvt_chan_t> d_chans;       // [GPSB200_TRK_MAX_CHAN]
    DeviceArray<int32_t> d_n;                      // [GPSB200_TRK_MAX_CHAN + 1]: nepochs, then nupdates
    DeviceArray<gpsb200_fix_t> d_fix;              // [max_updates]
    DeviceArray<gpsb200_vtrack_chan_t> d_out;      // [max_updates][nchan]
    DeviceArray<gpsb200_track_epoch_t> d_epochs;   // [nchan][max_epochs]
};

cudaError_t scratch_reserve(Scratch &sc, int nchan, int max_updates, int max_epochs);
// Enqueue the call on s with a cluster of `ctas` CTAs (0: min(nchan, 8)) and wait for the results.
cudaError_t launch(Scratch &sc, const int8_t *chips, const void *src, int64_t nsamples, int sample_size, int64_t base,
                   const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg, gpsb200_vtrack_state_t *state,
                   int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *out, int32_t *nupdates,
                   gpsb200_track_epoch_t *epochs, int max_epochs, int32_t *nepochs, int ctas, cudaStream_t s);

}  // namespace vtk
}  // namespace gpsb200
