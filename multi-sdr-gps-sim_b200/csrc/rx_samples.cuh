// Device helpers of the receiver-side kernels (acquire.cu, track.cu): the sample reduction and the carrier tables they
// share (include/gpsb200.h: acquisition and tracking contracts). The sine table also builds the synthesis's carrier
// tables (k_tables, synth_kernels.cu).
#pragma once
#include <stdint.h>

#include "synth_tables.h"

namespace gpsb200 {
namespace rx {

namespace {

__constant__ uint8_t c_qsine[128] = {GPSB200_QUARTER_SINE};

__device__ __forceinline__ int sine512(int k) {   // sinTable512[k] (gps.c:145-178)
    k &= 511;
    const int r = k & 255;
    const int v = c_qsine[r < 128 ? r : 255 - r];
    return k < 256 ? v : -v;
}

// Sample i of an interleaved I,Q buffer at the int8 scale: int8 as is, int16 reduced to clamp(x >> 4, -128, 127).
template <typename T>
__device__ __forceinline__ void load_iq(const T *iq, int64_t i, int &I, int &Q);
template <>
__device__ __forceinline__ void load_iq<int8_t>(const int8_t *iq, int64_t i, int &I, int &Q) {
    const char2 v = reinterpret_cast<const char2 *>(iq)[i];
    I = v.x;
    Q = v.y;
}
template <>
__device__ __forceinline__ void load_iq<int16_t>(const int16_t *iq, int64_t i, int &I, int &Q) {
    const short2 v = reinterpret_cast<const short2 *>(iq)[i];
    I = min(max(v.x >> 4, -128), 127);
    Q = min(max(v.y >> 4, -128), 127);
}

}  // namespace

}  // namespace rx
}  // namespace gpsb200
