// Device helpers of the receiver-side kernels (acquire.cu, track.cu, snapshot.cu): the sample reduction, the carrier
// table and its wipe-off, the early / prompt / late chips and the reduction of the correlator sums they share
// (include/gpsb200.h: acquisition, tracking and snapshot contracts). The sine table also builds the synthesis's carrier
// tables (k_tables, synth_kernels.cu).
#pragma once
#include <stdint.h>

#include "synth_tables.h"
#include "track.h"

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

// The carrier table tab[512] = (cos, sin) = (sinTable512[i + 128], sinTable512[i]), filled by threads 0..nthreads-1.
__device__ __forceinline__ void fill_carrier_table(int2 *tab, int nthreads) {
    for (int i = threadIdx.x; i < 512; i += nthreads) tab[i] = make_int2(sine512(i + 128), sine512(i));
}

// The carrier wipe-off of sample (I, Q) at carrier phase ph (2^-32 turns): (I cos + Q sin, Q cos - I sin).
__device__ __forceinline__ int2 wipe_off(const int2 *tab, uint32_t ph, int I, int Q) {
    const int2 cs = tab[ph >> 23];
    return make_int2(I * cs.x + Q * cs.y, Q * cs.x - I * cs.y);
}

// The early, prompt and late chips (+-1) of ca[1023] at code phase p < kM (2^-32 chips): p + kHalf, p and p - kHalf,
// folded into [0, kM).
__device__ __forceinline__ void epl_chips(const int8_t *ca, uint64_t p, int &ce, int &cp, int &cl) {
    uint64_t e = p + trk::kHalf;
    if (e >= trk::kM) e -= trk::kM;
    const uint64_t l = p >= trk::kHalf ? p - trk::kHalf : p + trk::kM - trk::kHalf;
    ce = ca[e >> 32];
    cp = ca[p >> 32];
    cl = ca[l >> 32];
}

// The N correlator sums a of every thread into the CTA's per-warp partials: each summed over its warp with shuffles (a
// fixed order), then lane 0 stores them to part[0..N), the warp's row.
template <int N>
__device__ __forceinline__ void warp_partials(int (&a)[N], int32_t *part) {
#pragma unroll
    for (int j = 0; j < N; j++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[j] += __shfl_xor_sync(0xffffffffu, a[j], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int j = 0; j < N; j++) part[j] = a[j];
}

// Sum j of the per-warp partials part[kWarps][6] over the warps, in warp order.
template <int kWarps>
__device__ __forceinline__ int warps_sum(const int32_t (*part)[6], int j) {
    int v = 0;
#pragma unroll
    for (int q = 0; q < kWarps; q++) v += part[q][j];
    return v;
}

}  // namespace

}  // namespace rx
}  // namespace gpsb200
