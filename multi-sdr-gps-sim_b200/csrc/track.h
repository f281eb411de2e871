// Code and carrier tracking loops (include/gpsb200.h: gpsb200_track; DESIGN §10). One coherent period per local C/A code
// epoch, exact integer arithmetic; the loop update below is the contract's, shared by the kernel and the host checks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/gpsb200.h"
#include "device_buffer.h"

namespace gpsb200 {
namespace trk {

constexpr uint64_t kM = 1023ull << 32;          // code phase modulus: 1023 chips in 2^-32 chip units
constexpr uint64_t kHalf = 1ull << 31;          // early / late offset: half a chip
constexpr int kMaxPeriod = 3001;                // samples of a period at most (header: 2999..3001)
constexpr int kThreads = 256;                   // threads of k_track
constexpr int kPerThread = (kMaxPeriod + kThreads - 1) / kThreads;   // 12 samples per thread and period
constexpr int64_t kFreqClamp = 1ll << 34;       // |F| bound, 2^-10 carrier step units (+-2^24 steps = +-11.7 kHz)
constexpr int kCordicSteps = 24;

// round(atan(2^-i) / (2 pi) * 2^32), i = 0..23 (tests/track_model.py checks the same list against the formula).
#define GPSB200_TRK_ATAN                                                                                     \
    536870912, 316933406, 167458907, 85004756, 42667331, 21354465, 10679838, 5340245, 2670163, 1335087, 667544, \
        333772, 166886, 83443, 41722, 20861, 10430, 5215, 2608, 1304, 652, 326, 163, 81

__host__ __device__ inline int64_t tdiv(int64_t a, int64_t b) { return a / b; }   // C++: truncation toward zero

__host__ __device__ inline int bitlen64(uint64_t v) {
#ifdef __CUDA_ARCH__
    return 64 - __clzll((long long) v);
#else
    return v ? 64 - __builtin_clzll(v) : 0;
#endif
}

// Angle of (x, y), x >= 0, in 2^-32 turns: normalised to 30 bits, then 24 CORDIC vectoring steps. The zero vector has
// angle 0 (the steps alone would give -0.277 turn), so that a period or window of zeros steers no loop.
__host__ __device__ inline int32_t angle(int64_t x, int64_t y) {
    if (x == 0 && y == 0) return 0;
    const int32_t A[kCordicSteps] = {GPSB200_TRK_ATAN};
    const uint64_t ay = y < 0 ? (uint64_t) (-y) : (uint64_t) y;
    const uint64_t mx = (uint64_t) x > ay ? (uint64_t) x : ay;
    const int s = bitlen64(mx) > 30 ? bitlen64(mx) - 30 : 0;
    x >>= s;
    y >>= s;
    int64_t z = 0;
    for (int i = 0; i < kCordicSteps; i++) {
        const int64_t xs = x >> i, ys = y >> i;
        if (y > 0) {
            x += ys;
            y -= xs;
            z += A[i];
        } else {
            x -= ys;
            y += xs;
            z -= A[i];
        }
    }
    return (int32_t) z;
}

// The code step at carrier step w and DLL discriminator D: NOM + w / 1540 + 2048 D / 3000 (carrier aided), clamped to
// GPSB200_TRK_CODE_STEP_MIN..MAX. A start state and the snapshot measurement take D = 0.
__host__ __device__ inline uint32_t code_step(int32_t w, int64_t D = 0) {
    int64_t u = (int64_t) GPSB200_TRK_CODE_STEP_NOM + tdiv(w, 1540) + tdiv(2048 * D, 3000);
    u = u < (int64_t) GPSB200_TRK_CODE_STEP_MIN ? (int64_t) GPSB200_TRK_CODE_STEP_MIN
                                                 : (u > (int64_t) GPSB200_TRK_CODE_STEP_MAX ? (int64_t) GPSB200_TRK_CODE_STEP_MAX : u);
    return (uint32_t) u;
}

// DLL discriminator of early and late powers E, L >= 0: both shifted to at most 40 bits, then (E - L) 2^14 / (E + L).
__host__ __device__ inline int64_t dll(int64_t E, int64_t L) {
    const int bl = bitlen64((uint64_t) (E + L));
    const int s = bl > 40 ? bl - 40 : 0;
    E >>= s;
    L >>= s;
    return (E + L) == 0 ? 0 : tdiv((E - L) * 16384, E + L);
}

// FLL terms of the prompt sums (i0, q0) and the next ones (i1, q1): cross and dot, both negated when dot < 0 (a data
// bit flipped between them). The loop takes the angle of one pair, the snapshot the angle of the sums over its chunks.
struct CrossDot {
    int64_t cross, dot;
};
__host__ __device__ inline CrossDot fll(int64_t i0, int64_t q0, int64_t i1, int64_t q1) {
    const int64_t cross = i0 * q1 - q0 * i1, dot = i0 * i1 + q0 * q1;
    return dot < 0 ? CrossDot{-cross, -dot} : CrossDot{cross, dot};
}

// The carrier step w = acq::phase_step(doppler_hz) and code step u = code_step(w) a channel starts from at an
// acquisition's Doppler (gpsb200_track_start, the snapshot measurement's seed).
void start_steps(double doppler_hz, int32_t &w, uint32_t &u);

// One loop update after a period with sums c[6] = E_I, E_Q, P_I, P_Q, L_I, L_Q. Updates carr_freq, carr_step, code_step,
// prev_*, lock_*, lock and epochs of st (the phases and sample are advanced by the caller).
__host__ __device__ inline void loop_update(gpsb200_track_state_t &st, const int32_t c[6]) {
    const int64_t pi = c[2], pq = c[3];
    // PLL: Costas discriminator
    const int32_t e = pi < 0 ? angle(-pi, -pq) : angle(pi, pq);
    int64_t F = st.carr_freq;
    // FLL assist during pull-in
    if (st.epochs >= 1 && st.epochs < GPSB200_TRK_FLL_EPOCHS) {
        const CrossDot f = fll(st.prev_i, st.prev_q, pi, pq);
        F += tdiv(64 * (int64_t) angle(f.dot, f.cross), 3000);
    }
    F += (int64_t) (e >> 12);
    F = F > kFreqClamp ? kFreqClamp : (F < -kFreqClamp ? -kFreqClamp : F);
    st.carr_freq = F;
    const int32_t w = (int32_t) ((F >> 10) + (int64_t) (e >> 16));
    st.carr_step = w;
    // DLL: normalised early-minus-late power, carrier aided
    const int64_t D = dll((int64_t) c[0] * c[0] + (int64_t) c[1] * c[1], (int64_t) c[4] * c[4] + (int64_t) c[5] * c[5]);
    st.code_step = code_step(w, D);
    // narrow-band lock indicator
    const int32_t api = (int32_t) (pi < 0 ? -pi : pi), apq = (int32_t) (pq < 0 ? -pq : pq);
    st.lock_i += (api - st.lock_i) >> 4;
    st.lock_q += (apq - st.lock_q) >> 4;
    st.lock = (int64_t) 3 * st.lock_q < (int64_t) st.lock_i ? 1 : 0;
    st.prev_i = (int32_t) pi;
    st.prev_q = (int32_t) pq;
    st.epochs += 1;
}

// Samples of the period that starts with code phase phi at code step u: ceil((M - phi) / u).
__host__ __device__ inline int period_len(uint64_t phi, uint32_t u) { return (int) ((kM - phi + u - 1) / u); }

// Empty when the states and call shape are well-formed (see the header); nsamples / base describe the buffer.
std::string check(const gpsb200_track_state_t *st, int nchan, int max_epochs, int64_t nsamples, int64_t base,
                  int sample_size);

// The [33][1023] C/A chips as +-1 (row 0 unused) that k_track and k_snapshot read, written into d.
cudaError_t chips_upload(DeviceArray<int8_t> &d);

// Device scratch of the tracking calls of one context, grown as needed.
struct Scratch {
    DeviceArray<gpsb200_track_state_t> d_state;    // [GPSB200_TRK_MAX_CHAN]
    DeviceArray<gpsb200_track_epoch_t> d_epochs;   // [nchan][max_epochs]
    DeviceArray<int32_t> d_n;                      // [GPSB200_TRK_MAX_CHAN]
};

cudaError_t scratch_reserve(Scratch &sc, int nchan, int max_epochs);
// Enqueue the tracking of the samples at `src` (stream sample `base` first) on s and wait for the results.
// chips: chips_upload's table.
cudaError_t launch(Scratch &sc, const int8_t *chips, const void *src, int64_t nsamples, int sample_size, int64_t base,
                   gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                   int32_t *nepochs, cudaStream_t s);

}  // namespace trk
}  // namespace gpsb200
