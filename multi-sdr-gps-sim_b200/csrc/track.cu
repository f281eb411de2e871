// Code and carrier tracking (include/gpsb200.h: gpsb200_track; DESIGN §10).
//
// k_track: one CTA per channel, 256 threads, looping over the channel's periods. Per period every thread wipes off and
// correlates samples m = tid + 256 r (r < 12, m < L) against the early, prompt and late replicas, the six int32 sums are
// reduced in a fixed order (warp shuffles, then warp 0 over the 8 warp partials), and thread 0 runs the loop update of
// track.h and publishes the next period's NCO state through shared memory. The loop is sequential in time: the figure
// of merit is the latency of one period, not bandwidth (every channel reads the same samples, which hit in L2).
#include <cstring>
#include <vector>

#include "acquire.h"
#include "device_buffer.h"
#include "rx_samples.cuh"
#include "synth_tables.h"
#include "track.h"

namespace gpsb200 {
namespace trk {

namespace {

using rx::load_iq;

constexpr int kWarps = kThreads / 32;

struct Smem {
    int2 tab[512];                  // (cos, sin)
    int8_t ca[1024];                // the channel's chips as +-1
    int32_t part[kWarps][6];        // warp partial sums
    gpsb200_track_state_t st;       // the loop state, owned by thread 0
    int L;                          // samples of the current period, 0: stop
};

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_track(const T *__restrict__ iq, int64_t nsamples, int64_t base, const int8_t *__restrict__ chips,
        gpsb200_track_state_t *__restrict__ states, int max_epochs, gpsb200_track_epoch_t *__restrict__ epochs,
        int32_t *__restrict__ nepochs) {
    __shared__ Smem sm;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int ch = blockIdx.x;
    rx::fill_carrier_table(sm.tab, kThreads);
    if (tid == 0) sm.st = states[ch];
    __syncthreads();
    for (int i = tid; i < GPSB200_CA_LEN; i += kThreads) sm.ca[i] = chips[sm.st.prn * GPSB200_CA_LEN + i];
    const int64_t end = base + nsamples;
    gpsb200_track_epoch_t *out = epochs + (size_t) ch * max_epochs;
    int k = 0;
    for (;;) {
        if (tid == 0) {
            const int L = period_len(sm.st.code_phase, sm.st.code_step);
            sm.L = (k < max_epochs && sm.st.sample + L <= end) ? L : 0;
        }
        __syncthreads();   // L and the NCO state published (and, at k = 0, the chips)
        const int L = sm.L;
        if (L == 0) break;
        const int64_t s = sm.st.sample - base;
        const uint64_t phi = sm.st.code_phase;
        const uint32_t u = sm.st.code_step, theta = sm.st.carr_phase, w = (uint32_t) sm.st.carr_step;
        int a[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int r = 0; r < kPerThread; r++) {
            const int m = tid + kThreads * r;
            if (m < L) {
                int I, Q;
                load_iq<T>(iq, s + m, I, Q);
                const int2 d = rx::wipe_off(sm.tab, theta + (uint32_t) m * w, I, Q);
                int ce, cp, cl;
                rx::epl_chips(sm.ca, phi + (uint64_t) m * u, ce, cp, cl);
                a[0] += ce * d.x;
                a[1] += ce * d.y;
                a[2] += cp * d.x;
                a[3] += cp * d.y;
                a[4] += cl * d.x;
                a[5] += cl * d.y;
            }
        }
        rx::warp_partials(a, sm.part[warp]);
        __syncthreads();
        if (tid == 0) {
            int32_t c[6];
            for (int j = 0; j < 6; j++) c[j] = rx::warps_sum<kWarps>(sm.part, j);
            gpsb200_track_state_t st = sm.st;
            const int64_t s_abs = st.sample;
            st.sample += L;
            st.carr_phase = theta + (uint32_t) L * w;
            st.code_phase = phi + (uint64_t) L * u - kM;
            loop_update(st, c);
            gpsb200_track_epoch_t ep;
            ep.sample = s_abs;
            ep.e_i = c[0];
            ep.e_q = c[1];
            ep.p_i = c[2];
            ep.p_q = c[3];
            ep.l_i = c[4];
            ep.l_q = c[5];
            ep.carr_phase = st.carr_phase;
            ep.carr_step = st.carr_step;
            ep.code_phase = (uint32_t) st.code_phase;
            ep.code_step = st.code_step;
            ep.lock = st.lock;
            ep.reserved = 0;
            out[k] = ep;
            sm.st = st;
        }
        k++;
    }
    if (tid == 0) {
        states[ch] = sm.st;
        nepochs[ch] = k;
    }
}

}  // namespace

std::string check(const gpsb200_track_state_t *st, int nchan, int max_epochs, int64_t nsamples, int64_t base,
                  int sample_size) {
    if (!st) return "state is NULL";
    if (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16) return "sample_size must be GPSB200_SC08 or GPSB200_SC16";
    if (nchan < 1 || nchan > GPSB200_TRK_MAX_CHAN) return "nchan must be 1..32";
    if (max_epochs < 1) return "max_epochs must be >= 1";
    if (nsamples < 0 || base < 0) return "nsamples and base must be >= 0";
    for (int c = 0; c < nchan; c++) {
        const gpsb200_track_state_t &s = st[c];
        const std::string at = "channel " + std::to_string(c) + ": ";
        if (s.prn < 1 || s.prn > 32) return at + "PRN outside 1..32";
        if (s.epochs < 0 || s.lock < 0 || s.lock > 1 || s.lock_i < 0 || s.lock_q < 0) return at + "bad loop state";
        if (s.code_step < GPSB200_TRK_CODE_STEP_MIN || s.code_step > GPSB200_TRK_CODE_STEP_MAX)
            return at + "code_step outside GPSB200_TRK_CODE_STEP_MIN..MAX";
        if (s.code_phase >= GPSB200_TRK_CODE_STEP_MAX) return at + "code_phase must be below GPSB200_TRK_CODE_STEP_MAX";
        if (s.carr_freq > kFreqClamp || s.carr_freq < -kFreqClamp) return at + "|carr_freq| above 2^34";
        if (s.sample < base) return at + "the next period starts before the buffer's first sample";
    }
    return std::string();
}

void start_steps(double doppler_hz, int32_t &w, uint32_t &u) {
    w = (int32_t) acq::phase_step(doppler_hz);
    u = code_step(w);
}

cudaError_t chips_upload(DeviceArray<int8_t> &d) {
    std::vector<int8_t> c((size_t) 33 * GPSB200_CA_LEN, 0);
    for (int prn = 1; prn <= 32; prn++) {
        uint8_t ca[GPSB200_CA_LEN];
        ca_code(prn, ca);
        for (int i = 0; i < GPSB200_CA_LEN; i++) c[(size_t) prn * GPSB200_CA_LEN + i] = (int8_t) (2 * ca[i] - 1);
    }
    CU_RET(d.grow(c.size()));
    return cudaMemcpy(d.get(), c.data(), c.size(), cudaMemcpyHostToDevice);
}

cudaError_t scratch_reserve(Scratch &sc, int nchan, int max_epochs) {
    CU_RET(sc.d_state.grow(GPSB200_TRK_MAX_CHAN));
    CU_RET(sc.d_n.grow(GPSB200_TRK_MAX_CHAN));
    return sc.d_epochs.grow((size_t) nchan * max_epochs);
}

cudaError_t launch(Scratch &sc, const int8_t *chips, const void *src, int64_t nsamples, int sample_size, int64_t base,
                   gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                   int32_t *nepochs, cudaStream_t s) {
    CU_RET(cudaMemcpyAsync(sc.d_state.get(), state, nchan * sizeof(gpsb200_track_state_t), cudaMemcpyHostToDevice, s));
    if (sample_size == GPSB200_SC08)
        k_track<int8_t><<<nchan, kThreads, 0, s>>>(static_cast<const int8_t *>(src), nsamples, base, chips,
                                                   sc.d_state.get(), max_epochs, sc.d_epochs.get(), sc.d_n.get());
    else
        k_track<int16_t><<<nchan, kThreads, 0, s>>>(static_cast<const int16_t *>(src), nsamples, base, chips,
                                                    sc.d_state.get(), max_epochs, sc.d_epochs.get(), sc.d_n.get());
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(nepochs, sc.d_n.get(), nchan * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaMemcpyAsync(state, sc.d_state.get(), nchan * sizeof(gpsb200_track_state_t), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaStreamSynchronize(s));
    // the epochs of channel c sit at c * max_epochs; copy only the written ones
    for (int c = 0; c < nchan; c++)
        if (nepochs[c] > 0)
            CU_RET(cudaMemcpyAsync(epochs + (size_t) c * max_epochs, sc.d_epochs.get() + (size_t) c * max_epochs,
                                   (size_t) nepochs[c] * sizeof(gpsb200_track_epoch_t), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

}  // namespace trk
}  // namespace gpsb200
