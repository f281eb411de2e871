// Snapshot measurement (include/gpsb200.h: gpsb200_snapshot_measure; DESIGN §11.5).
//
// k_snapshot: one CTA per PRN, 256 threads. A pass correlates the K chunks of 3000 samples from s0: every thread wipes
// off samples j = tid + 256 r (r < 12, j < 3000) of each chunk against the prompt replica (and, in the code passes, the
// early and late ones), the sums are reduced per chunk with warp shuffles into shared memory, then summed over the 8
// warps by one thread per chunk. Warp 0 reduces the chunks' int64 powers and thread 0 runs the header's update. Every
// sum is an exact integer sum, so its value does not depend on the order; there are no atomics. Pass 0 is the frequency
// pass (prompt only, at the seed), then one code pass per iteration.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "acquire.h"
#include "device_buffer.h"
#include "rx_samples.cuh"
#include "snapshot.h"
#include "track.h"

namespace gpsb200 {
namespace snap {

namespace {

using rx::load_iq;
using trk::kM;

constexpr int kWarps = kThreads / 32;

struct Smem {
    int2 tab[512];                                  // (cos, sin)
    int8_t ca[1024];                                // the PRN's chips as +-1
    int32_t part[GPSB200_ACQ_MAX_MS][kWarps][6];    // warp partials per chunk: E_I, E_Q, L_I, L_Q, P_I, P_Q
    int32_t p[GPSB200_ACQ_MAX_MS][2];               // the chunks' prompt sums (frequency pass)
    int64_t sq[GPSB200_ACQ_MAX_MS][3];              // the chunks' early, late and prompt powers (code passes)
    gpsb200_snapshot_t rec;                         // owned by thread 0
};

// One pass over the K chunks with the replica at phi + m u (mod M) and the wipe-off at m w: the warp partials of every
// chunk into sm.part (prompt only unless kCode).
template <typename T, bool kCode>
__device__ __forceinline__ void correlate(Smem &sm, const T *__restrict__ iq, int K, uint64_t phi, uint32_t u, uint32_t w) {
    const int tid = threadIdx.x, warp = tid >> 5;
    constexpr int kSums = kCode ? 6 : 2;
#pragma unroll 1
    for (int k = 0; k < K; k++) {
        const uint64_t base = (phi + (uint64_t) (kChunk * k) * u) % kM;
        int a[kSums];
#pragma unroll
        for (int j = 0; j < kSums; j++) a[j] = 0;
#pragma unroll
        for (int r = 0; r < kPerThread; r++) {
            const int j = tid + kThreads * r;
            if (j < kChunk) {
                const int m = kChunk * k + j;
                int I, Q;
                load_iq<T>(iq, m, I, Q);
                const int2 d = rx::wipe_off(sm.tab, (uint32_t) m * w, I, Q);
                uint64_t p = base + (uint64_t) j * u;   // base < M and j u <= 2999 u_max <= M: one fold
                if (p >= kM) p -= kM;
                int ce, cp, cl;   // the early and late chips are not read in the frequency pass
                rx::epl_chips(sm.ca, p, ce, cp, cl);
                a[kSums - 2] += cp * d.x;
                a[kSums - 1] += cp * d.y;
                if (kCode) {
                    a[0] += ce * d.x;
                    a[1] += ce * d.y;
                    a[2] += cl * d.x;
                    a[3] += cl * d.y;
                }
            }
        }
        rx::warp_partials(a, &sm.part[k][warp][6 - kSums]);
    }
}

// The body of k_snapshot and k_snapshot_batch, which differ only in where a CTA's samples start: record blockIdx.x.
template <typename T>
__device__ __forceinline__ void measure(Smem &sm, const T *__restrict__ iq, int K, const int8_t *__restrict__ chips,
                                        int iterations, gpsb200_snapshot_t *__restrict__ recs) {
    const int tid = threadIdx.x, lane = tid & 31;
    rx::fill_carrier_table(sm.tab, kThreads);
    if (tid == 0) sm.rec = recs[blockIdx.x];
    __syncthreads();
    if (sm.rec.status != GPSB200_SNAP_OK) return;   // WEAK: the seed record stays (the whole CTA leaves)
    for (int i = tid; i < GPSB200_CA_LEN; i += kThreads) sm.ca[i] = chips[sm.rec.prn * GPSB200_CA_LEN + i];
    __syncthreads();

    // header step 2: the frequency pass at the seed
    correlate<T, false>(sm, iq, K, sm.rec.code_phase, sm.rec.code_step, (uint32_t) sm.rec.carr_step);
    __syncthreads();
    if (tid < K) {
        sm.p[tid][0] = rx::warps_sum<kWarps>(sm.part[tid], 4);
        sm.p[tid][1] = rx::warps_sum<kWarps>(sm.part[tid], 5);
    }
    __syncthreads();
    if (tid == 0) {
        int64_t pw = 0, sc = 0, sd = 0;
        for (int k = 0; k < K; k++) {
            const int64_t pi = sm.p[k][0], pq = sm.p[k][1];
            pw += pi * pi + pq * pq;
            if (k + 1 < K) {
                const trk::CrossDot f = trk::fll(pi, pq, sm.p[k + 1][0], sm.p[k + 1][1]);
                sc += f.cross;
                sd += f.dot;
            }
        }
        sm.rec.power = (uint64_t) pw;
        if (K >= 2) {
            sm.rec.carr_step += (int32_t) trk::tdiv(trk::angle(sd, sc), 3000);
            sm.rec.code_step = trk::code_step(sm.rec.carr_step);
        }
    }
    __syncthreads();

    // header step 3: the code iterations at w1, u1
#pragma unroll 1
    for (int it = 0; it < iterations; it++) {
        correlate<T, true>(sm, iq, K, sm.rec.code_phase, sm.rec.code_step, (uint32_t) sm.rec.carr_step);
        __syncthreads();
        if (tid < K) {
            int64_t v[6];
#pragma unroll
            for (int j = 0; j < 6; j++) v[j] = rx::warps_sum<kWarps>(sm.part[tid], j);
            sm.sq[tid][0] = v[0] * v[0] + v[1] * v[1];
            sm.sq[tid][1] = v[2] * v[2] + v[3] * v[3];
            sm.sq[tid][2] = v[4] * v[4] + v[5] * v[5];
        }
        __syncthreads();
        if (tid < 32) {
            int64_t E = 0, L = 0, P = 0;
            for (int k = lane; k < K; k += 32) {
                E += sm.sq[k][0];
                L += sm.sq[k][1];
                P += sm.sq[k][2];
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                E += __shfl_xor_sync(0xffffffffu, E, o);
                L += __shfl_xor_sync(0xffffffffu, L, o);
                P += __shfl_xor_sync(0xffffffffu, P, o);
            }
            if (tid == 0) {
                const int64_t D = trk::dll(E, L);
                int64_t phi = (int64_t) sm.rec.code_phase + D * GPSB200_SNAP_GAIN;
                phi = phi < 0 ? phi + (int64_t) kM : (phi >= (int64_t) kM ? phi - (int64_t) kM : phi);
                sm.rec.code_phase = (uint64_t) phi;
                sm.rec.last_step = (int32_t) D;
                sm.rec.power = (uint64_t) P;
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        gpsb200_snapshot_t r = sm.rec;
        r.iterations = iterations;
        if (iterations > 0 && (r.last_step > GPSB200_SNAP_MAX_LAST_D || r.last_step < -GPSB200_SNAP_MAX_LAST_D))
            r.status = GPSB200_SNAP_NO_CONVERGENCE;
        recs[blockIdx.x] = r;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_snapshot(const T *__restrict__ iq, int K, const int8_t *__restrict__ chips,
                                                       int iterations, gpsb200_snapshot_t *__restrict__ recs) {
    __shared__ Smem sm;
    measure<T>(sm, iq, K, chips, iterations, recs);
}

// A batch of windows (gpsb200_snapshot_batch; DESIGN §11.6): record blockIdx.x = w nprn + q, window w's samples start
// win_off[w] samples from iq.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_snapshot_batch(const T *__restrict__ iq, const int64_t *__restrict__ win_off, int nprn, int K,
                 const int8_t *__restrict__ chips, int iterations, gpsb200_snapshot_t *__restrict__ recs) {
    __shared__ Smem sm;
    measure<T>(sm, iq + 2 * win_off[blockIdx.x / nprn], K, chips, iterations, recs);
}

}  // namespace

std::string check_config(const gpsb200_snapshot_config_t *cfg) {
    if (!(cfg->min_ratio >= 0.0) || !std::isfinite(cfg->min_ratio)) return "min_ratio must be finite and >= 0";
    if (cfg->iterations < 0 || cfg->iterations > GPSB200_SNAP_MAX_ITER) return "iterations must be 0..16";
    if (cfg->reserved != 0) return "snapshot config reserved must be 0";
    return std::string();
}

std::string check(const gpsb200_acq_config_t *acq, int64_t nsamples, int sample_size, const gpsb200_acq_result_t *res,
                  const gpsb200_snapshot_config_t *cfg) {
    if (!acq || !res || !cfg) return "NULL acquisition config, results or snapshot config";
    // the measurement reads s0, K, the PRNs and the window, never the bins: check the config with one neutral bin, so
    // that the config of a per-PRN window search (gpsb200_acquire_windows) is accepted as it stands
    gpsb200_acq_config_t one = *acq;
    one.f_lo_hz = 0.0;
    one.step_hz = 0.0;
    one.nbins = 1;
    const std::string bad = acq::check(&one, nsamples, sample_size);
    if (!bad.empty()) return bad;
    const std::string bad_cfg = check_config(cfg);
    if (!bad_cfg.empty()) return bad_cfg;
    for (int p = 0; p < acq->nprn; p++) {
        const gpsb200_acq_result_t &r = res[p];
        const std::string at = "result " + std::to_string(p) + ": ";
        if (r.prn != acq->prn[p]) return at + "prn differs from the search's PRN list";
        if (r.delay < 0 || r.delay >= kChunk) return at + "delay outside 0..2999";
        if (!(std::fabs(r.doppler_hz) <= 10000.0)) return at + "|doppler_hz| above 10 kHz";
    }
    return std::string();
}

void seed(const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res, const gpsb200_snapshot_config_t *cfg,
          gpsb200_snapshot_t *out) {
    for (int p = 0; p < acq->nprn; p++) {
        const gpsb200_acq_result_t &r = res[p];
        gpsb200_snapshot_t &o = out[p];
        memset(&o, 0, sizeof o);
        o.prn = r.prn;
        o.sample = acq->s0;
        trk::start_steps(r.doppler_hz, o.carr_step, o.code_step);
        o.code_phase = (kM - ((uint64_t) r.delay * o.code_step) % kM) % kM;
        o.ratio = r.ratio;
        o.status = r.ratio >= cfg->min_ratio ? GPSB200_SNAP_OK : GPSB200_SNAP_WEAK;
    }
}

int64_t batch_window_bytes(const gpsb200_acq_config_t *acq, int sample_size) {
    const int64_t rows = (int64_t) acq->nprn * acq->nbins;
    // a pair's PRN, first bin, result and record: 4 + 8 + 56 + 56 = 124 bytes, rounded up as the header states it
    const int64_t pair = 128;
    static_assert(sizeof(int32_t) + sizeof(double) + sizeof(gpsb200_acq_result_t) + sizeof(gpsb200_snapshot_t) <= 128,
                  "a pair's scratch");
    return rows * ((int64_t) acq::kCode * 8 + 3 * 8 + 4) + acq->nprn * pair + 8 +
           acq::window_samples(acq) * (sample_size == GPSB200_SC16 ? 4 : 2);
}

int batch_pass(const gpsb200_acq_config_t *acq, int sample_size, int nwin) {
    const int64_t w = GPSB200_SNAP_BATCH_SCRATCH / batch_window_bytes(acq, sample_size);
    return (int) std::max<int64_t>(1, std::min<int64_t>(w, nwin));
}

cudaError_t launch(Scratch &sc, const void *window, int sample_size, int K, int nprn, const int8_t *chips, int iterations,
                   gpsb200_snapshot_t *rec, cudaStream_t s) {
    CU_RET(sc.d_rec.grow(32));
    CU_RET(cudaMemcpyAsync(sc.d_rec.get(), rec, nprn * sizeof(gpsb200_snapshot_t), cudaMemcpyHostToDevice, s));
    if (sample_size == GPSB200_SC08)
        k_snapshot<int8_t><<<nprn, kThreads, 0, s>>>(static_cast<const int8_t *>(window), K, chips, iterations,
                                                     sc.d_rec.get());
    else
        k_snapshot<int16_t><<<nprn, kThreads, 0, s>>>(static_cast<const int16_t *>(window), K, chips, iterations,
                                                      sc.d_rec.get());
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(rec, sc.d_rec.get(), nprn * sizeof(gpsb200_snapshot_t), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

cudaError_t launch_batch(Scratch &sc, const void *src, int sample_size, int K, int nwin, int nprn,
                         const int64_t *d_win_off, const int8_t *chips, int iterations, gpsb200_snapshot_t *rec,
                         cudaStream_t s) {
    const int n = nwin * nprn;
    CU_RET(sc.d_brec.grow((size_t) n));
    CU_RET(cudaMemcpyAsync(sc.d_brec.get(), rec, n * sizeof(gpsb200_snapshot_t), cudaMemcpyHostToDevice, s));
    if (sample_size == GPSB200_SC08)
        k_snapshot_batch<int8_t><<<n, kThreads, 0, s>>>(static_cast<const int8_t *>(src), d_win_off, nprn, K, chips,
                                                        iterations, sc.d_brec.get());
    else
        k_snapshot_batch<int16_t><<<n, kThreads, 0, s>>>(static_cast<const int16_t *>(src), d_win_off, nprn, K, chips,
                                                         iterations, sc.d_brec.get());
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(rec, sc.d_brec.get(), n * sizeof(gpsb200_snapshot_t), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

}  // namespace snap
}  // namespace gpsb200
