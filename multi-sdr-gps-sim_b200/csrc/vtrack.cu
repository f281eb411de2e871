// Vector tracking (include/gpsb200.h: gpsb200_vtrack; DESIGN §10.1).
//
// k_vtrack: one thread-block cluster of K CTAs (256 threads each) per call; channel c runs on CTA c mod K, one channel
// after the other. A channel's period is k_track's: every thread wipes off and correlates samples m = tid + 256 r
// (r < 12, m < L), the sums are reduced in a fixed order (warp shuffles, then thread 0 over the 8 warp partials), and
// thread 0 advances the NCOs and adds the period to the interval's sums. When a CTA's channels have their N periods (or
// cannot run another), it writes their states into the leader CTA's (rank 0) shared memory through distributed shared
// memory; after one cluster.sync() warp 0 of the leader runs the filter (lanes = channels for the predictions and
// commands, lane 0 for the time update and the sequential measurement updates), and after a second one every CTA reads
// its channels' commands back. No atomics: every sum has one writer and a fixed order.
#include <cooperative_groups.h>

#include <cmath>
#include <cstring>

#include "device_buffer.h"
#include "orbit.cuh"
#include "rx_samples.cuh"
#include "track.h"
#include "vtrack.h"

namespace gpsb200 {
namespace vtk {

namespace {

namespace cg = cooperative_groups;
using trk::kM;
using trk::kPerThread;
using trk::kThreads;

constexpr int kWarps = kThreads / 32;
constexpr int kMaxChan = GPSB200_TRK_MAX_CHAN;
constexpr double kFs = 3e6;
constexpr double kLambdaChip = kC / 1.023e6;
constexpr double kLambdaL1 = kC / 1575.42e6;
constexpr double k2p32 = 4294967296.0;

struct Lead {                                   // the filter's shared memory, used in the leader CTA only
    gpsb200_vtrack_chan_state_t all[kMaxChan];  // every channel's state at the interval's end
    double X[8], P[64], Xp[8];
    double h[kMaxChan][3], yc[kMaxChan], yr[kMaxChan], vc[kMaxChan], vr[kMaxChan];
    int used[kMaxChan];
    int ready[kMaxCluster];
    int go;
    int seeded, updates;
    int64_t t_f;
};

struct Smem {
    int2 tab[512];
    int32_t part[kWarps][7];
    gpsb200_vtrack_chan_state_t loc[kMaxChan];  // this CTA's channels, j = 0.. (channel rank + j K)
    int32_t nep[kMaxChan];
    int L, go;
    Lead lead;
};

__device__ inline double frac(double x) { return x - floor(x); }

// Header "predict": code phase (chips), unit vector e and range rate of a channel at sample s from X at sample t_f.
__device__ void predict(const gpsb200_ephemeris_t &eph, const double *X, int64_t t_f, int64_t s, int64_t s0, double t0,
                        double &phi, double *e, double &rr) {
    const double dt = (double) (s - t_f) / kFs;
    double r[3];
    for (int i = 0; i < 3; i++) r[i] = X[i] + X[3 + i] * dt;
    const double b = X[6] + X[7] * dt;
    const int64_t d = s - s0;
    const int64_t q = d / 3000, m = d - 3000 * q;   // d >= 0
    const double t = t0 + (double) q / 1000.0 + (double) m / kFs - b / kC;
    double tau = 0.075, p[3], v[3], dts = 0.0, ddt = 0.0, l[3] = {0.0, 0.0, 0.0}, vr[3] = {0.0, 0.0, 0.0};
#pragma unroll 1
    for (int i = 0; i < 3; i++) {
        pvt::satellite(eph, t - tau, p, v, dts, ddt);
        double sth, cth;
        sincos(kOmegaE * tau, &sth, &cth);
        l[0] = p[0] * cth + p[1] * sth - r[0];
        l[1] = p[1] * cth - p[0] * sth - r[1];
        l[2] = p[2] - r[2];
        vr[0] = v[0] * cth + v[1] * sth;
        vr[1] = v[1] * cth - v[0] * sth;
        vr[2] = v[2];
        tau = sqrt(l[0] * l[0] + l[1] * l[1] + l[2] * l[2]) / kC;
    }
    const double F0 = frac(1000.0 * t0);
    phi = 1023.0 * frac(F0 + (double) m / 3000.0 + 1000.0 * (dts - tau - b / kC));
    const double rn = tau * kC;
    for (int i = 0; i < 3; i++) e[i] = l[i] / rn;
    rr = e[0] * (vr[0] - X[3]) + e[1] * (vr[1] - X[4]) + e[2] * (vr[2] - X[5]) - kC * ddt + X[7];
}

__device__ inline int32_t carrier_step(double rr) {
    double f = -rr / kLambdaL1;
    f = f < -10000.0 ? -10000.0 : (f > 10000.0 ? 10000.0 : f);
    return (int32_t) llround(f * k2p32 / kFs);
}

// Header "command": the next interval's u and w of a channel whose NCO code phase is phi_nco.
__device__ void command(double phi, double rr, uint64_t phi_nco, int N, uint32_t &u, int32_t &w) {
    w = carrier_step(rr);
    double err = phi * k2p32 - (double) phi_nco;
    const double half = 0.5 * (double) kM;
    if (err >= half) err -= (double) kM;
    else if (err < -half) err += (double) kM;
    const int64_t e = llround(err);
    int64_t uu = (int64_t) GPSB200_TRK_CODE_STEP_NOM + trk::tdiv(w, 1540) + trk::tdiv(e, 3000ll * N);
    uu = uu < (int64_t) GPSB200_TRK_CODE_STEP_MIN ? (int64_t) GPSB200_TRK_CODE_STEP_MIN
                                                  : (uu > (int64_t) GPSB200_TRK_CODE_STEP_MAX ? (int64_t) GPSB200_TRK_CODE_STEP_MAX : uu);
    u = (uint32_t) uu;
}

// Header "first", lane c of the leader's warp 0.
__device__ __noinline__ void first(Lead &L, const gpsb200_pvt_chan_t *chans, int nchan, int64_t s0, double t0) {
    const int c = threadIdx.x;
    if (c < nchan) {
        double phi, e[3], rr;
        predict(chans[c].eph, L.X, s0, s0, s0, t0, phi, e, rr);
        const int32_t w = carrier_step(rr);
        const uint32_t u = trk::code_step(w);
        const uint64_t phi0 = (uint64_t) llround(phi * k2p32) % kM;
        gpsb200_track_state_t &n = L.all[c].nco;
        if (phi0 == 0) {
            n.sample = s0;
            n.code_phase = 0;
        } else {
            const uint64_t len = (kM - phi0 + u - 1) / u;
            n.sample = s0 + (int64_t) len;
            n.code_phase = phi0 + len * u - kM;
        }
        n.carr_step = w;
        n.code_step = u;
        n.carr_phase = 0;
        L.all[c].start = n.sample;
    }
    if (c == 0) {
        L.t_f = s0;
        L.seeded = 1;
    }
    __syncwarp();
}

// Header "update", warp 0 of the leader: time update, measurements, sequential updates, outputs, commands.
__device__ __noinline__ void update(Lead &L, const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t &cfg, int nchan,
                       int64_t s0, double t0, gpsb200_fix_t *fix, gpsb200_vtrack_chan_t *out) {
    const int lane = threadIdx.x;
    const int N = cfg.periods;
    if (lane == 0) {
        int64_t tn = L.all[0].nco.sample;
        for (int c = 1; c < nchan; c++) tn = L.all[c].nco.sample > tn ? L.all[c].nco.sample : tn;
        const double dt = (double) (tn - L.t_f) / kFs;
        double F[64], FP[64], Q[64];
        for (int i = 0; i < 64; i++) {
            F[i] = (i % 9 == 0) ? 1.0 : 0.0;
            Q[i] = 0.0;
        }
        for (int i = 0; i < 3; i++) F[i * 8 + 3 + i] = dt;
        F[6 * 8 + 7] = dt;
        const double qa = cfg.accel_psd, qb = cfg.bias_psd, qd = cfg.drift_psd;
        const double d2 = dt * dt, d3 = d2 * dt;
        for (int i = 0; i < 3; i++) {
            Q[i * 8 + i] = qa * d3 / 3.0;
            Q[i * 8 + 3 + i] = Q[(3 + i) * 8 + i] = qa * d2 / 2.0;
            Q[(3 + i) * 8 + 3 + i] = qa * dt;
        }
        Q[6 * 8 + 6] = qb * dt + qd * d3 / 3.0;
        Q[6 * 8 + 7] = Q[7 * 8 + 6] = qd * d2 / 2.0;
        Q[7 * 8 + 7] = qd * dt;
        double X[8];
        for (int i = 0; i < 8; i++) {
            double a = 0.0;
            for (int k = 0; k < 8; k++) a += F[i * 8 + k] * L.X[k];
            X[i] = a;
        }
        for (int i = 0; i < 8; i++)
            for (int j = 0; j < 8; j++) {
                double a = 0.0;
                for (int k = 0; k < 8; k++) a += F[i * 8 + k] * L.P[k * 8 + j];
                FP[i * 8 + j] = a;
            }
        for (int i = 0; i < 8; i++)
            for (int j = 0; j < 8; j++) {
                double a = 0.0;
                for (int k = 0; k < 8; k++) a += FP[i * 8 + k] * F[j * 8 + k];
                L.P[i * 8 + j] = a + Q[i * 8 + j];
            }
        for (int i = 0; i < 8; i++) L.X[i] = L.Xp[i] = X[i];
        L.t_f = tn;
    }
    __syncwarp();
    if (lane < nchan) {
        const int c = lane;
        gpsb200_vtrack_chan_state_t &cs = L.all[c];
        const gpsb200_track_state_t &n = cs.nco;
        double phi, e[3], rr;
        predict(chans[c].eph, L.Xp, L.t_f, n.sample, s0, t0, phi, e, rr);
        const double q = cs.s ? (double) cs.p / (GPSB200_VTRK_NOISE_SCALE * (double) cs.s) : 0.0;
        const int used = q >= cfg.q_min ? 1 : 0;
        const int64_t D = trk::dll(cs.e, cs.l);
        const int64_t du = (int64_t) n.code_step - (int64_t) trk::code_step(n.carr_step);
        const int64_t nsamp = n.sample - cs.start;
        double r = (double) n.code_phase / k2p32 + (double) D / 65536.0 - (double) du * (double) nsamp / 8589934592.0 - phi;
        r = r + 511.5;
        r = r - 1023.0 * floor(r / 1023.0) - 511.5;
        const double yc = -kLambdaChip * r;
        const int32_t a = trk::angle(cs.dot, cs.cross);
        const double fm = (double) n.carr_step * kFs / k2p32 + (double) a * 1000.0 / k2p32;
        const double yr = -kLambdaL1 * fm - rr;
        gpsb200_vtrack_chan_t &o = out[c];
        o.sample = n.sample;
        o.e = cs.e;
        o.l = cs.l;
        o.p = cs.p;
        o.s = cs.s;
        o.dot = cs.dot;
        o.cross = cs.cross;
        o.prn = n.prn;
        o.used = used;
        o.q = q;
        o.code_res_m = yc;
        o.rate_res_mps = yr;
        const double vc = cfg.sigma_code_m * cfg.sigma_code_m / ((q - 1.0) * N);
        const double vr = cfg.sigma_rate_mps * cfg.sigma_rate_mps / ((q - 1.0) * N);
        o.sigma_code_m = used ? sqrt(vc) : INFINITY;
        o.sigma_rate_mps = used ? sqrt(vr) : INFINITY;
        for (int i = 0; i < 3; i++) L.h[c][i] = e[i];
        L.yc[c] = yc;
        L.yr[c] = yr;
        L.vc[c] = vc;
        L.vr[c] = vr;
        L.used[c] = used;
    }
    __syncwarp();
    if (lane == 0) {
        double X[8], P[64];
        for (int i = 0; i < 8; i++) X[i] = L.X[i];
        for (int i = 0; i < 64; i++) P[i] = L.P[i];
        for (int c = 0; c < nchan; c++) {
            if (!L.used[c]) continue;
            for (int kind = 0; kind < 2; kind++) {
                double h[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                for (int i = 0; i < 3; i++) h[kind * 3 + i] = -L.h[c][i];
                h[6 + kind] = 1.0;
                double y = kind ? L.yr[c] : L.yc[c];
                double hd = 0.0;
                for (int i = 0; i < 8; i++) hd += h[i] * (X[i] - L.Xp[i]);
                y -= hd;
                double g[8];
                for (int i = 0; i < 8; i++) {
                    double a = 0.0;
                    for (int k = 0; k < 8; k++) a += P[i * 8 + k] * h[k];
                    g[i] = a;
                }
                double s = 0.0;
                for (int i = 0; i < 8; i++) s += h[i] * g[i];
                s += kind ? L.vr[c] : L.vc[c];
                double K[8];
                for (int i = 0; i < 8; i++) K[i] = g[i] / s;
                for (int i = 0; i < 8; i++) X[i] += K[i] * y;
                for (int i = 0; i < 8; i++)
                    for (int j = 0; j < 8; j++) P[i * 8 + j] -= K[i] * g[j];
            }
        }
        for (int i = 0; i < 8; i++) L.X[i] = X[i];
        for (int i = 0; i < 64; i++) L.P[i] = P[i];
        // the fix record
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        gpsb200_fix_t f;
        f.sample = L.t_f;
        int nused = 0;
        uint32_t mask = 0;
        double ss = 0.0, G[16];
        for (int i = 0; i < 16; i++) G[i] = 0.0;
        for (int c = 0; c < nchan; c++) {
            if (!L.used[c]) continue;
            nused++;
            mask |= 1u << c;
            const double g4[4] = {-L.h[c][0], -L.h[c][1], -L.h[c][2], 1.0};
            double hd = 0.0;
            for (int i = 0; i < 3; i++) hd += g4[i] * (X[i] - L.Xp[i]);
            hd += X[6] - L.Xp[6];
            const double res = L.yc[c] - hd;
            ss += res * res;
            for (int i = 0; i < 4; i++)
                for (int j = 0; j < 4; j++) G[i * 4 + j] += g4[i] * g4[j];
        }
        f.status = nused >= 4 ? GPSB200_FIX_OK : GPSB200_FIX_FEW;
        f.nused = nused;
        f.mask = mask;
        f.iterations = 1;
        f.x = X[0];
        f.y = X[1];
        f.z = X[2];
        f.clock_m = X[6];
        f.t_rx = t0 + (double) (L.t_f - s0) / kFs - X[6] / kC;
        f.vx = X[3];
        f.vy = X[4];
        f.vz = X[5];
        f.drift = X[7];
        double lat, lon, hgt;
        pvt::ecef_llh(X, lat, lon, hgt);
        f.lat_deg = lat * 180.0 / kPi;
        f.lon_deg = lon * 180.0 / kPi;
        f.height = hgt;
        f.rms = nused ? sqrt(ss / nused) : nan;
        f.pdop = nan;
        if (nused >= 4) {   // Gauss-Jordan on the 4 x 4 normal matrix (positive definite with 4 independent rows)
            double A[16], Iv[16];
            for (int i = 0; i < 16; i++) {
                A[i] = G[i];
                Iv[i] = (i % 5 == 0) ? 1.0 : 0.0;
            }
            for (int k = 0; k < 4; k++) {
                const double piv = A[k * 4 + k];
                for (int j = 0; j < 4; j++) {
                    A[k * 4 + j] /= piv;
                    Iv[k * 4 + j] /= piv;
                }
                for (int i = 0; i < 4; i++) {
                    if (i == k) continue;
                    const double fct = A[i * 4 + k];
                    for (int j = 0; j < 4; j++) {
                        A[i * 4 + j] -= fct * A[k * 4 + j];
                        Iv[i * 4 + j] -= fct * Iv[k * 4 + j];
                    }
                }
            }
            f.pdop = sqrt(Iv[0] + Iv[5] + Iv[10]);
        }
        *fix = f;
        L.updates += 1;
    }
    __syncwarp();
    if (lane < nchan) {
        const int c = lane;
        gpsb200_vtrack_chan_state_t &cs = L.all[c];
        double phi, e[3], rr;
        predict(chans[c].eph, L.X, L.t_f, cs.nco.sample, s0, t0, phi, e, rr);
        uint32_t u;
        int32_t w;
        command(phi, rr, cs.nco.code_phase, N, u, w);
        out[c].code_step = u;
        out[c].carr_step = w;
        cs.nco.code_step = u;
        cs.nco.carr_step = w;
        cs.used = L.used[c];
        cs.start = cs.nco.sample;
        cs.e = cs.l = cs.p = cs.s = cs.dot = cs.cross = 0;
        cs.k = 0;
    }
    __syncwarp();
}

// Copy n bytes (a multiple of 8) between records of global or shared memory (either may be another CTA's) with the
// CTA's threads.
__device__ inline void copy8(void *dst, const void *src, int n) {
    long long *d = static_cast<long long *>(dst);
    const long long *s = static_cast<const long long *>(src);
    for (int i = threadIdx.x; i < n / 8; i += kThreads) d[i] = s[i];
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_vtrack(const T *__restrict__ iq, int64_t nsamples, int64_t base, const int8_t *__restrict__ chips,
         const gpsb200_pvt_chan_t *__restrict__ chans, const gpsb200_vtrack_config_t cfg,
         gpsb200_vtrack_state_t *__restrict__ state, int max_updates, gpsb200_fix_t *__restrict__ fixes,
         gpsb200_vtrack_chan_t *__restrict__ outs, gpsb200_track_epoch_t *__restrict__ epochs, int max_epochs,
         int32_t *__restrict__ counts) {
    __shared__ Smem sm;
    extern __shared__ int8_t ca[];   // [channels of this CTA][1024]
    cg::cluster_group cl = cg::this_cluster();
    const int K = (int) cl.num_blocks(), rank = (int) cl.block_rank();
    const int tid = threadIdx.x, warp = tid >> 5;
    Lead *lead = cl.map_shared_rank(&sm.lead, 0);
    const int nchan = state->nchan, N = cfg.periods;
    const int64_t s0 = state->s0;
    const double t0 = state->t0;
    rx::fill_carrier_table(sm.tab, kThreads);
    if (rank == 0) {
        copy8(sm.lead.all, state->ch, nchan * (int) sizeof(gpsb200_vtrack_chan_state_t));
        if (tid < 8) sm.lead.X[tid] = state->x[tid];
        if (tid < 64) sm.lead.P[tid] = state->P[tid];
        if (tid == 0) {
            sm.lead.t_f = state->t_f;
            sm.lead.seeded = state->seeded;
            sm.lead.updates = state->updates;
        }
        __syncthreads();
        if (!sm.lead.seeded && warp == 0) first(sm.lead, chans, nchan, s0, t0);
    }
    cl.sync();
    const int nmine = rank < nchan ? (nchan - rank + K - 1) / K : 0;
    for (int j = 0; j < nmine; j++) {
        copy8(&sm.loc[j], &lead->all[rank + j * K], (int) sizeof(gpsb200_vtrack_chan_state_t));
        if (tid == 0) sm.nep[j] = 0;
    }
    __syncthreads();
    for (int j = 0; j < nmine; j++)
        for (int i = tid; i < GPSB200_CA_LEN; i += kThreads) ca[j * 1024 + i] = chips[sm.loc[j].nco.prn * GPSB200_CA_LEN + i];
    const int64_t end = base + nsamples;
    for (int nupd = 0; nupd < max_updates; nupd++) {
        for (int j = 0; j < nmine; j++) {
            gpsb200_vtrack_chan_state_t &cs = sm.loc[j];
            const int8_t *caj = ca + j * 1024;
            for (;;) {
                if (tid == 0) {
                    const int L = trk::period_len(cs.nco.code_phase, cs.nco.code_step);
                    sm.L = (cs.k < N && cs.nco.sample + L <= end) ? L : 0;
                }
                __syncthreads();   // L and the NCO state published (and the chips)
                const int L = sm.L;
                if (L == 0) break;
                const int64_t s = cs.nco.sample - base;
                const uint64_t phi = cs.nco.code_phase;
                const uint32_t u = cs.nco.code_step, theta = cs.nco.carr_phase, w = (uint32_t) cs.nco.carr_step;
                int a[7] = {0, 0, 0, 0, 0, 0, 0};
#pragma unroll
                for (int r = 0; r < kPerThread; r++) {
                    const int m = tid + kThreads * r;
                    if (m < L) {
                        int I, Q;
                        rx::load_iq<T>(iq, s + m, I, Q);
                        const int2 d = rx::wipe_off(sm.tab, theta + (uint32_t) m * w, I, Q);
                        int ce, cp, cl_;
                        rx::epl_chips(caj, phi + (uint64_t) m * u, ce, cp, cl_);
                        a[0] += ce * d.x;
                        a[1] += ce * d.y;
                        a[2] += cp * d.x;
                        a[3] += cp * d.y;
                        a[4] += cl_ * d.x;
                        a[5] += cl_ * d.y;
                        a[6] += I * I + Q * Q;
                    }
                }
                rx::warp_partials(a, sm.part[warp]);
                __syncthreads();
                if (tid == 0) {
                    int32_t c[7];
                    for (int k = 0; k < 7; k++) {
                        int v = 0;
                        for (int q = 0; q < kWarps; q++) v += sm.part[q][k];
                        c[k] = v;
                    }
                    gpsb200_track_state_t &n = cs.nco;
                    const int64_t s_abs = n.sample;
                    n.sample += L;
                    n.carr_phase = theta + (uint32_t) L * w;
                    n.code_phase = phi + (uint64_t) L * u - kM;
                    cs.e += (int64_t) c[0] * c[0] + (int64_t) c[1] * c[1];
                    cs.l += (int64_t) c[4] * c[4] + (int64_t) c[5] * c[5];
                    cs.p += (int64_t) c[2] * c[2] + (int64_t) c[3] * c[3];
                    cs.s += c[6];
                    if (cs.k >= 1) {
                        const trk::CrossDot f = trk::fll(n.prev_i, n.prev_q, c[2], c[3]);
                        cs.cross += f.cross;
                        cs.dot += f.dot;
                    }
                    n.prev_i = c[2];
                    n.prev_q = c[3];
                    n.epochs += 1;
                    cs.k += 1;
                    if (epochs) {
                        gpsb200_track_epoch_t ep;
                        ep.sample = s_abs;
                        ep.e_i = c[0];
                        ep.e_q = c[1];
                        ep.p_i = c[2];
                        ep.p_q = c[3];
                        ep.l_i = c[4];
                        ep.l_q = c[5];
                        ep.carr_phase = n.carr_phase;
                        ep.carr_step = n.carr_step;
                        ep.code_phase = (uint32_t) n.code_phase;
                        ep.code_step = n.code_step;
                        ep.lock = cs.used;
                        ep.reserved = 0;
                        epochs[(size_t) (rank + j * K) * max_epochs + sm.nep[j]] = ep;
                        sm.nep[j] += 1;
                    }
                }
            }
        }
        // publish this CTA's channels to the leader
        for (int j = 0; j < nmine; j++) copy8(&lead->all[rank + j * K], &sm.loc[j], (int) sizeof(gpsb200_vtrack_chan_state_t));
        if (tid == 0) {
            int ready = 1;
            for (int j = 0; j < nmine; j++) ready &= sm.loc[j].k == N;
            lead->ready[rank] = ready;
        }
        cl.sync();
        if (rank == 0 && warp == 0) {
            int go = 1;
            for (int r = 0; r < K; r++) go &= sm.lead.ready[r];
            if (go) update(sm.lead, chans, cfg, nchan, s0, t0, fixes + nupd, outs + (size_t) nupd * nchan);
            if (tid == 0) sm.lead.go = go;
        }
        cl.sync();
        if (tid == 0) sm.go = lead->go;
        __syncthreads();
        if (!sm.go) break;
        for (int j = 0; j < nmine; j++) copy8(&sm.loc[j], &lead->all[rank + j * K], (int) sizeof(gpsb200_vtrack_chan_state_t));
        if (rank == 0 && tid == 0) counts[kMaxChan] = nupd + 1;
        __syncthreads();
    }
    for (int j = 0; j < nmine; j++) {
        copy8(&state->ch[rank + j * K], &sm.loc[j], (int) sizeof(gpsb200_vtrack_chan_state_t));
        if (tid == 0) counts[rank + j * K] = sm.nep[j];
    }
    if (rank == 0) {
        if (tid < 8) state->x[tid] = sm.lead.X[tid];
        if (tid < 64) state->P[tid] = sm.lead.P[tid];
        if (tid == 0) {
            state->t_f = sm.lead.t_f;
            state->seeded = sm.lead.seeded;
            state->updates = sm.lead.updates;
        }
    }
    cl.sync();   // the leader's shared memory outlives every read of it
}

template <typename T>
cudaError_t launch_k(int K, size_t dyn, cudaStream_t s, const T *iq, int64_t nsamples, int64_t base, const int8_t *chips,
                     const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t &cfg, gpsb200_vtrack_state_t *state,
                     int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *outs, gpsb200_track_epoch_t *epochs,
                     int max_epochs, int32_t *counts) {
    CU_RET(cudaFuncSetAttribute(k_vtrack<T>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CU_RET(cudaFuncSetAttribute(k_vtrack<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024));
    cudaLaunchConfig_t lc = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = K;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    lc.gridDim = dim3(K);
    lc.blockDim = dim3(kThreads);
    lc.dynamicSmemBytes = dyn;
    lc.stream = s;
    lc.attrs = attr;
    lc.numAttrs = 1;
    return cudaLaunchKernelEx(&lc, k_vtrack<T>, iq, nsamples, base, chips, chans, cfg, state, max_updates, fixes, outs,
                              epochs, max_epochs, counts);
}

}  // namespace

std::string check_config(const gpsb200_vtrack_config_t *cfg) {
    if (!cfg) return "config is NULL";
    if (cfg->periods < 1 || cfg->periods > GPSB200_VTRK_MAX_PERIODS) return "periods must be 1..100";
    if (cfg->reserved != 0) return "reserved must be 0";
    const double pos[] = {cfg->sigma_code_m, cfg->sigma_rate_mps, cfg->sigma_pos, cfg->sigma_vel, cfg->sigma_bias,
                          cfg->sigma_drift};
    for (double v : pos)
        if (!(v > 0.0) || !std::isfinite(v)) return "sigmas must be finite and > 0";
    if (!(cfg->q_min > 1.0) || !std::isfinite(cfg->q_min)) return "q_min must be finite and > 1";
    const double psd[] = {cfg->accel_psd, cfg->bias_psd, cfg->drift_psd};
    for (double v : psd)
        if (!(v >= 0.0) || !std::isfinite(v)) return "process noise densities must be finite and >= 0";
    return std::string();
}

std::string check(const gpsb200_vtrack_state_t *st, const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg,
                  int max_updates, bool epochs, int max_epochs, int64_t nsamples, int64_t base, int sample_size) {
    if (!st || !chans) return "state or chans is NULL";
    std::string bad = check_config(cfg);
    if (!bad.empty()) return bad;
    if (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16) return "sample_size must be GPSB200_SC08 or GPSB200_SC16";
    if (st->nchan < 1 || st->nchan > GPSB200_TRK_MAX_CHAN) return "state nchan must be 1..32";
    if (max_updates < 1) return "max_updates must be >= 1";
    if (epochs && (int64_t) max_epochs < ((int64_t) max_updates + 1) * cfg->periods)
        return "max_epochs must be >= (max_updates + 1) * periods";
    if (nsamples < 0 || base < 0) return "nsamples and base must be >= 0";
    if ((!st->seeded && st->s0 < base) || st->s0 < 0 || st->t_f < st->s0)
        return "s0 must be >= 0 (and >= base before the first call) and t_f >= s0";
    if (st->seeded != 0 && st->seeded != 1) return "seeded must be 0 or 1";
    if (!(st->t0 >= 0.0 && st->t0 < 604800.0 + 1.0)) return "t0 outside the week";
    for (int i = 0; i < 8; i++)
        if (!std::isfinite(st->x[i])) return "X is not finite";
    for (int i = 0; i < 64; i++)
        if (!std::isfinite(st->P[i])) return "P is not finite";
    uint32_t seen = 0;   // a repeated PRN would count one satellite's measurements twice and make G singular
    for (int c = 0; c < st->nchan; c++) {
        const gpsb200_vtrack_chan_state_t &cs = st->ch[c];
        const std::string at = "channel " + std::to_string(c) + ": ";
        if (cs.nco.prn < 1 || cs.nco.prn > 32) return at + "PRN outside 1..32";
        if (seen >> (cs.nco.prn - 1) & 1u) return at + "PRN already on an earlier channel";
        seen |= 1u << (cs.nco.prn - 1);
        if (chans[c].prn != cs.nco.prn) return at + "chans[c].prn is not the channel's PRN";
        if (!chans[c].eph.valid) return at + "no valid ephemeris";
        if (cs.k < 0 || cs.k > cfg->periods) return at + "k outside 0..periods";
        if (st->seeded) {
            if (cs.nco.code_step < GPSB200_TRK_CODE_STEP_MIN || cs.nco.code_step > GPSB200_TRK_CODE_STEP_MAX)
                return at + "code_step outside GPSB200_TRK_CODE_STEP_MIN..MAX";
            if (cs.nco.code_phase >= GPSB200_TRK_CODE_STEP_MAX) return at + "code_phase must be below GPSB200_TRK_CODE_STEP_MAX";
            if (cs.nco.sample < base || cs.start > cs.nco.sample || cs.start < st->s0)
                return at + "the next period starts before the buffer or the interval before s0";
            if (cs.e < 0 || cs.l < 0 || cs.p < 0 || cs.s < 0 || cs.dot < 0) return at + "negative interval sums";
        }
    }
    return std::string();
}

cudaError_t scratch_reserve(Scratch &sc, int nchan, int max_updates, int max_epochs) {
    CU_RET(sc.d_state.grow(1));
    CU_RET(sc.d_chans.grow(kMaxChan));
    CU_RET(sc.d_n.grow(kMaxChan + 1));
    CU_RET(sc.d_fix.grow((size_t) max_updates));
    CU_RET(sc.d_out.grow((size_t) max_updates * nchan));
    if (max_epochs > 0) CU_RET(sc.d_epochs.grow((size_t) nchan * max_epochs));
    return cudaSuccess;
}

cudaError_t launch(Scratch &sc, const int8_t *chips, const void *src, int64_t nsamples, int sample_size, int64_t base,
                   const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg, gpsb200_vtrack_state_t *state,
                   int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *out, int32_t *nupdates,
                   gpsb200_track_epoch_t *epochs, int max_epochs, int32_t *nepochs, int ctas, cudaStream_t s) {
    const int nchan = state->nchan;
    const int K = ctas > 0 ? (ctas < nchan ? ctas : nchan) : (nchan < 8 ? nchan : 8);
    const size_t dyn = (size_t) ((nchan + K - 1) / K) * 1024;
    CU_RET(cudaMemcpyAsync(sc.d_state.get(), state, sizeof(gpsb200_vtrack_state_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_chans.get(), chans, nchan * sizeof(gpsb200_pvt_chan_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemsetAsync(sc.d_n.get(), 0, (kMaxChan + 1) * sizeof(int32_t), s));
    gpsb200_track_epoch_t *dep = epochs ? sc.d_epochs.get() : nullptr;
    if (sample_size == GPSB200_SC08)
        CU_RET(launch_k<int8_t>(K, dyn, s, static_cast<const int8_t *>(src), nsamples, base, chips, sc.d_chans.get(),
                                *cfg, sc.d_state.get(), max_updates, sc.d_fix.get(), sc.d_out.get(), dep, max_epochs,
                                sc.d_n.get()));
    else
        CU_RET(launch_k<int16_t>(K, dyn, s, static_cast<const int16_t *>(src), nsamples, base, chips, sc.d_chans.get(),
                                 *cfg, sc.d_state.get(), max_updates, sc.d_fix.get(), sc.d_out.get(), dep, max_epochs,
                                 sc.d_n.get()));
    int32_t n[kMaxChan + 1];
    CU_RET(cudaMemcpyAsync(n, sc.d_n.get(), sizeof n, cudaMemcpyDeviceToHost, s));
    CU_RET(cudaMemcpyAsync(state, sc.d_state.get(), sizeof(gpsb200_vtrack_state_t), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaStreamSynchronize(s));
    *nupdates = n[kMaxChan];
    if (n[kMaxChan] > 0) {
        CU_RET(cudaMemcpyAsync(fixes, sc.d_fix.get(), (size_t) n[kMaxChan] * sizeof(gpsb200_fix_t),
                               cudaMemcpyDeviceToHost, s));
        CU_RET(cudaMemcpyAsync(out, sc.d_out.get(), (size_t) n[kMaxChan] * nchan * sizeof(gpsb200_vtrack_chan_t),
                               cudaMemcpyDeviceToHost, s));
    }
    if (epochs)
        for (int c = 0; c < nchan; c++) {
            nepochs[c] = n[c];
            if (n[c] > 0)
                CU_RET(cudaMemcpyAsync(epochs + (size_t) c * max_epochs, sc.d_epochs.get() + (size_t) c * max_epochs,
                                       (size_t) n[c] * sizeof(gpsb200_track_epoch_t), cudaMemcpyDeviceToHost, s));
        }
    return cudaStreamSynchronize(s);
}

}  // namespace vtk
}  // namespace gpsb200
