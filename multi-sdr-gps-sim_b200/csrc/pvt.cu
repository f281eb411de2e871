// Position, velocity and time (include/gpsb200.h: gpsb200_pvt; DESIGN §11).
//
// k_pvt: one warp per fix instant, lane = channel (nchan <= 32, so one warp holds every channel of the call). Each lane
// finds its code period by a binary search bracketed by the 2999..3001-sample period length, forms its measurement in
// integers, and evaluates its satellite once (Kepler, orbit, clock). Every Gauss-Newton iteration does the Earth rotation
// and the Klobuchar delay per lane and sums the normal equations over the warp with an XOR butterfly: both lanes of a
// pair add the same two values, so every lane ends with the same bits and solves the 4 x 4 system identically. No
// atomics, no shared memory; the kernel is bound by FP64 arithmetic (the trigonometry of the orbit and the iterations).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#include "device_buffer.h"
#include "orbit.cuh"
#include "pvt.h"
#include "synth_tables.h"

namespace gpsb200 {
namespace pvt {

namespace {

constexpr double kCms = 2.99792458e5;             // metres per ms of light time
constexpr double kCodeMod = 1023.0 * 4294967296.0;   // 2^-32 chips per code period
constexpr double kStepHz = 3e6 / 4294967296.0;    // carrier step unit, Hz
constexpr double kIonoMinRadius = 6e6;            // the Klobuchar term needs an estimate near the surface
constexpr double kConverged = 1e-4;               // m
constexpr double kRunaway = 1e8;                  // m from the Earth's centre: a diverging estimate, given up
constexpr unsigned kFull = 0xffffffffu;

struct Args {
    const gpsb200_track_epoch_t *ep;
    const gpsb200_pvt_chan_t *ch;
    const int32_t *n;
    int nchan, max_epochs, ref;
    int64_t ref_sample, ref_ms;
    gpsb200_pvt_config_t cfg;
    gpsb200_fix_t *fixes;
    double *res;
};

// The RAIM instantiation's arguments: the tables go up with the launch. Args comes first, so the fields the plain
// instantiation reads sit at the same parameter offsets in both.
struct RaimArgs : Args {
    gpsb200_raim_config_t raim;
    double T[GPSB200_RAIM_MAX_DOF], lambda[GPSB200_RAIM_MAX_DOF];
    gpsb200_raim_t *out;
};
// The ARAIM instantiation's: K_fa,H / K_fa,V for n = 5..32 go up with the launch, as the chi^2 tables do.
struct AraimArgs : Args {
    gpsb200_araim_config_t araim;
    double kh[GPSB200_RAIM_MAX_DOF], kv[GPSB200_RAIM_MAX_DOF];
    gpsb200_araim_t *out;
};
template <bool kRaim> using KernelArgs = typename std::conditional<kRaim, RaimArgs, Args>::type;

__constant__ double kUraNom[15] = {2.0, 2.8, 4.0, 5.7, 8.0, 11.3, 16.0, 32.0, 64.0, 128.0, 256.0, 512.0, 1024.0, 2048.0,
                                   4096.0};
constexpr double kTenDeg = 10.0 * M_PI / 180.0;

__device__ inline int64_t floor_div(int64_t a, int64_t b) {
    const int64_t q = a / b;
    return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

__device__ inline double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

__device__ inline double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, o));
    return v;
}

// The largest v over the warp and its lane j, the lowest lane on ties; every lane ends with the same pair.
__device__ inline void warp_argmax(double &v, int &j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(kFull, v, o);
        const int oj = __shfl_xor_sync(kFull, j, o);
        if (ov > v || (ov == v && oj < j)) {
            v = ov;
            j = oj;
        }
    }
}

// Cholesky solve of the symmetric N x N system, packed as its upper triangle row by row (N = 4: n00 n01 n02 n03 n11 n12
// n13 n22 n23 n33). factor is false when the system is not positive definite. solve<n> uses the leading n x n block,
// whose factor is the leading block of the whole factor.
template <int N> struct Chol {
    double l[N][N];
    __device__ bool factor(const double *P) {
        double a[N][N];
        if constexpr (N == 4) {
            // Loaded by the loop below, the 4 x 4 system moved the register allocation of k_pvt's RAIM instantiation:
            // 17.62-17.74 ms against 17.46-17.57 ms (tools/pvt_bench.py --raim, H100 80GB HBM3, 700 W).
            const double b[4][4] = {{P[0], P[1], P[2], P[3]}, {P[1], P[4], P[5], P[6]}, {P[2], P[5], P[7], P[8]},
                                    {P[3], P[6], P[8], P[9]}};
            for (int i = 0; i < 4; i++)
                for (int j = 0; j < 4; j++) a[i][j] = b[i][j];
        } else {
            int t = 0;
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = i; j < N; j++) a[i][j] = a[j][i] = P[t++];
        }
#pragma unroll
        for (int j = 0; j < N; j++) {
            double d = a[j][j];
#pragma unroll
            for (int k = 0; k < j; k++) d -= l[j][k] * l[j][k];
            if (!(d > 0.0)) return false;
            l[j][j] = sqrt(d);
#pragma unroll
            for (int i = j + 1; i < N; i++) {
                double v = a[i][j];
#pragma unroll
                for (int k = 0; k < j; k++) v -= l[i][k] * l[j][k];
                l[i][j] = v / l[j][j];
            }
        }
        return true;
    }
    template <int n = N> __device__ void solve(const double *b, double *x) const {
        double y[n];
#pragma unroll
        for (int i = 0; i < n; i++) {
            double v = b[i];
#pragma unroll
            for (int k = 0; k < i; k++) v -= l[i][k] * y[k];
            y[i] = v / l[i][i];
        }
#pragma unroll
        for (int i = n - 1; i >= 0; i--) {
            double v = y[i];
#pragma unroll
            for (int k = i + 1; k < n; k++) v -= l[k][i] * x[k];
            x[i] = v / l[i][i];
        }
    }
};

// The Klobuchar delay in metres (the reference's ionosphericDelay, gps.c:1893-1964, with a valid alpha / beta set).
// Fm (not NULL): receives the obliquity factor F and the geomagnetic latitude phi_m (semicircles) as well.
__device__ double klobuchar(const gpsb200_pvt_config_t &cfg, double lat, double lon, double az, double el, double t,
                            double *Fm = nullptr) {
    const double E = el / kPi, phi_u = lat / kPi, lam_u = lon / kPi;
    const double om = 0.53 - E;
    const double F = 1.0 + 16.0 * om * om * om;
    const double psi = 0.0137 / (E + 0.11) - 0.022;
    double phi_i = phi_u + psi * cos(az);
    phi_i = phi_i > 0.416 ? 0.416 : (phi_i < -0.416 ? -0.416 : phi_i);
    const double lam_i = lam_u + psi * sin(az) / cos(phi_i * kPi);
    const double phi_m = phi_i + 0.064 * cos((lam_i - 1.617) * kPi);
    if (Fm) {
        Fm[0] = F;
        Fm[1] = phi_m;
    }
    const double pm2 = phi_m * phi_m, pm3 = pm2 * phi_m;
    double amp = cfg.alpha[0] + cfg.alpha[1] * phi_m + cfg.alpha[2] * pm2 + cfg.alpha[3] * pm3;
    if (amp < 0.0) amp = 0.0;
    double per = cfg.beta[0] + cfg.beta[1] * phi_m + cfg.beta[2] * pm2 + cfg.beta[3] * pm3;
    if (per < 72000.0) per = 72000.0;
    double tl = 43200.0 * lam_i + t;
    tl -= 86400.0 * floor(tl / 86400.0);
    const double X = 2.0 * kPi * (tl - 50400.0) / per;
    if (fabs(X) < 1.57) {
        const double X2 = X * X;
        return F * (5.0e-9 + amp * (1.0 - X2 / 2.0 + X2 * X2 / 24.0)) * kC;
    }
    return F * 5.0e-9 * kC;
}

// The code period k >= 1 of a channel holding sample s (epochs[k].sample <= s < epochs[k + 1].sample), -1 if none.
__device__ int find_period(const gpsb200_track_epoch_t *e, int n, int64_t s) {
    if (n < 3 || s < e[1].sample || s >= e[n - 1].sample) return -1;
    // periods hold 2999..3001 samples, so k lies within [d / 3001 - 1, d / 2999 + 1]; check, else search everything
    const int64_t d = s - e[0].sample;
    int lo = (int) max((int64_t) 1, d / 3001 - 1), hi = (int) min((int64_t) (n - 2), d / 2999 + 1);
    for (int pass = 0; pass < 2; pass++) {
        if (lo <= hi) {
            int L = lo, H = hi;
            while (L < H) {
                const int mid = (L + H + 1) >> 1;
                if (e[mid].sample <= s) L = mid;
                else H = mid - 1;
            }
            if (e[L].sample <= s && s < e[L + 1].sample) return L;
        }
        lo = 1;
        hi = n - 2;
    }
    return -1;
}

// The eligibility test of a lane's channel at sample s: a valid, healthy ephemeris and a code period k >= 1 holding s
// whose two epochs are locked. Returns k, with the code phase at s (frac, ms) and the range rate (m/s) of that period;
// -1 when the channel fails the test.
__device__ __forceinline__ int locked_period(const Args &a, int lane, int64_t s, double &frac, double &rate) {
    const gpsb200_pvt_chan_t &c = a.ch[lane];
    const gpsb200_track_epoch_t *e = a.ep + (size_t) lane * a.max_epochs;
    const int k = c.eph.valid && c.eph.health == 0 ? find_period(e, a.n[lane], s) : -1;
    if (!(k >= 1 && e[k - 1].lock && e[k].lock)) return -1;
    const uint64_t phi = (uint64_t) e[k - 1].code_phase + (uint64_t) (s - e[k].sample) * e[k - 1].code_step;
    frac = (double) phi / kCodeMod;
    rate = -kLambda * ((double) e[k - 1].carr_step * kStepHz);
    return k;
}

// The measurement of a lane's channel at sample s for a fix with the time anchor (DESIGN §11): q whole ms and m samples
// after the reference channel's anchor, the pseudorange rho, the range rate and the satellite (position, velocity,
// clock offset and drift) at its transmit time. false, with nothing written, when the channel fails locked_period (or,
// with ura, has URA index 15) or the transmit time lies more than 2 h from toe.
__device__ __forceinline__ bool measure(const Args &a, int lane, int64_t s, int64_t q, int64_t m, bool ura, double &rho,
                                        double &rate, double *p, double *v, double &dtsv, double &ddtsv) {
    if (lane >= a.nchan || a.ref < 0) return false;
    const gpsb200_pvt_chan_t &c = a.ch[lane];
    if (ura && !(c.eph.ura >= 0 && c.eph.ura < 15)) return false;
    double frac, rt;
    const int k = locked_period(a, lane, s, frac, rt);
    if (k < 1) return false;
    const int64_t T = (((c.anchor_ms + k - c.anchor_epoch) % kWeekMs) + kWeekMs) % kWeekMs;
    const double tsv = (double) T * 1e-3 + frac * 1e-3;
    if (!(fabs(wrap_half_week(tsv - c.eph.toe)) <= 7200.0)) return false;
    int64_t D = (a.ref_ms + 75 + q - T) % kWeekMs;
    D = D >= kWeekMs / 2 ? D - kWeekMs : (D < -kWeekMs / 2 ? D + kWeekMs : D);
    rho = (double) D * kCms + ((double) m / 3000.0 - frac) * kCms;
    rate = rt;
    const double d0 = wrap_half_week(tsv - c.eph.toc);
    const double tt = tsv - (c.eph.af0 + d0 * (c.eph.af1 + d0 * c.eph.af2));
    satellite(c.eph, tt, p, v, dtsv, ddtsv);
    return true;
}

// A lane's row at the estimate X: the satellite at p, v (ECEF at its transmit time) turned by the Earth's rotation over
// the flight time. Gives the line of sight l, its length R and the turned velocity pv; with enu, also l's azimuth and
// elevation in the frame g (az and el are left as they are without).
__device__ __forceinline__ void sight(const double *p, const double *v, const double *X, const Geo &g, bool enu,
                                      double *l, double &R, double *pv, double &az, double &el) {
    const double g0 = p[0] - X[0], g1 = p[1] - X[1], g2 = p[2] - X[2];
    const double tau = sqrt(g0 * g0 + g1 * g1 + g2 * g2) / kC;
    double sth, cth;
    sincos(kOmegaE * tau, &sth, &cth);
    const double px = p[0] * cth + p[1] * sth, py = p[1] * cth - p[0] * sth;
    pv[0] = v[0] * cth + v[1] * sth;
    pv[1] = v[1] * cth - v[0] * sth;
    pv[2] = v[2];
    l[0] = px - X[0];
    l[1] = py - X[1];
    l[2] = p[2] - X[2];
    R = sqrt(l[0] * l[0] + l[1] * l[1] + l[2] * l[2]);
    if (enu) {
        const double nn = -g.sla * g.clo * l[0] - g.sla * g.slo * l[1] + g.cla * l[2];
        const double ee = -g.slo * l[0] + g.clo * l[1];
        const double uu = g.cla * g.clo * l[0] + g.cla * g.slo * l[1] + g.sla * l[2];
        az = atan2(ee, nn);
        if (az < 0.0) az += 2.0 * kPi;
        el = atan2(uu, sqrt(nn * nn + ee * ee));
    }
}

// The record of a fix instant before its solve, and of one without a fix: NaN fields, the status and the channels used.
__device__ inline void no_fix(gpsb200_fix_t &f, int64_t s, int nused, unsigned mask, int status) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    f.sample = s;
    f.nused = nused;
    f.mask = mask;
    f.iterations = 0;
    f.status = status;
    f.x = f.y = f.z = f.clock_m = f.t_rx = f.vx = f.vy = f.vz = f.drift = nan;
    f.lat_deg = f.lon_deg = f.height = f.pdop = f.rms = nan;
}

// The record of a converged fix X (position and clock first), ch the factor of its last iteration and trx its receive
// time before the fold into the week: velocity and drift on the rows h of the lanes in use, y weighted by wy; PDOP; the
// rms of the post-fit residuals resid; latitude / longitude (also returned, rad) and height.
template <int N>
__device__ __forceinline__ void finish(const Chol<N> &ch, const double *X, double trx, bool use, const double *h,
                                       const double *pv, double rate, double ddtsv, double wy, double resid, int nused,
                                       gpsb200_fix_t &f, double &lat, double &lon) {
    const double y = use ? (rate + kC * ddtsv + (h[0] * pv[0] + h[1] * pv[1] + h[2] * pv[2])) * wy : 0.0;
    const double bv[4] = {warp_sum(h[0] * y), warp_sum(h[1] * y), warp_sum(h[2] * y), warp_sum(y)};
    double V[4];
    ch.template solve<4>(bv, V);
    const double ss = warp_sum(use ? resid * resid : 0.0);
    double Q[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double ei[N] = {}, xi[N];
        ei[i] = 1.0;
        ch.solve(ei, xi);
        Q[i] = xi[i];
    }
    f.status = GPSB200_FIX_OK;
    f.x = X[0];
    f.y = X[1];
    f.z = X[2];
    f.clock_m = X[3];
    f.t_rx = trx < 0.0 ? trx + 604800.0 : (trx >= 604800.0 ? trx - 604800.0 : trx);
    f.vx = V[0];
    f.vy = V[1];
    f.vz = V[2];
    f.drift = V[3];
    double hgt;
    ecef_llh(X, lat, lon, hgt);
    f.lat_deg = lat * (180.0 / M_PI);
    f.lon_deg = lon * (180.0 / M_PI);
    f.height = hgt;
    f.pdop = sqrt(Q[0] + Q[1] + Q[2]);
    f.rms = sqrt(ss / (double) nused);
}

// ---- ARAIM (DESIGN §11.2) --------------------------------------------------------------------------------------------
__device__ inline double q_tail(double x) { return 0.5 * erfc(x / M_SQRT2); }          // the standard normal upper tail
__device__ inline double q_inv(double p) { return M_SQRT2 * erfcinv(2.0 * p); }

// One solution-separation pass at a fix (header, step 5-6): this lane's fault hypothesis k and hypothesis 0.
struct Ss {
    double dx[3], T[3], b[3], s[3];   // east, north, up of hypothesis k (this lane's channel, when in the set)
    double b0[3], s0[3];              // hypothesis 0 (the same on every lane)
    double ratio;                     // max_q |dx_q| / T_q; -1 outside the set
    bool pass;                        // |dx_q| <= T_q for every q (true outside the set)
    bool pd;                          // G^T W(k) G positive definite (true outside the set)
};

// use: this lane's channel is in the set; h, sw (= 1 / sigma_int), r: its row, weight and prefit residual of the last
// Gauss-Newton iteration, acc2 = sigma_acc^2; N, ch: that iteration's normal matrix and its factor; X: the fix. The
// subset solutions come from N_k = N - w_k g_k g_k^T, which each lane factors itself; the sums over the other channels'
// rows run in one loop over the lanes (__shfl_sync), O(n^2) per fix. Returns sigma_acc,U.
__device__ double mhss(const AraimArgs &a, bool use, int n, const double *h, double sw, double r, double acc2,
                       const double *N, const Chol<4> &ch, const double *X, Ss &o) {
    const int lane = threadIdx.x & 31;
    Geo g;
    g.set(X);
    const double u[3][3] = {{-g.slo, g.clo, 0.0}, {-g.sla * g.clo, -g.sla * g.slo, g.cla},
                            {g.cla * g.clo, g.cla * g.slo, g.sla}};
    // the normal matrix less this lane's row
    const double w0 = use ? h[0] * sw : 0.0, w1 = use ? h[1] * sw : 0.0, w2 = use ? h[2] * sw : 0.0, wc = use ? sw : 0.0;
    const double Nk[10] = {N[0] - w0 * w0, N[1] - w0 * w1, N[2] - w0 * w2, N[3] - w0 * wc, N[4] - w1 * w1,
                           N[5] - w1 * w2, N[6] - w1 * wc, N[7] - w2 * w2, N[8] - w2 * wc, N[9] - wc * wc};
    Chol<4> ck;
    const bool fk = use && ck.factor(Nk);
    o.pd = !use || fk;
    double z[3][4], z0[3][4];   // N_k^-1 u_q and N^-1 u_q
#pragma unroll
    for (int q = 0; q < 3; q++) {
        const double e[4] = {u[q][0], u[q][1], u[q][2], 0.0};
        ch.solve(e, z0[q]);
        o.s0[q] = sqrt(e[0] * z0[q][0] + e[1] * z0[q][1] + e[2] * z0[q][2]);
        if (fk) {
            ck.solve(e, z[q]);
            o.s[q] = sqrt(e[0] * z[q][0] + e[1] * z[q][1] + e[2] * z[q][2]);
        } else {
            z[q][0] = z[q][1] = z[q][2] = z[q][3] = 0.0;
            o.s[q] = 0.0;
        }
    }
    // S(k)_qi = w_i z_q . g_i (i != k), S0_qi = w_i z0_q . g_i, summed over the set's channels i
    const double wself = use ? sw * sw : 0.0;
    double bb[3] = {0, 0, 0}, ss[3] = {0, 0, 0}, dx[3] = {0, 0, 0};
#pragma unroll 1
    for (int i = 0; i < a.nchan; i++) {
        const double g0 = __shfl_sync(kFull, h[0], i), g1 = __shfl_sync(kFull, h[1], i), g2 = __shfl_sync(kFull, h[2], i);
        const double wi = __shfl_sync(kFull, wself, i), yi = __shfl_sync(kFull, r, i), ai = __shfl_sync(kFull, acc2, i);
#pragma unroll
        for (int q = 0; q < 3; q++) {
            const double Sk = i == lane ? 0.0 : wi * (z[q][0] * g0 + z[q][1] * g1 + z[q][2] * g2 + z[q][3]);
            const double dS = Sk - wi * (z0[q][0] * g0 + z0[q][1] * g1 + z0[q][2] * g2 + z0[q][3]);
            bb[q] += fabs(Sk);
            ss[q] += dS * dS * ai;
            dx[q] += dS * yi;
        }
    }
    const double kfa[3] = {a.kh[n - 5], a.kh[n - 5], a.kv[n - 5]};
    o.pass = true;
    o.ratio = -1.0;
    double sacc = 0.0;
#pragma unroll
    for (int q = 0; q < 3; q++) {
        const double S0 = wself * (z0[q][0] * h[0] + z0[q][1] * h[1] + z0[q][2] * h[2] + z0[q][3]);
        o.b0[q] = a.araim.b_nom * warp_sum(fabs(S0));
        if (q == 2) sacc = sqrt(warp_sum(S0 * S0 * acc2));
        o.dx[q] = dx[q];
        o.b[q] = a.araim.b_nom * bb[q];
        o.T[q] = kfa[q] * sqrt(ss[q]);
        if (use) {
            o.pass = o.pass && fabs(dx[q]) <= o.T[q];
            o.ratio = fmax(o.ratio, fabs(dx[q]) / o.T[q]);
        }
    }
    return sacc;
}

// The smallest level L with 2 Q((L - b0) / s0) + sum over the set's lanes of p_sat Q((L - T - b) / s) <= rhs, by
// bisection to 1e-3 m (header, step 8). Every lane takes the same branches: the sums are butterflies.
__device__ double protection_level(double rhs, double b0, double s0, bool use, double T, double b, double s,
                                   double p_sat, int n) {
    const double m = (double) (n + 1);
    double lo = b0 + s0 * q_inv(rhs / 2.0), hi = b0 + s0 * q_inv(rhs / m / 2.0);
    lo = fmax(lo, warp_max(use && rhs < p_sat ? T + b + s * q_inv(rhs / p_sat) : -HUGE_VAL));
    hi = fmax(hi, warp_max(use && rhs / m < p_sat ? T + b + s * q_inv(rhs / m / p_sat) : -HUGE_VAL));
#pragma unroll 1
    for (int it = 0; it < 200 && hi - lo > 1e-3; it++) {
        const double mid = 0.5 * (lo + hi);
        const double lhs = 2.0 * q_tail((mid - b0) / s0) + warp_sum(use ? p_sat * q_tail((mid - T - b) / s) : 0.0);
        if (lhs <= rhs) hi = mid;
        else lo = mid;
    }
    return hi;
}

// P_NM = 1 - (1 - p)^n - n p (1 - p)^(n-1), summed as the binomial tail sum_{j >= 2} C(n, j) p^j (1 - p)^(n-j), which
// has no cancellation.
__device__ double p_not_monitored(double p, int n) {
    double t = 0.5 * n * (n - 1) * p * p * pow(1.0 - p, (double) (n - 2)), sum = 0.0;
#pragma unroll 1
    for (int j = 2; j <= n; j++) {
        sum += t;
        t *= (double) (n - j) / (double) (j + 1) * (p / (1.0 - p));
    }
    return sum;
}

// kRaim: the RAIM stage of gpsb200_pvt_raim after the solve (DESIGN §11.1). Each lane keeps two flags: `has` (a
// measurement) and `use` (in the solve). An excluded lane still evaluates its row every iteration, with weight 0, so the
// same warp sums serve every pass, and its residual against the final fix comes out of the same formula. The RAIM
// instantiation is held to 128 registers (4 CTAs per SM, as the plain one) at the price of some spills: at its natural
// 160 it ran 3 CTAs per SM and 15 % slower (DESIGN §11.1).
template <bool kRaim>
__global__ void __launch_bounds__(kWarps * 32, kRaim ? 4 : 0) k_pvt(const KernelArgs<kRaim> a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;   // the whole warp leaves together
    const int64_t s = a.cfg.s0 + fi * a.cfg.step;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);

    // ---- the measurement of this lane's channel (integers), its satellite (FP64) ----
    double rho = 0.0, rate = 0.0, dtsv = 0.0, ddtsv = 0.0, p[3] = {0, 0, 0}, v[3] = {0, 0, 0};
    // the nominal receive time: whole ms of week and the sub-ms sample offset from the reference channel's anchor
    const int64_t ds = s - a.ref_sample;
    const int64_t q = floor_div(ds, 3000), m = ds - 3000 * q;
    const int64_t nom_ms = (((a.ref_ms + 75 + q) % kWeekMs) + kWeekMs) % kWeekMs;
    bool use = measure(a, lane, s, q, m, false, rho, rate, p, v, dtsv, ddtsv);
    const bool has = use;
    unsigned mask = __ballot_sync(kFull, use);
    int nused = __popc(mask);
    gpsb200_fix_t f;
    no_fix(f, s, nused, mask, nused < 4 ? GPSB200_FIX_FEW : GPSB200_FIX_NO_CONVERGENCE);
    double resid = nan;
    // RAIM: the record, and this lane's N^-1 g (position part) and 1 - h_jj of the last pass
    int verdict = GPSB200_RAIM_UNAVAILABLE, dof = 0;
    unsigned excluded = 0;
    double stat = nan, thr = nan, hpl = nan, vpl = nan, xg[3] = {0, 0, 0}, omh = 0.0;
    if (nused >= 4) {
        double X[4] = {0.0, 0.0, 0.0, 0.0};
        double h[3] = {0, 0, 0}, r = 0.0, pr_v[3] = {0, 0, 0};
        Chol<4> ch;
        bool ok = false;
        double dX[4] = {0, 0, 0, 0};
        int it0 = 0;   // iterations of the earlier passes
#pragma unroll 1
        for (;;) {     // Gauss-Newton passes: one, or (RAIM) one more per exclusion, from the previous pass's fix
#pragma unroll 1
        for (int j = 0; j < GPSB200_PVT_MAX_ITER; j++) {
            const double rad = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
            const bool iono = a.cfg.iono && rad >= kIonoMinRadius;
            Geo g;
            if (iono) g.set(X);
            h[0] = h[1] = h[2] = 0.0;
            r = 0.0;
            if (has) {
                double l[3], R, az = 0.0, el = 0.0, I = 0.0;
                sight(p, v, X, g, iono, l, R, pr_v, az, el);
                if (iono)
                    I = klobuchar(a.cfg, g.lat, g.lon, az, el, (double) nom_ms * 1e-3 + (double) m / 3e6 - X[3] / kC);
                r = rho - (R + X[3] - kC * dtsv + I);
                h[0] = -l[0] / R;
                h[1] = -l[1] / R;
                h[2] = -l[2] / R;
            }
            // an excluded lane's row enters with weight 0
            const double w0 = kRaim && !use ? 0.0 : h[0], w1 = kRaim && !use ? 0.0 : h[1], w2 = kRaim && !use ? 0.0 : h[2];
            const double N[10] = {warp_sum(w0 * w0), warp_sum(w0 * w1), warp_sum(w0 * w2), warp_sum(w0),
                                  warp_sum(w1 * w1), warp_sum(w1 * w2), warp_sum(w1),
                                  warp_sum(w2 * w2), warp_sum(w2), (double) nused};
            const double b[4] = {warp_sum(w0 * r), warp_sum(w1 * r), warp_sum(w2 * r), warp_sum(use ? r : 0.0)};
            f.iterations = it0 + j + 1;
            if (!ch.factor(N)) break;
            ch.solve(b, dX);
#pragma unroll
            for (int i = 0; i < 4; i++) X[i] += dX[i];
            if (sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]) > kRunaway) break;
            if (sqrt(dX[0] * dX[0] + dX[1] * dX[1] + dX[2] * dX[2]) < kConverged) {
                ok = true;
                break;
            }
        }
        if constexpr (!kRaim) {
            break;
        } else {
            // the test of the set just solved; an exclusion goes round again
            if (!ok) {
                if (excluded) verdict = GPSB200_RAIM_ALERT;   // a re-solve that failed; else the first: UNAVAILABLE
                break;
            }
            if (nused < 5) break;                          // UNAVAILABLE (only the first set can be this small)
            const double e = r - (h[0] * dX[0] + h[1] * dX[1] + h[2] * dX[2] + dX[3]);
            const double g[4] = {h[0], h[1], h[2], 1.0};
            double x[4];
            ch.solve(g, x);
            omh = 1.0 - (g[0] * x[0] + g[1] * x[1] + g[2] * x[2] + g[3] * x[3]);
            xg[0] = x[0];
            xg[1] = x[1];
            xg[2] = x[2];
            stat = warp_sum(use ? e * e : 0.0) / (a.raim.sigma * a.raim.sigma);
            dof = nused - 4;
            thr = a.T[dof - 1];
            if (!(stat > thr)) {
                verdict = excluded ? GPSB200_RAIM_EXCLUDED : GPSB200_RAIM_PASS;
                break;
            }
            verdict = GPSB200_RAIM_ALERT;
            if (nused < 6 || __popc(excluded) >= a.raim.max_exclude) break;
            double key = use && omh > 1e-9 ? e * e / omh : -1.0;
            int worst = lane;
            warp_argmax(key, worst);
            if (key < 0.0) break;                          // no candidate
            excluded |= 1u << worst;
            if (lane == worst) use = false;
            mask = __ballot_sync(kFull, use);
            nused = __popc(mask);
            f.mask = mask;
            f.nused = nused;
            it0 = f.iterations;
            ok = false;
        }
        }   // passes (the iteration loop inside keeps its indentation)
        if (ok) {
            // post-fit residuals of the last iteration, velocity and drift on the same rows
            if (has) resid = r - (h[0] * dX[0] + h[1] * dX[1] + h[2] * dX[2] + dX[3]);
            double lat, lon;
            finish(ch, X, (double) nom_ms * 1e-3 + ((double) m / 3e6 - X[3] / kC), use, h, pr_v, rate, ddtsv, 1.0,
                   resid, nused, f, lat, lon);
            if constexpr (kRaim) {
                if (verdict != GPSB200_RAIM_UNAVAILABLE) {
                    // Brown's slopes: N^-1 g in east / north / up at the fix
                    double sla, cla, slo, clo;
                    sincos(lat, &sla, &cla);
                    sincos(lon, &slo, &clo);
                    const double xe = -slo * xg[0] + clo * xg[1];
                    const double xn = -sla * clo * xg[0] - sla * slo * xg[1] + cla * xg[2];
                    const double xu = cla * clo * xg[0] + cla * slo * xg[1] + sla * xg[2];
                    const double inf = __longlong_as_double(0x7ff0000000000000ll);
                    const bool flat = !(omh > 1e-9);
                    const double hs = use ? (flat ? inf : sqrt(xe * xe + xn * xn) / sqrt(omh)) : 0.0;
                    const double vs = use ? (flat ? inf : fabs(xu) / sqrt(omh)) : 0.0;
                    const double k = a.raim.sigma * sqrt(a.lambda[dof - 1]);
                    hpl = warp_max(hs) * k;
                    vpl = warp_max(vs) * k;
                }
            }
        }
    }
    if (lane == 0) a.fixes[fi] = f;
    if (a.res && lane < a.nchan) a.res[fi * a.nchan + lane] = has ? resid : nan;
    if constexpr (kRaim) {
        if (lane == 0) {
            gpsb200_raim_t o;
            o.verdict = verdict;
            o.excluded = excluded;
            o.dof = dof;
            o.reserved = 0;
            o.stat = stat;
            o.threshold = thr;
            o.hpl = hpl;
            o.vpl = vpl;
            a.out[fi] = o;
        }
    }
}

// k_pvt_araim: gpsb200_pvt_araim (DESIGN §11.2). The measurement and the Gauss-Newton pass are k_pvt's with the
// weights; `use` is the set, so a masked or excluded lane's row enters with weight 0. Rows and residuals are scaled by
// sw = 1 / sigma_int, computed per iteration at the estimate's elevation. Solution separation and the protection levels
// run where the test of a set is final, inside the pass loop, so that nothing of them stays live across a re-solve.
// kAraimMinBlocks: DESIGN §11.2.
constexpr int kAraimMinBlocks = 4;
__global__ void __launch_bounds__(kWarps * 32, kAraimMinBlocks) k_pvt_araim(const AraimArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;   // the whole warp leaves together
    const int64_t s = a.cfg.s0 + fi * a.cfg.step;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);

    // ---- the measurement of this lane's channel (integers), its satellite (FP64), its URA sigmas ----
    double rho = 0.0, rate = 0.0, dtsv = 0.0, ddtsv = 0.0, p[3] = {0, 0, 0}, v[3] = {0, 0, 0};
    double sura2 = 0.0, sure2 = 0.0;
    const int64_t ds = s - a.ref_sample;
    const int64_t q = floor_div(ds, 3000), m = ds - 3000 * q;
    const int64_t nom_ms = (((a.ref_ms + 75 + q) % kWeekMs) + kWeekMs) % kWeekMs;
    // header step 1: URA index 15 never enters the set
    bool use = measure(a, lane, s, q, m, true, rho, rate, p, v, dtsv, ddtsv);
    if (use) {
        const double sura = fmax(a.araim.sigma_ura, kUraNom[a.ch[lane].eph.ura]);
        const double sure = sura * a.araim.sigma_ure / a.araim.sigma_ura;
        sura2 = sura * sura;
        sure2 = sure * sure;
    }
    const bool has = use;
    unsigned mask = __ballot_sync(kFull, use);
    int nused = __popc(mask);
    gpsb200_fix_t f;
    no_fix(f, s, nused, mask, nused < 4 ? GPSB200_FIX_FEW : GPSB200_FIX_NO_CONVERGENCE);
    double resid = nan;
    // the record; this lane's 1 / sigma_int, elevation and sigma^2 other than URA / URE of the last iteration
    int verdict = GPSB200_RAIM_UNAVAILABLE;
    unsigned excluded = 0, masked = 0;
    bool mask_done = false;
    double hpl = nan, vpl = nan, ratio = nan, emt = nan, sacc_v = nan, pnm = nan;
    double sw = 1.0, el = 0.5 * M_PI, rest2 = 0.0;
    if (nused >= 4) {
        double X[4] = {0.0, 0.0, 0.0, 0.0};
        double h[3] = {0, 0, 0}, r = 0.0, pr_v[3] = {0, 0, 0};
        double N[10];   // the weighted normal matrix of the last iteration
        Chol<4> ch;
        bool ok = false;
        double dX[4] = {0, 0, 0, 0};
        int it0 = 0;   // iterations of the earlier passes
#pragma unroll 1
        for (;;) {     // Gauss-Newton passes: the first, one after the mask, one after an exclusion
#pragma unroll 1
            for (int j = 0; j < GPSB200_PVT_MAX_ITER; j++) {
                const double rad = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
                const bool near = rad >= kIonoMinRadius, iono = a.cfg.iono && near;
                Geo g;
                if (near) g.set(X);   // the elevation weighs with or without the Klobuchar term
                h[0] = h[1] = h[2] = 0.0;
                r = 0.0;
                if (has) {
                    double l[3], R, az = 0.0, I = 0.0, Fm[2] = {1.0, 0.0};
                    el = 0.5 * M_PI;
                    sight(p, v, X, g, near, l, R, pr_v, az, el);
                    if (iono)
                        I = klobuchar(a.cfg, g.lat, g.lon, az, el, (double) nom_ms * 1e-3 + (double) m / 3e6 - X[3] / kC,
                                      Fm);
                    r = rho - (R + X[3] - kC * dtsv + I);
                    h[0] = -l[0] / R;
                    h[1] = -l[1] / R;
                    h[2] = -l[2] / R;
                    // header step 2
                    const double se = sin(el);
                    const double st = 0.12 * 1.001 / sqrt(0.002001 + se * se);
                    const double mp = 0.13 + 0.53 * exp(-el / kTenDeg);
                    const double pm = fabs(Fm[1]) * 180.0;   // semicircles -> deg
                    const double si = iono ? fmax(I / 5.0, Fm[0] * (pm <= 20.0 ? 9.0 : (pm <= 55.0 ? 4.5 : 6.0))) : 0.0;
                    rest2 = st * st + (a.araim.sigma_noise * a.araim.sigma_noise + mp * mp) + si * si;
                    sw = 1.0 / sqrt(sura2 + rest2);
                }
                // rows and residuals scaled by 1 / sigma_int; a lane outside the set weighs 0
                const double w0 = use ? h[0] * sw : 0.0, w1 = use ? h[1] * sw : 0.0, w2 = use ? h[2] * sw : 0.0;
                const double wc = use ? sw : 0.0, wr = use ? r * sw : 0.0;
                N[0] = warp_sum(w0 * w0);
                N[1] = warp_sum(w0 * w1);
                N[2] = warp_sum(w0 * w2);
                N[3] = warp_sum(w0 * wc);
                N[4] = warp_sum(w1 * w1);
                N[5] = warp_sum(w1 * w2);
                N[6] = warp_sum(w1 * wc);
                N[7] = warp_sum(w2 * w2);
                N[8] = warp_sum(w2 * wc);
                N[9] = warp_sum(wc * wc);
                const double b[4] = {warp_sum(w0 * wr), warp_sum(w1 * wr), warp_sum(w2 * wr), warp_sum(wc * wr)};
                f.iterations = it0 + j + 1;
                if (!ch.factor(N)) break;
                ch.solve(b, dX);
#pragma unroll
                for (int i = 0; i < 4; i++) X[i] += dX[i];
                if (sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]) > kRunaway) break;
                if (sqrt(dX[0] * dX[0] + dX[1] * dX[1] + dX[2] * dX[2]) < kConverged) {
                    ok = true;
                    break;
                }
            }
            // the test of the set just solved; the mask or an exclusion goes round again
            if (!ok) {
                if (excluded) verdict = GPSB200_RAIM_ALERT;   // a re-solve after an exclusion that failed
                break;
            }
            if (!mask_done) {                              // header step 4, once, after the first converged solve
                mask_done = true;
                const bool low = use && el < a.araim.mask_deg * (M_PI / 180.0);
                masked = __ballot_sync(kFull, low);
                if (masked) {
                    if (low) use = false;
                    mask = __ballot_sync(kFull, use);
                    nused = __popc(mask);
                    f.mask = mask;
                    f.nused = nused;
                    it0 = f.iterations;
                    ok = false;
                    if (nused < 4) {
                        f.status = GPSB200_FIX_FEW;
                        break;
                    }
                    continue;
                }
            }
            if (nused < 5) break;                          // UNAVAILABLE
            Ss o;
            const double sacc = mhss(a, use, nused, h, sw, r, sure2 + rest2, N, ch, X, o);
            if (__any_sync(kFull, !o.pd)) break;           // UNAVAILABLE
            double key = o.ratio;
            int worst = lane;
            warp_argmax(key, worst);
            ratio = key;
            emt = warp_max(use ? o.T[2] : 0.0);
            sacc_v = sacc;
            const bool pass = __all_sync(kFull, o.pass);
            if (!pass && !excluded && a.araim.max_exclude == 1 && nused >= 6) {   // header step 7
                excluded = 1u << worst;
                if (lane == worst) use = false;
                mask = __ballot_sync(kFull, use);
                nused = __popc(mask);
                f.mask = mask;
                f.nused = nused;
                it0 = f.iterations;
                ok = false;
                continue;
            }
            verdict = pass ? (excluded ? GPSB200_RAIM_EXCLUDED : GPSB200_RAIM_PASS) : GPSB200_RAIM_ALERT;
            // header step 8, over this final set
            const double ps = a.araim.p_sat, pv = a.araim.p_hmi_vert, ph = a.araim.p_hmi_horz;
            pnm = p_not_monitored(ps, nused);
            if (!(pnm < pv + ph)) {
                verdict = GPSB200_RAIM_UNAVAILABLE;
                break;
            }
            const double sc = 1.0 - pnm / (pv + ph);
            vpl = protection_level(pv * sc, o.b0[2], o.s0[2], use, o.T[2], o.b[2], o.s[2], ps, nused);
            const double he = protection_level(ph / 2.0 * sc, o.b0[0], o.s0[0], use, o.T[0], o.b[0], o.s[0], ps, nused);
            const double hn = protection_level(ph / 2.0 * sc, o.b0[1], o.s0[1], use, o.T[1], o.b[1], o.s[1], ps, nused);
            hpl = sqrt(he * he + hn * hn);
            break;
        }
        if (ok) {
            // post-fit residuals of the last iteration; velocity and drift on its weighted rows
            if (has) resid = r - (h[0] * dX[0] + h[1] * dX[1] + h[2] * dX[2] + dX[3]);
            double lat, lon;
            finish(ch, X, (double) nom_ms * 1e-3 + ((double) m / 3e6 - X[3] / kC), use, h, pr_v, rate, ddtsv, sw * sw,
                   resid, nused, f, lat, lon);
        }
    }
    if (lane == 0) {
        a.fixes[fi] = f;
        gpsb200_araim_t o;
        o.verdict = verdict;
        o.excluded = excluded;
        o.masked = masked;
        o.n = nused;
        o.test_ratio = ratio;
        o.hpl = hpl;
        o.vpl = vpl;
        o.emt = emt;
        o.sigma_acc_v = sacc_v;
        o.p_nm = pnm;
        a.out[fi] = o;
    }
    if (a.res && lane < a.nchan) a.res[fi * a.nchan + lane] = has ? resid : nan;
}

// ---- coarse-time fixes (DESIGN §11.3) -------------------------------------------------------------------------------
struct CoarseArgs : Args {
    gpsb200_coarse_config_t ap;
    gpsb200_coarse_t *out;
    int64_t *ms;
};
// Fixes from snapshot records (DESIGN §11.5): the records [nfix][nchan] in place of the epochs.
struct SnapCoarseArgs : CoarseArgs {
    const gpsb200_snapshot_t *meas;
};

// The coarse record of an instant without a coarse-time fix.
__device__ inline void no_coarse(gpsb200_coarse_t &o, int ref) {
    o.delta = o.pdop = __longlong_as_double(0x7ff8000000000000ll);
    o.ref = ref;
    o.week = -1;
    o.changed = 0;
    o.reserved = 0;
}

// The two measurements of the coarse-time solve (header step 2 of gpsb200_pvt_coarse). Each gives a fix's instant
// and, per lane: used, whether the channel is used at sample s and a-priori time tas; take, for a used channel, use =
// true, its ephemeris, code phase (frac, ms), range rate (m/s) and the prediction of step 3 at x_a (pred, sel), and
// nothing for the others. The body of take sits in each measurement so that the tracked one compiles as it did before
// the snapshot one existed.
// From tracked epochs at the instants s0 + i step.
struct FromEpochs {
    __device__ __forceinline__ int64_t instant(const Args &a, int64_t fi) const { return a.cfg.s0 + fi * a.cfg.step; }
    __device__ __forceinline__ bool used(const Args &a, int lane, int64_t s, double tas,
                                         const gpsb200_ephemeris_t &eph) const {
        double frac, rate;
        return locked_period(a, lane, s, frac, rate) >= 1 && fabs(wrap_half_week(tas - eph.toe)) <= 7200.0;
    }
    // locked_period, restated: calling it here made k_pvt_coarse take 25.55-25.60 ms against 25.22-25.48 ms and the
    // 12-channel search 8 094 ms against 8 078 ms (tools/pvt_bench.py --coarse / --search, H100 80GB HBM3, 700 W).
    __device__ __forceinline__ void take(const Args &a, int lane, int64_t s, double tas, const double *x_a,
                                         const double *up, bool &use, const gpsb200_ephemeris_t *&eph, double &frac,
                                         double &rate, double &pred, double &sel) const {
        if (lane < a.nchan) {
            const gpsb200_pvt_chan_t &c = a.ch[lane];
            const gpsb200_track_epoch_t *e = a.ep + (size_t) lane * a.max_epochs;
            const int k = c.eph.valid && c.eph.health == 0 ? find_period(e, a.n[lane], s) : -1;
            if (k >= 1 && e[k - 1].lock && e[k].lock && fabs(wrap_half_week(tas - c.eph.toe)) <= 7200.0) {
                use = true;
                eph = &c.eph;
                const uint64_t phi = (uint64_t) e[k - 1].code_phase + (uint64_t) (s - e[k].sample) * e[k - 1].code_step;
                frac = (double) phi / kCodeMod;
                rate = -kLambda * ((double) e[k - 1].carr_step * kStepHz);
                pred = predict(*eph, x_a, tas, up, sel);
            }
        }
    }
};
// From the snapshot records of one fix instant (row: the instant's nchan records); the instant is their sample.
struct FromSnapshots {
    const gpsb200_snapshot_t *row;
    __device__ __forceinline__ int64_t instant(const Args &, int64_t) const { return row[0].sample; }
    __device__ __forceinline__ bool used(const Args &a, int lane, int64_t, double tas,
                                         const gpsb200_ephemeris_t &eph) const {
        const gpsb200_snapshot_t &r = row[lane];
        return r.status == GPSB200_SNAP_OK && r.prn == a.ch[lane].prn && eph.valid && eph.health == 0 &&
               fabs(wrap_half_week(tas - eph.toe)) <= 7200.0;
    }
    __device__ __forceinline__ void take(const Args &a, int lane, int64_t s, double tas, const double *x_a,
                                         const double *up, bool &use, const gpsb200_ephemeris_t *&eph, double &frac,
                                         double &rate, double &pred, double &sel) const {
        if (lane < a.nchan && used(a, lane, s, tas, a.ch[lane].eph)) {
            use = true;
            eph = &a.ch[lane].eph;
            frac = (double) row[lane].code_phase / kCodeMod;
            rate = -kLambda * ((double) row[lane].carr_step * kStepHz);
            pred = predict(*eph, x_a, tas, up, sel);
        }
    }
};

// gpsb200_pvt_coarse's header steps 1-9 at sample s from the a-priori config ap: one warp, lane = channel, as k_pvt. The satellite is evaluated in every iteration, at the transmit time moved by the current delta. The fix and
// coarse records come out uniform over the warp; resid, Nw and has are this lane's (channel's). meas: the measurement
// of step 2 (FromEpochs or FromSnapshots).
template <class Meas>
__device__ __forceinline__ void coarse_solve(const Args &a, const Meas &meas, const gpsb200_coarse_config_t &ap,
                                             int64_t s, int lane, gpsb200_fix_t &f, gpsb200_coarse_t &o, double &resid,
                                             int64_t &Nw, bool &has) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    // header step 1
    const int64_t ds = s - ap.s_a;
    const int64_t q = floor_div(ds, 3000), m = ds - 3000 * q;
    const double u = ap.t_a + (double) ds / 3e6;
    const double kw = floor(u / 604800.0);
    const double tas = u - 604800.0 * kw;
    const double W = floor(ap.t_a), F = ap.t_a - W;
    const double sub = F * 1000.0 + (double) m / 3000.0;   // ms

    // header steps 2-4: measurement, prediction at x_a, reference channel
    bool use = false;
    double frac = 0.0, rate = 0.0, pred = 0.0, sel = -2.0;
    const gpsb200_ephemeris_t *eph = nullptr;
    Geo ga;
    ga.set(ap.x_a);
    const double up[3] = {ga.cla * ga.clo, ga.cla * ga.slo, ga.sla};
    meas.take(a, lane, s, tas, ap.x_a, up, use, eph, frac, rate, pred, sel);
    has = use;
    const unsigned mask = __ballot_sync(kFull, use);
    const int nused = __popc(mask);
    double key = use ? sel : -2.0;
    int r = lane;
    warp_argmax(key, r);
    const int ref = nused ? r : -1;
    const double pred_r = __shfl_sync(kFull, pred, r), frac_r = __shfl_sync(kFull, frac, r);
    // header step 5
    const int64_t Nr = (int64_t) round_half_up(pred_r - frac_r);
    const int64_t dN = (int64_t) round_half_up((pred - pred_r) - (frac - frac_r));
    Nw = (((Nr + dN) % kWeekMs) + kWeekMs) % kWeekMs;
    // header step 6
    double rho = 0.0, tsv = 0.0;
    if (has) {
        int64_t D = ((int64_t) W * 1000 + q - Nw) % kWeekMs;
        D = D >= kWeekMs / 2 ? D - kWeekMs : (D < -kWeekMs / 2 ? D + kWeekMs : D);
        rho = (double) D * kCms + (sub - frac) * kCms;
        tsv = (double) Nw * 1e-3 + frac * 1e-3;
    }

    no_fix(f, s, nused, mask, nused < 5 ? GPSB200_FIX_FEW : GPSB200_FIX_NO_CONVERGENCE);
    no_coarse(o, ref);
    resid = nan;
    if (nused >= 5) {
        double X[5] = {ap.x_a[0], ap.x_a[1], ap.x_a[2], 0.0, 0.0};
        double h[4] = {0, 0, 0, 0}, rr = 0.0, pr_v[3] = {0, 0, 0}, ddtsv = 0.0;
        Chol<5> ch;
        bool ok = false;
        double dX[5] = {0, 0, 0, 0, 0};
#pragma unroll 1
        for (int j = 0; j < GPSB200_PVT_MAX_ITER; j++) {
            const double rad = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
            const bool iono = a.cfg.iono && rad >= kIonoMinRadius;
            Geo g;
            if (iono) g.set(X);
            h[0] = h[1] = h[2] = h[3] = 0.0;
            rr = 0.0;
            if (has) {
                const gpsb200_ephemeris_t &e = *eph;
                const double t = tsv + X[4];
                const double d0 = wrap_half_week(t - e.toc);
                const double tt = t - (e.af0 + d0 * (e.af1 + d0 * e.af2));
                double p[3], v[3], dtsv, l[3], R, az = 0.0, el = 0.0, I = 0.0;
                satellite(e, tt, p, v, dtsv, ddtsv);
                sight(p, v, X, g, iono, l, R, pr_v, az, el);
                if (iono) I = klobuchar(a.cfg, g.lat, g.lon, az, el, tas + X[4] - X[3] / kC);
                rr = rho - (R + X[3] - kC * dtsv + I);
                h[0] = -l[0] / R;
                h[1] = -l[1] / R;
                h[2] = -l[2] / R;
                h[3] = (l[0] * pr_v[0] + l[1] * pr_v[1] + l[2] * pr_v[2]) / R - kC * ddtsv;
            }
            const double N[15] = {warp_sum(h[0] * h[0]), warp_sum(h[0] * h[1]), warp_sum(h[0] * h[2]), warp_sum(h[0]),
                                  warp_sum(h[0] * h[3]), warp_sum(h[1] * h[1]), warp_sum(h[1] * h[2]), warp_sum(h[1]),
                                  warp_sum(h[1] * h[3]), warp_sum(h[2] * h[2]), warp_sum(h[2]), warp_sum(h[2] * h[3]),
                                  (double) nused, warp_sum(h[3]), warp_sum(h[3] * h[3])};
            const double b[5] = {warp_sum(h[0] * rr), warp_sum(h[1] * rr), warp_sum(h[2] * rr), warp_sum(rr),
                                 warp_sum(h[3] * rr)};
            f.iterations = j + 1;
            if (!ch.factor(N)) break;
            ch.solve(b, dX);
#pragma unroll
            for (int i = 0; i < 5; i++) X[i] += dX[i];
            if (sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]) > kRunaway) break;
            if (sqrt(dX[0] * dX[0] + dX[1] * dX[1] + dX[2] * dX[2]) < kConverged) {
                ok = true;
                break;
            }
        }
        if (ok) {
            // header step 8, at the fix, with the same reference channel
            const double trx = tas + X[4] - X[3] / kC;
            double dummy, pred2 = 0.0;
            if (has) pred2 = predict(*eph, X, trx, up, dummy);
            const double pred2_r = __shfl_sync(kFull, pred2, r);
            const bool moved = has && (int64_t) round_half_up((pred2 - pred2_r) - (frac - frac_r)) != dN;
            o.changed = __ballot_sync(kFull, moved);
            if (has) resid = rr - (h[0] * dX[0] + h[1] * dX[1] + h[2] * dX[2] + dX[3] + h[3] * dX[4]);
            if (o.changed || __any_sync(kFull, has && !(fabs(resid) <= GPSB200_COARSE_MAX_RESIDUAL))) {
                f.status = GPSB200_FIX_AMBIGUOUS;
                resid = nan;
            } else {
                // velocity and drift on the rows' first four columns, 5-state PDOP; t_rx's fold carries into the week
                double lat, lon;
                finish(ch, X, trx, has, h, pr_v, rate, ddtsv, 1.0, resid, nused, f, lat, lon);
                o.delta = X[4];
                o.pdop = f.pdop;
                o.week = ap.week + (int) (trx < 0.0 ? kw - 1.0 : (trx >= 604800.0 ? kw + 1.0 : kw));
            }
        }
    }
}

// k_pvt_coarse: gpsb200_pvt_coarse (DESIGN §11.3), one warp per fix. kCoarseMinBlocks: held to 128 registers (some
// spills) it ran 10 % faster than at its natural 168 with 3 CTAs per SM (DESIGN §11.3).
constexpr int kCoarseMinBlocks = 4;
template <class Meas>
__device__ __forceinline__ void coarse_fix(const CoarseArgs &a, const Meas &meas, int64_t fi, int lane) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    gpsb200_fix_t f;
    gpsb200_coarse_t o;
    double resid;
    int64_t Nw;
    bool has;
    coarse_solve(a, meas, a.ap, meas.instant(a, fi), lane, f, o, resid, Nw, has);
    if (lane == 0) {
        a.fixes[fi] = f;
        a.out[fi] = o;
    }
    if (a.res && lane < a.nchan) a.res[fi * a.nchan + lane] = has ? resid : nan;
    if (a.ms && lane < a.nchan) a.ms[fi * a.nchan + lane] = has ? Nw : -1;
}
__global__ void __launch_bounds__(kWarps * 32, kCoarseMinBlocks) k_pvt_coarse(const CoarseArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;   // the whole warp leaves together
    coarse_fix(a, FromEpochs(), fi, lane);
}
// gpsb200_pvt_snapshot: the same fixes from snapshot records.
__global__ void __launch_bounds__(kWarps * 32, kCoarseMinBlocks) k_pvt_snapshot(const SnapCoarseArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;
    coarse_fix(a, FromSnapshots{a.meas + fi * a.nchan}, fi, lane);
}

// ---- position search: coarse-time fixes from every node of a global grid (DESIGN §11.4) -----------------------------
// An OK node's solution, appended to its fix instant's list (SearchArgs::hits) in whatever order the warps finish; only
// order-free reductions read the list, so the results do not depend on scheduling.
struct SearchHit {
    double rms, x, y, z;
    int32_t node, reserved;
};
static_assert(sizeof(SearchHit) == 5 * sizeof(double), "Scratch::d_hits holds SearchHit records as 5 doubles");
static_assert(sizeof(SearchHit) == GPSB200_SEARCH_HIT_BYTES_PER_OK, "the header states the list's size");

// Instants per pass of k_pvt_search and k_search_pick: as many as one GPSB200_SEARCH_HIT_BYTES list holds, at most 65535
// (blockIdx.y).
inline int search_pass(int nodes) {
    const int64_t per = (int64_t) GPSB200_SEARCH_MAX_OK(nodes) * (int64_t) sizeof(SearchHit);
    return (int) std::max<int64_t>(1, std::min<int64_t>(65535, (int64_t) GPSB200_SEARCH_HIT_BYTES / per));
}
struct SearchArgs : Args {
    gpsb200_search_config_t sc;
    double sin_min;            // sin(GPSB200_SEARCH_MIN_ELEV_DEG)
    double *sat;               // [nfix][32][3]: each channel's satellite at t_a(s) - 0.075 s, unrotated
    uint32_t *used;            // [nfix]: the used channels (header step 2)
    int32_t *searched, *nok;   // [nfix]: nodes searched, OK nodes (also counts those the list could not hold)
    SearchHit *hits;           // [instants of this pass][max_ok]
    double *node_rms;          // [nfix][nodes] or NULL
    gpsb200_search_t *out;
    int64_t *ms;
    int f0, nf;                // the instants f0 .. f0 + nf - 1 of this pass (k_pvt_search, k_search_pick)
    int max_ok;                // the list's length per instant: GPSB200_SEARCH_MAX_OK(nodes)
};
struct SnapSearchArgs : SearchArgs {
    const gpsb200_snapshot_t *meas;   // [nfix][nchan]
};

// Node i of the n-node grid (header step 1): ECEF position x and the up vector at its geodetic latitude / longitude.
__host__ __device__ inline void search_node(int64_t i, int n, double *x, double *up) {
    constexpr double kGolden = 0x1.8722191a02d61p-2;   // the double nearest (3 - sqrt(5)) / 2
    const double z = 1.0 - (2.0 * (double) i + 1.0) / (double) n;
    const double t = (double) i * kGolden;
    const double lat = asin(z), lon = 2.0 * M_PI * (t - floor(t));
    const double sla = sin(lat), cla = cos(lat), slo = sin(lon), clo = cos(lon);
    const double N = kWgsA / sqrt(1.0 - kWgsE * kWgsE * sla * sla);
    x[0] = N * cla * clo;
    x[1] = N * cla * slo;
    x[2] = N * (1.0 - kWgsE * kWgsE) * sla;
    up[0] = cla * clo;
    up[1] = cla * slo;
    up[2] = sla;
}

// Per fix instant (one warp, lane = channel): header step 2's used channels and step 3's satellite positions; clears the
// instant's counters.
template <class Meas>
__device__ __forceinline__ void search_sats(const SearchArgs &a, const Meas &meas, int64_t fi, int lane) {
    const int64_t s = meas.instant(a, fi);
    const int64_t ds = s - a.sc.s_a;
    const double u = a.sc.t_a + (double) ds / 3e6;
    const double tas = u - 604800.0 * floor(u / 604800.0);
    bool use = false;
    double p[3] = {0.0, 0.0, 0.0};
    if (lane < a.nchan) {
        const gpsb200_ephemeris_t &eph = a.ch[lane].eph;
        if (meas.used(a, lane, s, tas, eph)) {
            use = true;
            double v[3], dt, ddt;
            satellite(eph, tas - 0.075, p, v, dt, ddt);
        }
    }
    for (int i = 0; i < 3; i++) a.sat[(fi * 32 + lane) * 3 + i] = p[i];
    const unsigned mask = __ballot_sync(kFull, use);
    if (lane == 0) {
        a.used[fi] = mask;
        a.searched[fi] = 0;
        a.nok[fi] = 0;
    }
}
__global__ void __launch_bounds__(kWarps * 32) k_search_sats(const SearchArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;
    search_sats(a, FromEpochs(), fi, lane);
}
__global__ void __launch_bounds__(kWarps * 32) k_snapshot_sats(const SnapSearchArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;
    search_sats(a, FromSnapshots{a.meas + fi * a.nchan}, fi, lane);
}

// Header steps 3-4 over the grid: one warp per 32 nodes of one fix instant (blockIdx.y). Each lane tests its own node's
// visibility; the warp then solves the visible nodes one after another, lane = channel, and appends the OK ones to the
// instant's list. Testing 32 nodes per warp keeps the warps busy although most nodes fail the test.
constexpr int kSearchMinBlocks = 4;
template <class Meas>
__device__ __forceinline__ void search_nodes_of(const SearchArgs &a, const Meas &meas, int64_t fi, int lane) {
    const int64_t base = ((int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5)) * 32;
    const int n = a.sc.nodes;
    if (base >= n) return;
    const unsigned used = a.used[fi];
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const int64_t node = base + lane;
    double x[3], up[3];
    search_node(node, n, x, up);
    bool vis = node < n;
    // too few channels: nothing is searched (every node's rms stays NaN)
    for (unsigned m = __popc(used) >= GPSB200_SEARCH_MIN_CHANNELS ? used : 0u; m; m &= m - 1) {
        const double *p = a.sat + (fi * 32 + __ffs(m) - 1) * 3;
        const double l0 = p[0] - x[0], l1 = p[1] - x[1], l2 = p[2] - x[2];
        vis &= (up[0] * l0 + up[1] * l1 + up[2] * l2) / sqrt(l0 * l0 + l1 * l1 + l2 * l2) >= a.sin_min;
    }
    unsigned todo = __ballot_sync(kFull, vis && __popc(used) >= GPSB200_SEARCH_MIN_CHANNELS);
    if (lane == 0 && todo) atomicAdd(a.searched + fi, __popc(todo));
    double my_rms = nan;
    const int64_t s = meas.instant(a, fi);
    gpsb200_coarse_config_t ap;
    ap.t_a = a.sc.t_a;
    ap.s_a = a.sc.s_a;
    ap.week = a.sc.week;
    ap.reserved = 0;
    for (; todo; todo &= todo - 1) {
        const int j = __ffs(todo) - 1;
        for (int i = 0; i < 3; i++) ap.x_a[i] = __shfl_sync(kFull, x[i], j);
        gpsb200_fix_t f;
        gpsb200_coarse_t o;
        double resid;
        int64_t Nw;
        bool has;
        coarse_solve(a, meas, ap, s, lane, f, o, resid, Nw, has);
        if (f.status != GPSB200_FIX_OK) continue;
        if (lane == j) my_rms = f.rms;
        if (lane == 0) {
            const int k = atomicAdd(a.nok + fi, 1);
            if (k < a.max_ok) a.hits[(fi - a.f0) * a.max_ok + k] = SearchHit{f.rms, f.x, f.y, f.z,
                                                                                              (int32_t) (base + j), 0};
        }
    }
    if (a.node_rms && node < n) a.node_rms[fi * n + node] = my_rms;
}
__global__ void __launch_bounds__(kWarps * 32, kSearchMinBlocks) k_pvt_search(const SearchArgs a) {
    const int64_t fi = (int64_t) a.f0 + blockIdx.y;
    search_nodes_of(a, FromEpochs(), fi, threadIdx.x & 31);
}
__global__ void __launch_bounds__(kWarps * 32, kSearchMinBlocks) k_snapshot_search(const SnapSearchArgs a) {
    const int64_t fi = (int64_t) a.f0 + blockIdx.y;
    search_nodes_of(a, FromSnapshots{a.meas + fi * a.nchan}, fi, threadIdx.x & 31);
}

// The winner's ordering key (header step 5): rms in whole millimetres, rounded down.
__device__ inline double rms_key(double rms) { return floor(rms * 1000.0); }

// (key, node) lexicographic minimum over the warp, carrying the list index k; every lane ends with the same triple.
__device__ inline void warp_argmin_hit(double &key, int &node, int &k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double okey = __shfl_xor_sync(kFull, key, o);
        const int onode = __shfl_xor_sync(kFull, node, o), ok = __shfl_xor_sync(kFull, k, o);
        if (okey < key || (okey == key && onode < node)) {
            key = okey;
            node = onode;
            k = ok;
        }
    }
}

// Header steps 5-6 per fix instant (one warp, lane = channel): the winner and its support from the list, then the
// winner's coarse solve again for the records. br / ar hold rms_key values.
template <class Meas>
__device__ __forceinline__ void search_pick(const SearchArgs &a, const Meas &meas, int64_t fi, int lane) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll), inf = __longlong_as_double(0x7ff0000000000000ll);
    const int64_t s = meas.instant(a, fi);
    const unsigned used = a.used[fi];
    const int nused = __popc(used), nok = a.nok[fi];
    gpsb200_search_t r;
    r.winner = -1;
    r.searched = a.searched[fi];
    r.ok = nok;
    r.support = 0;
    r.alt_rms = r.alt_dist = nan;
    r.reserved = 0;
    if (nused >= GPSB200_SEARCH_MIN_CHANNELS && nok >= 1 && nok <= a.max_ok) {
        const SearchHit *h = a.hits + (fi - a.f0) * a.max_ok;
        double br = inf;
        int bn = 0x7fffffff, bk = -1;
        for (int k = lane; k < nok; k += 32)
            if (rms_key(h[k].rms) < br || (rms_key(h[k].rms) == br && h[k].node < bn)) {
                br = rms_key(h[k].rms);
                bn = h[k].node;
                bk = k;
            }
        warp_argmin_hit(br, bn, bk);
        const double wx = h[bk].x, wy = h[bk].y, wz = h[bk].z;
        double ar = inf;
        int an = 0x7fffffff, ak = -1, near = 0;
        for (int k = lane; k < nok; k += 32) {
            const double dx = h[k].x - wx, dy = h[k].y - wy, dz = h[k].z - wz;
            if (sqrt(dx * dx + dy * dy + dz * dz) <= GPSB200_SEARCH_DISTINCT) near++;
            else if (rms_key(h[k].rms) < ar || (rms_key(h[k].rms) == ar && h[k].node < an)) {
                ar = rms_key(h[k].rms);
                an = h[k].node;
                ak = k;
            }
        }
        warp_argmin_hit(ar, an, ak);
        r.winner = bn;
        r.support = __reduce_add_sync(kFull, near);
        if (ak >= 0) {
            const double dx = h[ak].x - wx, dy = h[ak].y - wy, dz = h[ak].z - wz;
            r.alt_rms = h[ak].rms;
            r.alt_dist = sqrt(dx * dx + dy * dy + dz * dz);
        }
    }
    gpsb200_fix_t f;
    gpsb200_coarse_t o;
    double resid = nan;
    int64_t Nw = -1;
    bool has = false;
    if (r.winner >= 0) {
        gpsb200_coarse_config_t ap;
        double up[3];
        search_node(r.winner, a.sc.nodes, ap.x_a, up);
        ap.t_a = a.sc.t_a;
        ap.s_a = a.sc.s_a;
        ap.week = a.sc.week;
        ap.reserved = 0;
        coarse_solve(a, meas, ap, s, lane, f, o, resid, Nw, has);
        if (!isnan(r.alt_rms)) f.status = GPSB200_FIX_AMBIGUOUS;
    } else {
        no_fix(f, s, nused, used,
               nused < GPSB200_SEARCH_MIN_CHANNELS ? GPSB200_FIX_FEW
               : nok > a.max_ok                    ? GPSB200_FIX_AMBIGUOUS
                                                   : GPSB200_FIX_NO_CONVERGENCE);
        no_coarse(o, -1);
    }
    r.delta = o.delta;
    r.pdop = o.pdop;
    r.ref = o.ref;
    r.week = o.week;
    r.changed = o.changed;
    if (lane == 0) {
        a.fixes[fi] = f;
        a.out[fi] = r;
    }
    if (a.res && lane < a.nchan) a.res[fi * a.nchan + lane] = has ? resid : nan;
    if (a.ms && lane < a.nchan) a.ms[fi * a.nchan + lane] = has ? Nw : -1;
}
__global__ void __launch_bounds__(kWarps * 32) k_search_pick(const SearchArgs a) {
    const int64_t local = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (local >= a.nf) return;
    search_pick(a, FromEpochs(), a.f0 + local, threadIdx.x & 31);
}
__global__ void __launch_bounds__(kWarps * 32) k_snapshot_pick(const SnapSearchArgs a) {
    const int64_t local = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (local >= a.nf) return;
    const int64_t fi = a.f0 + local;
    search_pick(a, FromSnapshots{a.meas + fi * a.nchan}, fi, threadIdx.x & 31);
}

void fill(Args &a, const Scratch &sc) {
    a.ep = sc.d_epochs.get();
    a.ch = sc.d_chans.get();
    a.n = sc.d_n.get();
    a.nchan = sc.nchan;
    a.max_epochs = sc.max_epochs;
    a.ref = sc.ref;
    a.ref_sample = sc.ref_sample;
    a.ref_ms = sc.ref_ms;
    a.cfg = sc.cfg;
    a.fixes = sc.d_fixes.get();
    a.res = sc.want_res ? sc.d_res.get() : nullptr;
}

// gpsb200_pvt_search: the satellite table, then the grid and the pick in passes of search_pass(nodes) instants, each
// pass reusing one OK list of GPSB200_SEARCH_HIT_BYTES at most.
template <bool kSnap>
cudaError_t launch_search(const Scratch &sc, cudaStream_t s) {
    typename std::conditional<kSnap, SnapSearchArgs, SearchArgs>::type a;
    fill(a, sc);
    if constexpr (kSnap) a.meas = sc.d_meas.get();
    a.sc = sc.search_cfg;
    a.sin_min = std::sin(GPSB200_SEARCH_MIN_ELEV_DEG * (M_PI / 180.0));
    a.sat = sc.d_sat.get();
    a.used = sc.d_used.get();
    a.searched = sc.d_searched.get();
    a.nok = sc.d_nok.get();
    a.hits = reinterpret_cast<SearchHit *>(sc.d_hits.get());
    a.node_rms = sc.want_node_rms ? sc.d_node_rms.get() : nullptr;
    a.out = sc.d_search.get();
    a.ms = sc.want_ms ? sc.d_ms.get() : nullptr;
    a.max_ok = GPSB200_SEARCH_MAX_OK(a.sc.nodes);
    const unsigned fix_blocks = (unsigned) (((int64_t) sc.cfg.nfix + kWarps - 1) / kWarps);
    if constexpr (kSnap) k_snapshot_sats<<<fix_blocks, kWarps * 32, 0, s>>>(a);
    else k_search_sats<<<fix_blocks, kWarps * 32, 0, s>>>(a);
    const unsigned node_blocks = (unsigned) ((a.sc.nodes + kWarps * 32 - 1) / (kWarps * 32));
    const int per_pass = search_pass(a.sc.nodes);
    for (int f0 = 0; f0 < sc.cfg.nfix; f0 += per_pass) {
        a.f0 = f0;
        a.nf = std::min(per_pass, sc.cfg.nfix - f0);
        const unsigned pick_blocks = (unsigned) ((a.nf + kWarps - 1) / kWarps);
        if constexpr (kSnap) {
            k_snapshot_search<<<dim3(node_blocks, (unsigned) a.nf), kWarps * 32, 0, s>>>(a);
            k_snapshot_pick<<<pick_blocks, kWarps * 32, 0, s>>>(a);
        } else {
            k_pvt_search<<<dim3(node_blocks, (unsigned) a.nf), kWarps * 32, 0, s>>>(a);
            k_search_pick<<<pick_blocks, kWarps * 32, 0, s>>>(a);
        }
    }
    return cudaGetLastError();
}

cudaError_t launch(const Scratch &sc, cudaStream_t s) {
    const unsigned blocks = (unsigned) (((int64_t) sc.cfg.nfix + kWarps - 1) / kWarps);
    switch (sc.mode) {
    case Mode::plain: {
        Args a;
        fill(a, sc);
        k_pvt<false><<<blocks, kWarps * 32, 0, s>>>(a);
        break;
    }
    case Mode::raim: {
        RaimArgs a;
        fill(a, sc);
        a.raim = sc.raim_cfg;
        memcpy(a.T, sc.tab_T, sizeof a.T);
        memcpy(a.lambda, sc.tab_lambda, sizeof a.lambda);
        a.out = sc.d_raim.get();
        k_pvt<true><<<blocks, kWarps * 32, 0, s>>>(a);
        break;
    }
    case Mode::araim: {
        AraimArgs a;
        fill(a, sc);
        a.araim = sc.araim_cfg;
        memcpy(a.kh, sc.kfa_h, sizeof a.kh);
        memcpy(a.kv, sc.kfa_v, sizeof a.kv);
        a.out = sc.d_araim.get();
        k_pvt_araim<<<blocks, kWarps * 32, 0, s>>>(a);
        break;
    }
    case Mode::coarse: {
        CoarseArgs a;
        fill(a, sc);
        a.ap = sc.coarse_cfg;
        a.out = sc.d_coarse.get();
        a.ms = sc.want_ms ? sc.d_ms.get() : nullptr;
        k_pvt_coarse<<<blocks, kWarps * 32, 0, s>>>(a);
        break;
    }
    case Mode::snapshot: {
        SnapCoarseArgs a;
        fill(a, sc);
        a.ap = sc.coarse_cfg;
        a.out = sc.d_coarse.get();
        a.ms = sc.want_ms ? sc.d_ms.get() : nullptr;
        a.meas = sc.d_meas.get();
        k_pvt_snapshot<<<blocks, kWarps * 32, 0, s>>>(a);
        break;
    }
    case Mode::search:
        return launch_search<false>(sc, s);
    case Mode::snapshot_search:
        return launch_search<true>(sc, s);
    }
    return cudaGetLastError();
}

}  // namespace

std::string check_coarse(const gpsb200_coarse_config_t &c) {
    for (int i = 0; i < 3; i++)
        if (!std::isfinite(c.x_a[i])) return "coarse x_a must be finite";
    if (!(c.t_a >= 0.0 && c.t_a < 604800.0)) return "coarse t_a must lie in 0 <= t_a < 604800";
    if (c.s_a < 0 || c.s_a > (1ll << 62)) return "coarse s_a outside 0..2^62";
    if (c.week < 0) return "coarse week must be >= 0";
    if (c.reserved != 0) return "coarse reserved must be 0";
    return std::string();
}

std::string check(const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs, const int32_t *nepochs,
                  int max_epochs, const gpsb200_pvt_config_t *cfg, const Stage &st) {
    const gpsb200_raim_config_t *raim = st.raim;
    const gpsb200_araim_config_t *araim = st.araim;
    const gpsb200_coarse_config_t *coarse = st.coarse;
    const gpsb200_search_config_t *search = st.search;
    if (st.meas) {
        if (!chans || !cfg) return "NULL chans, meas or cfg";
    } else if (!chans || !epochs || !nepochs || !cfg) {
        return "NULL chans, epochs, nepochs or cfg";
    }
    if (search) {
        const gpsb200_search_config_t &c = *search;
        if (!(c.t_a >= 0.0 && c.t_a < 604800.0)) return "search t_a must lie in 0 <= t_a < 604800";
        if (c.s_a < 0 || c.s_a > (1ll << 62)) return "search s_a outside 0..2^62";
        if (c.week < 0) return "search week must be >= 0";
        if (c.nodes < GPSB200_SEARCH_MIN_NODES || c.nodes > GPSB200_SEARCH_MAX_NODES)
            return "search nodes outside 64..4194304";
        if (c.reserved != 0) return "search reserved must be 0";
    }
    if (coarse) {
        const std::string bad = check_coarse(*coarse);
        if (!bad.empty()) return bad;
    }
    if (araim) {
        const gpsb200_araim_config_t &r = *araim;
        const auto in = [](double v, double lo, double hi) { return v >= lo && v <= hi; };   // false for NaN
        if (!in(r.mask_deg, 0.0, 90.0)) return "araim mask_deg must lie in 0..90";
        if (!in(r.sigma_ura, 0.0, 100.0) || !(r.sigma_ura > 0.0)) return "araim sigma_ura must lie in (0, 100]";
        if (!in(r.sigma_ure, 0.0, r.sigma_ura) || !(r.sigma_ure > 0.0)) return "araim sigma_ure must lie in (0, sigma_ura]";
        if (!in(r.sigma_noise, 0.0, 100.0) || !in(r.b_nom, 0.0, 100.0)) return "araim sigma_noise and b_nom must lie in 0..100";
        if (!in(r.p_sat, 1e-12, 1e-2)) return "araim p_sat must lie in 1e-12..1e-2";
        if (!in(r.p_hmi_vert, 1e-12, 0.5) || !in(r.p_hmi_horz, 1e-12, 0.5) || !in(r.p_fa_vert, 1e-12, 0.5) ||
            !in(r.p_fa_horz, 1e-12, 0.5))
            return "araim p_hmi_vert, p_hmi_horz, p_fa_vert and p_fa_horz must lie in 1e-12..0.5";
        if (r.max_exclude != 0 && r.max_exclude != 1) return "araim max_exclude must be 0 or 1";
        if (r.reserved[0] || r.reserved[1] || r.reserved[2]) return "araim reserved must be 0";
    }
    if (raim) {
        if (!std::isfinite(raim->sigma) || !(raim->sigma > 0.0)) return "raim sigma must be finite and > 0";
        if (!(raim->p_fa >= 1e-12 && raim->p_fa <= 0.5) || !(raim->p_md >= 1e-12 && raim->p_md <= 0.5))
            return "raim p_fa and p_md must lie in 1e-12..0.5";
        if (raim->max_exclude < 0 || raim->max_exclude > GPSB200_RAIM_MAX_EXCLUDE) return "raim max_exclude must be 0..4";
        if (raim->reserved != 0) return "raim reserved must be 0";
    }
    if (nchan < 1 || nchan > GPSB200_TRK_MAX_CHAN) return "nchan must be 1..32";
    if (max_epochs < 1) return "max_epochs must be >= 1";
    if (cfg->nfix < 1) return "nfix must be >= 1";
    if (!st.meas && cfg->step < 1) return "step must be >= 1";
    if (cfg->iono != 0 && cfg->iono != 1) return "iono must be 0 or 1";
    const int64_t kLast = 1ll << 62;   // fix instants stay far from int64 overflow
    if (!st.meas && (cfg->s0 < 0 || cfg->s0 > kLast || (int64_t) (cfg->nfix - 1) > (kLast - cfg->s0) / cfg->step))
        return "fix instants outside 0..2^62";
    if (st.meas) {   // snapshot records: each row's common sample is its fix instant
        for (int64_t i = 0; i < cfg->nfix; i++) {
            const gpsb200_snapshot_t *row = st.meas + i * nchan;
            const std::string at = "snapshot " + std::to_string(i) + ": ";
            if (row[0].sample < 0 || row[0].sample > kLast) return at + "sample outside 0..2^62";
            for (int c = 1; c < nchan; c++)
                if (row[c].sample != row[0].sample) return at + "records of different samples";
        }
    }
    for (int i = 0; i < 4; i++)
        if (!std::isfinite(cfg->alpha[i]) || !std::isfinite(cfg->beta[i])) return "alpha / beta must be finite";
    for (int c = 0; c < nchan; c++) {
        const gpsb200_pvt_chan_t &ch = chans[c];
        const std::string at = "channel " + std::to_string(c) + ": ";
        if (!st.meas && (nepochs[c] < 0 || nepochs[c] > max_epochs)) return at + "nepochs outside 0..max_epochs";
        if (ch.eph.valid != 0 && ch.eph.valid != 1) return at + "eph.valid must be 0 or 1";
        if (!ch.eph.valid || coarse || search) continue;   // never used, or a coarse-time call: no anchor read
        if (ch.anchor_epoch < 0 || ch.anchor_epoch >= nepochs[c]) return at + "anchor_epoch outside the channel's epochs";
        if (ch.anchor_ms < 0 || ch.anchor_ms >= kWeekMs) return at + "anchor_ms outside 0..604799999";
        if (araim && (ch.eph.ura < 0 || ch.eph.ura > 15)) return at + "eph.ura outside 0..15";
    }
    return std::string();
}

cudaError_t run(Scratch &sc, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg, gpsb200_fix_t *fixes,
                double *residuals, const Stage &st, cudaStream_t s) {
    const size_t nf = (size_t) cfg->nfix;
    sc.have_last = false;
    CU_RET(sc.d_chans.grow(GPSB200_TRK_MAX_CHAN));
    CU_RET(sc.d_n.grow(GPSB200_TRK_MAX_CHAN));
    if (st.meas) CU_RET(sc.d_meas.grow(nf * nchan));
    else CU_RET(sc.d_epochs.grow((size_t) nchan * max_epochs));
    CU_RET(sc.d_fixes.grow(nf));
    if (residuals) CU_RET(sc.d_res.grow(nf * nchan));
    if (st.ms) CU_RET(sc.d_ms.grow(nf * nchan));
    sc.mode = st.mode();
    if (st.raim) {
        CU_RET(sc.d_raim.grow(nf));
        sc.raim_cfg = *st.raim;
        if (st.raim->p_fa != sc.tab_p_fa || st.raim->p_md != sc.tab_p_md) {   // the tables take 20-80 ms of host time
            raim_thresholds(st.raim->p_fa, st.raim->p_md, sc.tab_T, sc.tab_lambda);
            sc.tab_p_fa = st.raim->p_fa;
            sc.tab_p_md = st.raim->p_md;
        }
    }
    if (st.araim) {
        CU_RET(sc.d_araim.grow(nf));
        sc.araim_cfg = *st.araim;
        araim_kfa(st.araim->p_fa_vert, st.araim->p_fa_horz, sc.kfa_h, sc.kfa_v);
    }
    if (st.coarse) {
        CU_RET(sc.d_coarse.grow(nf));
        sc.coarse_cfg = *st.coarse;
    }
    if (st.search) {
        const int nodes = st.search->nodes;
        CU_RET(sc.d_search.grow(nf));
        CU_RET(sc.d_sat.grow(nf * 32 * 3));
        CU_RET(sc.d_used.grow(nf));
        CU_RET(sc.d_searched.grow(nf));
        CU_RET(sc.d_nok.grow(nf));
        const size_t pass = (size_t) std::min<int64_t>(search_pass(nodes), cfg->nfix);
        CU_RET(sc.d_hits.grow(pass * GPSB200_SEARCH_MAX_OK(nodes) * sizeof(SearchHit) / sizeof(double)));
        if (st.node_rms) CU_RET(sc.d_node_rms.grow(nf * nodes));
        sc.search_cfg = *st.search;
    }
    sc.want_ms = st.ms != nullptr;
    sc.want_node_rms = st.node_rms != nullptr;
    // the reference channel of the nominal receive time: the lowest with a valid, healthy ephemeris (a coarse-time call
    // has no anchors and no nominal receive time)
    sc.ref = -1;
    for (int c = 0; c < nchan && sc.ref < 0 && !st.coarse && !st.search; c++)
        if (chans[c].eph.valid && chans[c].eph.health == 0) sc.ref = c;
    sc.ref_sample = sc.ref >= 0 ? epochs[(size_t) sc.ref * max_epochs + chans[sc.ref].anchor_epoch].sample : 0;
    sc.ref_ms = sc.ref >= 0 ? chans[sc.ref].anchor_ms : 0;
    sc.nchan = nchan;
    sc.max_epochs = max_epochs;
    sc.cfg = *cfg;
    sc.want_res = residuals != nullptr;
    if (st.meas) {
        CU_RET(cudaMemcpyAsync(sc.d_meas.get(), st.meas, nf * nchan * sizeof(gpsb200_snapshot_t),
                               cudaMemcpyHostToDevice, s));
    } else {
        CU_RET(cudaMemcpyAsync(sc.d_epochs.get(), epochs, (size_t) nchan * max_epochs * sizeof(gpsb200_track_epoch_t),
                               cudaMemcpyHostToDevice, s));
        CU_RET(cudaMemcpyAsync(sc.d_n.get(), nepochs, nchan * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    }
    CU_RET(cudaMemcpyAsync(sc.d_chans.get(), chans, nchan * sizeof(gpsb200_pvt_chan_t), cudaMemcpyHostToDevice, s));
    CU_RET(launch(sc, s));
    const auto down = [&](void *dst, const void *src, size_t bytes) {
        return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s);
    };
    CU_RET(down(fixes, sc.d_fixes.get(), nf * sizeof(gpsb200_fix_t)));
    if (residuals) CU_RET(down(residuals, sc.d_res.get(), nf * nchan * sizeof(double)));
    if (st.raim) CU_RET(down(st.raim_out, sc.d_raim.get(), nf * sizeof(gpsb200_raim_t)));
    if (st.araim) CU_RET(down(st.araim_out, sc.d_araim.get(), nf * sizeof(gpsb200_araim_t)));
    if (st.coarse) CU_RET(down(st.coarse_out, sc.d_coarse.get(), nf * sizeof(gpsb200_coarse_t)));
    if (st.search) CU_RET(down(st.search_out, sc.d_search.get(), nf * sizeof(gpsb200_search_t)));
    if (st.ms) CU_RET(down(st.ms, sc.d_ms.get(), nf * nchan * sizeof(int64_t)));
    if (st.node_rms) CU_RET(down(st.node_rms, sc.d_node_rms.get(), nf * st.search->nodes * sizeof(double)));
    CU_RET(cudaStreamSynchronize(s));
    sc.have_last = true;
    return cudaSuccess;
}

cudaError_t replay(Scratch &sc, cudaStream_t s) { return launch(sc, s); }

void search_nodes(int n, double *xyz) {
    for (int i = 0; i < n; i++) {
        double up[3];
        search_node(i, n, xyz + 3 * (size_t) i, up);
    }
}

}  // namespace pvt
}  // namespace gpsb200
