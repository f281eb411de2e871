// Position, velocity and time (include/gpsb200.h: gpsb200_pvt; DESIGN §11).
//
// k_pvt: one warp per fix instant, lane = channel (nchan <= 32, so one warp holds every channel of the call). Each lane
// finds its code period by a binary search bracketed by the 2999..3001-sample period length, forms its measurement in
// integers, and evaluates its satellite once (Kepler, orbit, clock). Every Gauss-Newton iteration does the Earth rotation
// and the Klobuchar delay per lane and sums the normal equations over the warp with an XOR butterfly: both lanes of a
// pair add the same two values, so every lane ends with the same bits and solves the 4 x 4 system identically. No
// atomics, no shared memory; the kernel is bound by FP64 arithmetic (the trigonometry of the orbit and the iterations).
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#include "device_buffer.h"
#include "pvt.h"
#include "synth_tables.h"

namespace gpsb200 {
namespace pvt {

namespace {

constexpr double kCms = 2.99792458e5;             // metres per ms of light time
constexpr double kRelF = -4.442807633e-10;        // relativistic clock term, s / m^1/2
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
template <bool kRaim> using KernelArgs = typename std::conditional<kRaim, RaimArgs, Args>::type;

__device__ inline double wrap_half_week(double d) { return d > 302400.0 ? d - 604800.0 : (d < -302400.0 ? d + 604800.0 : d); }

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

// Cholesky solve of the symmetric 4 x 4 system N x = b, N packed as n00 n01 n02 n03 n11 n12 n13 n22 n23 n33.
// false when N is not positive definite.
struct Chol {
    double l[4][4];
    __device__ bool factor(const double *N) {
        const double a[4][4] = {{N[0], N[1], N[2], N[3]}, {N[1], N[4], N[5], N[6]}, {N[2], N[5], N[7], N[8]},
                                {N[3], N[6], N[8], N[9]}};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            double d = a[j][j];
#pragma unroll
            for (int k = 0; k < j; k++) d -= l[j][k] * l[j][k];
            if (!(d > 0.0)) return false;
            l[j][j] = sqrt(d);
#pragma unroll
            for (int i = j + 1; i < 4; i++) {
                double v = a[i][j];
#pragma unroll
                for (int k = 0; k < j; k++) v -= l[i][k] * l[j][k];
                l[i][j] = v / l[j][j];
            }
        }
        return true;
    }
    __device__ void solve(const double *b, double *x) const {
        double y[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            double v = b[i];
#pragma unroll
            for (int k = 0; k < i; k++) v -= l[i][k] * y[k];
            y[i] = v / l[i][i];
        }
#pragma unroll
        for (int i = 3; i >= 0; i--) {
            double v = y[i];
#pragma unroll
            for (int k = i + 1; k < 4; k++) v -= l[k][i] * x[k];
            x[i] = v / l[i][i];
        }
    }
};

// WGS-84 latitude, longitude (rad) and height of an ECEF point: six fixed-point steps of
// lat = atan2(z + e^2 N(lat) sin lat, p) from lat = atan2(z, p (1 - e^2)).
__device__ void ecef_llh(const double *x, double &lat, double &lon, double &h) {
    const double e2 = kWgsE * kWgsE;
    const double p = sqrt(x[0] * x[0] + x[1] * x[1]);
    lon = atan2(x[1], x[0]);
    lat = atan2(x[2], p * (1.0 - e2));
    double N = kWgsA;
#pragma unroll 1
    for (int it = 0; it < 6; it++) {
        const double sl = sin(lat);
        N = kWgsA / sqrt(1.0 - e2 * sl * sl);
        lat = atan2(x[2] + e2 * N * sl, p);
    }
    double sl, cl;
    sincos(lat, &sl, &cl);
    h = p * cl + x[2] * sl - kWgsA * sqrt(1.0 - e2 * sl * sl);
}

// The Klobuchar delay in metres (the reference's ionosphericDelay, gps.c:1893-1964, with a valid alpha / beta set).
__device__ double klobuchar(const gpsb200_pvt_config_t &cfg, double lat, double lon, double az, double el, double t) {
    const double E = el / kPi, phi_u = lat / kPi, lam_u = lon / kPi;
    const double om = 0.53 - E;
    const double F = 1.0 + 16.0 * om * om * om;
    const double psi = 0.0137 / (E + 0.11) - 0.022;
    double phi_i = phi_u + psi * cos(az);
    phi_i = phi_i > 0.416 ? 0.416 : (phi_i < -0.416 ? -0.416 : phi_i);
    const double lam_i = lam_u + psi * sin(az) / cos(phi_i * kPi);
    const double phi_m = phi_i + 0.064 * cos((lam_i - 1.617) * kPi);
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

// Satellite position, velocity (ECEF) at GPS time t and clock offset / drift (IS-GPS-200 20.3.3.3.3, 20.3.3.4.3).
__device__ void satellite(const gpsb200_ephemeris_t &e, double t, double *p, double *v, double &dt, double &ddt) {
    const double tk = wrap_half_week(t - e.toe);
    const double A = e.sqrta * e.sqrta;
    const double n = sqrt(kGM / (A * A * A)) + e.deltan;
    const double M = e.m0 + n * tk;
    double E = M;
#pragma unroll 1
    for (int it = 0; it < 10; it++) {
        double sE, cE;
        sincos(E, &sE, &cE);
        const double dE = (M - E + e.ecc * sE) / (1.0 - e.ecc * cE);
        E += dE;
        if (fabs(dE) <= 1e-14) break;
    }
    double sE, cE;
    sincos(E, &sE, &cE);
    const double om = 1.0 - e.ecc * cE;
    const double Edot = n / om;
    const double sq = sqrt(1.0 - e.ecc * e.ecc);
    const double pk = atan2(sq * sE, cE - e.ecc) + e.aop;
    const double pkdot = sq * Edot / om;
    double s2, c2;
    sincos(2.0 * pk, &s2, &c2);
    const double uk = pk + e.cus * s2 + e.cuc * c2;
    const double ukdot = pkdot * (1.0 + 2.0 * (e.cus * c2 - e.cuc * s2));
    const double rk = A * om + e.crc * c2 + e.crs * s2;
    const double rkdot = A * e.ecc * sE * Edot + 2.0 * pkdot * (e.crs * c2 - e.crc * s2);
    const double ik = e.inc0 + e.idot * tk + e.cic * c2 + e.cis * s2;
    const double ikdot = e.idot + 2.0 * pkdot * (e.cis * c2 - e.cic * s2);
    double su, cu, si, ci;
    sincos(uk, &su, &cu);
    sincos(ik, &si, &ci);
    const double xp = rk * cu, yp = rk * su;
    const double xpdot = rkdot * cu - yp * ukdot, ypdot = rkdot * su + xp * ukdot;
    const double odot = e.omgdot - kOmegaE;
    const double ok = e.omg0 + tk * odot - kOmegaE * e.toe;
    double so, co;
    sincos(ok, &so, &co);
    p[0] = xp * co - yp * ci * so;
    p[1] = xp * so + yp * ci * co;
    p[2] = yp * si;
    const double tmp = ypdot * ci - yp * si * ikdot;
    v[0] = -odot * p[1] + xpdot * co - tmp * so;
    v[1] = odot * p[0] + xpdot * so + tmp * co;
    v[2] = yp * ci * ikdot + ypdot * si;
    const double d = wrap_half_week(t - e.toc);
    dt = e.af0 + d * (e.af1 + d * e.af2) + kRelF * e.ecc * e.sqrta * sE - e.tgd;
    ddt = e.af1 + 2.0 * d * e.af2;
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

// kRaim: the RAIM stage of gpsb200_pvt_raim after the solve (DESIGN §11.1). Each lane keeps two flags: `has` (a
// measurement) and `use` (in the solve). An excluded lane still evaluates its row every iteration, with weight 0, so the
// same warp sums serve every pass, and its residual against the final fix comes out of the same formula. The RAIM
// instantiation is held to 128 registers (4 CTAs per SM, as the plain one) at the price of some spills: at its natural
// 160 it ran 3 CTAs per SM and 15 % slower. The plain one keeps its bounds and instructions (DESIGN §11.1).
template <bool kRaim>
__global__ void __launch_bounds__(kWarps * 32, kRaim ? 4 : 0) k_pvt(const KernelArgs<kRaim> a) {
    const int lane = threadIdx.x & 31;
    const int64_t fi = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (fi >= a.cfg.nfix) return;   // the whole warp leaves together
    const int64_t s = a.cfg.s0 + fi * a.cfg.step;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);

    // ---- the measurement of this lane's channel (integers), its satellite (FP64) ----
    bool use = false;
    double rho = 0.0, rate = 0.0, dtsv = 0.0, ddtsv = 0.0, p[3] = {0, 0, 0}, v[3] = {0, 0, 0};
    // the nominal receive time: whole ms of week and the sub-ms sample offset from the reference channel's anchor
    const int64_t ds = s - a.ref_sample;
    const int64_t q = floor_div(ds, 3000), m = ds - 3000 * q;
    const int64_t nom_ms = (((a.ref_ms + 75 + q) % kWeekMs) + kWeekMs) % kWeekMs;
    if (lane < a.nchan && a.ref >= 0) {
        const gpsb200_pvt_chan_t &c = a.ch[lane];
        const gpsb200_track_epoch_t *e = a.ep + (size_t) lane * a.max_epochs;
        const int k = c.eph.valid && c.eph.health == 0 ? find_period(e, a.n[lane], s) : -1;
        if (k >= 1 && e[k - 1].lock && e[k].lock) {
            const uint64_t phi = (uint64_t) e[k - 1].code_phase + (uint64_t) (s - e[k].sample) * e[k - 1].code_step;
            const int64_t T = (((c.anchor_ms + k - c.anchor_epoch) % kWeekMs) + kWeekMs) % kWeekMs;
            const double frac = (double) phi / kCodeMod;               // ms
            const double tsv = (double) T * 1e-3 + frac * 1e-3;
            if (fabs(wrap_half_week(tsv - c.eph.toe)) <= 7200.0) {
                use = true;
                int64_t D = (a.ref_ms + 75 + q - T) % kWeekMs;
                D = D >= kWeekMs / 2 ? D - kWeekMs : (D < -kWeekMs / 2 ? D + kWeekMs : D);
                rho = (double) D * kCms + ((double) m / 3000.0 - frac) * kCms;
                rate = -kLambda * ((double) e[k - 1].carr_step * kStepHz);
                const double d0 = wrap_half_week(tsv - c.eph.toc);
                const double tt = tsv - (c.eph.af0 + d0 * (c.eph.af1 + d0 * c.eph.af2));
                satellite(c.eph, tt, p, v, dtsv, ddtsv);
            }
        }
    }
    const bool has = use;
    unsigned mask = __ballot_sync(kFull, use);
    int nused = __popc(mask);
    gpsb200_fix_t f;
    f.sample = s;
    f.nused = nused;
    f.mask = mask;
    f.iterations = 0;
    f.status = nused < 4 ? GPSB200_FIX_FEW : GPSB200_FIX_NO_CONVERGENCE;
    f.x = f.y = f.z = f.clock_m = f.t_rx = f.vx = f.vy = f.vz = f.drift = nan;
    f.lat_deg = f.lon_deg = f.height = f.pdop = f.rms = nan;
    double resid = nan;
    // RAIM: the record, and this lane's N^-1 g (position part) and 1 - h_jj of the last pass
    int verdict = GPSB200_RAIM_UNAVAILABLE, dof = 0;
    unsigned excluded = 0;
    double stat = nan, thr = nan, hpl = nan, vpl = nan, xg[3] = {0, 0, 0}, omh = 0.0;
    if (nused >= 4) {
        double X[4] = {0.0, 0.0, 0.0, 0.0};
        double h[3] = {0, 0, 0}, r = 0.0, pr_v[3] = {0, 0, 0};
        Chol ch;
        bool ok = false;
        double dX[4] = {0, 0, 0, 0};
        int it0 = 0;   // iterations of the earlier passes
#pragma unroll 1
        for (;;) {     // Gauss-Newton passes: one, or (RAIM) one more per exclusion, from the previous pass's fix
#pragma unroll 1
        for (int j = 0; j < GPSB200_PVT_MAX_ITER; j++) {
            const double rad = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
            const bool iono = a.cfg.iono && rad >= kIonoMinRadius;
            double lat = 0.0, lon = 0.0, hgt = 0.0, sla = 0.0, cla = 0.0, slo = 0.0, clo = 0.0;
            if (iono) {
                ecef_llh(X, lat, lon, hgt);
                sincos(lat, &sla, &cla);
                sincos(lon, &slo, &clo);
            }
            h[0] = h[1] = h[2] = 0.0;
            r = 0.0;
            if (has) {
                const double g0 = p[0] - X[0], g1 = p[1] - X[1], g2 = p[2] - X[2];
                const double tau = sqrt(g0 * g0 + g1 * g1 + g2 * g2) / kC;
                double sth, cth;
                sincos(kOmegaE * tau, &sth, &cth);
                const double px = p[0] * cth + p[1] * sth, py = p[1] * cth - p[0] * sth;
                pr_v[0] = v[0] * cth + v[1] * sth;
                pr_v[1] = v[1] * cth - v[0] * sth;
                pr_v[2] = v[2];
                const double l0 = px - X[0], l1 = py - X[1], l2 = p[2] - X[2];
                const double R = sqrt(l0 * l0 + l1 * l1 + l2 * l2);
                double I = 0.0;
                if (iono) {
                    const double nn = -sla * clo * l0 - sla * slo * l1 + cla * l2;
                    const double ee = -slo * l0 + clo * l1;
                    const double uu = cla * clo * l0 + cla * slo * l1 + sla * l2;
                    double az = atan2(ee, nn);
                    if (az < 0.0) az += 2.0 * kPi;
                    const double el = atan2(uu, sqrt(nn * nn + ee * ee));
                    const double trx = (double) nom_ms * 1e-3 + (double) m / 3e6 - X[3] / kC;
                    I = klobuchar(a.cfg, lat, lon, az, el, trx);
                }
                r = rho - (R + X[3] - kC * dtsv + I);
                h[0] = -l0 / R;
                h[1] = -l1 / R;
                h[2] = -l2 / R;
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
            const double y = use ? rate + kC * ddtsv + (h[0] * pr_v[0] + h[1] * pr_v[1] + h[2] * pr_v[2]) : 0.0;
            const double bv[4] = {warp_sum(h[0] * y), warp_sum(h[1] * y), warp_sum(h[2] * y), warp_sum(y)};
            double V[4];
            ch.solve(bv, V);
            const double ss = warp_sum(use ? resid * resid : 0.0);
            double Q[3];
#pragma unroll
            for (int i = 0; i < 3; i++) {
                double ei[4] = {0, 0, 0, 0}, xi[4];
                ei[i] = 1.0;
                ch.solve(ei, xi);
                Q[i] = xi[i];
            }
            f.status = GPSB200_FIX_OK;
            f.x = X[0];
            f.y = X[1];
            f.z = X[2];
            f.clock_m = X[3];
            double trx = (double) nom_ms * 1e-3 + ((double) m / 3e6 - X[3] / kC);
            f.t_rx = trx < 0.0 ? trx + 604800.0 : (trx >= 604800.0 ? trx - 604800.0 : trx);
            f.vx = V[0];
            f.vy = V[1];
            f.vz = V[2];
            f.drift = V[3];
            double lat, lon, hgt;
            ecef_llh(X, lat, lon, hgt);
            f.lat_deg = lat * (180.0 / M_PI);
            f.lon_deg = lon * (180.0 / M_PI);
            f.height = hgt;
            f.pdop = sqrt(Q[0] + Q[1] + Q[2]);
            f.rms = sqrt(ss / (double) nused);
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

template <bool kRaim> void fill(KernelArgs<kRaim> &a, const Scratch &sc);
template <> void fill<false>(Args &a, const Scratch &sc) {
    a.ep = sc.d_epochs;
    a.ch = sc.d_chans;
    a.n = sc.d_n;
    a.nchan = sc.nchan;
    a.max_epochs = sc.max_epochs;
    a.ref = sc.ref;
    a.ref_sample = sc.ref_sample;
    a.ref_ms = sc.ref_ms;
    a.cfg = sc.cfg;
    a.fixes = sc.d_fixes;
    a.res = sc.want_res ? sc.d_res : nullptr;
}
template <> void fill<true>(RaimArgs &a, const Scratch &sc) {
    fill<false>(a, sc);
    a.raim = sc.raim_cfg;
    memcpy(a.T, sc.tab_T, sizeof a.T);
    memcpy(a.lambda, sc.tab_lambda, sizeof a.lambda);
    a.out = sc.d_raim;
}

template <bool kRaim> cudaError_t launch_as(const Scratch &sc, cudaStream_t s) {
    KernelArgs<kRaim> a;
    fill<kRaim>(a, sc);
    const int64_t blocks = ((int64_t) sc.cfg.nfix + kWarps - 1) / kWarps;
    k_pvt<kRaim><<<(unsigned) blocks, kWarps * 32, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch(const Scratch &sc, cudaStream_t s) {
    return sc.raim ? launch_as<true>(sc, s) : launch_as<false>(sc, s);
}

}  // namespace

std::string check(const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs, const int32_t *nepochs,
                  int max_epochs, const gpsb200_pvt_config_t *cfg, const gpsb200_raim_config_t *raim) {
    if (!chans || !epochs || !nepochs || !cfg) return "NULL chans, epochs, nepochs or cfg";
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
    if (cfg->step < 1) return "step must be >= 1";
    if (cfg->iono != 0 && cfg->iono != 1) return "iono must be 0 or 1";
    const int64_t kLast = 1ll << 62;   // fix instants stay far from int64 overflow
    if (cfg->s0 < 0 || cfg->s0 > kLast || (int64_t) (cfg->nfix - 1) > (kLast - cfg->s0) / cfg->step)
        return "fix instants outside 0..2^62";
    for (int i = 0; i < 4; i++)
        if (!std::isfinite(cfg->alpha[i]) || !std::isfinite(cfg->beta[i])) return "alpha / beta must be finite";
    for (int c = 0; c < nchan; c++) {
        const gpsb200_pvt_chan_t &ch = chans[c];
        const std::string at = "channel " + std::to_string(c) + ": ";
        if (nepochs[c] < 0 || nepochs[c] > max_epochs) return at + "nepochs outside 0..max_epochs";
        if (ch.eph.valid != 0 && ch.eph.valid != 1) return at + "eph.valid must be 0 or 1";
        if (!ch.eph.valid) continue;   // never used: its anchor is not read
        if (ch.anchor_epoch < 0 || ch.anchor_epoch >= nepochs[c]) return at + "anchor_epoch outside the channel's epochs";
        if (ch.anchor_ms < 0 || ch.anchor_ms >= kWeekMs) return at + "anchor_ms outside 0..604799999";
    }
    return std::string();
}

void scratch_free(Scratch &sc) {
    cudaFree(sc.d_epochs);
    cudaFree(sc.d_chans);
    cudaFree(sc.d_n);
    cudaFree(sc.d_fixes);
    cudaFree(sc.d_res);
    cudaFree(sc.d_raim);
    sc = Scratch();
}

cudaError_t run(Scratch &sc, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
                const gpsb200_raim_config_t *raim, gpsb200_fix_t *fixes, double *residuals, gpsb200_raim_t *out,
                cudaStream_t s) {
    sc.have_last = false;
    if (!sc.d_chans) {
        CU_RET(cudaMalloc(&sc.d_chans, GPSB200_TRK_MAX_CHAN * sizeof(gpsb200_pvt_chan_t)));
        CU_RET(cudaMalloc(&sc.d_n, GPSB200_TRK_MAX_CHAN * sizeof(int32_t)));
    }
    CU_RET(grow(sc.d_epochs, sc.epoch_cap, (size_t) nchan * max_epochs));
    CU_RET(grow(sc.d_fixes, sc.fix_cap, (size_t) cfg->nfix));
    if (residuals) CU_RET(grow(sc.d_res, sc.res_cap, (size_t) cfg->nfix * nchan));
    sc.raim = raim != nullptr;
    if (raim) {
        CU_RET(grow(sc.d_raim, sc.raim_cap, (size_t) cfg->nfix));
        sc.raim_cfg = *raim;
        if (raim->p_fa != sc.tab_p_fa || raim->p_md != sc.tab_p_md) {   // the tables take 20-80 ms of host time
            raim_thresholds(raim->p_fa, raim->p_md, sc.tab_T, sc.tab_lambda);
            sc.tab_p_fa = raim->p_fa;
            sc.tab_p_md = raim->p_md;
        }
    }
    // the reference channel of the nominal receive time: the lowest with a valid, healthy ephemeris
    sc.ref = -1;
    for (int c = 0; c < nchan && sc.ref < 0; c++)
        if (chans[c].eph.valid && chans[c].eph.health == 0) sc.ref = c;
    sc.ref_sample = sc.ref >= 0 ? epochs[(size_t) sc.ref * max_epochs + chans[sc.ref].anchor_epoch].sample : 0;
    sc.ref_ms = sc.ref >= 0 ? chans[sc.ref].anchor_ms : 0;
    sc.nchan = nchan;
    sc.max_epochs = max_epochs;
    sc.cfg = *cfg;
    sc.want_res = residuals != nullptr;
    CU_RET(cudaMemcpyAsync(sc.d_epochs, epochs, (size_t) nchan * max_epochs * sizeof(gpsb200_track_epoch_t),
                           cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_chans, chans, nchan * sizeof(gpsb200_pvt_chan_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_n, nepochs, nchan * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU_RET(launch(sc, s));
    CU_RET(cudaMemcpyAsync(fixes, sc.d_fixes, (size_t) cfg->nfix * sizeof(gpsb200_fix_t), cudaMemcpyDeviceToHost, s));
    if (residuals)
        CU_RET(cudaMemcpyAsync(residuals, sc.d_res, (size_t) cfg->nfix * nchan * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (raim)
        CU_RET(cudaMemcpyAsync(out, sc.d_raim, (size_t) cfg->nfix * sizeof(gpsb200_raim_t), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaStreamSynchronize(s));
    sc.have_last = true;
    return cudaSuccess;
}

cudaError_t replay(Scratch &sc, cudaStream_t s) { return launch(sc, s); }

}  // namespace pvt
}  // namespace gpsb200
