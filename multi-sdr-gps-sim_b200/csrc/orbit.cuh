// Device pieces of the fix kernels (pvt.cu) that collective detection (collective.cu) shares: the satellite from its
// ephemeris, the WGS-84 conversion and frame, and the coarse-time prediction of a transmit time. They live in pvt's
// unnamed namespace in every translation unit that includes them, so pvt.cu compiles them as it did when they were its
// own.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gpsb200.h"
#include "synth_tables.h"

namespace gpsb200 {
namespace pvt {
namespace {

constexpr double kRelF = -4.442807633e-10;        // relativistic clock term, s / m^1/2

__device__ inline double wrap_half_week(double d) { return d > 302400.0 ? d - 604800.0 : (d < -302400.0 ? d + 604800.0 : d); }

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

// The geodetic frame at an ECEF point: latitude and longitude (rad) and their sines and cosines; all 0 until set.
struct Geo {
    double lat = 0.0, lon = 0.0, sla = 0.0, cla = 0.0, slo = 0.0, clo = 0.0;
    __device__ void set(const double *x) {
        double hgt;
        ecef_llh(x, lat, lon, hgt);
        sincos(lat, &sla, &cla);
        sincos(lon, &slo, &clo);
    }
};

// gpsb200_pvt_coarse's header step 3: the predicted transmit time (ms, satellite time) of a satellite at position x and
// receive time t, and sin(elevation) seen along the up vector `up` (unit, ECEF). kRate: also the range rate e . v_rot
// of a static receiver (m/s; e = l / (c tau), v_rot the satellite velocity turned as p is) and the satellite clock
// drift (s/s), both of the last step (collective detection's Doppler, gpsb200_collective step 5).
template <bool kRate>
__device__ __forceinline__ double predict_steps(const gpsb200_ephemeris_t &e, const double *x, double t,
                                                const double *up, double &sel, double *rate, double *drift) {
    double tau = 0.075, p[3], v[3], dt = 0.0, ddt;
    double l0 = 0.0, l1 = 0.0, l2 = 0.0, v0 = 0.0, v1 = 0.0;
#pragma unroll 1
    for (int i = 0; i < 3; i++) {
        satellite(e, t - tau, p, v, dt, ddt);
        double sth, cth;
        sincos(kOmegaE * tau, &sth, &cth);
        l0 = p[0] * cth + p[1] * sth - x[0];
        l1 = p[1] * cth - p[0] * sth - x[1];
        l2 = p[2] - x[2];
        if constexpr (kRate) {
            v0 = v[0] * cth + v[1] * sth;
            v1 = v[1] * cth - v[0] * sth;
        }
        tau = sqrt(l0 * l0 + l1 * l1 + l2 * l2) / kC;
    }
    sel = (up[0] * l0 + up[1] * l1 + up[2] * l2) / (tau * kC);
    if constexpr (kRate) {
        *rate = (l0 * v0 + l1 * v1 + l2 * v[2]) / (tau * kC);
        *drift = ddt;
    }
    return 1000.0 * (t - tau + dt);
}

__device__ double predict(const gpsb200_ephemeris_t &e, const double *x, double t, const double *up, double &sel) {
    return predict_steps<false>(e, x, t, up, sel, nullptr, nullptr);
}

__device__ inline double round_half_up(double v) { return floor(v + 0.5); }

}  // namespace
}  // namespace pvt
}  // namespace gpsb200
