// Where each satellite is in the sky from an almanac (include/gpsb200.h: gpsb200_almanac_predict; DESIGN §9.1): the
// almanac orbit at the transmit time, the line of sight from a static receiver, its azimuth / elevation and the Doppler
// the acquisition search peaks at. A warm start searches a few bins around that Doppler per visible PRN instead of the
// whole grid (gpsb200_acquire_windows). Host code, shared by the CLI and Python; tests/almanac_model.py restates it.
#include <stdint.h>

#include <cmath>
#include <cstring>

#include "../../include/gpsb200.h"
#include "synth_tables.h"

namespace {

using gpsb200::kC;
using gpsb200::kGM;
using gpsb200::kLambda;
using gpsb200::kOmegaE;
using gpsb200::kPi;
using gpsb200::kWgsA;
using gpsb200::kWgsE;

// Position, velocity (ECEF) and clock offset of the almanac orbit at GPS time (week, sow).
void orbit(const gpsb200_almanac_record_t &r, int32_t week, double sow, double *p, double *v, double &dt) {
    const double tk = (double) (week - r.toa_week) * 604800.0 + (sow - r.toa_sec);
    const double A = r.sqrta * r.sqrta;
    const double n = std::sqrt(kGM / (A * A * A));
    const double M = r.m0 * kPi + n * tk;
    double E = M;
    for (int it = 0; it < 10; it++) {
        const double dE = (M - E + r.e * std::sin(E)) / (1.0 - r.e * std::cos(E));
        E += dE;
        if (std::fabs(dE) <= 1e-14) break;
    }
    const double sE = std::sin(E), cE = std::cos(E);
    const double om = 1.0 - r.e * cE;
    const double Edot = n / om;
    const double sq = std::sqrt(1.0 - r.e * r.e);
    const double uk = std::atan2(sq * sE, cE - r.e) + r.aop * kPi;
    const double ukdot = sq * Edot / om;
    const double rk = A * om, rkdot = A * r.e * sE * Edot;
    const double ik = (0.30 + r.delta_i) * kPi;
    const double su = std::sin(uk), cu = std::cos(uk), si = std::sin(ik), ci = std::cos(ik);
    const double xp = rk * cu, yp = rk * su;
    const double xpdot = rkdot * cu - yp * ukdot, ypdot = rkdot * su + xp * ukdot;
    const double odot = r.omegadot * kPi - kOmegaE;
    const double ok = r.omega0 * kPi + tk * odot - kOmegaE * r.toa_sec;
    const double so = std::sin(ok), co = std::cos(ok);
    p[0] = xp * co - yp * ci * so;
    p[1] = xp * so + yp * ci * co;
    p[2] = yp * si;
    const double tmp = ypdot * ci;
    v[0] = -odot * p[1] + xpdot * co - tmp * so;
    v[1] = odot * p[0] + xpdot * so + tmp * co;
    v[2] = ypdot * si;
    dt = r.af0 + r.af1 * tk;
}

double dist(const double *a, const double *b) {
    const double d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
    return std::sqrt(d0 * d0 + d1 * d1 + d2 * d2);
}

// WGS-84 latitude and longitude (rad) of an ECEF point: six fixed-point steps, as the fix kernels' ecef_llh.
void latlon(const double *x, double &lat, double &lon) {
    const double e2 = kWgsE * kWgsE;
    const double p = std::sqrt(x[0] * x[0] + x[1] * x[1]);
    lon = std::atan2(x[1], x[0]);
    lat = std::atan2(x[2], p * (1.0 - e2));
    for (int it = 0; it < 6; it++) {
        const double sl = std::sin(lat);
        const double N = kWgsA / std::sqrt(1.0 - e2 * sl * sl);
        lat = std::atan2(x[2] + e2 * N * sl, p);
    }
}

}  // namespace

extern "C" int gpsb200_almanac_predict(const gpsb200_almanac_record_t rec[32], int32_t week, double sow,
                                       const double x_a[3], gpsb200_sky_t out[32]) {
    if (!rec || !x_a || !out || !std::isfinite(sow) || !std::isfinite(x_a[0]) || !std::isfinite(x_a[1]) ||
        !std::isfinite(x_a[2]))
        return GPSB200_ERR_ARG;
    double lat, lon;
    latlon(x_a, lat, lon);
    const double sla = std::sin(lat), cla = std::cos(lat), slo = std::sin(lon), clo = std::cos(lon);
    for (int i = 0; i < 32; i++) {
        const gpsb200_almanac_record_t &r = rec[i];
        gpsb200_sky_t &o = out[i];
        memset(&o, 0, sizeof o);
        o.prn = i + 1;
        if (!r.valid || !r.svid || r.toa_week < 0) continue;
        double p[3], v[3], dt;
        orbit(r, week, sow, p, v, dt);
        const double tau1 = dist(p, x_a) / kC;
        orbit(r, week, sow - tau1, p, v, dt);
        // sight: turned by the Earth's rotation over the flight time
        const double tau = dist(p, x_a) / kC;
        const double sth = std::sin(kOmegaE * tau), cth = std::cos(kOmegaE * tau);
        const double l[3] = {p[0] * cth + p[1] * sth - x_a[0], p[1] * cth - p[0] * sth - x_a[1], p[2] - x_a[2]};
        const double pv[3] = {v[0] * cth + v[1] * sth, v[1] * cth - v[0] * sth, v[2]};
        const double R = std::sqrt(l[0] * l[0] + l[1] * l[1] + l[2] * l[2]);
        const double nn = -sla * clo * l[0] - sla * slo * l[1] + cla * l[2];
        const double ee = -slo * l[0] + clo * l[1];
        const double uu = cla * clo * l[0] + cla * slo * l[1] + sla * l[2];
        double az = std::atan2(ee, nn);
        if (az < 0.0) az += 2.0 * M_PI;
        o.valid = 1;
        o.az_deg = az * (180.0 / M_PI);
        o.el_deg = std::atan2(uu, std::sqrt(nn * nn + ee * ee)) * (180.0 / M_PI);
        o.range_m = R - kC * dt;
        const double rate = (l[0] * pv[0] + l[1] * pv[1] + l[2] * pv[2]) / R;
        o.doppler_hz = -(rate - kC * r.af1) / kLambda;
    }
    return GPSB200_OK;
}
