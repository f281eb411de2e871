"""Numpy statement of the almanac prediction (include/gpsb200.h: gpsb200_almanac_predict; DESIGN §9.1) and of the
almanac page layout (IS-GPS-200 20.3.3.5.1.2): the tests' reference. It shares no code with the library."""
import math

import numpy as np

GM = 3.986005e14
OMEGA_E = 7.2921151467e-5
PI = 3.1415926535898                 # the reference's pi, for semicircles
C = 2.99792458e8
LAMBDA_L1 = 0.190293672798365
WGS_A, WGS_E = 6378137.0, 0.0818191908426
WEEK_S = 604800.0

# the engine's almanac scales (the reference's gps.h literals): two of them are not exact powers of two
ENGINE_SCALE = {"e": 4.76837158203125e-007, "delta_i": 2.0 ** -19, "omegadot": 3.63797880709171e-012,
                "sqrta": 0.00048828125, "omega0": 1.19209289550781e-007, "aop": 1.19209289550781e-007,
                "m0": 1.19209289550781e-007, "af0": 9.5367431640625e-007, "af1": 3.63797880709171e-012}
# IS-GPS-200: bits, signed, exact scale
FIELDS = {"e": (16, False, 2.0 ** -21), "delta_i": (16, True, 2.0 ** -19), "omegadot": (16, True, 2.0 ** -38),
          "sqrta": (24, False, 2.0 ** -11), "omega0": (24, True, 2.0 ** -23), "aop": (24, True, 2.0 ** -23),
          "m0": (24, True, 2.0 ** -23), "af0": (11, True, 2.0 ** -20), "af1": (11, True, 2.0 ** -38)}


def engine_integer(name, sem_value):
    """The integer the engine transmits for a SEM value: C's (long) truncation of value / literal scale, kept to the
    field's width as two's complement."""
    bits = FIELDS[name][0]
    v = int(math.trunc(sem_value / ENGINE_SCALE[name]))
    v &= (1 << bits) - 1
    return v - (1 << bits) if FIELDS[name][1] and v >= 1 << (bits - 1) else v


def orbit(r, week, sow):
    """Position, velocity (ECEF) and clock offset of the almanac orbit of record r at GPS time (week, sow)."""
    tk = float(week - int(r["toa_week"])) * WEEK_S + (sow - float(r["toa_sec"]))
    A = float(r["sqrta"]) ** 2
    n = math.sqrt(GM / (A * A * A))
    M = float(r["m0"]) * PI + n * tk
    e = float(r["e"])
    E = M
    for _ in range(10):
        dE = (M - E + e * math.sin(E)) / (1.0 - e * math.cos(E))
        E += dE
        if abs(dE) <= 1e-14:
            break
    om = 1.0 - e * math.cos(E)
    Edot = n / om
    nu = math.atan2(math.sqrt(1.0 - e * e) * math.sin(E), math.cos(E) - e)
    u = nu + float(r["aop"]) * PI
    udot = math.sqrt(1.0 - e * e) * Edot / om
    rad, raddot = A * om, A * e * math.sin(E) * Edot
    inc = (0.30 + float(r["delta_i"])) * PI
    Om = float(r["omega0"]) * PI + (float(r["omegadot"]) * PI - OMEGA_E) * tk - OMEGA_E * float(r["toa_sec"])
    Omdot = float(r["omegadot"]) * PI - OMEGA_E
    # in-plane position and velocity, rotated into ECEF: R3(-Omega) R1(-i)
    xp, yp = rad * math.cos(u), rad * math.sin(u)
    vxp = raddot * math.cos(u) - rad * math.sin(u) * udot
    vyp = raddot * math.sin(u) + rad * math.cos(u) * udot
    R1 = np.array([[1, 0, 0], [0, math.cos(inc), -math.sin(inc)], [0, math.sin(inc), math.cos(inc)]])
    R3 = np.array([[math.cos(Om), -math.sin(Om), 0], [math.sin(Om), math.cos(Om), 0], [0, 0, 1]])
    p = R3 @ R1 @ np.array([xp, yp, 0.0])
    v = R3 @ R1 @ np.array([vxp, vyp, 0.0]) + np.cross([0.0, 0.0, Omdot], p)
    return p, v, float(r["af0"]) + float(r["af1"]) * tk


def geodetic_latlon(x):
    e2 = WGS_E ** 2
    p = math.hypot(x[0], x[1])
    lat = math.atan2(x[2], p * (1 - e2))
    for _ in range(6):
        N = WGS_A / math.sqrt(1 - e2 * math.sin(lat) ** 2)
        lat = math.atan2(x[2] + e2 * N * math.sin(lat), p)
    return lat, math.atan2(x[1], x[0])


def predict(rec, week, sow, x_a):
    """-> dict prn -> (el_deg, az_deg, range_m, doppler_hz) for every record predicted."""
    x = np.asarray(x_a, np.float64)
    lat, lon = geodetic_latlon(x)
    up = np.array([math.cos(lat) * math.cos(lon), math.cos(lat) * math.sin(lon), math.sin(lat)])
    north = np.array([-math.sin(lat) * math.cos(lon), -math.sin(lat) * math.sin(lon), math.cos(lat)])
    east = np.array([-math.sin(lon), math.cos(lon), 0.0])
    out = {}
    for i, r in enumerate(rec):
        if not (int(r["valid"]) and int(r["svid"]) and int(r["toa_week"]) >= 0):
            continue
        p, _, _ = orbit(r, week, sow)
        tau1 = np.linalg.norm(p - x) / C
        p, v, dt = orbit(r, week, sow - tau1)
        th = OMEGA_E * np.linalg.norm(p - x) / C
        rot = np.array([[math.cos(th), math.sin(th), 0], [-math.sin(th), math.cos(th), 0], [0, 0, 1]])
        l = rot @ p - x
        R = np.linalg.norm(l)
        el = math.degrees(math.atan2(l @ up, math.hypot(l @ north, l @ east)))
        az = math.degrees(math.atan2(l @ east, l @ north)) % 360.0
        rate = l @ (rot @ v) / R
        out[i + 1] = (el, az, R - C * dt, -(rate - C * float(r["af1"])) / LAMBDA_L1)
    return out


def llh_to_ecef(lat_deg, lon_deg, h):
    la, lo = math.radians(lat_deg), math.radians(lon_deg)
    e2 = WGS_E ** 2
    N = WGS_A / math.sqrt(1 - e2 * math.sin(la) ** 2)
    return np.array([(N + h) * math.cos(la) * math.cos(lo), (N + h) * math.cos(la) * math.sin(lo),
                     (N * (1 - e2) + h) * math.sin(la)])
