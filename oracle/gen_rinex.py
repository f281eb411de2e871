#!/usr/bin/env python3
"""TEST INFRASTRUCTURE -- deterministic synthetic RINEX-2 navigation files.

The reference repository bundles no ephemeris file (SURVEY.md finding 2), so the
scenarios of BASELINE.json are driven by formulaic "sky-N" constellations: N GPS
satellites (PRN 1..N) on i = 55 deg near-circular orbits whose sub-satellite
points at toe are spread over the sky of the receiver, so that all N are above
the horizon of the static Tokyo location for the whole run.  No RNG anywhere.

--rx LAT,LON centres the same rings on another receiver (night, polar and
southern skies for the ionosphere term); --no-iono leaves out ION ALPHA and
ION BETA, so that the reader finds DELTA-UTC and LEAP SECONDS only and takes
the ionosphere parameters as invalid (gps.c:1255-1257).

Layout follows what readRinex2 parses (reference gps.c:1131-1505): header labels
at column 60, ION ALPHA/BETA 2X,4D12.4, DELTA-UTC 3X,2D19.12,2I9, LEAP SECONDS
I6; records I2,1X,I2.2,4(1X,I2),F5.1,3D19.12 then seven lines of 3X,4D19.12.
"""
import argparse
import math

GM = 3.986005e14
OMEGA_E = 7.2921151467e-5
TOE_SOW = 7200.0          # 2024-01-07 02:00:00 = GPS week 2296, sow 7200
WEEK = 2296
RX_LAT, RX_LON = 35.681298, 139.766247


def d19(v):
    """Fortran D19.12: ' 0.123456789012D+01'."""
    if v == 0.0:
        return " 0.000000000000D+00"
    s = "-" if v < 0 else " "
    a = abs(v)
    e = int(math.floor(math.log10(a))) + 1
    m = a / 10.0 ** e
    ms = "%.12f" % m
    if ms.startswith("1."):          # rounding carried to 1.0
        e += 1
        ms = "%.12f" % (a / 10.0 ** e)
    return "%s%sD%s%02d" % (s, ms, "+" if e >= 0 else "-", abs(e))


def d12(v):
    """Fortran D12.4."""
    if v == 0.0:
        return "  0.0000D+00"
    s = "-" if v < 0 else " "
    a = abs(v)
    e = int(math.floor(math.log10(a))) + 1
    ms = "%.4f" % (a / 10.0 ** e)
    if ms.startswith("1."):
        e += 1
        ms = "%.4f" % (a / 10.0 ** e)
    return " %s%sD%s%02d" % (s, ms, "+" if e >= 0 else "-", abs(e))


def sub_points(n, rx=(RX_LAT, RX_LON)):
    """n sub-satellite points (lat, lon in deg) around the receiver rx: rings of
    great-circle radius 10/24/38/52/62 deg, azimuths staggered, |latitude| kept
    below 52 deg so an i = 55 deg orbit can reach it."""
    rings = [(10.0, 3), (24.0, 6), (38.0, 8), (52.0, 8), (62.0, 7)]
    pts = []
    for r_deg, cnt in rings:
        for k in range(cnt):
            az = 360.0 * (k + 0.5 * (len(pts) % 2)) / cnt + 7.0 * r_deg
            pts.append((r_deg, az % 360.0))
    out = []
    lat0, lon0 = math.radians(rx[0]), math.radians(rx[1])
    for r_deg, az in pts:
        # fold azimuths that would push the point beyond 52 deg latitude toward the equator
        r, a = math.radians(r_deg), math.radians(az)
        lat = math.asin(math.sin(lat0) * math.cos(r) + math.cos(lat0) * math.sin(r) * math.cos(a))
        if abs(math.degrees(lat)) > 52.0:
            a = math.pi - a          # mirror north <-> south, keeps east/west component
            lat = math.asin(math.sin(lat0) * math.cos(r) + math.cos(lat0) * math.sin(r) * math.cos(a))
        lon = lon0 + math.atan2(math.sin(a) * math.sin(r) * math.cos(lat0),
                                math.cos(r) - math.sin(lat0) * math.sin(lat))
        out.append((math.degrees(lat), math.degrees(lon)))
    assert len(out) >= n
    return out[:n]


def elements(prn, lat_deg, lon_deg):
    inc = math.radians(55.0)
    ecc = 0.0005 + 1e-4 * prn
    sqrta = 5153.6 + 0.01 * prn
    aop = 0.0
    s = math.sin(math.radians(lat_deg)) / math.sin(inc)
    u = math.asin(max(-1.0, min(1.0, s)))
    if prn % 2 == 0:                 # alternate ascending / descending passes
        u = math.pi - u
    # longitude of the ascending node in the Earth-fixed frame at toe
    omg_e = math.radians(lon_deg) - math.atan2(math.cos(inc) * math.sin(u), math.cos(u))
    omg0 = omg_e + OMEGA_E * TOE_SOW          # satpos: ok = omg0 + tk*omgkdot - OMEGA_EARTH*toe.sec
    omg0 = (omg0 + math.pi) % (2 * math.pi) - math.pi
    nu = u - aop                               # true anomaly
    E = 2.0 * math.atan2(math.sqrt(1 - ecc) * math.sin(nu / 2), math.sqrt(1 + ecc) * math.cos(nu / 2))
    m0 = E - ecc * math.sin(E)
    m0 = (m0 + math.pi) % (2 * math.pi) - math.pi
    return dict(inc=inc, ecc=ecc, sqrta=sqrta, aop=aop, omg0=omg0, m0=m0)


def d17(v):
    """Fortran D17.10 (RINEX 3 TIME SYSTEM CORR a0)."""
    if v == 0.0:
        return " 0.0000000000D+00"
    sgn = "-" if v < 0 else " "
    a = abs(v)
    e = int(math.floor(math.log10(a))) + 1
    ms = "%.10f" % (a / 10.0 ** e)
    if ms.startswith("1."):
        e += 1
        ms = "%.10f" % (a / 10.0 ** e)
    return "%s%sD%s%02d" % (sgn, ms, "+" if e >= 0 else "-", abs(e))


def d16(v):
    """Fortran D16.9 (RINEX 3 TIME SYSTEM CORR a1)."""
    if v == 0.0:
        return " 0.000000000D+00"
    sgn = "-" if v < 0 else " "
    a = abs(v)
    e = int(math.floor(math.log10(a))) + 1
    ms = "%.9f" % (a / 10.0 ** e)
    if ms.startswith("1."):
        e += 1
        ms = "%.9f" % (a / 10.0 ** e)
    return "%s%sD%s%02d" % (sgn, ms, "+" if e >= 0 else "-", abs(e))


def write3(path, nsat, rx=(RX_LAT, RX_LON), iono=True):
    """RINEX 3 flavour of the same constellation, laid out as readRinex3 parses it
    (reference gps.c:1512-1891): IONOSPHERIC CORR GPSA/GPSB 4D12.4 at column 5, TIME SYSTEM CORR
    GPUT D17.10,D16.9,I7,I5, records 'Gnn yyyy mm dd hh mm ss' + 3D19.12, orbit lines 4X,4D19.12."""
    L = []

    def hdr(body, label):
        L.append("%-60s%-20s" % (body, label))

    hdr("     3.04           N: GNSS NAV DATA    G: GPS", "RINEX VERSION / TYPE")
    hdr("gpsb200 gen_rinex   synthetic sky-%-3d   20240107 020000 UTC" % nsat, "PGM / RUN BY / DATE")
    if iono:
        hdr("GPSA " + d12(1.118e-8) + d12(7.451e-9) + d12(-5.96e-8) + d12(-5.96e-8), "IONOSPHERIC CORR")
        hdr("GPSB " + d12(9.011e4) + d12(1.638e4) + d12(-1.966e5) + d12(-6.554e4), "IONOSPHERIC CORR")
    hdr("GPUT " + d17(9.313225746155e-10) + d16(8.881784197001e-16) + "%7d%5d" % (61440, WEEK), "TIME SYSTEM CORR")
    hdr("%6d" % 18, "LEAP SECONDS")
    hdr("", "END OF HEADER")
    for prn, (lat, lon) in zip(range(1, nsat + 1), sub_points(nsat, rx)):
        el = elements(prn, lat, lon)
        L.append("G%02d 2024 01 07 02 00 00" % prn + d19(1e-5 * prn) + d19(1e-12 * prn) + d19(0.0))
        rows = [
            (float(prn), 10.0 + prn, 4.5e-9, el["m0"]),
            (1e-6, el["ecc"], 5e-6, el["sqrta"]),
            (TOE_SOW, 1e-8 * prn, el["omg0"], -1e-8 * prn),
            (el["inc"], 200.0 + prn, el["aop"], -8e-9),
            (1e-10, 1.0, float(WEEK), 0.0),
            (0.0, 0.0, -1e-8, float(prn)),
            (TOE_SOW - 30.0, 4.0, 0.0, 0.0),
        ]
        for r in rows:
            L.append("    " + "".join(d19(v) for v in r))
    with open(path, "w") as f:
        f.write("\n".join(L) + "\n")


def propagate(el, prn, hours):
    """The same orbit re-expressed at toe + hours (continuous with the first set): M0 and OMEGA0 advance
    with their rates (satpos, reference gps.c:361-460)."""
    if hours == 0:
        return dict(el), 1e-5 * prn
    dt = 3600.0 * hours
    n = math.sqrt(GM / (el["sqrta"] ** 2) ** 3) + 4.5e-9
    e2 = dict(el)
    e2["m0"] = (el["m0"] + n * dt + math.pi) % (2 * math.pi) - math.pi
    e2["omg0"] = (el["omg0"] + (-8e-9) * dt + math.pi) % (2 * math.pi) - math.pi
    return e2, 1e-5 * prn + 1e-12 * prn * dt


def write(path, nsat, sets=1, rx=(RX_LAT, RX_LON), iono=True):
    L = []

    def hdr(body, label):
        L.append("%-60s%-20s" % (body, label))

    hdr("     2.10           N: GPS NAV DATA", "RINEX VERSION / TYPE")
    hdr("gpsb200 gen_rinex   synthetic sky-%-3d   20240107 020000 UTC" % nsat, "PGM / RUN BY / DATE")
    if iono:
        hdr("  " + d12(1.118e-8) + d12(7.451e-9) + d12(-5.96e-8) + d12(-5.96e-8), "ION ALPHA")
        hdr("  " + d12(9.011e4) + d12(1.638e4) + d12(-1.966e5) + d12(-6.554e4), "ION BETA")
    hdr("   " + d19(9.313225746155e-10) + d19(8.881784197001e-16) + "%9d%9d" % (61440, WEEK), "DELTA-UTC: A0,A1,T,W")
    hdr("%6d" % 18, "LEAP SECONDS")
    hdr("", "END OF HEADER")
    # one record set every two hours (the reference starts a new set when toc advances by more than an hour,
    # gps.c:1380-1392, and rolls to it one hour before its toc, gps.c:2890-2905)
    for k in range(sets):
        for prn, (lat, lon) in zip(range(1, nsat + 1), sub_points(nsat, rx)):
            el, af0 = propagate(elements(prn, lat, lon), prn, 2 * k)
            toe = TOE_SOW + 7200.0 * k
            L.append("%2d 24  1  7 %2d  0  0.0" % (prn, 2 + 2 * k) + d19(af0) + d19(1e-12 * prn) + d19(0.0))
            rows = [
                (float(prn + 40 * k), 10.0 + prn, 4.5e-9, el["m0"]),            # IODE Crs dn M0
                (1e-6, el["ecc"], 5e-6, el["sqrta"]),                           # Cuc e Cus sqrtA
                (toe, 1e-8 * prn, el["omg0"], -1e-8 * prn),                     # toe Cic OMEGA0 Cis
                (el["inc"], 200.0 + prn, el["aop"], -8e-9),                     # i0 Crc omega OMEGADOT
                (1e-10, 1.0, float(WEEK), 0.0),                                 # IDOT codesL2 week L2P
                (0.0, 0.0, -1e-8, float(prn + 40 * k)),                         # sva svh tgd iodc
                (toe - 30.0, 4.0, 0.0, 0.0),                                    # tx time, fit
            ]
            for r in rows:
                L.append("   " + "".join(d19(v) for v in r))
    with open(path, "w") as f:
        f.write("\n".join(L) + "\n")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--nsat", type=int, default=12)
    ap.add_argument("--out", required=True)
    ap.add_argument("--v3", action="store_true", help="write RINEX 3 instead of RINEX 2")
    ap.add_argument("--sets", type=int, default=1, help="ephemeris sets, two hours apart (RINEX 2 only)")
    ap.add_argument("--rx", default="%r,%r" % (RX_LAT, RX_LON), help="LAT,LON [deg] of the receiver the sky is centred on")
    ap.add_argument("--no-iono", action="store_true", help="leave out the Klobuchar alpha / beta header lines")
    a = ap.parse_args()
    rx = tuple(float(v) for v in a.rx.split(","))
    if a.v3:
        write3(a.out, a.nsat, rx, not a.no_iono)
    else:
        write(a.out, a.nsat, a.sets, rx, not a.no_iono)
