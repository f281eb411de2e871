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

--varied gives the broadcast terms the default sky leaves at one value: the
argument of perigee spread over (-pi, pi], e from 0.001 to 0.03, toe = toc +
16 j s (toc stays on the record epoch), both signs of the clock, group-delay,
harmonic and rate terms, every signed field at its most negative and most
positive integer on PRNs 1-12, IODC >= 256, non-zero URA index and health. Its
sub-satellite points are placed at 03:00:00 (VARIED_AT), between the two sets of
--sets 2, so that a run starting an hour from either toc sees the whole sky.

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


def records(nsat, sets, rx):
    """The default sky's records: -> [(set, prn, (af0, af1, af2), seven orbit rows)] with toc on the record epoch
    TOE_SOW + 7200 set."""
    out = []
    for k in range(sets):
        for prn, (lat, lon) in zip(range(1, nsat + 1), sub_points(nsat, rx)):
            el, af0 = propagate(elements(prn, lat, lon), prn, 2 * k)
            toe = TOE_SOW + 7200.0 * k
            rows = [
                (float(prn + 40 * k), 10.0 + prn, 4.5e-9, el["m0"]),            # IODE Crs dn M0
                (1e-6, el["ecc"], 5e-6, el["sqrta"]),                           # Cuc e Cus sqrtA
                (toe, 1e-8 * prn, el["omg0"], -1e-8 * prn),                     # toe Cic OMEGA0 Cis
                (el["inc"], 200.0 + prn, el["aop"], -8e-9),                     # i0 Crc omega OMEGADOT
                (1e-10, 1.0, float(WEEK), 0.0),                                 # IDOT codesL2 week L2P
                (0.0, 0.0, -1e-8, float(prn + 40 * k)),                         # sva svh tgd iodc
                (toe - 30.0, 4.0, 0.0, 0.0),                                    # tx time, fit
            ]
            out.append((k, prn, (af0, 1e-12 * prn, 0.0), rows))
    return out


VARIED_AT = 10800.0       # 03:00:00: --varied places the sub-satellite points here, an hour from either toc
# the signed fields of eph2sbf (reference gps.c:617-705): name, bits, scale (x pi for the semicircle ones)
SIGNED = [("af0", 22, 2.0 ** -31), ("af1", 16, 2.0 ** -43), ("af2", 8, 2.0 ** -55), ("tgd", 8, 2.0 ** -31),
          ("crs", 16, 2.0 ** -5), ("crc", 16, 2.0 ** -5), ("cuc", 16, 2.0 ** -29), ("cus", 16, 2.0 ** -29),
          ("cic", 16, 2.0 ** -29), ("cis", 16, 2.0 ** -29), ("deltan", 16, 2.0 ** -43 * math.pi),
          ("idot", 14, 2.0 ** -43 * math.pi)]


def limit_value(name, at_max):
    """The value of a signed field that eph2sbf's truncation toward zero turns into its most negative (at_max False)
    or most positive integer k: (k -+ 0.5) x scale, half an integer from either neighbour whatever D19.12 rounds."""
    bits, scale = next((b, sc) for f, b, sc in SIGNED if f == name)
    k = (1 << (bits - 1)) - 1 if at_max else -(1 << (bits - 1))
    return (k + (0.5 if at_max else -0.5)) * scale


def limits_of(prn):
    """--varied: PRN p in 1..12 carries SIGNED[p - 1] at its most negative integer and SIGNED[(p + 5) % 12] at its most
    positive one, in every set; so each field reaches both ends on the twelve-satellite sky."""
    if not 1 <= prn <= len(SIGNED):
        return {}
    return {SIGNED[prn - 1][0]: limit_value(SIGNED[prn - 1][0], False),
            SIGNED[(prn + 5) % len(SIGNED)][0]: limit_value(SIGNED[(prn + 5) % len(SIGNED)][0], True)}


def varied_terms(prn):
    """--varied: the terms of PRN prn other than the orbit's placement; both signs across the PRNs of every signed
    field, at magnitudes of the real constellation."""
    sg = lambda i: 1.0 if (prn + i) % 2 else -1.0
    t = dict(af0=sg(0) * 2e-5 * prn, af1=sg(1) * 3e-12 * prn, af2=sg(2) * 3e-17 * prn, tgd=sg(3) * 4e-10 * prn,
             crs=sg(4) * (12.0 + 3.5 * prn), crc=sg(5) * (150.0 + 6.0 * prn), cuc=sg(6) * (1e-6 + 2.5e-7 * prn),
             cus=sg(7) * (2e-6 + 2e-7 * prn), cic=sg(8) * (2e-8 + 1e-8 * prn), cis=sg(9) * (1e-8 + 1.5e-8 * prn),
             deltan=sg(10) * (3.5e-9 + 5e-11 * prn), idot=sg(11) * (1e-10 + 1.5e-11 * prn))
    t.update(limits_of(prn))
    # a clock term held at its limit in every set cannot be re-expressed at the next toc; the terms above it are 0 there,
    # so that every clock still continues across the sets
    if "af0" in limits_of(prn):
        t["af1"] = t["af2"] = 0.0
    if "af1" in limits_of(prn):
        t["af2"] = 0.0
    m = (prn - 1) // 2                                           # omega: +-pi (1 - (2 i + 1) / 32), never 0
    t["aop"] = (1.0 if prn % 2 else -1.0) * math.pi * (1.0 - (2 * ((7 * m) % 16) + 1) / 32.0)
    t["ecc"] = 0.001 + 0.029 * ((7 * prn) % 32) / 31.0
    t["dtoe"] = 16.0 * ((29 * prn) % 225 - 112)                  # toe - toc: 16 j s, |j| <= 112
    t["iodc"] = prn + 256 * (prn % 4)
    t["sva"] = float(prn % 7)
    t["svh"] = float(prn if prn % 8 == 3 else (32 + prn if prn % 8 == 6 else 0))
    t["omgdot"] = -(7.6e-9 + 2e-11 * prn)
    return t


def varied_records(nsat, sets, rx):
    """--varied records (same layout as records()): each orbit placed so that its sub-satellite point is sub_points()'s
    at VARIED_AT, the later sets the same orbit and clock re-expressed at their own toe / toc (M0, OMEGA0 and i0 advanced
    by their rates, af0 and af1 by af1 and af2), so that both sets give the same satellite on either side of the roll."""
    out = []
    for prn, (lat, lon) in zip(range(1, nsat + 1), sub_points(nsat, rx)):
        t = varied_terms(prn)
        ecc, aop, sqrta = t["ecc"], t["aop"], 5153.6 + 0.01 * prn
        toe0 = TOE_SOW + t["dtoe"]
        n = math.sqrt(GM / (sqrta ** 2) ** 3) + t["deltan"]
        tk = VARIED_AT - toe0
        inc = math.radians(55.0)                                 # the inclination at VARIED_AT
        s = math.sin(math.radians(lat)) / math.sin(inc)
        u = math.asin(max(-1.0, min(1.0, s)))
        if prn % 2 == 0:
            u = math.pi - u
        nu = u - aop
        E = 2.0 * math.atan2(math.sqrt(1 - ecc) * math.sin(nu / 2), math.sqrt(1 + ecc) * math.cos(nu / 2))
        m_at = E - ecc * math.sin(E)
        omg_e = math.radians(lon) - math.atan2(math.cos(inc) * math.sin(u), math.cos(u))
        for k in range(sets):
            dt = 7200.0 * k                                      # from set 0's toe (and toc) to set k's
            toc, toe = TOE_SOW + dt, toe0 + dt
            tk_k = VARIED_AT - toe
            wrap = lambda a: (a + math.pi) % (2 * math.pi) - math.pi
            m0 = wrap(m_at - n * tk_k)
            # satpos: Omega = omg0 + tk (omgdot - OMEGA_E) - OMEGA_E toe
            omg0 = wrap(omg_e - tk_k * (t["omgdot"] - OMEGA_E) + OMEGA_E * toe)
            inc0 = inc - t["idot"] * tk_k
            lim = limits_of(prn)
            af0 = lim.get("af0", t["af0"] + dt * (t["af1"] + dt * t["af2"]))     # the clock polynomial re-expressed
            af1 = lim.get("af1", t["af1"] + 2.0 * dt * t["af2"])                # at toc (a limit value stays put)
            iodc = t["iodc"] + 40 * k
            rows = [
                (float(iodc & 0xFF), t["crs"], t["deltan"], m0),                # IODE Crs dn M0
                (t["cuc"], ecc, t["cus"], sqrta),                               # Cuc e Cus sqrtA
                (toe, t["cic"], omg0, t["cis"]),                                # toe Cic OMEGA0 Cis
                (inc0, t["crc"], aop, t["omgdot"]),                             # i0 Crc omega OMEGADOT
                (t["idot"], 1.0, float(WEEK), 0.0),                             # IDOT codesL2 week L2P
                (t["sva"], t["svh"], t["tgd"], float(iodc)),                    # sva svh tgd iodc
                (toc - 30.0, 4.0, 0.0, 0.0),                                    # tx time, fit
            ]
            out.append((k, prn, (af0, af1, t["af2"]), rows))
    out.sort(key=lambda r: (r[0], r[1]))
    for k, prn, clk, rows in out:                                # every integer fits its field: nothing wraps
        v = dict(zip(("af0", "af1", "af2"), clk), crs=rows[0][1], deltan=rows[0][2], cuc=rows[1][0], cus=rows[1][2],
                 cic=rows[2][1], cis=rows[2][3], crc=rows[3][1], idot=rows[4][0], tgd=rows[5][2])
        for f, bits, scale in SIGNED:
            q = math.trunc(v[f] / scale)
            assert -(1 << (bits - 1)) <= q < (1 << (bits - 1)), (prn, k, f, q)
        assert 0 < rows[5][3] < 1024 and rows[2][0] % 16 == 0, (prn, k)
    return out


def header(L, nsat, v3, iono):
    def hdr(body, label):
        L.append("%-60s%-20s" % (body, label))

    if v3:
        hdr("     3.04           N: GNSS NAV DATA    G: GPS", "RINEX VERSION / TYPE")
    else:
        hdr("     2.10           N: GPS NAV DATA", "RINEX VERSION / TYPE")
    hdr("gpsb200 gen_rinex   synthetic sky-%-3d   20240107 020000 UTC" % nsat, "PGM / RUN BY / DATE")
    if iono and v3:
        hdr("GPSA " + d12(1.118e-8) + d12(7.451e-9) + d12(-5.96e-8) + d12(-5.96e-8), "IONOSPHERIC CORR")
        hdr("GPSB " + d12(9.011e4) + d12(1.638e4) + d12(-1.966e5) + d12(-6.554e4), "IONOSPHERIC CORR")
    elif iono:
        hdr("  " + d12(1.118e-8) + d12(7.451e-9) + d12(-5.96e-8) + d12(-5.96e-8), "ION ALPHA")
        hdr("  " + d12(9.011e4) + d12(1.638e4) + d12(-1.966e5) + d12(-6.554e4), "ION BETA")
    if v3:
        hdr("GPUT " + d17(9.313225746155e-10) + d16(8.881784197001e-16) + "%7d%5d" % (61440, WEEK), "TIME SYSTEM CORR")
    else:
        hdr("   " + d19(9.313225746155e-10) + d19(8.881784197001e-16) + "%9d%9d" % (61440, WEEK),
            "DELTA-UTC: A0,A1,T,W")
    hdr("%6d" % 18, "LEAP SECONDS")
    hdr("", "END OF HEADER")


def write3(path, nsat, sets=1, rx=(RX_LAT, RX_LON), iono=True, varied=False):
    """RINEX 3 flavour of the same constellation, laid out as readRinex3 parses it
    (reference gps.c:1512-1891): IONOSPHERIC CORR GPSA/GPSB 4D12.4 at column 5, TIME SYSTEM CORR
    GPUT D17.10,D16.9,I7,I5, records 'Gnn yyyy mm dd hh mm ss' + 3D19.12, orbit lines 4X,4D19.12."""
    L = []
    header(L, nsat, True, iono)
    for k, prn, clk, rows in (varied_records if varied else records)(nsat, sets, rx):
        L.append("G%02d 2024 01 07 %02d 00 00" % (prn, 2 + 2 * k) + "".join(d19(v) for v in clk))
        for r in rows:
            L.append("    " + "".join(d19(v) for v in r))
    with open(path, "w") as f:
        f.write("\n".join(L) + "\n")


def write(path, nsat, sets=1, rx=(RX_LAT, RX_LON), iono=True, varied=False):
    L = []
    header(L, nsat, False, iono)
    # one record set every two hours (the reference starts a new set when toc advances by more than an hour,
    # gps.c:1380-1392, and rolls to it one hour before its toc, gps.c:2890-2905)
    for k, prn, clk, rows in (varied_records if varied else records)(nsat, sets, rx):
        L.append("%2d 24  1  7 %2d  0  0.0" % (prn, 2 + 2 * k) + "".join(d19(v) for v in clk))
        for r in rows:
            L.append("   " + "".join(d19(v) for v in r))
    with open(path, "w") as f:
        f.write("\n".join(L) + "\n")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--nsat", type=int, default=12)
    ap.add_argument("--out", required=True)
    ap.add_argument("--v3", action="store_true", help="write RINEX 3 instead of RINEX 2")
    ap.add_argument("--sets", type=int, default=1, help="ephemeris sets, two hours apart")
    ap.add_argument("--rx", default="%r,%r" % (RX_LAT, RX_LON), help="LAT,LON [deg] of the receiver the sky is centred on")
    ap.add_argument("--no-iono", action="store_true", help="leave out the Klobuchar alpha / beta header lines")
    ap.add_argument("--varied", action="store_true", help="vary the broadcast terms across the PRNs (module docstring)")
    a = ap.parse_args()
    rx = tuple(float(v) for v in a.rx.split(","))
    (write3 if a.v3 else write)(a.out, a.nsat, a.sets, rx, not a.no_iono, a.varied)
