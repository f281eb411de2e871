#!/usr/bin/env python3
"""TEST INFRASTRUCTURE -- deterministic SEM almanac files for the sky-N constellations of gen_rinex.py.

The almanac covers all 32 PRNs (so that subframe 4 pages 2-5 and 7-10, PRN 25-32, carry data too), computed from the
orbits gen_rinex.py writes for sky-32 (sky-N uses the first N of them): eccentricity, sqrt(A), rate of right
ascension, and M0 / OMEGA0 propagated from toe to toa. Angles are in semicircles, as SEM files hold them. The week is
written modulo 1024 (2296 -> 248) as Celestrak writes it; toa is 8192 s, the first multiple of 4096 s after the
02:00:00 start. Numbers use Celestrak's " %.14E" layout with three-digit exponents.

Two fields are test values rather than orbit data, chosen so that both signs of every signed almanac field are
written: delta_i (inclination relative to 0.30 semicircles) alternates by +-0.01 semicircles around 55 deg, and
af0 / af1 are negative for even PRNs. PRN 5 has a blank SVN line.

Edge files (one option each): --truncate K cuts the file inside PRN K's record, in the middle of its second orbit
line; --malformed puts a non-numeric URA into PRN 3's record; --bad-ids writes PRN 1's record with id 0 and PRN 32's
with id 40; --duplicate repeats PRN 7's record (with a different M0) after PRN 10's and announces 33 records;
--full-week writes the full week number; --week / --toa override the header.
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_rinex  # noqa: E402

TOA = 8192


def e14(v):
    """Celestrak SEM number: ' 5.12599945068359E-003' / '-1.52323007583618E-001'."""
    s = "%.14E" % v
    mant, exp = s.split("E")
    return "%s%sE%s%03d" % ("" if v < 0 else " ", mant, "-" if int(exp) < 0 else "+", abs(int(exp)))


def wrap_semi(x_rad):
    """radians -> semicircles in [-1, 1)."""
    return ((x_rad + math.pi) % (2 * math.pi) - math.pi) / math.pi


def records(toa=TOA):
    out = []
    dt = toa - gen_rinex.TOE_SOW
    omegadot = -8e-9                                    # rad/s, as in the RINEX records
    for prn, (lat, lon) in zip(range(1, 33), gen_rinex.sub_points(32)):
        el = gen_rinex.elements(prn, lat, lon)
        n = math.sqrt(gen_rinex.GM / (el["sqrta"] ** 2) ** 3) + 4.5e-9
        sign = -1.0 if prn % 2 == 0 else 1.0
        out.append(dict(
            prn=prn, svn=None if prn == 5 else 40 + prn, ura=0,
            e=el["ecc"], delta_i=el["inc"] / math.pi - 0.30 - sign * 0.01, omegadot=omegadot / math.pi,
            sqrta=el["sqrta"], omega0=wrap_semi(el["omg0"] + omegadot * dt), aop=el["aop"] / math.pi,
            m0=wrap_semi(el["m0"] + n * dt), af0=sign * 1e-5 * prn, af1=sign * 1e-11 * prn,
            health=0, config=11))
    return out


def record_lines(r, rid=None):
    return ["", "%d" % (r["prn"] if rid is None else rid), "" if r["svn"] is None else "%d" % r["svn"], "%d" % r["ura"],
            "  ".join(e14(r[k]) for k in ("e", "delta_i", "omegadot")),
            "  ".join(e14(r[k]) for k in ("sqrta", "omega0", "aop")),
            "  ".join(e14(r[k]) for k in ("m0", "af0", "af1")),
            "%d" % r["health"], "%d" % r["config"]]


def sem_text(week=gen_rinex.WEEK % 1024, toa=TOA, truncate=None, malformed=False, bad_ids=False, duplicate=False):
    recs = records(toa)
    body = []
    for r in recs:
        rid = None
        if bad_ids and r["prn"] == 1:
            rid = 0
        elif bad_ids and r["prn"] == 32:
            rid = 40
        lines = record_lines(r, rid)
        if malformed and r["prn"] == 3:
            lines[3] = "x"
        if truncate == r["prn"]:
            cut = lines[:5] + [lines[5][:len(lines[5]) // 2]]
            body += cut
            return "\n".join(["%d GPSB200.ALM" % len(recs), " %d %d" % (week, toa)] + body)   # no final newline
        body += lines
        if duplicate and r["prn"] == 10:
            d = dict(recs[6])
            d["m0"] = wrap_semi(d["m0"] * math.pi + 0.5)
            body += record_lines(d)
    count = len(recs) + (1 if duplicate else 0)
    return "\n".join(["%d GPSB200.ALM" % count, " %d %d" % (week, toa)] + body) + "\n"


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--week", type=int, default=gen_rinex.WEEK % 1024, help="header week (default: modulo 1024)")
    ap.add_argument("--full-week", action="store_true", help="write the full GPS week number")
    ap.add_argument("--toa", type=int, default=TOA, help="header time of applicability [s of week]")
    ap.add_argument("--truncate", type=int, default=None, metavar="PRN", help="end the file inside this PRN's record")
    ap.add_argument("--malformed", action="store_true")
    ap.add_argument("--bad-ids", action="store_true")
    ap.add_argument("--duplicate", action="store_true")
    a = ap.parse_args()
    week = gen_rinex.WEEK if a.full_week else a.week
    with open(a.out, "w") as f:
        f.write(sem_text(week, a.toa, a.truncate, a.malformed, a.bad_ids, a.duplicate))
