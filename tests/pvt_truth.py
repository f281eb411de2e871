"""Truth for position fixes from the scenario: the broadcast ephemeris as the RINEX file holds it and as eph2sbf
quantises it, "ideal epochs" (what a perfect tracking loop would record) from the scenario's channel records, and the
true receiver position, velocity and time at any sample.

Time: sample s of a run is received at GPS time start + s / 3e6 (block b is made at receive time start + 0.1 b).
Position: block b's records are computed at xyz[b] and their code phase and frequency carry the range linearly to
xyz[b + 1] (gps.c:2703-2744), so the position at sample s is xyz[b] moved linearly towards xyz[b + 1]. Static runs
have xyz[b] = the -l point for every b; motion runs the motion file's rows."""
import numpy as np

import pvt_model as PM

BLOCK = 300000
FS = 3e6
WEEK_MS = 604800000


# ---- the RINEX file of oracle/gen_rinex.py -------------------------------------------------------------------------
def _d(s):
    return float(s.replace("D", "E"))


def _sow(y, m, d, hh, mi, sec):
    """GPS second of week of a record epoch (UTC taken as GPS time, as the reference's date2gps does)."""
    import datetime
    dt = datetime.datetime(y, m, d, hh, mi) - datetime.datetime(1980, 1, 6)
    return (dt.days * 86400 + dt.seconds) % 604800 + sec


def read_rinex_sets(path):
    """-> ([{prn: record} per set], ion_alpha[4], ion_beta[4]) of a RINEX-2 or RINEX-3 navigation file as gen_rinex
    writes it. A record holds every broadcast field by name (sva and svh as written, before the reader's +32), and toc,
    the second of week of its epoch line. A set starts where the epoch passes the set's first by more than an hour, as the
    reference groups them (gps.c:1380-1392)."""
    lines = open(path).read().splitlines()
    v3 = float(lines[0][:9]) >= 3.0
    alpha = beta = None
    i = 0
    while "END OF HEADER" not in lines[i]:
        label, ln = lines[i][60:].strip(), lines[i]
        if label == "ION ALPHA" or (label == "IONOSPHERIC CORR" and ln.startswith("GPSA")):
            alpha = [_d(ln[(5 if v3 else 2) + 12 * k:(17 if v3 else 14) + 12 * k]) for k in range(4)]
        if label == "ION BETA" or (label == "IONOSPHERIC CORR" and ln.startswith("GPSB")):
            beta = [_d(ln[(5 if v3 else 2) + 12 * k:(17 if v3 else 14) + 12 * k]) for k in range(4)]
        i += 1
    i += 1
    sets, first = [], None
    names = ["iode", "crs", "deltan", "m0", "cuc", "ecc", "cus", "sqrta", "toe", "cic", "omg0", "cis", "inc0", "crc",
             "aop", "omgdot", "idot", "codes", "week", "l2p", "sva", "svh", "tgd", "iodc", "ttx", "fit", "sp1", "sp2"]
    c0 = 4 if v3 else 3
    while i + 7 < len(lines) + 1 and i < len(lines):
        head = lines[i]
        if v3:
            prn, y, m, d, hh, mi, sec = (int(head[1:3]), int(head[4:8]), int(head[9:11]), int(head[12:14]),
                                         int(head[15:17]), int(head[18:20]), float(head[21:23]))
            c = 23
        else:
            prn, y, m, d, hh, mi, sec = (int(head[0:2]), 2000 + int(head[3:5]), int(head[6:8]), int(head[9:11]),
                                         int(head[12:14]), int(head[15:17]), float(head[17:22]))
            c = 22
        r = dict(af0=_d(head[c:c + 19]), af1=_d(head[c + 19:c + 38]), af2=_d(head[c + 38:c + 57]))
        vals = []
        for k in range(1, 8):
            ln = lines[i + k]
            vals += [_d(ln[c0 + 19 * j:c0 + 19 + 19 * j]) for j in range(4)]
        r.update(zip(names, vals))
        r["toc"] = _sow(y, m, d, hh, mi, sec)
        if first is None or r["toc"] - first > 3600.0:
            first = r["toc"]
            sets.append({})
        sets[-1].setdefault(prn, r)
        i += 8
    return sets, np.array(alpha), np.array(beta)


def read_rinex(path):
    """-> (records {prn: dict}, ion_alpha[4], ion_beta[4]) of the first set of a navigation file (read_rinex_sets)."""
    sets, alpha, beta = read_rinex_sets(path)
    return sets[0], alpha, beta


# integer field of eph2sbf (gps.c:662-684: truncation toward zero) and its scale; x pi for semicircles
EPH_FIELDS = {"toc": 16.0, "toe": 16.0, "af0": 2.0 ** -31, "af1": 2.0 ** -43, "af2": 2.0 ** -55, "tgd": 2.0 ** -31,
              "crs": 2.0 ** -5, "crc": 2.0 ** -5, "cuc": 2.0 ** -29, "cus": 2.0 ** -29, "cic": 2.0 ** -29,
              "cis": 2.0 ** -29, "ecc": 2.0 ** -33, "sqrta": 2.0 ** -19, "deltan": 2.0 ** -43 * PM.PI,
              "m0": 2.0 ** -31 * PM.PI, "omg0": 2.0 ** -31 * PM.PI, "inc0": 2.0 ** -31 * PM.PI,
              "aop": 2.0 ** -31 * PM.PI, "omgdot": 2.0 ** -43 * PM.PI, "idot": 2.0 ** -43 * PM.PI}
SEMICIRCLE = {"deltan": 2.0 ** -43, "m0": 2.0 ** -31, "omg0": 2.0 ** -31, "inc0": 2.0 ** -31, "aop": 2.0 ** -31,
              "omgdot": 2.0 ** -43, "idot": 2.0 ** -43}


def eph2sbf_value(rec, f):
    """What the broadcast field f of a RINEX record decodes to: eph2sbf's integer times the scale."""
    if f in SEMICIRCLE:
        return float(np.trunc(rec[f] / SEMICIRCLE[f] / PM.PI)) * SEMICIRCLE[f] * PM.PI
    return float(np.trunc(rec[f] / EPH_FIELDS[f])) * EPH_FIELDS[f]


def klobuchar_broadcast(alpha, beta):
    """alpha / beta as page 18 carries them (gps.c:686-693: rounded to the scale)."""
    sa = [2.0 ** -30, 2.0 ** -27, 2.0 ** -24, 2.0 ** -24]
    sb = [2048.0, 16384.0, 65536.0, 65536.0]
    return (np.array([np.round(a / s) * s for a, s in zip(alpha, sa)]),
            np.array([np.round(b / s) * s for b, s in zip(beta, sb)]))


# ---- ideal epochs and anchors ------------------------------------------------------------------------------------
def frame_ms0(frames, f):
    """Transmit time (ms of week) of the start of NAV frame slot f: word 11 is subframe 1's HOW, first bit at
    6 TOW - 5.4 s, 6.6 s into the slot."""
    slot = next(s for s in frames[f] if s.any())
    how = (int(slot[11]) >> 6) & 0xFFFFFF
    if int(slot[10]) & 1:
        how ^= 0xFFFFFF
    tow = (how >> 7) & 0x1FFFF
    return 6000 * tow - 12000


def ideal_epochs(ch, prn, frames, frame_of_block):
    """The epoch records a perfect loop would make for prn over the blocks of ch (consecutive from sample 0): a period
    starts at each sample where the signal's code phase has just wrapped; code_phase (at the next period's start, 2^-32
    chips) and code_step / carr_step (of the next period) from the records' code_phase + f_code t and f_carr; lock 1.
    -> (epochs TRACK_EPOCH array, anchor_epoch 0, anchor_ms of epoch 0)."""
    import track_model as T
    blk, slot = np.nonzero(ch["prn"] == prn)
    rec = ch[blk, slot]
    cp0, fc, fcar = (rec[f].astype(np.float64)[:, None] for f in ("code_phase", "f_code", "f_carr"))
    base = (blk * BLOCK)[:, None]
    j = np.arange(0, 102)[None, :]
    sj = np.ceil(base + (1023.0 * j - cp0) * FS / fc).astype(np.int64)
    inside = (sj >= base) & (sj < base + BLOCK)    # j = 0: a wrap less than a sample before the block start
    cp = cp0 + fc * (sj - base) / FS
    ms0 = np.array([frame_ms0(frames, f) for f in range(len(frames))], np.int64)
    total = (rec["iword"].astype(np.int64) * 600 + rec["ibit"] * 20 + rec["icode"])[:, None] + j
    tx = np.mod(ms0[np.asarray(frame_of_block)[blk]][:, None] + total, WEEK_MS)[inside]
    n = int(inside.sum())
    e = np.zeros(n, T.EPOCH_DTYPE)
    e["sample"] = sj[inside]
    phases = np.maximum(0, np.round((cp - 1023.0 * j) * 2.0 ** 32)).astype(np.int64)[inside]
    e["code_phase"][:-1] = phases[1:] % (1 << 32)
    e["code_step"][:-1] = np.broadcast_to(np.round(fc / FS * 2.0 ** 32), sj.shape)[inside][1:]
    e["carr_step"][:-1] = np.broadcast_to(np.round(fcar * 2.0 ** 32 / FS), sj.shape)[inside][1:]
    e["lock"] = 1
    assert np.all(np.mod(np.diff(tx), WEEK_MS) == 1)
    return e, 0, int(tx[0])


def truth_xyz(xyz_rows, s):
    """True receiver ECEF at samples s from the per-block positions xyz_rows[b] (block b moves to xyz_rows[b + 1])."""
    s = np.asarray(s, np.int64)
    b = s // BLOCK
    f = (s - b * BLOCK) / BLOCK
    a = xyz_rows[np.minimum(b, len(xyz_rows) - 1)]
    c = xyz_rows[np.minimum(b + 1, len(xyz_rows) - 1)]
    return a + f[:, None] * (c - a), (c - a) / 0.1


def truth_time(start_sow, s):
    return np.mod(start_sow + np.asarray(s, np.int64) / FS, 604800.0)
