"""Truth of a tracked channel from the scenario's channel records: code phase, Doppler, bit boundaries and the NAV words
a receiver should read, at any sample of a stream made from consecutive block records (CHAN_DTYPE rows)."""
import datetime

import numpy as np

BLOCK = 300000
FS = 3e6


def slot_of(ch, prn):
    """Slot of prn in every block (-1 where it is not held)."""
    hit = ch["prn"] == prn
    return np.where(hit.any(1), hit.argmax(1), -1)


def at(ch, prn, s):
    """(record, t, cp): the record of prn in the block holding sample s, t = s - block start, cp = its code phase at s in
    chips counted from the block start's code period (unwrapped: cp >= 1023 after the first code boundary)."""
    b = int(s) // BLOCK
    k = int(np.nonzero(ch[b]["prn"] == prn)[0][0])
    rec = ch[b][k]
    t = int(s) - b * BLOCK
    return rec, b, k, float(rec["code_phase"]) + float(rec["f_code"]) * t / FS


def code_error_chips(ch, prn, s, phi):
    """Signal code phase minus local prompt phase phi (2^-32 chips) at sample s, in chips, wrapped to [-511.5, 511.5)."""
    _, _, _, cp = at(ch, prn, s)
    d = (cp % 1023.0) - float(phi) / 2 ** 32
    return (d + 511.5) % 1023.0 - 511.5


def ms_index(ch, prn, s):
    """(block, slot, total ms since the record's NAV frame start, distance in chips from a code boundary) of a sample s
    that should sit at a code boundary."""
    rec, b, k, cp = at(ch, prn, s)
    j = int(round(cp / 1023.0))
    total = int(rec["iword"]) * 600 + int(rec["ibit"]) * 20 + int(rec["icode"]) + j
    return b, k, total, cp - 1023.0 * j


def gps_sow(y, mo, d, h, mi, sec):
    """GPS seconds of week of a calendar date (no leap seconds: the scenario's time is GPS time)."""
    t = datetime.datetime(y, mo, d, h, mi) - datetime.datetime(1980, 1, 6)
    return (t.total_seconds() + sec) % (7 * 86400)


def epoch_errors(ch, prn, ep, phi0=0):
    """Per epoch: (code error in chips at the period start, Doppler error in Hz of the updated carrier step against the
    record's f_carr)."""
    phis = np.concatenate([[phi0], ep["code_phase"][:-1].astype(np.int64)])
    cerr = np.array([code_error_chips(ch, prn, s, p) for s, p in zip(ep["sample"], phis)])
    ferr = np.array([float(e["carr_step"]) * FS / 2 ** 32 - float(at(ch, prn, e["sample"])[0]["f_carr"]) for e in ep])
    return cerr, ferr


def word_failures(ch, prn, words, frames, frame_of_block, bits=None):
    """The decoded words against the scenario's: each word's first sample at a word boundary (whole 600 ms from the
    record's frame start) and its 30 bits equal to the NAV word the scenario sent there. -> list of failure strings."""
    bad = []
    for w in words:
        b, k, total, dist = ms_index(ch, prn, int(w["sample"]))
        if total % 600 != 0:
            bad.append("word %d at sample %d: %d ms into the frame, not at a word boundary" % (w["index"], w["sample"], total))
            continue
        widx = total // 600
        want = int(frames[int(frame_of_block[b])][k][widx]) & 0x3FFFFFFF
        if int(w["raw"]) != want or not w["parity_ok"]:
            bad.append("word %d (frame %d word %d): got %08x want %08x parity %d" % (
                w["index"], frame_of_block[b], widx, w["raw"], want, w["parity_ok"]))
    return bad
