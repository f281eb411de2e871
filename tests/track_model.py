"""Numpy statement of the tracking loops (include/gpsb200.h: gpsb200_track; DESIGN §10): the tests' reference.

It shares no code with the library: samples, carrier tables, phase-step rounding and C/A codes come from acq_model (its
own Gold-code generator, the reference's tables from the golden fixtures). The loop runs vectorised over channels and
sequentially over periods, in int64 arithmetic; C's truncating division is `tdiv` (numpy's // floors), C's arithmetic
right shift is numpy's >> (both floor)."""
import math

import numpy as np

import acq_model as A

M = 1023 << 32                       # code phase modulus, 2^-32 chips
H = 1 << 31                          # half a chip
CODE_STEP_NOM = 1464583848           # round(1.023e6 / 3e6 * 2^32)
CODE_STEP_MIN = 1464095816           # ceil(M / 3001)
CODE_STEP_MAX = 1465072205           # floor(M / 2999)
FLL_EPOCHS = 200
FREQ_CLAMP = 1 << 34
MAX_PERIOD = 3001
# round(atan(2^-i) / (2 pi) * 2^32), i = 0..23, as listed in the library (test_track checks it against the formula)
ATAN = [536870912, 316933406, 167458907, 85004756, 42667331, 21354465, 10679838, 5340245, 2670163, 1335087, 667544,
        333772, 166886, 83443, 41722, 20861, 10430, 5215, 2608, 1304, 652, 326, 163, 81]

STATE_DTYPE = np.dtype([("prn", "<i4"), ("epochs", "<i4"), ("sample", "<i8"), ("code_phase", "<u8"),
                        ("carr_freq", "<i8"), ("carr_phase", "<u4"), ("carr_step", "<i4"), ("code_step", "<u4"),
                        ("prev_i", "<i4"), ("prev_q", "<i4"), ("lock_i", "<i4"), ("lock_q", "<i4"), ("lock", "<i4")])
EPOCH_DTYPE = np.dtype([("sample", "<i8"), ("e_i", "<i4"), ("e_q", "<i4"), ("p_i", "<i4"), ("p_q", "<i4"),
                        ("l_i", "<i4"), ("l_q", "<i4"), ("carr_phase", "<u4"), ("carr_step", "<i4"),
                        ("code_phase", "<u4"), ("code_step", "<u4"), ("lock", "<i4"), ("reserved", "<i4")])


def atan_table():
    return [int(round(math.atan(2.0 ** -i) / (2 * math.pi) * 2 ** 32)) for i in range(24)]


def tdiv(a, b):
    """C's integer division (truncation toward zero) of int64 arrays."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    q = np.abs(a) // np.abs(b)
    return np.where((a < 0) != (b < 0), -q, q)


def excess_bits(v, keep):
    """max(0, bitlen(v) - keep) of non-negative int64 v."""
    v = np.asarray(v, np.int64)
    s = np.zeros(v.shape, np.int64)
    for k in range(64 - keep):
        s += (v >> (keep + k)) > 0
    return s


def angle(x, y):
    """Angle of (x, y), x >= 0, in 2^-32 turns: both shifted to 30 bits, 24 CORDIC vectoring steps; 0 for (0, 0)."""
    x, y = np.asarray(x, np.int64).copy(), np.asarray(y, np.int64).copy()
    zero = (x == 0) & (y == 0)
    s = excess_bits(np.maximum(x, np.abs(y)), 30)
    x, y = x >> s, y >> s
    z = np.zeros(x.shape, np.int64)
    for i, a in enumerate(ATAN):
        xs, ys = x >> i, y >> i
        pos = y > 0
        x, y, z = np.where(pos, x + ys, x - ys), np.where(pos, y - xs, y + xs), np.where(pos, z + a, z - a)
    return np.where(zero, 0, z)


def code_step_of(w, D=0):
    """The code step at carrier step w and DLL discriminator D (D = 0: a start state and the snapshot measurement)."""
    return np.clip(CODE_STEP_NOM + tdiv(w, 1540) + tdiv(2048 * np.asarray(D, np.int64), 3000), CODE_STEP_MIN,
                   CODE_STEP_MAX)


def dll(E, L):
    """DLL discriminator of early and late powers E, L >= 0: both shifted to 40 bits, then (E - L) 2^14 / (E + L)."""
    E, L = np.asarray(E, np.int64), np.asarray(L, np.int64)
    s = excess_bits(E + L, 40)
    E, L = E >> s, L >> s
    tot = E + L
    return np.where(tot == 0, 0, tdiv((E - L) * 16384, np.where(tot == 0, 1, tot)))


def start(prn, doppler_hz, sample):
    """The contract's start state of a channel from an acquisition."""
    st = np.zeros(1, STATE_DTYPE)[0]
    w = A.phase_step(doppler_hz)
    w = w - (1 << 32) if w >= 1 << 31 else w
    st["prn"], st["sample"], st["carr_step"], st["carr_freq"] = prn, sample, w, w * 1024
    st["code_step"] = int(code_step_of(np.int64(w)))
    return st


def loop_update(S, c):
    """One update of the loop state S (dict of int64 arrays) from the sums c[6] (int64 arrays)."""
    pi, pq = c[2], c[3]
    neg = pi < 0
    e = angle(np.where(neg, -pi, pi), np.where(neg, -pq, pq))
    F = S["carr_freq"].copy()
    fll = (S["epochs"] >= 1) & (S["epochs"] < FLL_EPOCHS)
    cross = S["prev_i"] * pq - S["prev_q"] * pi
    dot = S["prev_i"] * pi + S["prev_q"] * pq
    flip = dot < 0
    d = angle(np.where(flip, -dot, dot), np.where(flip, -cross, cross))
    F = F + np.where(fll, tdiv(64 * d, 3000), 0)
    F = np.clip(F + (e >> 12), -FREQ_CLAMP, FREQ_CLAMP)
    S["carr_freq"] = F
    w = (F >> 10) + (e >> 16)
    S["carr_step"] = w
    S["code_step"] = code_step_of(w, dll(c[0] * c[0] + c[1] * c[1], c[4] * c[4] + c[5] * c[5]))
    S["lock_i"] = S["lock_i"] + ((np.abs(pi) - S["lock_i"]) >> 4)
    S["lock_q"] = S["lock_q"] + ((np.abs(pq) - S["lock_q"]) >> 4)
    S["lock"] = (3 * S["lock_q"] < S["lock_i"]).astype(np.int64)
    S["prev_i"], S["prev_q"] = pi.copy(), pq.copy()
    S["epochs"] = S["epochs"] + 1


_CODES = {}


def code_pm(prn):
    """Chips of prn as +-1 (int64), padded with a 0 at index 1023."""
    if prn not in _CODES:
        _CODES[prn] = np.concatenate([2 * A.ca_code(prn).astype(np.int64) - 1, [0]])
    return _CODES[prn]


def track(iq, sample_size, base, states, max_epochs=None):
    """Run the contract over the buffer iq (interleaved I,Q; stream sample `base` first) from `states`
    (STATE_DTYPE[nchan]). -> (list of EPOCH_DTYPE arrays per channel, states after)."""
    I, Q = A.samples(iq, sample_size)
    N = I.size
    end = base + N
    cos, sin = A.tables()
    st = np.array(states, STATE_DTYPE).reshape(-1)
    nch = st.size
    S = {f: st[f].astype(np.int64) for f in STATE_DTYPE.names}
    codes = np.stack([code_pm(int(p)) for p in st["prn"]])
    me = N // 2999 + 1 if max_epochs is None else int(max_epochs)
    out = [[] for _ in range(nch)]
    active = np.ones(nch, bool)
    m = np.arange(MAX_PERIOD, dtype=np.int64)
    k = 0
    rows = np.arange(nch)[:, None]
    while True:
        L = (M - S["code_phase"] + S["code_step"] - 1) // S["code_step"]
        active &= (k < me) & (S["sample"] + L <= end)
        if not active.any():
            break
        a = np.nonzero(active)[0]
        Sa = {f: v[a] for f, v in S.items()}
        La = L[a]
        valid = m[None, :] < La[:, None]
        idx = np.minimum((Sa["sample"] - base)[:, None] + m[None, :], N - 1)
        Ii, Qi = I[idx], Q[idx]
        th = (Sa["carr_phase"][:, None] + m[None, :] * (Sa["carr_step"] & 0xFFFFFFFF)[:, None]) & 0xFFFFFFFF
        t = th >> 23
        cc, ss = cos[t], sin[t]
        dI = np.where(valid, Ii * cc + Qi * ss, 0)
        dQ = np.where(valid, Qi * cc - Ii * ss, 0)
        p = Sa["code_phase"][:, None] + m[None, :] * Sa["code_step"][:, None]
        e = p + H
        e = np.where(e >= M, e - M, e)
        l_ = np.where(p >= H, p - H, p + M - H)
        ca = codes[a]
        r = rows[:a.size]
        ce, cp, cl = (ca[r, np.minimum(x >> 32, 1023)] for x in (e, p, l_))
        c = [(ce * dI).sum(1), (ce * dQ).sum(1), (cp * dI).sum(1), (cp * dQ).sum(1), (cl * dI).sum(1), (cl * dQ).sum(1)]
        s_abs = Sa["sample"].copy()
        Sa["sample"] = Sa["sample"] + La
        Sa["carr_phase"] = (Sa["carr_phase"] + La * (Sa["carr_step"] & 0xFFFFFFFF)) & 0xFFFFFFFF
        Sa["code_phase"] = Sa["code_phase"] + La * Sa["code_step"] - M
        loop_update(Sa, c)
        for f, v in Sa.items():
            S[f][a] = v
        for j, ch in enumerate(a):
            out[ch].append((s_abs[j], c[0][j], c[1][j], c[2][j], c[3][j], c[4][j], c[5][j], Sa["carr_phase"][j],
                            Sa["carr_step"][j], Sa["code_phase"][j], Sa["code_step"][j], Sa["lock"][j], 0))
        k += 1
    res = np.zeros(nch, STATE_DTYPE)
    for f in STATE_DTYPE.names:
        res[f] = S[f]
    return [np.array(o, EPOCH_DTYPE) if o else np.zeros(0, EPOCH_DTYPE) for o in out], res


def record_at(rec, s):
    """Code phase (chips, unwrapped from the block start) and carrier Doppler of a channel record at sample s of its
    block."""
    return float(rec["code_phase"]) + float(rec["f_code"]) * s / 3e6, float(rec["f_carr"])
