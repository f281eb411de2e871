"""Numpy statement of the acquisition search (include/gpsb200.h: gpsb200_acquire; DESIGN §9): the tests' reference.

It shares no code with the library: the C/A codes come from its own Gold-code generator, the carrier tables from the
reference's tables as dumped into the golden fixtures. The correlation is computed by float64 FFT and rounded to
integers, which is exact here (|C| < 2^28, length 6000, rounding error far below 0.5); `method="direct"` computes it
by the defining sum, to check the FFT path on small grids.
"""
import os

import numpy as np

CODE = 3000                      # samples per C/A period at 3 Msps
EXCLUDE = 3                      # P2 ignores delays within +-3 samples of the peak
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

RESULT_DTYPE = np.dtype([("prn", "<i4"), ("bin", "<i4"), ("delay", "<i4"), ("reserved", "<i4"),
                         ("doppler_hz", "<f8"), ("delay_chips", "<f8"), ("p1", "<u8"), ("p2", "<u8"), ("ratio", "<f8")])

_G2_DELAY = [5, 6, 7, 8, 17, 18, 139, 140, 141, 251, 252, 254, 255, 256, 257, 258,
             469, 470, 471, 472, 473, 474, 509, 512, 513, 514, 515, 516, 859, 860, 861, 862]   # IS-GPS-200 Table 3-Ia


def ca_code(prn):
    """0/1 chips of PRN prn: G1 = 1 + x^3 + x^10, G2 = 1 + x^2 + x^3 + x^6 + x^8 + x^9 + x^10, G2 delayed."""
    g1, g2 = [1] * 10, [1] * 10
    o1, o2 = np.zeros(1023, np.uint8), np.zeros(1023, np.uint8)
    for i in range(1023):
        o1[i], o2[i] = g1[9], g2[9]
        f1 = g1[2] ^ g1[9]
        f2 = g2[1] ^ g2[2] ^ g2[5] ^ g2[7] ^ g2[8] ^ g2[9]
        g1 = [f1] + g1[:9]
        g2 = [f2] + g2[:9]
    d = _G2_DELAY[prn - 1]
    return o1 ^ np.roll(o2, d)


def replica(prn):
    """c_p[n] = 2 ca_p[(n * 1023) / 3000] - 1, n < 3000 (int64)."""
    n = np.arange(CODE, dtype=np.int64)
    return 2 * ca_code(prn)[(n * 1023) // CODE].astype(np.int64) - 1


def tables():
    """(cos512, sin512) of the reference, int64."""
    g = np.load(os.path.join(GOLD, "sky12_static_10s_i8.npz"))
    return g["cos512"].astype(np.int64), g["sin512"].astype(np.int64)


def phase_step(f_hz):
    """(uint32) llround(f * 2^32 / 3e6): rounding half away from zero, then modulo 2^32."""
    v = float(f_hz) * 4294967296.0 / 3e6
    r = int(np.floor(abs(v) + 0.5))
    return (r if v >= 0 else -r) % (1 << 32)


def samples(iq, sample_size):
    """Interleaved I,Q -> (I, Q) int64 at the int8 scale: int16 reduced to clamp(x >> 4, -128, 127)."""
    x = np.asarray(iq)
    if sample_size == 2:
        x = np.clip(x.astype(np.int64) >> 4, -128, 127)
    x = x.astype(np.int64)
    return x[0::2], x[1::2]


def wipe(I, Q, u, m0=0):
    """Carrier wipe-off of samples m0, m0 + 1, ... at phase step u -> (I_d, Q_d) int64."""
    cos, sin = tables()
    m = np.arange(m0, m0 + I.size, dtype=np.uint64)
    idx = ((m * np.uint64(u)) & np.uint64(0xFFFFFFFF)) >> np.uint64(23)
    c, s = cos[idx.astype(np.int64)], sin[idx.astype(np.int64)]
    return I * c + Q * s, Q * c - I * s


def correlate(Id, Qd, c, method="fft"):
    """C_I, C_Q (int64 [3000]) of one period: sum_n c[n] x[tau + n], x = the 5999 samples of the period."""
    assert Id.size == 2 * CODE - 1
    if method == "direct":
        w = np.lib.stride_tricks.sliding_window_view
        return w(Id, CODE)[:CODE] @ c, w(Qd, CODE)[:CODE] @ c
    n = 2 * CODE
    x = np.fft.fft(Id.astype(np.float64) + 1j * Qd.astype(np.float64), n)
    y = np.fft.ifft(x * np.conj(np.fft.fft(c.astype(np.float64), n)))[:CODE]
    return np.rint(y.real).astype(np.int64), np.rint(y.imag).astype(np.int64)


def grid(iq, sample_size, s0, K, prns, f_lo, step, nbins, method="fft"):
    """P[nprn][nbins][3000] uint64 of the search. iq: the whole buffer (interleaved); the window must lie inside it."""
    I, Q = samples(iq, sample_size)
    W = CODE * K + CODE - 1
    if not (1 <= K <= 100 and 0 <= s0 and s0 + W <= I.size):
        raise ValueError("window outside the buffer or K outside 1..100")
    I, Q = I[s0:s0 + W], Q[s0:s0 + W]
    reps = [replica(p) for p in prns]
    out = np.zeros((len(prns), nbins, CODE), np.uint64)
    for j in range(nbins):
        Id, Qd = wipe(I, Q, phase_step(f_lo + j * step))
        for k in range(K):
            a, b = Id[CODE * k:CODE * (k + 2) - 1], Qd[CODE * k:CODE * (k + 2) - 1]
            if method == "fft":
                n = 2 * CODE
                x = np.fft.fft(a.astype(np.float64) + 1j * b.astype(np.float64), n)
                C = np.fft.ifft(x[None, :] * np.conj(np.fft.fft(np.array(reps, np.float64), n, axis=1)), axis=1)[:, :CODE]
                cI, cQ = np.rint(C.real).astype(np.int64), np.rint(C.imag).astype(np.int64)
            else:
                pairs = [correlate(a, b, c, "direct") for c in reps]
                cI, cQ = np.array([p[0] for p in pairs]), np.array([p[1] for p in pairs])
            out[:, j, :] += (cI * cI + cQ * cQ).astype(np.uint64)
    return out


def reduce(P, prns, f_lo, step):
    """Per PRN: argmax (lowest j, then lowest tau on ties), P1, P2 outside +-3 samples (circular) in the peak's row."""
    res = np.zeros(len(prns), RESULT_DTYPE)
    tau = np.arange(CODE)
    for i, prn in enumerate(prns):
        j1, t1 = divmod(int(np.argmax(P[i].reshape(-1))), CODE)
        d = np.abs(tau - t1)
        d = np.minimum(d, CODE - d)
        row = P[i, j1]
        p2 = int(row[d > EXCLUDE].max())
        p1 = int(row[t1])
        res[i] = (prn, j1, t1, 0, f_lo + j1 * step, t1 * 1023.0 / 3000.0, p1, p2,
                  float(p1) / float(p2) if p2 else np.inf)
    return res


def search(iq, sample_size, s0, K, prns, f_lo=-5000.0, step=250.0, nbins=41, method="fft", want_grid=False):
    P = grid(iq, sample_size, s0, K, prns, f_lo, step, nbins, method)
    res = reduce(P, prns, f_lo, step)
    return (res, P) if want_grid else res


def truth(rec, s0=0):
    """Doppler and code-delay truth of one channel record at sample s0 of its block: (f_carr, tau_true in samples)
    where the signal's chip 0 starts, modulo the code period."""
    cp0 = (float(rec["code_phase"]) + float(rec["f_code"]) * s0 / 3e6) % 1023.0
    period = 1023.0 * 3e6 / float(rec["f_code"])
    return float(rec["f_carr"]), (((1023.0 - cp0) % 1023.0) * 3e6 / float(rec["f_code"])) % period


def circ_dist(a, b):
    d = abs(int(a) - int(b)) % CODE
    return min(d, CODE - d)


def truth_failures(res, recs, f_lo, step, r_present, r_absent, s0=0, edge=None):
    """The truth checks of one search over block records `recs` (CHAN rows of the searched block): every allocated PRN
    within step/2 of its f_carr (within step when f_carr lies within `edge` Hz of a bin edge, default step/10), within
    one sample of its code delay, with P1/P2 >= r_present; every other searched PRN below r_absent.
    -> list of failure strings (empty: all hold)."""
    edge = step / 10 if edge is None else edge
    bad = []
    held = {int(r["prn"]): r for r in recs if int(r["prn"]) > 0}
    for r in res:
        prn = int(r["prn"])
        if prn in held:
            f, t = truth(held[prn], s0)
            x = (f - f_lo) / step
            tol = step if abs((x - np.floor(x)) - 0.5) * step <= edge else step / 2
            if abs(r["doppler_hz"] - f) > tol:
                bad.append("PRN %d: Doppler %.1f vs f_carr %.1f" % (prn, r["doppler_hz"], f))
            if circ_dist(r["delay"], int(np.rint(t)) % CODE) > 1:
                bad.append("PRN %d: delay %d vs %.2f" % (prn, r["delay"], t))
            if not r["ratio"] >= r_present:
                bad.append("PRN %d present: P1/P2 %.3f < %.2f" % (prn, r["ratio"], r_present))
        elif not r["ratio"] < r_absent:
            bad.append("PRN %d absent: P1/P2 %.3f >= %.2f" % (prn, r["ratio"], r_absent))
    return bad
