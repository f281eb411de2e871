"""Numpy statement of the snapshot measurement (include/gpsb200.h: gpsb200_snapshot_measure; DESIGN §11.5) and of the
fixes from snapshot records (gpsb200_pvt_snapshot / gpsb200_pvt_snapshot_search): the tests' reference.

It shares no code with the library: samples, carrier tables, phase-step rounding and C/A codes come from acq_model, the
CORDIC angle, truncating division, the code-step rule and the DLL discriminator from track_model. Everything runs in
int64 (Python ints where a product could leave it). The fixes restate only the measurement step; the solve is coarse_model's, run at each
snapshot's instant with its measurement step replaced by the one below."""
import numpy as np

import acq_model as A
import track_model as T

M, H = T.M, T.H
CHUNK = 3000
MAX_ITER = 16
GAIN = 1 << 15
MAX_LAST_D = 131               # |D| of the last iteration: D * 2^15 <= 2^32 / 1000, a thousandth of a chip
OK, WEAK, NO_CONVERGENCE = 0, 1, 2
SNAPSHOT_DTYPE = np.dtype([("prn", "<i4"), ("status", "<i4"), ("sample", "<i8"), ("code_phase", "<u8"),
                           ("code_step", "<u4"), ("carr_step", "<i4"), ("iterations", "<i4"), ("last_step", "<i4"),
                           ("power", "<u8"), ("ratio", "<f8")])
assert SNAPSHOT_DTYPE.itemsize == 56


def seed(res_row, s0):
    """Step 1: (w0, u0, phi0) of one acquisition result."""
    w = A.phase_step(float(res_row["doppler_hz"]))
    w = w - (1 << 32) if w >= 1 << 31 else w
    u = int(T.code_step_of(np.int64(w)))
    phi = (-int(res_row["delay"]) * u) % M
    return w, u, phi


def sums(I, Q, prn, K, phi, u, w, code=True):
    """Chunk sums over the K chunks of 3000 samples from the window start (I, Q: the window, int64) with the replica at
    phi + m u (mod M) and the wipe-off at m w. -> dict of int64 [K]: pi, pq and, with code, ei, eq, li, lq."""
    cos, sin = A.tables()
    n = CHUNK * K
    m = np.arange(n, dtype=np.int64)
    idx = ((m.astype(np.uint64) * np.uint64(w & 0xFFFFFFFF)) & np.uint64(0xFFFFFFFF)) >> np.uint64(23)
    c, s = cos[idx.astype(np.int64)], sin[idx.astype(np.int64)]
    i, q = I[:n], Q[:n]
    dI, dQ = i * c + q * s, q * c - i * s
    p = (np.int64(phi) + m * np.int64(u)) % M
    ca = T.code_pm(int(prn))
    out = {}
    reps = [("p", p)]
    if code:
        reps += [("e", (p + H) % M), ("l", (p + M - H) % M)]
    for name, x in reps:
        cc = ca[x >> 32]
        out[name + "i"] = (cc * dI).reshape(K, CHUNK).sum(1)
        out[name + "q"] = (cc * dQ).reshape(K, CHUNK).sum(1)
    return out


def freq_step(pi, pq):
    """Step 2: the carrier-step correction from the prompt sums of consecutive chunks (d / 3000, truncated)."""
    pi, pq = [int(v) for v in pi], [int(v) for v in pq]
    sc = sd = 0
    for k in range(len(pi) - 1):
        cross = pi[k] * pq[k + 1] - pq[k] * pi[k + 1]
        dot = pi[k] * pi[k + 1] + pq[k] * pq[k + 1]
        if dot < 0:
            cross, dot = -cross, -dot
        sc += cross
        sd += dot
    assert abs(sc) < 2 ** 63 and sd < 2 ** 63
    d = int(T.angle(np.int64(sd), np.int64(sc)))
    return int(T.tdiv(np.int64(d), 3000))


def dll(ei, eq, li, lq):
    """Step 3's discriminator D of one iteration."""
    E = sum(int(a) * int(a) + int(b) * int(b) for a, b in zip(ei, eq))
    L = sum(int(a) * int(a) + int(b) * int(b) for a, b in zip(li, lq))
    assert E + L < 2 ** 63
    return int(T.dll(E, L))


def power(pi, pq):
    return sum(int(a) * int(a) + int(b) * int(b) for a, b in zip(pi, pq))


def measure(iq, sample_size, s0, K, res, min_ratio=2.5, iterations=12, trace=None):
    """The snapshot records of the acquisition results `res` (ACQ_RESULT rows, in the search's PRN order) over the
    window of K chunks from s0 of the buffer iq (interleaved I,Q). trace: None or a list that receives each refined
    PRN's per-iteration D values. -> SNAPSHOT_DTYPE[nprn]."""
    I, Q = A.samples(iq, sample_size)
    I, Q = I[s0:s0 + CHUNK * K], Q[s0:s0 + CHUNK * K]
    assert I.size == CHUNK * K
    out = np.zeros(len(res), SNAPSHOT_DTYPE)
    for j, r in enumerate(res):
        w, u, phi = seed(r, s0)
        rec = out[j]
        rec["prn"], rec["sample"], rec["ratio"] = int(r["prn"]), s0, float(r["ratio"])
        rec["code_phase"], rec["code_step"], rec["carr_step"] = phi, u, w
        if not float(r["ratio"]) >= min_ratio:
            rec["status"] = WEAK
            continue
        prn = int(r["prn"])
        f = sums(I, Q, prn, K, phi, u, w, code=False)
        pw = power(f["pi"], f["pq"])
        if K >= 2:
            w = w + freq_step(f["pi"], f["pq"])
            u = int(T.code_step_of(np.int64(w)))
        D = 0
        ds = []
        for _ in range(iterations):
            c = sums(I, Q, prn, K, phi, u, w)
            D = dll(c["ei"], c["eq"], c["li"], c["lq"])
            pw = power(c["pi"], c["pq"])
            phi = (phi + D * GAIN) % M
            ds.append(D)
        if trace is not None:
            trace.append(ds)
        rec["code_phase"], rec["code_step"], rec["carr_step"] = phi, u, w
        rec["iterations"], rec["last_step"], rec["power"] = iterations, D, pw
        rec["status"] = NO_CONVERGENCE if abs(D) > MAX_LAST_D else OK
    return out


# ---- fixes from snapshot records -------------------------------------------------------------------------------------
def snapshot_meas(chans, meas, tas):
    """The measurement step of gpsb200_pvt_snapshot: meas [F, C] SNAPSHOT records, tas [F] a-priori times.
    -> dict of [F, C]: use, frac (ms), w."""
    meas = np.asarray(meas, SNAPSHOT_DTYPE)
    nf, nc = meas.shape
    use = np.zeros((nf, nc), bool)
    for c in range(nc):
        eph = chans[c]["eph"]
        if not eph["valid"] or eph["health"] != 0:
            continue
        use[:, c] = ((meas[:, c]["status"] == OK) & (meas[:, c]["prn"] == chans[c]["prn"])
                     & (np.abs(T_wrap(tas - eph["toe"])) <= 7200.0))
    frac = meas["code_phase"].astype(np.float64) / (1023.0 * 4294967296.0)
    return dict(use=use, frac=frac, w=meas["carr_step"].astype(np.int64))


def T_wrap(d):
    d = np.asarray(d, np.float64)
    return np.where(d > 302400.0, d - 604800.0, np.where(d < -302400.0, d + 604800.0, d))


def _per_snapshot(solve, chans, meas, cfg, conf):
    """Run solve (coarse_model.coarse or search_model.search) once per snapshot at its instant, with coarse_model's
    measurement step replaced by snapshot_meas on that snapshot's records; concatenate the results."""
    import coarse_model as CM
    meas = np.asarray(meas, SNAPSHOT_DTYPE)
    outs = []
    for i in range(meas.shape[0]):
        row = meas[i:i + 1]
        c1 = np.array(cfg).copy()
        c1["s0"], c1["step"], c1["nfix"] = int(row[0, 0]["sample"]), 1, 1
        saved = CM.measure
        CM.measure = lambda ch, ep, s, tas: {k: np.broadcast_to(v, (np.size(s), v.shape[1]))
                                             for k, v in snapshot_meas(ch, row, np.atleast_1d(tas)[:1]).items()}
        try:
            outs.append(solve(chans, [None] * meas.shape[1], c1, conf))
        finally:
            CM.measure = saved
    return tuple({k: np.concatenate([np.atleast_1d(o[j][k]) for o in outs]) for k in outs[0][j]}
                 if isinstance(outs[0][j], dict) else np.concatenate([o[j] for o in outs]) for j in range(len(outs[0])))


def coarse(chans, meas, cfg, ap):
    """gpsb200_pvt_snapshot on the model: coarse_model's solve at each snapshot's instant with the measurement above.
    meas [F, C]. -> coarse_model.coarse's tuple over the F snapshots."""
    import coarse_model as CM
    return _per_snapshot(CM.coarse, chans, meas, cfg, ap)


def search(chans, meas, cfg, sc):
    """gpsb200_pvt_snapshot_search on the model: search_model's search at each snapshot's instant with the measurement
    above. meas [F, C]. -> search_model.search's tuple over the F snapshots."""
    import search_model as SM
    return _per_snapshot(SM.search, chans, meas, cfg, sc)
