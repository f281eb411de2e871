"""Numpy statement of collective detection (include/gpsb200.h: gpsb200_collective; DESIGN §11.7): the tests' reference.

It shares no code with the library. The satellite and the WGS-84 conversion are pvt_model's; the prediction is
coarse_model's step 3 restated with the range rate and clock drift of its last step. The search's grid comes from
acq_model (or, on the GPU, from the device's own search). Every integer stage (normalisation, scores, pick, seeds) is
exact, so given the same table of (bin, delay) cells the model's scores, record and seeds equal the device's bit for
bit, but for the winner's latitude, longitude and height (numpy's transcendentals differ from CUDA's by ulps); the table
itself agrees except where a continuous delay or bin lies within ulps of a rounding boundary."""
import numpy as np

import acq_model as A
import pvt_model as PM
from pvt_model import C, OMEGA_E, satellite, wrap_half_week

OK, FEW, AMBIGUOUS = 0, 1, 2
MIN_USED, Q_SHIFT, Q_CAP, AMBIGUOUS_PCT = 4, 8, 8192, 90
LAMBDA = 0.190293672798365
CODE = A.CODE

RECORD_DTYPE = np.dtype([("status", "<i4"), ("nused", "<i4"), ("used", "<u4"), ("shift", "<i4"), ("winner", "<i4"),
                         ("runner", "<i4"), ("score", "<u4"), ("runner_score", "<u4"), ("o_t", "<f8"),
                         ("x", "<f8", 3), ("lat_deg", "<f8"), ("lon_deg", "<f8"), ("height", "<f8"),
                         ("runner_dist", "<f8")])


def frame(x_a):
    """(E, N, U) unit vectors at x_a's WGS-84 latitude / longitude."""
    lat, lon, _ = PM.ecef_llh(np.asarray(x_a, np.float64))
    sla, cla, slo, clo = np.sin(lat), np.cos(lat), np.sin(lon), np.cos(lon)
    return np.array([-slo, clo, 0.0]), np.array([-sla * clo, -sla * slo, cla]), np.array([cla * clo, cla * slo, sla])


def predict(eph, x, t, up):
    """Step 3 of gpsb200_pvt_coarse with the last step's range rate and drift: eph [..] broadcast with x [.., 3] and
    t [..]. -> (pred ms, sin(elevation), range rate m/s, drift s/s)."""
    tau = np.full(np.broadcast_shapes(np.shape(eph), np.shape(t)), 0.075)
    for _ in range(3):
        p, v, dt, ddt = satellite(eph, t - tau)
        sth, cth = np.sin(OMEGA_E * tau), np.cos(OMEGA_E * tau)
        l = np.stack([p[..., 0] * cth + p[..., 1] * sth - x[..., 0], p[..., 1] * cth - p[..., 0] * sth - x[..., 1],
                      p[..., 2] - x[..., 2]], -1)
        vr = np.stack([v[..., 0] * cth + v[..., 1] * sth, v[..., 1] * cth - v[..., 0] * sth, v[..., 2]], -1)
        tau = np.sqrt(l[..., 0] * l[..., 0] + l[..., 1] * l[..., 1] + l[..., 2] * l[..., 2]) / C
    sel = (up[..., 0] * l[..., 0] + up[..., 1] * l[..., 1] + up[..., 2] * l[..., 2]) / (tau * C)
    rate = (l[..., 0] * vr[..., 0] + l[..., 1] * vr[..., 1] + l[..., 2] * vr[..., 2]) / (tau * C)
    return 1000.0 * (t - tau + dt), sel, rate, ddt


def t0_of(ap, s0):
    return float(ap["t_a"]) + float(int(s0) - int(ap["s_a"])) / 3e6


def normalise(P):
    """Step 3: P [nprn][nbins][3000] uint64 -> (mu [nprn] Python ints, q uint16 of P's shape)."""
    nprn, nbins, _ = P.shape
    mu = []
    q = np.zeros(P.shape, np.uint16)
    for p in range(nprn):
        x = P[p].reshape(-1)
        s = int((x & np.uint64(0xffffffff)).sum(dtype=np.uint64)) + (int((x >> np.uint64(32)).sum(dtype=np.uint64)) << 32)
        m = s // (nbins * CODE)
        mu.append(m)
        if m == 0:
            continue
        a = x // np.uint64(m)
        r = x - a * np.uint64(m)
        v = a.astype(np.uint64)
        for _ in range(Q_SHIFT):
            r = r << np.uint64(1)
            v = v << np.uint64(1)
            ge = r >= np.uint64(m)
            r = np.where(ge, r - np.uint64(m), r)
            v = v | ge.astype(np.uint64)
        v = np.where(a >= np.uint64(1 << (16 - Q_SHIFT)), np.uint64(Q_CAP), np.minimum(v, np.uint64(Q_CAP)))
        q[p] = v.reshape(nbins, CODE).astype(np.uint16)
    return mu, q


def used(eph, prns, ap, s0, mask_deg, mu):
    """Step 2 -> bool [nprn]."""
    t0 = t0_of(ap, s0)
    _, _, U = frame(ap["x_a"])
    out = np.zeros(len(prns), bool)
    for p, prn in enumerate(prns):
        e = eph[prn - 1]
        if not (e["valid"] and e["health"] == 0 and abs(wrap_half_week(t0 - e["toe"])) <= 7200.0 and mu[p] > 0):
            continue
        _, sel, _, _ = predict(e, np.asarray(ap["x_a"], np.float64), t0, U)
        out[p] = sel >= np.sin(float(mask_deg) * PM.PI / 180.0)
    return out


def offsets(cfg, h):
    """Step 4: the offsets [len(h), 4] (east, north, up m; time s) of hypotheses h."""
    h = np.asarray(h, np.int64).copy()
    o = np.zeros((h.size, 4))
    for a in range(4):
        n = int(cfg["n"][a])
        i = h % n
        h //= n
        if n > 1:
            o[:, a] = (i.astype(np.float64) - float(n - 1) * 0.5) * float(cfg["step"][a])
    return o


def positions(ap, cfg, h):
    E, N, U = frame(ap["x_a"])
    o = offsets(cfg, h)
    xa = np.asarray(ap["x_a"], np.float64)
    x = np.stack([xa[i] + o[:, 0] * E[i] + o[:, 1] * N[i] + o[:, 2] * U[i] for i in range(3)], -1)
    return x, o


def table(eph, prns, use, ap, s0, cfg, f_lo_p, step_hz, nbins, h=None):
    """Step 5 -> (cells int32 [H, nprn, 2] (bin, delay) as the device's table, the continuous delay and bin [H, nprn]
    before rounding, NaN where unused). h: the hypotheses (default all)."""
    nhyp = int(np.prod(cfg["n"].astype(np.int64)))
    h = np.arange(nhyp) if h is None else np.asarray(h, np.int64)
    x, o = positions(ap, cfg, h)
    _, _, U = frame(ap["x_a"])
    t = t0_of(ap, s0) + o[:, 3]
    cells = np.full((h.size, len(prns), 2), -1, np.int32)
    dc, jc = np.full((h.size, len(prns)), np.nan), np.full((h.size, len(prns)), np.nan)
    for p, prn in enumerate(prns):
        if not use[p]:
            continue
        pred, _, rate, drift = predict(eph[prn - 1], x, t, U)
        dv = 3000.0 * (1.0 - (pred - np.floor(pred)))
        d = np.floor(dv + 0.5).astype(np.int64) % CODE
        f = -(rate - C * drift) / LAMBDA
        jv = (f - f_lo_p[p]) / step_hz if nbins > 1 else np.zeros(h.size)
        j = np.floor(jv + 0.5) if nbins > 1 else np.zeros(h.size)
        cells[:, p, 0] = np.where((j >= 0) & (j < nbins), j, -1)
        cells[:, p, 1] = d
        dc[:, p], jc[:, p] = dv, jv
    return cells, dc, jc


def score(q, cells):
    """Step 6 -> (S [H] uint32, b [H] int32)."""
    H, nprn, _ = cells.shape
    b = np.arange(CODE)
    S = np.zeros((H, CODE), np.uint32)
    for p in range(nprn):
        j, d = cells[:, p, 0], cells[:, p, 1]
        on = j >= 0
        if not on.any():
            continue
        rows = q[p][j[on]]                                   # [h, 3000]
        idx = (d[on][:, None] + b[None, :]) % CODE
        S[on] += np.take_along_axis(rows, idx, 1).astype(np.uint32)
    best = np.argmax(S, 1)                                   # the first (lowest) shift among equal maxima
    return S[np.arange(H), best], best.astype(np.int32)


def pick(S, b, cfg, ap, use):
    """Step 7 and the record (a RECORD_DTYPE row)."""
    r = np.zeros(1, RECORD_DTYPE)[0]
    r["nused"] = int(use.sum())
    r["used"] = int((use.astype(np.int64) << np.arange(use.size)).sum())
    r["shift"] = r["winner"] = r["runner"] = -1
    for f in ("o_t", "lat_deg", "lon_deg", "height", "runner_dist"):
        r[f] = np.nan
    r["x"] = np.nan
    if use.sum() < MIN_USED:
        r["status"] = FEW
        return r
    w = int(np.argmax(S))
    o = offsets(cfg, np.arange(S.size))
    dist = np.sqrt((o[:, 0] - o[w, 0]) ** 2 + (o[:, 1] - o[w, 1]) ** 2 + (o[:, 2] - o[w, 2]) ** 2)
    far = dist > float(cfg["distinct_m"])
    x, ow = positions(ap, cfg, [w])
    lat, lon, hgt = PM.ecef_llh(x[0])
    r["status"], r["winner"], r["score"], r["shift"], r["o_t"] = OK, w, S[w], b[w], ow[0, 3]
    r["x"], r["lat_deg"], r["lon_deg"], r["height"] = x[0], lat * (180.0 / np.pi), lon * (180.0 / np.pi), hgt
    if far.any():
        cand = np.where(far, S.astype(np.int64), -1)
        k = int(np.argmax(cand))
        r["runner"], r["runner_score"], r["runner_dist"] = k, S[k], dist[k]
        if 100 * int(S[k]) >= AMBIGUOUS_PCT * int(S[w]):
            r["status"] = AMBIGUOUS
    return r


def seeds(res, P, rec, cells_w, f_lo_p, step_hz):
    """Step 8: res [nprn] and the winner's cells [nprn, 2] -> seeds [nprn]."""
    out = np.array(res, copy=True)
    for p in range(len(out)):
        j = int(cells_w[p, 0]) if rec["winner"] >= 0 else -1
        if j < 0:
            out[p]["ratio"] = -1.0
            continue
        d = (int(cells_w[p, 1]) + int(rec["shift"])) % CODE
        row = P[p, j]
        dd = np.abs(np.arange(CODE) - d)
        dd = np.minimum(dd, CODE - dd)
        p1, p2 = int(row[d]), int(row[dd > A.EXCLUDE].max())
        out[p]["bin"], out[p]["delay"] = j, d
        out[p]["doppler_hz"] = f_lo_p[p] + j * step_hz
        out[p]["delay_chips"] = d * 1023.0 / 3000.0
        out[p]["p1"], out[p]["p2"] = p1, p2
        out[p]["ratio"] = float(p1) / float(p2) if p2 else np.inf
    return out


def collective(P, res, eph, prns, ap, s0, cfg, f_lo_p, step_hz, cells=None):
    """Steps 2-8 on a search's grid P and results res. f_lo_p: each PRN's first bin. cells: the table to score (default
    the model's own). -> (record, seeds, S [H], b [H], cells [H, nprn, 2])."""
    nbins = P.shape[1]
    mu, q = normalise(P)
    use = used(eph, prns, ap, s0, cfg["mask_deg"], mu)
    nhyp = int(np.prod(cfg["n"].astype(np.int64)))
    if use.sum() < MIN_USED:
        rec = pick(None, None, cfg, ap, use)
        return rec, seeds(res, P, rec, None, f_lo_p, step_hz), np.zeros(nhyp, np.uint32), np.zeros(nhyp, np.int32), \
            np.full((nhyp, len(prns), 2), -1, np.int32)
    if cells is None:
        cells, _, _ = table(eph, prns, use, ap, s0, cfg, f_lo_p, step_hz, nbins)
    S, b = score(q, cells)
    rec = pick(S, b, cfg, ap, use)
    return rec, seeds(res, P, rec, cells[int(rec["winner"])], f_lo_p, step_hz), S, b, cells
