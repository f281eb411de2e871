"""Numpy statement of the position fix (include/gpsb200.h: gpsb200_pvt; DESIGN §11): the tests' reference.

It shares no code with the library. The measurement is formed in Python integers / int64 exactly as the contract states;
the satellite, the Earth rotation, the Klobuchar delay and the Gauss-Newton / least-squares solutions in float64,
vectorised over fix instants and channels. Sums run in another order than the kernel's warp butterfly and numpy's
transcendental functions differ from CUDA's by ulps, so fixes agree to well under a micrometre, not bit for bit."""
import numpy as np

C = 2.99792458e8
C_MS = 2.99792458e5
GM = 3.986005e14
OMEGA_E = 7.2921151467e-5
PI = 3.1415926535898
WGS_A = 6378137.0
WGS_E = 0.0818191908426
LAMBDA_L1 = 0.190293672798365
REL_F = -4.442807633e-10
CODE_MOD = 1023.0 * 2.0 ** 32
STEP_HZ = 3e6 / 2.0 ** 32
WEEK_MS = 604800000
MAX_ITER = 12
IONO_MIN_RADIUS = 6e6
CONVERGED = 1e-4
RUNAWAY = 1e8
FIX_OK, FIX_FEW, FIX_NO_CONVERGENCE = 0, 1, 2


def wrap_half_week(d):
    d = np.asarray(d, np.float64)
    return np.where(d > 302400.0, d - 604800.0, np.where(d < -302400.0, d + 604800.0, d))


def measure(chans, epochs, s):
    """The integer part of the contract for fix instants s (int64[F]) and channels chans (PVT_CHAN fields) with epochs
    (list of arrays). -> dict of [F, C] arrays: use (bool), k, phi (uint64), T (int64 ms of week), w (carrier step)."""
    s = np.asarray(s, np.int64)
    nf, nc = s.size, len(epochs)
    out = {f: np.zeros((nf, nc), dt) for f, dt in (("use", bool), ("k", np.int64), ("phi", np.uint64), ("T", np.int64),
                                                    ("w", np.int64), ("tsv", np.float64), ("frac", np.float64))}
    for c, e in enumerate(epochs):
        eph = chans[c]["eph"]
        n = len(e)
        if n < 3 or not eph["valid"] or eph["health"] != 0:
            continue
        smp = e["sample"].astype(np.int64)
        k = np.searchsorted(smp, s, side="right") - 1
        ok = (k >= 1) & (k <= n - 2)
        kk = np.clip(k, 1, max(1, n - 2))
        ok &= (e["lock"][kk - 1] != 0) & (e["lock"][kk] != 0)
        phi = e["code_phase"][kk - 1].astype(np.uint64) + (s - smp[kk]).astype(np.uint64) * e["code_step"][kk - 1].astype(np.uint64)
        T = np.mod(int(chans[c]["anchor_ms"]) + kk - int(chans[c]["anchor_epoch"]), WEEK_MS)
        frac = phi.astype(np.float64) / CODE_MOD
        tsv = T.astype(np.float64) * 1e-3 + frac * 1e-3
        ok &= np.abs(wrap_half_week(tsv - eph["toe"])) <= 7200.0
        for f, v in (("use", ok), ("k", kk), ("phi", phi), ("T", T), ("w", e["carr_step"][kk - 1]), ("tsv", tsv),
                     ("frac", frac)):
            out[f][:, c] = v
    return out


def satellite(eph, t):
    """Position, velocity (ECEF, [.., 3]), clock offset and drift of ephemeris records eph (broadcast with t) at GPS time t."""
    g = lambda f: np.asarray(eph[f], np.float64)
    tk = wrap_half_week(t - g("toe"))
    A = g("sqrta") ** 2
    n = np.sqrt(GM / (A * A * A)) + g("deltan")
    M = g("m0") + n * tk
    e = g("ecc")
    E = M.copy()
    done = np.zeros(E.shape, bool)
    for _ in range(10):
        dE = (M - E + e * np.sin(E)) / (1.0 - e * np.cos(E))
        E = np.where(done, E, E + dE)
        done |= np.abs(dE) <= 1e-14
        if done.all():
            break
    sE, cE = np.sin(E), np.cos(E)
    om = 1.0 - e * cE
    Edot = n / om
    sq = np.sqrt(1.0 - e * e)
    pk = np.arctan2(sq * sE, cE - e) + g("aop")
    pkdot = sq * Edot / om
    s2, c2 = np.sin(2.0 * pk), np.cos(2.0 * pk)
    uk = pk + g("cus") * s2 + g("cuc") * c2
    ukdot = pkdot * (1.0 + 2.0 * (g("cus") * c2 - g("cuc") * s2))
    rk = A * om + g("crc") * c2 + g("crs") * s2
    rkdot = A * e * sE * Edot + 2.0 * pkdot * (g("crs") * c2 - g("crc") * s2)
    ik = g("inc0") + g("idot") * tk + g("cic") * c2 + g("cis") * s2
    ikdot = g("idot") + 2.0 * pkdot * (g("cis") * c2 - g("cic") * s2)
    xp, yp = rk * np.cos(uk), rk * np.sin(uk)
    xpdot = rkdot * np.cos(uk) - yp * ukdot
    ypdot = rkdot * np.sin(uk) + xp * ukdot
    odot = g("omgdot") - OMEGA_E
    ok = g("omg0") + tk * odot - OMEGA_E * g("toe")
    so, co, si, ci = np.sin(ok), np.cos(ok), np.sin(ik), np.cos(ik)
    p = np.stack([xp * co - yp * ci * so, xp * so + yp * ci * co, yp * si], -1)
    tmp = ypdot * ci - yp * si * ikdot
    v = np.stack([-odot * p[..., 1] + xpdot * co - tmp * so, odot * p[..., 0] + xpdot * so + tmp * co,
                  yp * ci * ikdot + ypdot * si], -1)
    d = wrap_half_week(t - g("toc"))
    dt = g("af0") + d * (g("af1") + d * g("af2")) + REL_F * e * g("sqrta") * sE - g("tgd")
    return p, v, dt, g("af1") + 2.0 * d * g("af2")


def ecef_llh(x):
    """WGS-84 latitude, longitude (rad), height of ECEF points x[.., 3]: the contract's six fixed-point steps."""
    e2 = WGS_E * WGS_E
    p = np.hypot(x[..., 0], x[..., 1])
    lon = np.arctan2(x[..., 1], x[..., 0])
    lat = np.arctan2(x[..., 2], p * (1.0 - e2))
    for _ in range(6):
        sl = np.sin(lat)
        N = WGS_A / np.sqrt(1.0 - e2 * sl * sl)
        lat = np.arctan2(x[..., 2] + e2 * N * sl, p)
    sl, cl = np.sin(lat), np.cos(lat)
    return lat, lon, p * cl + x[..., 2] * sl - WGS_A * np.sqrt(1.0 - e2 * sl * sl)


def llh_ecef(lat_deg, lon_deg, h):
    """ECEF of a WGS-84 point (the -l location of a static scenario)."""
    lat, lon = np.radians(lat_deg), np.radians(lon_deg)
    N = WGS_A / np.sqrt(1.0 - WGS_E ** 2 * np.sin(lat) ** 2)
    return np.array([(N + h) * np.cos(lat) * np.cos(lon), (N + h) * np.cos(lat) * np.sin(lon),
                     (N * (1.0 - WGS_E ** 2) + h) * np.sin(lat)])


def klobuchar(alpha, beta, lat, lon, az, el, t, trace=None):
    """IS-GPS-200 20.3.3.5.2.5 as the reference evaluates it (gps.c:1893-1964), in metres. trace: see pvt()."""
    E, phi_u, lam_u = el / PI, lat / PI, lon / PI
    F = 1.0 + 16.0 * (0.53 - E) ** 3
    psi = 0.0137 / (E + 0.11) - 0.022
    phi_i = np.clip(phi_u + psi * np.cos(az), -0.416, 0.416)
    lam_i = lam_u + psi * np.sin(az) / np.cos(phi_i * PI)
    phi_m = phi_i + 0.064 * np.cos((lam_i - 1.617) * PI)
    amp = np.maximum(alpha[0] + alpha[1] * phi_m + alpha[2] * phi_m ** 2 + alpha[3] * phi_m ** 3, 0.0)
    per = np.maximum(beta[0] + beta[1] * phi_m + beta[2] * phi_m ** 2 + beta[3] * phi_m ** 3, 72000.0)
    tl = np.mod(43200.0 * lam_i + t, 86400.0)
    X = 2.0 * PI * (tl - 50400.0) / per
    if trace is not None:
        trace["klobuchar_x"].append(np.ravel(X))
    return np.where(np.abs(X) < 1.57, F * (5.0e-9 + amp * (1.0 - X * X / 2.0 + X ** 4 / 24.0)) * C, F * 5.0e-9 * C)


def pvt(chans, epochs, cfg, trace=None):
    """The fixes of the contract. chans: PVT_CHAN records; epochs: list of TRACK_EPOCH arrays; cfg: PVT_CONFIG record.
    trace: None, or a dict whose lists "radius", "runaway", "step" and "klobuchar_x" receive, per iteration, the values
    the model compares with IONO_MIN_RADIUS, RUNAWAY, CONVERGED and the Klobuchar |X| < 1.57 branch (so that a caller can
    check that no decision sits on its threshold).
    -> (fix dict of arrays [F] with the FIX_DTYPE field names, residuals [F, C], measurement dict of measure())."""
    nf, nc = int(cfg["nfix"]), len(epochs)
    s = int(cfg["s0"]) + np.arange(nf, dtype=np.int64) * int(cfg["step"])
    ms = measure(chans, epochs, s)
    use = ms["use"]
    ref = next((c for c in range(nc) if chans[c]["eph"]["valid"] and chans[c]["eph"]["health"] == 0), -1)
    if ref < 0:
        use[:] = False
        ref_sample = ref_ms = 0
    else:
        ref_sample = int(epochs[ref]["sample"][int(chans[ref]["anchor_epoch"])])
        ref_ms = int(chans[ref]["anchor_ms"])
    q = np.floor_divide(s - ref_sample, 3000)
    m = (s - ref_sample) - 3000 * q
    nom_ms = np.mod(ref_ms + 75 + q, WEEK_MS)
    D = np.mod(ref_ms + 75 + q[:, None] - ms["T"], WEEK_MS)
    D = np.where(D >= WEEK_MS // 2, D - WEEK_MS, D)
    rho = D.astype(np.float64) * C_MS + (m[:, None] / 3000.0 - ms["frac"]) * C_MS
    rate = -LAMBDA_L1 * (ms["w"].astype(np.float64) * STEP_HZ)
    eph = np.stack([chans[c]["eph"] for c in range(nc)])[None, :]
    d0 = wrap_half_week(ms["tsv"] - eph["toc"])
    tt = ms["tsv"] - (eph["af0"] + d0 * (eph["af1"] + d0 * eph["af2"]))
    P, V, dtsv, ddtsv = satellite(eph, tt)
    nused = use.sum(1)
    mask = (use * (1 << np.arange(nc, dtype=np.int64))).sum(1)
    X = np.zeros((nf, 4))
    status = np.where(nused < 4, FIX_FEW, FIX_NO_CONVERGENCE)
    iters = np.zeros(nf, np.int32)
    active = nused >= 4
    res = np.full((nf, nc), np.nan)
    H = np.zeros((nf, nc, 4))
    r = np.zeros((nf, nc))
    Vr = np.zeros((nf, nc, 3))
    dX = np.zeros((nf, 4))
    Nmat = np.zeros((nf, 4, 4))
    w = use.astype(np.float64)
    for j in range(MAX_ITER):
        a = np.nonzero(active)[0]
        if a.size == 0:
            break
        x = X[a]
        g = P[a] - x[:, None, :3]
        tau = np.linalg.norm(g, axis=-1) / C
        sth, cth = np.sin(OMEGA_E * tau), np.cos(OMEGA_E * tau)
        pa, va = P[a], V[a]
        pr = np.stack([pa[..., 0] * cth + pa[..., 1] * sth, pa[..., 1] * cth - pa[..., 0] * sth, pa[..., 2]], -1)
        Vr[a] = np.stack([va[..., 0] * cth + va[..., 1] * sth, va[..., 1] * cth - va[..., 0] * sth, va[..., 2]], -1)
        los = pr - x[:, None, :3]
        R = np.linalg.norm(los, axis=-1)
        I = np.zeros(R.shape)
        rad = np.linalg.norm(x[:, :3], axis=-1)
        iono = bool(cfg["iono"]) & (rad >= IONO_MIN_RADIUS)
        if iono.any():
            lat, lon, _ = ecef_llh(x[:, :3])
            sla, cla, slo, clo = (f(v)[:, None] for f, v in ((np.sin, lat), (np.cos, lat), (np.sin, lon), (np.cos, lon)))
            nn = -sla * clo * los[..., 0] - sla * slo * los[..., 1] + cla * los[..., 2]
            ee = -slo * los[..., 0] + clo * los[..., 1]
            uu = cla * clo * los[..., 0] + cla * slo * los[..., 1] + sla * los[..., 2]
            az = np.arctan2(ee, nn)
            az = np.where(az < 0.0, az + 2.0 * PI, az)
            el = np.arctan2(uu, np.hypot(nn, ee))
            trx = (nom_ms[a] * 1e-3 + m[a] / 3e6 - x[:, 3] / C)[:, None]
            I = np.where(iono[:, None], klobuchar(cfg["alpha"], cfg["beta"], lat[:, None], lon[:, None], az, el, trx,
                                                      trace), 0.0)
        ra = (rho[a] - (R + x[:, 3:4] - C * dtsv[a] + I)) * w[a]
        Ha = np.concatenate([-los / R[..., None], np.ones(R.shape + (1,))], -1) * w[a][..., None]
        H[a], r[a] = Ha, ra
        N = np.einsum("fci,fcj->fij", Ha, Ha)
        b = np.einsum("fci,fc->fi", Ha, ra)
        iters[a] = j + 1
        pd = np.all(np.linalg.eigvalsh(N) > 0, axis=-1)
        bad = a[~pd]
        active[bad] = False
        a, N, b = a[pd], N[pd], b[pd]
        d = np.linalg.solve(N, b[..., None])[..., 0]
        X[a] += d
        dX[a] = d
        Nmat[a] = N
        out, step = np.linalg.norm(X[a, :3], axis=-1), np.linalg.norm(d[:, :3], axis=-1)
        if trace is not None:
            for k, v in (("radius", rad), ("runaway", out), ("step", step)):
                trace[k].append(v)
        away = out > RUNAWAY
        active[a[away]] = False
        conv = (step < CONVERGED) & ~away
        status[a[conv]] = FIX_OK
        active[a[conv]] = False
    fix = {f: np.full(nf, np.nan) for f in ("x", "y", "z", "clock_m", "t_rx", "vx", "vy", "vz", "drift", "lat_deg",
                                             "lon_deg", "height", "pdop", "rms")}
    ok = np.nonzero(status == FIX_OK)[0]
    if ok.size:
        post = (r[ok] - np.einsum("fci,fi->fc", H[ok], dX[ok])) * w[ok]
        res[ok] = np.where(use[ok], post, np.nan)
        # rate + c drift_sv - e . v_sat, with the row's -e
        y = (rate[ok] + C * ddtsv[ok] + np.einsum("fci,fci->fc", H[ok][..., :3], Vr[ok])) * w[ok]
        vel = np.linalg.solve(Nmat[ok], np.einsum("fci,fc->fi", H[ok], y)[..., None])[..., 0]
        Q = np.linalg.inv(Nmat[ok])
        x = X[ok]
        lat, lon, h = ecef_llh(x[:, :3])
        trx = nom_ms[ok] * 1e-3 + (m[ok] / 3e6 - x[:, 3] / C)
        trx = np.where(trx < 0.0, trx + 604800.0, np.where(trx >= 604800.0, trx - 604800.0, trx))
        for f, v in (("x", x[:, 0]), ("y", x[:, 1]), ("z", x[:, 2]), ("clock_m", x[:, 3]), ("t_rx", trx),
                     ("vx", vel[:, 0]), ("vy", vel[:, 1]), ("vz", vel[:, 2]), ("drift", vel[:, 3]),
                     ("lat_deg", np.degrees(lat)), ("lon_deg", np.degrees(lon)), ("height", h),
                     ("pdop", np.sqrt(Q[:, 0, 0] + Q[:, 1, 1] + Q[:, 2, 2])),
                     ("rms", np.sqrt((np.nan_to_num(res[ok]) ** 2).sum(1) / nused[ok]))):
            fix[f][ok] = v
    fix.update(sample=s, status=status, nused=nused, mask=mask, iterations=iters)
    return fix, res, ms
