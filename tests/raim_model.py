"""Numpy statement of the RAIM stage (include/gpsb200.h: gpsb200_pvt_raim; DESIGN §11.1): the tests' reference.

It runs on pvt_model's measurement, satellite, Earth-rotation, Klobuchar and WGS-84 pieces. A pass is `solve`: the
Gauss-Newton fix of pvt_model.pvt, restated so that it takes each fix's channel set and start estimate (after an
exclusion, the previous fix) and returns the last iteration's rows, residuals, normal matrix and step. Without a mask
and a start it gives pvt_model.pvt's fixes and residuals bit for bit (tests/test_raim.py checks it on ideal epochs).
The chi^2 tables T / lambda come from the caller (gps.raim_thresholds; tests/test_raim.py checks them against scipy)."""
import numpy as np

import pvt_model as PM

PASS, EXCLUDED, ALERT, UNAVAILABLE = 0, 1, 2, 3
FLAT = 1e-9          # 1 - h_jj at or below this: never a candidate; +inf protection levels


def solve(chans, epochs, cfg, mask=None, x0=None):
    """pvt_model.pvt with mask (bool [F, C], optional: the channels each fix may use on top of the contract's rule) and
    x0 ([F, 4], optional: the start (x, y, z, b) of each fix instead of the Earth's centre).
    -> (fix dict, residuals [F, C], measurement dict of pvt_model.measure() plus the last iteration's unweighted rows
    "rows" [F, C, 4] and "r" [F, C] of every measured channel, its normal matrix "normal" [F, 4, 4] and step "dX" [F, 4])."""
    nf, nc = int(cfg["nfix"]), len(epochs)
    s = int(cfg["s0"]) + np.arange(nf, dtype=np.int64) * int(cfg["step"])
    ms = PM.measure(chans, epochs, s)
    use = ms["use"] if mask is None else ms["use"] & np.asarray(mask, bool)
    ref = next((c for c in range(nc) if chans[c]["eph"]["valid"] and chans[c]["eph"]["health"] == 0), -1)
    if ref < 0:
        use[:] = False
        ref_sample = ref_ms = 0
    else:
        ref_sample = int(epochs[ref]["sample"][int(chans[ref]["anchor_epoch"])])
        ref_ms = int(chans[ref]["anchor_ms"])
    q = np.floor_divide(s - ref_sample, 3000)
    m = (s - ref_sample) - 3000 * q
    nom_ms = np.mod(ref_ms + 75 + q, PM.WEEK_MS)
    D = np.mod(ref_ms + 75 + q[:, None] - ms["T"], PM.WEEK_MS)
    D = np.where(D >= PM.WEEK_MS // 2, D - PM.WEEK_MS, D)
    rho = D.astype(np.float64) * PM.C_MS + (m[:, None] / 3000.0 - ms["frac"]) * PM.C_MS
    rate = -PM.LAMBDA_L1 * (ms["w"].astype(np.float64) * PM.STEP_HZ)
    eph = np.stack([chans[c]["eph"] for c in range(nc)])[None, :]
    d0 = PM.wrap_half_week(ms["tsv"] - eph["toc"])
    tt = ms["tsv"] - (eph["af0"] + d0 * (eph["af1"] + d0 * eph["af2"]))
    P, V, dtsv, ddtsv = PM.satellite(eph, tt)
    nused = use.sum(1)
    bits = (use * (1 << np.arange(nc, dtype=np.int64))).sum(1)
    X = np.zeros((nf, 4)) if x0 is None else np.array(x0, np.float64)
    status = np.where(nused < 4, PM.FIX_FEW, PM.FIX_NO_CONVERGENCE)
    iters = np.zeros(nf, np.int32)
    active = nused >= 4
    res = np.full((nf, nc), np.nan)
    H, r = np.zeros((nf, nc, 4)), np.zeros((nf, nc))
    Hu, ru = np.zeros((nf, nc, 4)), np.zeros((nf, nc))
    Vr = np.zeros((nf, nc, 3))
    dX = np.zeros((nf, 4))
    Nmat = np.zeros((nf, 4, 4))
    w = use.astype(np.float64)
    for j in range(PM.MAX_ITER):
        a = np.nonzero(active)[0]
        if a.size == 0:
            break
        x = X[a]
        g = P[a] - x[:, None, :3]
        tau = np.linalg.norm(g, axis=-1) / PM.C
        sth, cth = np.sin(PM.OMEGA_E * tau), np.cos(PM.OMEGA_E * tau)
        pa, va = P[a], V[a]
        pr = np.stack([pa[..., 0] * cth + pa[..., 1] * sth, pa[..., 1] * cth - pa[..., 0] * sth, pa[..., 2]], -1)
        Vr[a] = np.stack([va[..., 0] * cth + va[..., 1] * sth, va[..., 1] * cth - va[..., 0] * sth, va[..., 2]], -1)
        los = pr - x[:, None, :3]
        R = np.linalg.norm(los, axis=-1)
        I = np.zeros(R.shape)
        iono = bool(cfg["iono"]) & (np.linalg.norm(x[:, :3], axis=-1) >= PM.IONO_MIN_RADIUS)
        if iono.any():
            lat, lon, _ = PM.ecef_llh(x[:, :3])
            sla, cla, slo, clo = (f(v)[:, None] for f, v in ((np.sin, lat), (np.cos, lat), (np.sin, lon), (np.cos, lon)))
            nn = -sla * clo * los[..., 0] - sla * slo * los[..., 1] + cla * los[..., 2]
            ee = -slo * los[..., 0] + clo * los[..., 1]
            uu = cla * clo * los[..., 0] + cla * slo * los[..., 1] + sla * los[..., 2]
            az = np.arctan2(ee, nn)
            az = np.where(az < 0.0, az + 2.0 * PM.PI, az)
            el = np.arctan2(uu, np.hypot(nn, ee))
            trx = (nom_ms[a] * 1e-3 + m[a] / 3e6 - x[:, 3] / PM.C)[:, None]
            I = np.where(iono[:, None], PM.klobuchar(cfg["alpha"], cfg["beta"], lat[:, None], lon[:, None], az, el, trx),
                         0.0)
        # every measured channel's row, unweighted; the normal equations take the set's rows only (an excluded
        # channel enters with weight 0, as in the kernel)
        Hu[a] = np.concatenate([-los / R[..., None], np.ones(R.shape + (1,))], -1)
        ru[a] = rho[a] - (R + x[:, 3:4] - PM.C * dtsv[a] + I)
        Ha, ra = Hu[a] * w[a][..., None], ru[a] * w[a]
        H[a], r[a] = Ha, ra
        N = np.einsum("fci,fcj->fij", Ha, Ha)
        b = np.einsum("fci,fc->fi", Ha, ra)
        iters[a] = j + 1
        pd = np.all(np.linalg.eigvalsh(N) > 0, axis=-1)
        active[a[~pd]] = False
        a, N, b = a[pd], N[pd], b[pd]
        d = np.linalg.solve(N, b[..., None])[..., 0]
        X[a] += d
        dX[a] = d
        Nmat[a] = N
        away = np.linalg.norm(X[a, :3], axis=-1) > PM.RUNAWAY
        active[a[away]] = False
        conv = (np.linalg.norm(d[:, :3], axis=-1) < PM.CONVERGED) & ~away
        status[a[conv]] = PM.FIX_OK
        active[a[conv]] = False
    fix = {f: np.full(nf, np.nan) for f in ("x", "y", "z", "clock_m", "t_rx", "vx", "vy", "vz", "drift", "lat_deg",
                                             "lon_deg", "height", "pdop", "rms")}
    ok = np.nonzero(status == PM.FIX_OK)[0]
    if ok.size:
        post = (r[ok] - np.einsum("fci,fi->fc", H[ok], dX[ok])) * w[ok]
        res[ok] = np.where(use[ok], post, np.nan)
        y = (rate[ok] + PM.C * ddtsv[ok] + np.einsum("fci,fci->fc", H[ok][..., :3], Vr[ok])) * w[ok]
        vel = np.linalg.solve(Nmat[ok], np.einsum("fci,fc->fi", H[ok], y)[..., None])[..., 0]
        Q = np.linalg.inv(Nmat[ok])
        x = X[ok]
        lat, lon, h = PM.ecef_llh(x[:, :3])
        trx = nom_ms[ok] * 1e-3 + (m[ok] / 3e6 - x[:, 3] / PM.C)
        trx = np.where(trx < 0.0, trx + 604800.0, np.where(trx >= 604800.0, trx - 604800.0, trx))
        for f, v in (("x", x[:, 0]), ("y", x[:, 1]), ("z", x[:, 2]), ("clock_m", x[:, 3]), ("t_rx", trx),
                     ("vx", vel[:, 0]), ("vy", vel[:, 1]), ("vz", vel[:, 2]), ("drift", vel[:, 3]),
                     ("lat_deg", np.degrees(lat)), ("lon_deg", np.degrees(lon)), ("height", h),
                     ("pdop", np.sqrt(Q[:, 0, 0] + Q[:, 1, 1] + Q[:, 2, 2])),
                     ("rms", np.sqrt((np.nan_to_num(res[ok]) ** 2).sum(1) / nused[ok]))):
            fix[f][ok] = v
    fix.update(sample=s, status=status, nused=nused, mask=bits, iterations=iters)
    ms.update(rows=Hu, r=ru, normal=Nmat, dX=dX)
    return fix, res, ms


def loo(ms, f):
    """Leave-one-out quantities of fix f from the last iteration of its pass: post-fit residuals e [C] of every
    measured channel, x_j = N^-1 g_j [C, 4] and 1 - h_jj [C]."""
    g = ms["rows"][f]
    e = ms["r"][f] - g @ ms["dX"][f]
    x = np.linalg.solve(ms["normal"][f], g.T).T
    return e, x, 1.0 - np.einsum("ci,ci->c", g, x)


def raim(chans, epochs, cfg, rcfg, T, lam):
    """-> (fix dict as solve gives for each fix's final set, residuals [F, C] as gpsb200_pvt_raim reports them,
    record dict of arrays [F] with the RAIM_DTYPE field names, and per fix the normalized residuals e^2 / (1 - h_jj) of
    every test run, for the tests' margin checks)."""
    sigma, max_ex = float(rcfg["sigma"]), int(rcfg["max_exclude"])
    fix, _, ms = solve(chans, epochs, cfg)
    nf, nc = fix["status"].size, len(epochs)
    has = ms["use"].copy()
    inset = has.copy()
    rec = dict(verdict=np.full(nf, UNAVAILABLE, np.int32), excluded=np.zeros(nf, np.uint32), dof=np.zeros(nf, np.int32),
               stat=np.full(nf, np.nan), threshold=np.full(nf, np.nan), hpl=np.full(nf, np.nan),
               vpl=np.full(nf, np.nan))
    tests = [[] for _ in range(nf)]
    state = {f: (fix, ms) for f in range(nf)}   # the pass each fix's final values come from
    iters = fix["iterations"].astype(np.int64).copy()
    todo = [f for f in range(nf) if fix["status"][f] == PM.FIX_OK and inset[f].sum() >= 5]
    while todo:
        resolve = []
        for f in todo:
            fx, m = state[f]
            e, _, omh = loo(m, f)
            n = int(inset[f].sum())
            stat = float((e[inset[f]] ** 2).sum()) / (sigma * sigma)
            rec["stat"][f], rec["dof"][f], rec["threshold"][f] = stat, n - 4, T[n - 5]
            key = np.where(inset[f] & (omh > FLAT), e * e / np.where(omh > FLAT, omh, 1.0), -1.0)
            tests[f].append((stat, T[n - 5], key))
            if not stat > T[n - 5]:
                rec["verdict"][f] = EXCLUDED if rec["excluded"][f] else PASS
                continue
            rec["verdict"][f] = ALERT
            if n < 6 or bin(int(rec["excluded"][f])).count("1") >= max_ex or key.max() < 0.0:
                continue
            j = int(np.argmax(key))              # the first maximum: the lowest channel on ties
            rec["excluded"][f] |= np.uint32(1 << j)
            inset[f, j] = False
            resolve.append(f)
        if not resolve:
            break
        x0 = np.zeros((nf, 4))
        for f in resolve:
            fx = state[f][0]
            x0[f] = [fx["x"][f], fx["y"][f], fx["z"][f], fx["clock_m"][f]]
        nfix, nms = solve(chans, epochs, cfg, mask=inset, x0=x0)[0::2]
        todo = []
        for f in resolve:
            state[f] = (nfix, nms)
            iters[f] += int(nfix["iterations"][f])
            if nfix["status"][f] == PM.FIX_OK:
                todo.append(f)
    # the final fixes, residuals and protection levels
    out = {k: np.array(v, copy=True) for k, v in fix.items()}
    res = np.full((nf, nc), np.nan)
    for f in range(nf):
        fx, m = state[f]
        for k in out:
            out[k][f] = fx[k][f]
        out["iterations"][f] = iters[f]
        if fx["status"][f] != PM.FIX_OK:
            continue
        e, x, omh = loo(m, f)
        res[f] = np.where(has[f], e, np.nan)
        if rec["verdict"][f] == UNAVAILABLE:
            continue
        lat, lon, _ = PM.ecef_llh(np.array([fx["x"][f], fx["y"][f], fx["z"][f]]))
        sla, cla, slo, clo = np.sin(lat), np.cos(lat), np.sin(lon), np.cos(lon)
        xe = -slo * x[:, 0] + clo * x[:, 1]
        xn = -sla * clo * x[:, 0] - sla * slo * x[:, 1] + cla * x[:, 2]
        xu = cla * clo * x[:, 0] + cla * slo * x[:, 1] + sla * x[:, 2]
        s = inset[f]
        flat = omh[s] <= FLAT
        k = sigma * np.sqrt(lam[rec["dof"][f] - 1])
        if flat.any():
            rec["hpl"][f] = rec["vpl"][f] = np.inf
        else:
            rec["hpl"][f] = np.max(np.hypot(xe[s], xn[s]) / np.sqrt(omh[s])) * k
            rec["vpl"][f] = np.max(np.abs(xu[s]) / np.sqrt(omh[s])) * k
    return out, res, rec, tests
