"""Numpy statement of the coarse-time fix (include/gpsb200.h: gpsb200_pvt_coarse; DESIGN §11.3): the tests' reference.

It shares no code with the library. The satellite, the Klobuchar delay and the WGS-84 conversion are pvt_model's (as
raim_model reuses them); the measurement, the whole-ms resolution and the five-state Gauss-Newton are restated here,
vectorised over fix instants and channels. numpy's transcendental functions differ from CUDA's by ulps, so the fixes
agree to well under a micrometre, and every integer decision the same unless it sits within ulps of a half."""
import numpy as np

import pvt_model as PM
from pvt_model import C, C_MS, OMEGA_E, WEEK_MS, ecef_llh, klobuchar, satellite, wrap_half_week

FIX_AMBIGUOUS = 3
TAU0 = 0.075
FLIGHT_STEPS = 3
MAX_RESIDUAL = 1000.0


def measure(chans, epochs, s, tas):
    """Header step 2 for fix instants s and a-priori times tas [F]. -> dict of [F, C]: use, frac (ms), w."""
    nf, nc = s.size, len(epochs)
    out = {f: np.zeros((nf, nc), dt) for f, dt in (("use", bool), ("frac", np.float64), ("w", np.int64))}
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
        ok &= np.abs(wrap_half_week(tas - eph["toe"])) <= 7200.0
        phi = e["code_phase"][kk - 1].astype(np.uint64) + (s - smp[kk]).astype(np.uint64) * e["code_step"][kk - 1].astype(np.uint64)
        out["use"][:, c] = ok
        out["frac"][:, c] = phi.astype(np.float64) / PM.CODE_MOD
        out["w"][:, c] = e["carr_step"][kk - 1]
    return out


def up_vector(x):
    lat, lon, _ = ecef_llh(np.asarray(x, np.float64))
    return np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], -1)


def predict(eph, x, t, up):
    """Header step 3: predicted transmit time (ms) and sin(elevation) of satellites eph [F, C] seen from x [F, 3] at
    receive times t [F] (up [F, 3])."""
    tau = np.full(eph.shape, TAU0)
    t = np.asarray(t, np.float64)[:, None]
    for _ in range(FLIGHT_STEPS):
        p, _, dt, _ = satellite(eph, t - tau)
        sth, cth = np.sin(OMEGA_E * tau), np.cos(OMEGA_E * tau)
        l = np.stack([p[..., 0] * cth + p[..., 1] * sth - x[:, None, 0], p[..., 1] * cth - p[..., 0] * sth - x[:, None, 1],
                      p[..., 2] - x[:, None, 2]], -1)
        tau = np.sqrt((l * l).sum(-1)) / C
    sel = (up[:, None, :] * l).sum(-1) / (tau * C)
    return 1000.0 * (t - tau + dt), sel


def round_half_up(v):
    return np.floor(v + 0.5)


def coarse(chans, epochs, cfg, ap, trace=None):
    """The fixes of the contract. chans: PVT_CHAN records; epochs: list of TRACK_EPOCH arrays; cfg: PVT_CONFIG record;
    ap: COARSE_CONFIG record. trace: None, or a dict whose list "half" receives the distance (ms) of every rounding
    argument from its nearest half, "residual" the converged fixes' |post-fit residuals| (m) and "step" / "runaway" the
    convergence and runaway figures per iteration.
    -> (fix dict [F] with FIX_DTYPE names, coarse dict [F] with COARSE_DTYPE names, residuals [F, C], ms [F, C])."""
    nf, nc = int(cfg["nfix"]), len(epochs)
    s = int(cfg["s0"]) + np.arange(nf, dtype=np.int64) * int(cfg["step"])
    ds = s - int(ap["s_a"])
    q = np.floor_divide(ds, 3000)
    m = ds - 3000 * q
    u = float(ap["t_a"]) + ds.astype(np.float64) / 3e6
    kw = np.floor(u / 604800.0)
    tas = u - 604800.0 * kw
    W = np.floor(float(ap["t_a"]))
    F = float(ap["t_a"]) - W
    sub = F * 1000.0 + m.astype(np.float64) / 3000.0
    ms_ = measure(chans, epochs, s, tas)
    use, frac = ms_["use"], ms_["frac"]
    eph = np.broadcast_to(np.stack([chans[c]["eph"] for c in range(nc)])[None, :], (nf, nc))
    xa = np.broadcast_to(np.asarray(ap["x_a"], np.float64), (nf, 3))
    up = up_vector(xa)
    pred, sel = predict(eph, xa, tas, up)
    nused = use.sum(1)
    mask = (use * (1 << np.arange(nc, dtype=np.int64))).sum(1)
    key = np.where(use, sel, -2.0)
    r = np.argmax(key, axis=1)                       # the first (lowest) channel among equal maxima
    ref = np.where(nused > 0, r, -1)
    fi = np.arange(nf)
    pred_r, frac_r = pred[fi, r][:, None], frac[fi, r][:, None]
    a0 = pred_r - frac_r
    a1 = (pred - pred_r) - (frac - frac_r)
    Nr = round_half_up(a0).astype(np.int64)
    dN = round_half_up(a1).astype(np.int64)
    Nw = np.mod(Nr + dN, WEEK_MS)
    if trace is not None:
        trace["half"].append(np.abs(a0 - np.floor(a0) - 0.5)[nused > 0].ravel())
        trace["half"].append(np.abs(a1 - np.floor(a1) - 0.5)[use].ravel())
    D = np.mod(int(W) * 1000 + q[:, None] - Nw, WEEK_MS)
    D = np.where(D >= WEEK_MS // 2, D - WEEK_MS, D)
    rho = D.astype(np.float64) * C_MS + (sub[:, None] - frac) * C_MS
    tsv = Nw.astype(np.float64) * 1e-3 + frac * 1e-3
    rate = -PM.LAMBDA_L1 * (ms_["w"].astype(np.float64) * PM.STEP_HZ)

    X = np.concatenate([xa, np.zeros((nf, 2))], 1)
    status = np.where(nused < 5, PM.FIX_FEW, PM.FIX_NO_CONVERGENCE)
    iters = np.zeros(nf, np.int32)
    active = nused >= 5
    H = np.zeros((nf, nc, 5))
    rr = np.zeros((nf, nc))
    Vr = np.zeros((nf, nc, 3))
    ddt = np.zeros((nf, nc))
    dX = np.zeros((nf, 5))
    Nmat = np.zeros((nf, 5, 5))
    w = use.astype(np.float64)
    for j in range(PM.MAX_ITER):
        a = np.nonzero(active)[0]
        if a.size == 0:
            break
        x = X[a]
        e = eph[a]
        t = tsv[a] + x[:, 4:5]
        d0 = wrap_half_week(t - e["toc"])
        P, V, dtsv, ddtsv = satellite(e, t - (e["af0"] + d0 * (e["af1"] + d0 * e["af2"])))
        g = P - x[:, None, :3]
        tau = np.sqrt((g * g).sum(-1)) / C
        sth, cth = np.sin(OMEGA_E * tau), np.cos(OMEGA_E * tau)
        pr = np.stack([P[..., 0] * cth + P[..., 1] * sth, P[..., 1] * cth - P[..., 0] * sth, P[..., 2]], -1)
        vr = np.stack([V[..., 0] * cth + V[..., 1] * sth, V[..., 1] * cth - V[..., 0] * sth, V[..., 2]], -1)
        los = pr - x[:, None, :3]
        R = np.sqrt((los * los).sum(-1))
        I = np.zeros(R.shape)
        rad = np.sqrt((x[:, :3] ** 2).sum(-1))
        iono = bool(cfg["iono"]) & (rad >= PM.IONO_MIN_RADIUS)
        if iono.any():
            lat, lon, _ = ecef_llh(x[:, :3])
            sla, cla, slo, clo = (f(v)[:, None] for f, v in ((np.sin, lat), (np.cos, lat), (np.sin, lon), (np.cos, lon)))
            nn = -sla * clo * los[..., 0] - sla * slo * los[..., 1] + cla * los[..., 2]
            ee = -slo * los[..., 0] + clo * los[..., 1]
            uu = cla * clo * los[..., 0] + cla * slo * los[..., 1] + sla * los[..., 2]
            az = np.arctan2(ee, nn)
            az = np.where(az < 0.0, az + 2.0 * PM.PI, az)
            el = np.arctan2(uu, np.sqrt(nn * nn + ee * ee))
            trx = (tas[a] + x[:, 4] - x[:, 3] / C)[:, None]
            I = np.where(iono[:, None], klobuchar(cfg["alpha"], cfg["beta"], lat[:, None], lon[:, None], az, el, trx),
                         0.0)
        ra = (rho[a] - (R + x[:, 3:4] - C * dtsv + I)) * w[a]
        hd = (los * vr).sum(-1) / R - C * ddtsv
        Ha = np.concatenate([-los / R[..., None], np.ones(R.shape + (1,)), hd[..., None]], -1) * w[a][..., None]
        H[a], rr[a], Vr[a], ddt[a] = Ha, ra, vr, ddtsv
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
        out, step = np.sqrt((X[a, :3] ** 2).sum(-1)), np.sqrt((d[:, :3] ** 2).sum(-1))
        if trace is not None:
            trace["step"].append(step)
            trace["runaway"].append(out)
        away = out > PM.RUNAWAY
        active[a[away]] = False
        conv = (step < PM.CONVERGED) & ~away
        status[a[conv]] = PM.FIX_OK
        active[a[conv]] = False

    changed = np.zeros(nf, np.int64)
    fix = {f: np.full(nf, np.nan) for f in ("x", "y", "z", "clock_m", "t_rx", "vx", "vy", "vz", "drift", "lat_deg",
                                             "lon_deg", "height", "pdop", "rms")}
    co = dict(delta=np.full(nf, np.nan), pdop=np.full(nf, np.nan), ref=ref.astype(np.int32),
              week=np.full(nf, -1, np.int32), changed=changed)
    res = np.full((nf, nc), np.nan)
    ok = np.nonzero(status == PM.FIX_OK)[0]
    if ok.size:
        x = X[ok]
        trx = tas[ok] + x[:, 4] - x[:, 3] / C
        pred2, _ = predict(eph[ok], x[:, :3], trx, up[ok])
        a2 = (pred2 - pred2[np.arange(ok.size), r[ok]][:, None]) - (frac[ok] - frac_r[ok])
        if trace is not None:
            trace["half"].append(np.abs(a2 - np.floor(a2) - 0.5)[use[ok]].ravel())
        moved = use[ok] & (round_half_up(a2).astype(np.int64) != dN[ok])
        changed[ok] = (moved * (1 << np.arange(nc, dtype=np.int64))).sum(1)
        post = (rr[ok] - np.einsum("fci,fi->fc", H[ok], dX[ok])) * w[ok]
        if trace is not None:
            trace["residual"].append(np.abs(post[use[ok]]))
        big = (use[ok] & ~(np.abs(post) <= MAX_RESIDUAL)).any(1)
        amb = (changed[ok] != 0) | big
        status[ok[amb]] = FIX_AMBIGUOUS
        ok, x, trx, post = ok[~amb], x[~amb], trx[~amb], post[~amb]
    if ok.size:
        res[ok] = np.where(use[ok], post, np.nan)
        y = (rate[ok] + C * ddt[ok] + np.einsum("fci,fci->fc", H[ok][..., :3], Vr[ok])) * w[ok]
        N4 = Nmat[ok][:, :4, :4]
        vel = np.linalg.solve(N4, np.einsum("fci,fc->fi", H[ok][..., :4], y)[..., None])[..., 0]
        Q = np.linalg.inv(Nmat[ok])
        lat, lon, h = ecef_llh(x[:, :3])
        wk = kw[ok].copy()
        t = trx.copy()
        lo, hi = t < 0.0, t >= 604800.0
        t = np.where(lo, t + 604800.0, np.where(hi, t - 604800.0, t))
        wk = np.where(lo, wk - 1.0, np.where(hi, wk + 1.0, wk))
        pdop = np.sqrt(Q[:, 0, 0] + Q[:, 1, 1] + Q[:, 2, 2])
        for f, v in (("x", x[:, 0]), ("y", x[:, 1]), ("z", x[:, 2]), ("clock_m", x[:, 3]), ("t_rx", t),
                     ("vx", vel[:, 0]), ("vy", vel[:, 1]), ("vz", vel[:, 2]), ("drift", vel[:, 3]),
                     ("lat_deg", np.degrees(lat)), ("lon_deg", np.degrees(lon)), ("height", h), ("pdop", pdop),
                     ("rms", np.sqrt((np.nan_to_num(res[ok]) ** 2).sum(1) / nused[ok]))):
            fix[f][ok] = v
        co["delta"][ok] = x[:, 4]
        co["pdop"][ok] = pdop
        co["week"][ok] = int(ap["week"]) + wk.astype(np.int64)
    fix.update(sample=s, status=status, nused=nused, mask=mask, iterations=iters)
    ms = np.where(use, Nw, -1)
    return fix, co, res, ms
