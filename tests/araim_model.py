"""Numpy statement of the ARAIM stage (include/gpsb200.h: gpsb200_pvt_araim; DESIGN §11.2): the tests' reference.

It runs on pvt_model's measurement, satellite, Klobuchar and WGS-84 pieces and restates the rest per fix instant: the
weighted Gauss-Newton pass, the elevation mask, and the solution separation from explicit per-subset matrices
S(k) = (G_k^T W_k G_k)^-1 G_k^T W_k (no rank-one downdate, unlike the kernel). The protection levels use scipy's erfc
and erfcinv. K_fa comes from the caller (gps.araim_kfa; tests/test_araim.py checks it against scipy)."""
import numpy as np
from scipy import special, stats

import pvt_model as PM

PASS, EXCLUDED, ALERT, UNAVAILABLE = 0, 1, 2, 3
URA_NOM = np.array([2.0, 2.8, 4.0, 5.7, 8.0, 11.3, 16.0, 32.0, 64.0, 128.0, 256.0, 512.0, 1024.0, 2048.0, 4096.0])


def q_tail(x):
    return 0.5 * special.erfc(x / np.sqrt(2.0))


def q_inv(p):
    return np.sqrt(2.0) * special.erfcinv(2.0 * p)


def klobuchar_f_phim(lat, lon, az, el):
    """The Klobuchar obliquity factor F and geomagnetic latitude phi_m (semicircles), as pvt_model.klobuchar forms them."""
    E, phi_u, lam_u = el / PM.PI, lat / PM.PI, lon / PM.PI
    F = 1.0 + 16.0 * (0.53 - E) ** 3
    psi = 0.0137 / (E + 0.11) - 0.022
    phi_i = np.clip(phi_u + psi * np.cos(az), -0.416, 0.416)
    lam_i = lam_u + psi * np.sin(az) / np.cos(phi_i * PM.PI)
    return F, phi_i + 0.064 * np.cos((lam_i - 1.617) * PM.PI)


def enu(X):
    lat, lon, _ = PM.ecef_llh(np.asarray(X[:3], np.float64))
    sla, cla, slo, clo = np.sin(lat), np.cos(lat), np.sin(lon), np.cos(lon)
    return np.array([[-slo, clo, 0.0], [-sla * clo, -sla * slo, cla], [cla * clo, cla * slo, sla]])


def protection_level(rhs, b0, s0, T, b, s, p_sat):
    """The smallest L with 2 Q((L - b0) / s0) + sum_k p_sat Q((L - T_k - b_k) / s_k) <= rhs, by the header's bisection."""
    m = len(T) + 1
    lo, hi = b0 + s0 * q_inv(rhs / 2.0), b0 + s0 * q_inv(rhs / m / 2.0)
    if rhs < p_sat:
        lo = max(lo, float(np.max(T + b + s * q_inv(rhs / p_sat))))
    if rhs / m < p_sat:
        hi = max(hi, float(np.max(T + b + s * q_inv(rhs / m / p_sat))))
    for _ in range(200):
        if not hi - lo > 1e-3:
            break
        mid = 0.5 * (lo + hi)
        if 2.0 * q_tail((mid - b0) / s0) + float(np.sum(p_sat * q_tail((mid - T - b) / s))) <= rhs:
            hi = mid
        else:
            lo = mid
    return hi


def pl_lhs(L, b0, s0, T, b, s, p_sat):
    """The left side of the protection-level equation with scipy.stats.norm.sf (for the tests)."""
    return 2.0 * stats.norm.sf((L - b0) / s0) + float(np.sum(p_sat * stats.norm.sf((L - T - b) / s)))


def p_nm(p, n):
    return float(stats.binom.sf(1, n, p))


class Inputs:
    """The measurement of every fix instant: pseudorange, range rate and satellite state per channel."""

    def __init__(self, chans, epochs, cfg):
        nf, nc = int(cfg["nfix"]), len(epochs)
        self.cfg, self.nf, self.nc = cfg, nf, nc
        self.s = int(cfg["s0"]) + np.arange(nf, dtype=np.int64) * int(cfg["step"])
        ms = PM.measure(chans, epochs, self.s)
        ura = np.array([int(chans[c]["eph"]["ura"]) for c in range(nc)])
        ok = (ura >= 0) & (ura < 15)
        use = ms["use"] & ok[None, :]
        ref = next((c for c in range(nc) if chans[c]["eph"]["valid"] and chans[c]["eph"]["health"] == 0), -1)
        if ref < 0:
            use[:] = False
            ref_sample = ref_ms = 0
        else:
            ref_sample = int(epochs[ref]["sample"][int(chans[ref]["anchor_epoch"])])
            ref_ms = int(chans[ref]["anchor_ms"])
        q = np.floor_divide(self.s - ref_sample, 3000)
        self.m = (self.s - ref_sample) - 3000 * q
        self.nom_ms = np.mod(ref_ms + 75 + q, PM.WEEK_MS)
        D = np.mod(ref_ms + 75 + q[:, None] - ms["T"], PM.WEEK_MS)
        D = np.where(D >= PM.WEEK_MS // 2, D - PM.WEEK_MS, D)
        self.rho = D.astype(np.float64) * PM.C_MS + (self.m[:, None] / 3000.0 - ms["frac"]) * PM.C_MS
        self.rate = -PM.LAMBDA_L1 * (ms["w"].astype(np.float64) * PM.STEP_HZ)
        eph = np.stack([chans[c]["eph"] for c in range(nc)])[None, :]
        d0 = PM.wrap_half_week(ms["tsv"] - eph["toc"])
        tt = ms["tsv"] - (eph["af0"] + d0 * (eph["af1"] + d0 * eph["af2"]))
        self.P, self.V, self.dtsv, self.ddtsv = PM.satellite(eph, tt)
        self.use = use
        self.ura = ura


def gauss_newton(inp, acfg, f, S, X, trace=None):
    """One weighted pass of fix f on the channel set S (bool [C]) from X. -> (ok, X, iterations, last-iteration dict)."""
    cfg, has = inp.cfg, inp.use[f]
    sig_ura = np.maximum(float(acfg["sigma_ura"]), URA_NOM[np.clip(inp.ura, 0, 14)])
    sura2 = sig_ura ** 2
    sure2 = (sig_ura * float(acfg["sigma_ure"]) / float(acfg["sigma_ura"])) ** 2
    X = np.array(X, np.float64)
    it = 0
    for _ in range(PM.MAX_ITER):
        P, V = inp.P[f], inp.V[f]
        tau = np.linalg.norm(P - X[:3], axis=-1) / PM.C
        sth, cth = np.sin(PM.OMEGA_E * tau), np.cos(PM.OMEGA_E * tau)
        pr = np.stack([P[:, 0] * cth + P[:, 1] * sth, P[:, 1] * cth - P[:, 0] * sth, P[:, 2]], -1)
        vr = np.stack([V[:, 0] * cth + V[:, 1] * sth, V[:, 1] * cth - V[:, 0] * sth, V[:, 2]], -1)
        los = pr - X[:3]
        R = np.linalg.norm(los, axis=-1)
        near = np.linalg.norm(X[:3]) >= PM.IONO_MIN_RADIUS
        iono = bool(cfg["iono"]) and near
        I, el, sig_iono = np.zeros(inp.nc), np.full(inp.nc, 0.5 * np.pi), np.zeros(inp.nc)
        if near:
            lat, lon, _ = PM.ecef_llh(X[:3])
            sla, cla, slo, clo = np.sin(lat), np.cos(lat), np.sin(lon), np.cos(lon)
            nn = -sla * clo * los[:, 0] - sla * slo * los[:, 1] + cla * los[:, 2]
            ee = -slo * los[:, 0] + clo * los[:, 1]
            uu = cla * clo * los[:, 0] + cla * slo * los[:, 1] + sla * los[:, 2]
            az = np.arctan2(ee, nn)
            az = np.where(az < 0.0, az + 2.0 * PM.PI, az)
            el = np.arctan2(uu, np.hypot(nn, ee))
            if iono:
                trx = inp.nom_ms[f] * 1e-3 + inp.m[f] / 3e6 - X[3] / PM.C
                I = PM.klobuchar(cfg["alpha"], cfg["beta"], lat, lon, az, el, trx)
                F, phim = klobuchar_f_phim(lat, lon, az, el)
                pm = np.abs(phim) * 180.0
                sig_iono = np.maximum(I / 5.0, F * np.where(pm <= 20.0, 9.0, np.where(pm <= 55.0, 4.5, 6.0)))
        r = inp.rho[f] - (R + X[3] - PM.C * inp.dtsv[f] + I)
        g = np.concatenate([-los / R[:, None], np.ones((inp.nc, 1))], -1)
        st = 0.12 * 1.001 / np.sqrt(0.002001 + np.sin(el) ** 2)
        mp = 0.13 + 0.53 * np.exp(-el / np.radians(10.0))
        rest2 = st * st + (float(acfg["sigma_noise"]) ** 2 + mp * mp) + sig_iono ** 2
        sw = 1.0 / np.sqrt(sura2 + rest2)
        w = np.where(S, sw, 0.0)
        Gw = g * w[:, None]
        N, b = Gw.T @ Gw, Gw.T @ (r * w)
        it += 1
        if not np.all(np.linalg.eigvalsh(N) > 0):
            return False, X, it, None
        d = np.linalg.solve(N, b)
        x_last, X = X, X + d
        if np.linalg.norm(X[:3]) > PM.RUNAWAY:
            return False, X, it, None
        if np.linalg.norm(d[:3]) < PM.CONVERGED:
            last = dict(g=g, r=r, d=d, N=N, el=el, int2=sura2 + rest2, acc2=sure2 + rest2, vr=vr, has=has)
            return True, X, it, last
    return False, X, it, None


def mhss(last, S, X, n, acfg, kh, kv, trace=None):
    """Solution separation at fix X over the set S (header step 5-6) from explicit subset matrices."""
    idx = np.nonzero(S)[0]
    G, y = last["g"][idx], last["r"][idx]
    W = np.diag(1.0 / last["int2"][idx])
    Ci, Ca = np.diag(last["int2"][idx]), np.diag(last["acc2"][idx])
    E = enu(X)
    S0 = E @ (np.linalg.inv(G.T @ W @ G) @ G.T @ W)[:3]
    out = dict(idx=idx, dx=np.zeros((n, 3)), s=np.zeros((n, 3)), ss=np.zeros((n, 3)), b=np.zeros((n, 3)), pd=True)
    for kk in range(n):
        keep = np.arange(n) != kk
        Gk, Wk = G[keep], W[np.ix_(keep, keep)]
        Nk = Gk.T @ Wk @ Gk
        if not np.all(np.linalg.eigvalsh(Nk) > 0):
            out["pd"] = False
            return out
        Sk = np.zeros((3, n))
        Sk[:, keep] = E @ (np.linalg.inv(Nk) @ Gk.T @ Wk)[:3]
        dS = Sk - S0
        out["dx"][kk] = dS @ y
        out["s"][kk] = np.sqrt(np.diag(Sk @ Ci @ Sk.T))
        out["ss"][kk] = np.sqrt(np.diag(dS @ Ca @ dS.T))
        out["b"][kk] = np.abs(Sk).sum(1) * float(acfg["b_nom"])
    out["S0"] = S0
    out["b0"] = np.abs(S0).sum(1) * float(acfg["b_nom"])
    out["s0"] = np.sqrt(np.diag(S0 @ Ci @ S0.T))
    out["sacc_v"] = float(np.sqrt((S0 @ Ca @ S0.T)[2, 2]))
    kfa = np.array([kh[n - 5], kh[n - 5], kv[n - 5]])
    out["T"] = kfa[None, :] * out["ss"]
    ratio = np.abs(out["dx"]) / out["T"]
    out["key"] = ratio.max(1)
    out["pass"] = bool(np.all(np.abs(out["dx"]) <= out["T"]))
    if trace is not None:
        trace["test"].append(np.ravel(ratio))
        trace["argmax"].append(out["key"])
    return out


def araim(chans, epochs, cfg, acfg, kh, kv, trace=None):
    """-> (fix dict as pvt_model gives, residuals [F, C], record dict with the ARAIM_DTYPE field names, and per fix the
    last MHSS dict and the rhs of each protection level (for the tests)). trace: None, or a dict of lists "mask", "test"
    and "argmax" that receive the elevations / mask, |dx| / T and the exclusion keys (margin checks)."""
    inp = Inputs(chans, epochs, cfg)
    nf, nc = inp.nf, inp.nc
    mask_rad = float(acfg["mask_deg"]) * np.pi / 180.0
    names = ("x", "y", "z", "clock_m", "t_rx", "vx", "vy", "vz", "drift", "lat_deg", "lon_deg", "height", "pdop", "rms")
    fix = {k: np.full(nf, np.nan) for k in names}
    fix.update(sample=inp.s, status=np.zeros(nf, np.int32), nused=np.zeros(nf, np.int32), mask=np.zeros(nf, np.int64),
               iterations=np.zeros(nf, np.int32))
    rec = dict(verdict=np.full(nf, UNAVAILABLE, np.int32), excluded=np.zeros(nf, np.uint32),
               masked=np.zeros(nf, np.uint32), n=np.zeros(nf, np.int32))
    for k in ("test_ratio", "hpl", "vpl", "emt", "sigma_acc_v", "p_nm"):
        rec[k] = np.full(nf, np.nan)
    res = np.full((nf, nc), np.nan)
    extra = [None] * nf
    bits = 1 << np.arange(nc, dtype=np.int64)
    for f in range(nf):
        S = inp.use[f].copy()
        n = int(S.sum())
        status = PM.FIX_FEW if n < 4 else PM.FIX_NO_CONVERGENCE
        iters, X, last, ok = 0, np.zeros(4), None, False
        if n >= 4:
            ok, X, it, last = gauss_newton(inp, acfg, f, S, X)
            iters += it
            if ok:
                if trace is not None:
                    trace["mask"].append(last["el"][S] / mask_rad)
                low = S & (last["el"] < mask_rad)
                rec["masked"][f] = int((low * bits).sum())
                if low.any():
                    S &= ~low
                    n = int(S.sum())
                    if n < 4:
                        ok, status = False, PM.FIX_FEW
                    else:
                        ok, X, it, last = gauss_newton(inp, acfg, f, S, X)
                        iters += it
            if ok and n >= 5:
                o = mhss(last, S, X, n, acfg, kh, kv, trace)
                verdict = UNAVAILABLE
                if o["pd"]:
                    rec["test_ratio"][f], rec["emt"][f], rec["sigma_acc_v"][f] = o["key"].max(), o["T"][:, 2].max(), \
                        o["sacc_v"]
                    verdict = PASS if o["pass"] else ALERT
                    if not o["pass"] and int(acfg["max_exclude"]) == 1 and n >= 6:
                        j = int(o["idx"][int(np.argmax(o["key"]))])     # the first maximum: the lowest channel
                        rec["excluded"][f] = 1 << j
                        S[j] = False
                        n -= 1
                        ok, X, it, last = gauss_newton(inp, acfg, f, S, X)
                        iters += it
                        verdict = ALERT
                        o = None
                        if ok:
                            o = mhss(last, S, X, n, acfg, kh, kv, trace)
                            if not o["pd"]:
                                verdict, o = UNAVAILABLE, None
                            else:
                                rec["test_ratio"][f], rec["emt"][f], rec["sigma_acc_v"][f] = \
                                    o["key"].max(), o["T"][:, 2].max(), o["sacc_v"]
                                verdict = EXCLUDED if o["pass"] else ALERT
                    if o is not None:
                        ps, pv, ph = float(acfg["p_sat"]), float(acfg["p_hmi_vert"]), float(acfg["p_hmi_horz"])
                        rec["p_nm"][f] = p_nm(ps, n)
                        if not rec["p_nm"][f] < pv + ph:
                            verdict = UNAVAILABLE
                        else:
                            sc = 1.0 - rec["p_nm"][f] / (pv + ph)
                            rhs = (pv * sc, ph / 2.0 * sc, ph / 2.0 * sc)
                            pl = [protection_level(r, o["b0"][q], o["s0"][q], o["T"][:, q], o["b"][:, q],
                                                   o["s"][:, q], ps) for q, r in zip((2, 0, 1), rhs)]
                            rec["vpl"][f], rec["hpl"][f] = pl[0], np.hypot(pl[1], pl[2])
                            extra[f] = (o, rhs, pl)
                rec["verdict"][f] = verdict
        rec["n"][f] = n
        fix["nused"][f], fix["mask"][f], fix["iterations"][f] = n, int((S * bits).sum()), iters
        if ok:
            status = PM.FIX_OK
            g, d, w2 = last["g"], last["d"], np.where(S, 1.0 / last["int2"], 0.0)
            e = last["r"] - g @ d
            res[f] = np.where(last["has"], e, np.nan)
            yv = inp.rate[f] + PM.C * inp.ddtsv[f] + np.einsum("ci,ci->c", g[:, :3], last["vr"])
            vel = np.linalg.solve(last["N"], (g * (w2 * yv)[:, None]).sum(0))
            Q = np.linalg.inv(last["N"])
            lat, lon, h = PM.ecef_llh(X[:3])
            trx = inp.nom_ms[f] * 1e-3 + (inp.m[f] / 3e6 - X[3] / PM.C)
            trx = trx + 604800.0 if trx < 0.0 else (trx - 604800.0 if trx >= 604800.0 else trx)
            for k, v in (("x", X[0]), ("y", X[1]), ("z", X[2]), ("clock_m", X[3]), ("t_rx", trx), ("vx", vel[0]),
                         ("vy", vel[1]), ("vz", vel[2]), ("drift", vel[3]), ("lat_deg", np.degrees(lat)),
                         ("lon_deg", np.degrees(lon)), ("height", h), ("pdop", np.sqrt(Q[0, 0] + Q[1, 1] + Q[2, 2])),
                         ("rms", np.sqrt(np.sum(e[S] ** 2) / n))):
                fix[k][f] = v
        fix["status"][f] = status
    return fix, res, rec, extra
