"""Numpy statement of vector tracking (include/gpsb200.h: gpsb200_vtrack; DESIGN §10.1): the tests' reference.

The periods are track_model's correlator with the NCO steps held over an update interval; the satellite is pvt_model's.
The filter is restated here in FP64 numpy. numpy's transcendental functions differ from CUDA's by ulps, so the
filter agrees with the kernel to far below a micrometre, but a command that rounds a double can differ by one unit:
`run` can therefore replay the kernel's commands (u, w per channel and update) to compare the correlators bit for bit."""
import numpy as np

import acq_model as A
import pvt_model as PM
import track_model as T

C = PM.C
FS = 3e6
LAMBDA_CHIP = C / 1.023e6
LAMBDA = C / 1575.42e6
NOISE_SCALE = 62500.0
W_MAX_HZ = 10000.0
M = T.M

CONFIG_DTYPE = np.dtype([("periods", "<i4"), ("reserved", "<i4"), ("sigma_code_m", "<f8"), ("sigma_rate_mps", "<f8"),
                         ("q_min", "<f8"), ("accel_psd", "<f8"), ("bias_psd", "<f8"), ("drift_psd", "<f8"),
                         ("sigma_pos", "<f8"), ("sigma_vel", "<f8"), ("sigma_bias", "<f8"), ("sigma_drift", "<f8")])
CHAN_STATE_DTYPE = np.dtype([("nco", T.STATE_DTYPE), ("start", "<i8"), ("e", "<i8"), ("l", "<i8"), ("p", "<i8"),
                             ("s", "<i8"), ("dot", "<i8"), ("cross", "<i8"), ("k", "<i4"), ("used", "<i4")])
STATE_DTYPE = np.dtype([("s0", "<i8"), ("t0", "<f8"), ("nchan", "<i4"), ("seeded", "<i4"), ("updates", "<i4"),
                        ("reserved", "<i4"), ("t_f", "<i8"), ("x", "<f8", 8), ("P", "<f8", (8, 8)),
                        ("ch", CHAN_STATE_DTYPE, 32)])
CHAN_DTYPE = np.dtype([("sample", "<i8"), ("e", "<i8"), ("l", "<i8"), ("p", "<i8"), ("s", "<i8"), ("dot", "<i8"),
                       ("cross", "<i8"), ("prn", "<i4"), ("used", "<i4"), ("code_step", "<u4"), ("carr_step", "<i4"),
                       ("q", "<f8"), ("code_res_m", "<f8"), ("rate_res_mps", "<f8"), ("sigma_code_m", "<f8"),
                       ("sigma_rate_mps", "<f8")])
assert (CONFIG_DTYPE.itemsize, CHAN_STATE_DTYPE.itemsize, STATE_DTYPE.itemsize, CHAN_DTYPE.itemsize) == (88, 128, 4712, 112)


def config(periods=20, sigma_code_m=50.0, sigma_rate_mps=10.0, q_min=1.2, accel_psd=1.0, bias_psd=0.1, drift_psd=0.01,
           sigma_pos=100.0, sigma_vel=1.0, sigma_bias=10.0, sigma_drift=1.0):
    c = np.zeros(1, CONFIG_DTYPE)[0]
    for k, v in locals().items():
        if k != "c":
            c[k] = v
    return c


def seed(cfg, x8, t_rx, s0, prns):
    st = np.zeros(1, STATE_DTYPE)[0]
    st["s0"], st["nchan"], st["t_f"] = s0, len(prns), s0
    st["x"] = x8
    st["t0"] = t_rx + x8[6] / C
    sd = [cfg["sigma_pos"]] * 3 + [cfg["sigma_vel"]] * 3 + [cfg["sigma_bias"], cfg["sigma_drift"]]
    st["P"] = np.diag(np.square(sd))
    for c, p in enumerate(prns):
        st["ch"][c]["nco"]["prn"] = p
    return st


def frac(x):
    return x - np.floor(x)


def predict(st, X, t_f, eph, s):
    """Header 'predict' for one channel at sample s from X at filter sample t_f. -> (phi chips, e[3], rr m/s)."""
    dt = (s - t_f) / FS
    r = X[0:3] + X[3:6] * dt
    b = X[6] + X[7] * dt
    d = s - int(st["s0"])
    q = d // 3000
    m = d - 3000 * q
    t0 = float(st["t0"])
    t = t0 + q / 1000.0 + m / FS - b / C
    tau = 0.075
    for _ in range(3):
        p, v, dts, ddt = PM.satellite(eph, np.float64(t - tau))
        sth, cth = np.sin(PM.OMEGA_E * tau), np.cos(PM.OMEGA_E * tau)
        l = np.array([p[0] * cth + p[1] * sth - r[0], p[1] * cth - p[0] * sth - r[1], p[2] - r[2]])
        vr = np.array([v[0] * cth + v[1] * sth, v[1] * cth - v[0] * sth, v[2]])
        tau = np.sqrt(l[0] * l[0] + l[1] * l[1] + l[2] * l[2]) / C
    F0 = frac(1000.0 * t0)
    phi = 1023.0 * frac(F0 + m / 3000.0 + 1000.0 * (float(dts) - tau - b / C))
    rn = tau * C
    e = l / rn
    rr = e[0] * (vr[0] - X[3]) + e[1] * (vr[1] - X[4]) + e[2] * (vr[2] - X[5]) - C * float(ddt) + X[7]
    return phi, e, rr


def command(phi, rr, phi_nco, N):
    """-> (u, w) from the predicted code phase phi (chips), range rate rr and the NCO's code phase phi_nco."""
    f = min(max(-rr / LAMBDA, -W_MAX_HZ), W_MAX_HZ)
    w = llround(f * 2.0 ** 32 / FS)
    err = phi * 2.0 ** 32 - float(phi_nco)
    if err >= M / 2:
        err -= M
    elif err < -M / 2:
        err += M
    e = llround(err)
    u = int(np.clip(T.CODE_STEP_NOM + int(T.tdiv(w, 1540)) + int(T.tdiv(e, 3000 * N)), T.CODE_STEP_MIN, T.CODE_STEP_MAX))
    return u, w


def llround(x):
    """C's llround: half away from zero."""
    return int(np.sign(x) * np.floor(abs(x) + 0.5))


def first(st, eph, N):
    """Header 'first': every channel started at s0 from X."""
    s0 = int(st["s0"])
    for c in range(int(st["nchan"])):
        phi, e, rr = predict(st, st["x"], s0, eph[c], s0)
        f = min(max(-rr / LAMBDA, -W_MAX_HZ), W_MAX_HZ)
        w = llround(f * 2.0 ** 32 / FS)
        u = int(T.code_step_of(np.int64(w)))
        phi0 = llround(phi * 2.0 ** 32) % M
        n = st["ch"][c]["nco"]
        if phi0 == 0:
            n["sample"], n["code_phase"] = s0, 0
        else:
            L = (M - phi0 + u - 1) // u
            n["sample"], n["code_phase"] = s0 + L, phi0 + L * u - M
        n["carr_step"], n["code_step"], n["carr_phase"] = w, u, 0
        st["ch"][c]["start"] = n["sample"]
    st["t_f"], st["seeded"] = s0, 1


def time_update(X, P, dt, cfg):
    F = np.eye(8)
    for i in range(3):
        F[i, 3 + i] = dt
    F[6, 7] = dt
    qa, qb, qd = float(cfg["accel_psd"]), float(cfg["bias_psd"]), float(cfg["drift_psd"])
    Q = np.zeros((8, 8))
    for i in range(3):
        Q[i, i], Q[i, 3 + i], Q[3 + i, i], Q[3 + i, 3 + i] = qa * dt ** 3 / 3, qa * dt ** 2 / 2, qa * dt ** 2 / 2, qa * dt
    Q[6, 6], Q[6, 7], Q[7, 6], Q[7, 7] = qb * dt + qd * dt ** 3 / 3, qd * dt ** 2 / 2, qd * dt ** 2 / 2, qd * dt
    return F @ X, F @ P @ F.T + Q


def update(st, eph, cfg, trace=None):
    """Header 'update' on the sums in st (every channel at k = N). -> (fix record dict, CHAN_DTYPE[nchan]); st updated
    with the new X, P, t_f and commands."""
    N = int(cfg["periods"])
    nch = int(st["nchan"])
    ch = st["ch"][:nch]
    ends = ch["nco"]["sample"].astype(np.int64)
    t_new = int(ends.max())
    X, P = time_update(st["x"].astype(np.float64), st["P"].astype(np.float64), (t_new - int(st["t_f"])) / FS, cfg)
    Xp = X.copy()
    out = np.zeros(nch, CHAN_DTYPE)
    rows = []
    for c in range(nch):
        cs = ch[c]
        n = cs["nco"]
        phi, e, rr = predict(st, Xp, t_new, eph[c], int(n["sample"]))
        S = int(cs["s"])
        q = float(cs["p"]) / (NOISE_SCALE * S) if S else 0.0
        used = q >= float(cfg["q_min"])
        D = int(T.dll(np.int64(cs["e"]), np.int64(cs["l"])))
        u, w = int(n["code_step"]), int(n["carr_step"])
        du = u - int(T.code_step_of(np.int64(w)))
        nsamp = int(n["sample"]) - int(cs["start"])
        r = float(n["code_phase"]) / 2.0 ** 32 + D / 65536.0 - du * nsamp / 2.0 ** 33 - phi
        r = (r + 511.5) % 1023.0 - 511.5
        yc = -LAMBDA_CHIP * r
        a = int(T.angle(np.int64(cs["dot"]), np.int64(cs["cross"])))
        fm = w * FS / 2.0 ** 32 + a * 1000.0 / 2.0 ** 32
        yr = -LAMBDA * fm - rr
        o = out[c]
        for f in ("e", "l", "p", "s", "dot", "cross"):
            o[f] = cs[f]
        o["sample"], o["prn"], o["used"], o["q"], o["code_res_m"], o["rate_res_mps"] = n["sample"], n["prn"], used, q, yc, yr
        if used:
            vc = float(cfg["sigma_code_m"]) ** 2 / ((q - 1.0) * N)
            vr = float(cfg["sigma_rate_mps"]) ** 2 / ((q - 1.0) * N)
            o["sigma_code_m"], o["sigma_rate_mps"] = np.sqrt(vc), np.sqrt(vr)
            hc = np.array([-e[0], -e[1], -e[2], 0, 0, 0, 1.0, 0])
            hr = np.array([0, 0, 0, -e[0], -e[1], -e[2], 0, 1.0])
            rows += [(c, hc, yc, vc), (c, hr, yr, vr)]
        else:
            o["sigma_code_m"] = o["sigma_rate_mps"] = np.inf
    for c, h, y, var in rows:
        yy = y - h @ (X - Xp)
        g = P @ h
        s = h @ g + var
        K = g / s
        X = X + K * yy
        P = P - np.outer(K, g)
    used_c = [(c, h, y) for c, h, y, _ in rows[0::2]]
    res = np.array([y - h @ (X - Xp) for _, h, y in used_c])
    fix = dict(sample=t_new, nused=len(used_c), mask=sum(1 << c for c, _, _ in used_c), x=X.copy(),
               rms=float(np.sqrt(np.mean(res ** 2))) if res.size else np.nan,
               t_rx=float(st["t0"]) + (t_new - int(st["s0"])) / FS - X[6] / C, pdop=np.nan)
    fix["status"] = 0 if len(used_c) >= 4 else 1
    if len(used_c) >= 4:
        G = np.zeros((4, 4))
        for _, h, _ in used_c:
            g4 = np.array([h[0], h[1], h[2], 1.0])
            G += np.outer(g4, g4)
        fix["pdop"] = float(np.sqrt(np.trace(np.linalg.inv(G)[:3, :3])))
    if trace is not None:
        trace.append(dict(X_prior=Xp, X=X.copy(), P=P.copy()))
    st["x"], st["P"], st["t_f"] = X, P, t_new
    for c in range(nch):
        cs = ch[c]
        n = cs["nco"]
        phi, e, rr = predict(st, X, t_new, eph[c], int(n["sample"]))
        u, w = command(phi, rr, int(n["code_phase"]), N)
        out[c]["code_step"], out[c]["carr_step"] = u, w
        n["code_step"], n["carr_step"] = u, w
        cs["used"] = int(out[c]["used"])
        cs["start"] = n["sample"]
        for f in ("e", "l", "p", "s", "dot", "cross", "k"):
            cs[f] = 0
    st["ch"][:nch] = ch
    st["updates"] += 1
    return fix, out


def periods(I, Q, base, st, N, codes, cos, sin, epochs):
    """Run every channel's periods until it has N in the interval or its next period leaves the buffer."""
    nch = int(st["nchan"])
    ch = st["ch"][:nch]
    n = ch["nco"]
    end = base + I.size
    m = np.arange(T.MAX_PERIOD, dtype=np.int64)
    rows = np.arange(nch)
    while True:
        L = (M - n["code_phase"].astype(np.int64) + n["code_step"].astype(np.int64) - 1) // n["code_step"].astype(np.int64)
        act = (ch["k"] < N) & (n["sample"] + L <= end)
        if not act.any():
            break
        a = np.nonzero(act)[0]
        La = L[a]
        valid = m[None, :] < La[:, None]
        idx = np.minimum((n["sample"][a] - base)[:, None] + m[None, :], I.size - 1)
        Ii, Qi = I[idx], Q[idx]
        w = n["carr_step"][a].astype(np.int64) & 0xFFFFFFFF
        th = (n["carr_phase"][a].astype(np.int64)[:, None] + m[None, :] * w[:, None]) & 0xFFFFFFFF
        t = th >> 23
        cc, ss = cos[t], sin[t]
        dI = np.where(valid, Ii * cc + Qi * ss, 0)
        dQ = np.where(valid, Qi * cc - Ii * ss, 0)
        u = n["code_step"][a].astype(np.int64)
        p = n["code_phase"][a].astype(np.int64)[:, None] + m[None, :] * u[:, None]
        e = p + T.H
        e = np.where(e >= M, e - M, e)
        l_ = np.where(p >= T.H, p - T.H, p + M - T.H)
        ca = codes[a]
        r = rows[:a.size][:, None]
        ce, cp, cl = (ca[r, np.minimum(x >> 32, 1023)] for x in (e, p, l_))
        c6 = [(ce * dI).sum(1), (ce * dQ).sum(1), (cp * dI).sum(1), (cp * dQ).sum(1), (cl * dI).sum(1), (cl * dQ).sum(1)]
        S = np.where(valid, Ii * Ii + Qi * Qi, 0).sum(1)
        for j, c in enumerate(a):
            cs = st["ch"][c]
            nc = cs["nco"]
            s_abs = int(nc["sample"])
            Lc = int(La[j])
            nc["sample"] = s_abs + Lc
            nc["carr_phase"] = (int(nc["carr_phase"]) + Lc * int(w[j])) & 0xFFFFFFFF
            nc["code_phase"] = int(nc["code_phase"]) + Lc * int(u[j]) - M
            pi, pq = int(c6[2][j]), int(c6[3][j])
            cs["e"] += int(c6[0][j]) ** 2 + int(c6[1][j]) ** 2
            cs["l"] += int(c6[4][j]) ** 2 + int(c6[5][j]) ** 2
            cs["p"] += pi * pi + pq * pq
            cs["s"] += int(S[j])
            if cs["k"] >= 1:
                i0, q0 = int(nc["prev_i"]), int(nc["prev_q"])
                cross, dot = i0 * pq - q0 * pi, i0 * pi + q0 * pq
                if dot < 0:
                    cross, dot = -cross, -dot
                cs["cross"] += cross
                cs["dot"] += dot
            nc["prev_i"], nc["prev_q"] = pi, pq
            nc["epochs"] += 1
            cs["k"] += 1
            if epochs is not None:
                epochs[c].append((s_abs, c6[0][j], c6[1][j], pi, pq, c6[4][j], c6[5][j], nc["carr_phase"],
                                  nc["carr_step"], int(nc["code_phase"]) & 0xFFFFFFFF, nc["code_step"], cs["used"], 0))
        n = st["ch"][:nch]["nco"]
        ch = st["ch"][:nch]


def run(iq, sample_size, base, state, chans, cfg, max_updates, replay=None, trace=None):
    """The contract over the buffer from `state` (STATE_DTYPE), chans: PVT_CHAN_DTYPE[nchan] (eph read).
    replay: CHAN_DTYPE[updates][nchan] of a kernel run whose (code_step, carr_step) replace the model's commands in the
    NCOs; the returned records keep the model's own commands, so that they can be compared with the kernel's.
    -> (fixes list of dicts, CHAN_DTYPE[updates][nchan], epochs list per channel (EPOCH_DTYPE), state after)."""
    st = np.array(state, STATE_DTYPE).reshape(())[()].copy()
    st = np.array([st], STATE_DTYPE)[0]
    I, Q = A.samples(iq, sample_size)
    cos, sin = A.tables()
    nch = int(st["nchan"])
    eph = [chans[c]["eph"] for c in range(nch)]
    N = int(cfg["periods"])
    codes = np.stack([T.code_pm(int(p)) for p in st["ch"]["nco"]["prn"][:nch]])
    if not st["seeded"]:
        first(st, eph, N)
    eps = [[] for _ in range(nch)]
    fixes, outs = [], []
    while len(fixes) < max_updates:
        periods(I, Q, base, st, N, codes, cos, sin, eps)
        if not (st["ch"]["k"][:nch] == N).all():
            break
        fix, out = update(st, eph, cfg, trace)
        if replay is not None and len(fixes) < len(replay):
            rp = replay[len(fixes)]
            for c in range(nch):
                st["ch"][c]["nco"]["code_step"], st["ch"][c]["nco"]["carr_step"] = rp[c]["code_step"], rp[c]["carr_step"]
        fixes.append(fix)
        outs.append(out)
    E = [np.array(e, T.EPOCH_DTYPE) if e else np.zeros(0, T.EPOCH_DTYPE) for e in eps]
    return fixes, (np.array(outs, CHAN_DTYPE) if outs else np.zeros((0, nch), CHAN_DTYPE)), E, st
