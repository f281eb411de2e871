"""Vector tracking's numpy model (tests/vtrack_model.py) on the CPU oracle's streams against the scenario's truth.

The seed is the truth moved by 100 m on every axis, 1 m/s on every velocity axis and 30 ns of clock. On the model, over
the first 0.5 s of sky12_static_35s: every channel's code error is below 0.55 chip at the start (the seed's 173 m of
range) and below 0.01 chip at 0.5 s; the fixes settle within 8 m of the truth (the clock takes the common part of the
ionosphere, which the filter does not model). The bounds below are the issue's: 0.125 chip and test_coarse's TRACKED
position bound (30 m), both after the first second."""
import numpy as np
import pytest

import pvt_model as PM
import scenario
import track_truth as TT
import vtrack_model as V
from scenario import gps
from test_acquire import golden_rows
from test_coarse import TRACKED, WEEK
from test_pvt import rinex
from test_scenario import LOC
from test_track import START_SOW

CERR_MAX = 0.125          # chips
SETTLE = 1.0              # s after the seed
GAP_BACK = 10             # intervals after a gap by which every channel is back within CERR_MAX
OFFSET = (100.0, 1.0, 30e-9)
WEAK_PRNS = (1, 2, 3, 4, 5, 6, 7, 8)
WEAK_GAIN = 0.12          # DESIGN §10.1's measurement: the largest g of the ladder where the scalar loops lose half
SCALAR_LOCK = 400         # epochs: a scalar channel is held when locked for good by then with code error <= 0.5 chip


def stream(name, nblk, gap=None, weak=None):
    """nblk blocks of a fixture re-synthesised by the CPU oracle; gap: a sample range set to zeros; weak: the gain
    factor of WEAK_PRNS in every block."""
    g = scenario.load_golden(name)
    ch = golden_rows(g, range(nblk))
    if weak is not None:
        for b in range(nblk):
            for c in range(ch.shape[1]):
                if int(ch[b, c]["prn"]) in WEAK_PRNS:
                    ch[b, c]["gain"] *= weak
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], int(g["sample_size"]))
    if gap is not None:
        iq[2 * gap[0]:2 * gap[1]] = 0
    return g, ch, iq


def chans_of(tmp_path, nsat, prns):
    nav, _, _ = rinex(tmp_path, nsat)
    eph = gps.rinex_ephemeris(nav, WEEK, START_SOW)
    ch = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    for c, p in enumerate(prns):
        ch[c]["eph"], ch[c]["prn"] = eph[p - 1], p
    return ch


def seed_x(x0, v0=np.zeros(3)):
    dp, dv, db = OFFSET
    return np.concatenate([x0 + dp, v0 + dv, [db * V.C, 0.0]])


def code_errors(ch, prn, e):
    """Code error (chips) at the start of every period but the first, from the epochs of one channel."""
    phis = e["code_phase"][:-1].astype(np.int64)
    return np.array([TT.code_error_chips(ch, prn, s, p) for s, p in zip(e["sample"][1:], phis)]), e["sample"][1:]


def check_truth(ch, prns, eps, fixes_xyz, fix_samples, x_true, pos_max=TRACKED["pos"], skip_samples=None):
    settle = int(SETTLE * TT.FS)
    for p, e in zip(prns, eps):
        cerr, smp = code_errors(ch, p, e)
        keep = smp >= settle if skip_samples is None else (smp >= settle) & ~skip_samples(smp)
        assert np.abs(cerr[keep]).max() <= CERR_MAX, (p, np.abs(cerr[keep]).max())
    late = fix_samples >= settle
    err = np.linalg.norm(fixes_xyz[late] - x_true(fix_samples[late]), axis=1)
    assert err.max() <= pos_max, err.max()
    return err


@pytest.fixture(scope="module")
def clean5(tmp_path_factory):
    g, ch, iq = stream("sky12_static_35s_i8", 50)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    return g, ch, iq, prns, chans_of(tmp_path_factory.mktemp("nav"), 12, prns)


def test_model_tracks_the_clean_stream(clean5):
    g, ch, iq, prns, chans = clean5
    x0 = PM.llh_ecef(*LOC)
    cfg = V.config()
    st = V.seed(cfg, seed_x(x0), START_SOW, 0, prns)
    fixes, outs, eps, _ = V.run(iq, 1, 0, st, chans, cfg, 10000)
    assert len(fixes) >= 240
    assert all(f["status"] == 0 and f["nused"] == 12 for f in fixes)
    xyz = np.array([f["x"][:3] for f in fixes])
    smp = np.array([f["sample"] for f in fixes])
    check_truth(ch, prns, eps, xyz, smp, lambda s: np.broadcast_to(x0, (s.size, 3)))
    vel = np.array([f["x"][3:6] for f in fixes])[smp >= SETTLE * TT.FS]
    assert np.abs(vel).max() <= TRACKED["vel"]


def scalar_lost(ch, prns, iq, ss):
    """The PRNs the scalar loops (track_model) lose from the truth's cell (100 Hz bins): not locked for good by epoch
    SCALAR_LOCK, or a code error above 0.5 chip after it."""
    import acq_model as A
    import track_model as T
    sts = []
    for c, p in enumerate(prns):
        f, tau = A.truth(ch[0][c], 0)
        sts.append(T.start(p, round(f / 100.0) * 100.0, int(np.rint(tau)) % A.CODE))
    eps, _ = T.track(iq, ss, 0, np.array(sts))
    lost = []
    for p, e in zip(prns, eps):
        un = np.nonzero(e["lock"] == 0)[0]
        pull = int(un[-1]) + 1 if un.size else 0
        cerr, _ = TT.epoch_errors(ch, p, e)
        if pull > SCALAR_LOCK or np.abs(cerr[SCALAR_LOCK:]).max() > 0.5:
            lost.append(p)
    return lost


def check_weak(ch, prns, fixes_xyz, fix_samples, masks, eps, x0):
    """Every weak channel within CERR_MAX and in the mask of every fix after SETTLE; the fixes within the bound."""
    check_truth(ch, prns, eps, fixes_xyz, fix_samples, lambda s: np.broadcast_to(x0, (s.size, 3)))
    weak_bits = sum(1 << c for c, p in enumerate(prns) if p in WEAK_PRNS)
    late = fix_samples >= SETTLE * TT.FS
    assert all((int(m) & weak_bits) == weak_bits for m in np.asarray(masks)[late])


def test_model_holds_the_weakened_stream(tmp_path):
    """PRNs 1-8 at a gain of WEAK_GAIN in every block, 5 s: the scalar loops lose at least half of them; the vector
    model holds all eight within CERR_MAX, uses them in every fix after SETTLE, and fixes within 30 m."""
    g, ch, iq = stream("sky12_static_35s_i8", 50, weak=WEAK_GAIN)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    lost = scalar_lost(ch, prns, iq, 1)
    assert len(set(lost) & set(WEAK_PRNS)) >= 4, lost
    chans = chans_of(tmp_path, 12, prns)
    x0 = PM.llh_ecef(*LOC)
    cfg = V.config()
    fixes, outs, eps, _ = V.run(iq, 1, 0, V.seed(cfg, seed_x(x0), START_SOW, 0, prns), chans, cfg, 10000)
    check_weak(ch, prns, np.array([f["x"][:3] for f in fixes]), np.array([f["sample"] for f in fixes]),
               [f["mask"] for f in fixes], eps, x0)


def test_model_coasts_through_a_gap(clean5, tmp_path):
    """200 ms of zeros from 2 s on: every sum in the gap is 0, so no channel is used and the filter coasts; after it
    every channel is back within CERR_MAX within GAP_BACK intervals."""
    g, ch, _, prns, chans = clean5
    gap = (6000000, 6600000)
    _, _, iq = stream("sky12_static_35s_i8", 30, gap=gap)
    x0 = PM.llh_ecef(*LOC)
    cfg = V.config()
    st = V.seed(cfg, seed_x(x0), START_SOW, 0, prns)
    fixes, outs, eps, _ = V.run(iq, 1, 0, st, chans, cfg, 10000)
    inside = (outs["sample"][:, 0] > gap[0] + 3001 * 20) & (outs["sample"][:, 0] <= gap[1])
    assert inside.sum() >= 8
    assert (outs[inside]["p"] == 0).all() and (outs[inside]["s"] == 0).all() and (outs[inside]["used"] == 0).all()
    back = gap[1] + GAP_BACK * 20 * 3001
    check_truth(ch, prns, eps, np.array([f["x"][:3] for f in fixes]), np.array([f["sample"] for f in fixes]),
                lambda s: np.broadcast_to(x0, (s.size, 3)),
                skip_samples=lambda s: (s >= gap[0]) & (s < back))


def batch_update(Xp, P, rows):
    """The measurement update of a whole interval in matrix form: S = H P H^T + R, K = P H^T S^-1, X = Xp + K y."""
    if not rows:
        return Xp, P
    H = np.array([h for h, _, _ in rows])
    y = np.array([y for _, y, _ in rows])
    R = np.diag([v for _, _, v in rows])
    S = H @ P @ H.T + R
    K = P @ H.T @ np.linalg.inv(S)
    return Xp + K @ y, P - K @ H @ P


def c_div(a, b):
    """C's integer division: truncation toward zero."""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def restated_predict(st, X, t_f, eph, s):
    """The header's 'predict', written out again: (code phase in chips, unit vector, range rate) at sample s."""
    dt = (s - t_f) / V.FS
    r, v_rx = X[:3] + X[3:6] * dt, X[3:6]
    b = X[6] + X[7] * dt
    q, m = divmod(s - int(st["s0"]), 3000)
    t = float(st["t0"]) + q / 1000.0 + m / V.FS - b / V.C
    tau = 0.075
    for _ in range(3):
        p, v, dts, ddt = PM.satellite(eph, np.float64(t - tau))
        a = PM.OMEGA_E * tau
        R = np.array([[np.cos(a), np.sin(a), 0.0], [-np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
        los, vsat = R @ p - r, R @ v
        tau = np.linalg.norm(los) / V.C
    ms = (1000.0 * float(st["t0"])) % 1.0 + m / 3000.0 + 1000.0 * (float(dts) - tau - b / V.C)
    e = los / np.linalg.norm(los)
    return 1023.0 * (ms % 1.0), e, float(e @ (vsat - v_rx)) - V.C * float(ddt) + X[7]


def restated_rows(before, after, out, chans, cfg, Xp, t_new):
    """The header's measurement rows of an interval, recomputed from its sums (out) and the NCO states before and
    after it, at the prior X. -> list of (row, innovation, variance) of the used channels, and every channel's
    (y_c, y_r)."""
    N = int(cfg["periods"])
    rows, ys = [], []
    for c, o in enumerate(out):
        nb, na = before["ch"][c], after["ch"][c]["nco"]
        u, w = int(nb["nco"]["code_step"]), int(nb["nco"]["carr_step"])
        E, L = int(o["e"]), int(o["l"])
        sh = max(0, (E + L).bit_length() - 40)
        E, L = E >> sh, L >> sh
        D = 0 if E + L == 0 else c_div((E - L) * 16384, E + L)
        nominal = min(max(V.T.CODE_STEP_NOM + c_div(w, 1540), V.T.CODE_STEP_MIN), V.T.CODE_STEP_MAX)
        n = int(o["sample"]) - int(nb["start"])
        phi, e, rr = restated_predict(before, Xp, t_new, chans[c]["eph"], int(o["sample"]))
        r = int(na["code_phase"]) / 2.0 ** 32 + D / 65536.0 - (u - nominal) * n / 2.0 ** 33 - phi
        r = (r + 511.5) % 1023.0 - 511.5
        yc = -V.LAMBDA_CHIP * r
        a = int(V.T.angle(np.int64(o["dot"]), np.int64(o["cross"])))
        yr = -V.LAMBDA * (w * V.FS / 2.0 ** 32 + a * 1000.0 / 2.0 ** 32) - rr
        ys.append((yc, yr))
        if not o["used"]:
            continue
        vc = float(cfg["sigma_code_m"]) ** 2 / ((o["q"] - 1.0) * N)
        vr = float(cfg["sigma_rate_mps"]) ** 2 / ((o["q"] - 1.0) * N)
        rows.append((np.concatenate([-e, np.zeros(3), [1.0, 0.0]]), yc, vc))
        rows.append((np.concatenate([np.zeros(3), -e, [0.0, 1.0]]), yr, vr))
    return rows, ys


def test_each_update_against_its_restatement(clean5):
    """Every update of 1 s of the clean stream, recomputed from the previous state and the interval's sums by a
    restatement of the header's equations: the innovations from the sums and NCO states (dll, the correction term
    du n / 2^33, the wrap, angle() to f_m, the range rate), and the update in matrix form (batch gain), within 1e-6 m
    (and 1e-6 m/s, 1e-9 s x C of clock)."""
    g, ch, iq, prns, chans = clean5
    x0 = PM.llh_ecef(*LOC)
    cfg = V.config()
    st = V.seed(cfg, seed_x(x0), START_SOW, 0, prns)
    V.first(st, [chans[c]["eph"] for c in range(len(prns))], int(cfg["periods"]))
    trace = []
    n = 0
    for _ in range(50):
        before = np.array([st], V.STATE_DTYPE)[0]
        fixes, outs, _, st = V.run(iq, 1, 0, st, chans, cfg, 1, trace=trace)
        assert len(fixes) == 1
        t_new = int(fixes[0]["sample"])
        Xp, Pp = V.time_update(before["x"].astype(np.float64), before["P"].astype(np.float64),
                               (t_new - int(before["t_f"])) / V.FS, cfg)
        assert np.allclose(Xp, trace[-1]["X_prior"], rtol=0, atol=1e-9)
        rows, ys = restated_rows(before, st, outs[0], chans, cfg, Xp, t_new)
        assert len(rows) == 24
        for (yc, yr), o in zip(ys, outs[0]):
            assert abs(yc - o["code_res_m"]) <= 1e-6 and abs(yr - o["rate_res_mps"]) <= 1e-6, (yc, yr, o)
        X, P = batch_update(Xp, Pp, rows)
        assert np.abs(X[:6] - st["x"][:6]).max() <= 1e-6, X - st["x"]
        assert np.abs(X[6:] - st["x"][6:]).max() <= 1e-9 * V.C
        n += 1
    assert n == 50
