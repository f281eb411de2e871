"""Vector tracking at the edges of its contract, on the model (tests/vtrack_model.py): the constructions that
test_vtrack_edges_gpu runs on the kernel, each shown here to reach its edge.

- 50-digit references of the fix record's t_rx and geodetic coordinates (mpmath), and the model's against them.
- Open loop on zeros (S = 0, so q = 0 and no channel is used): a seed a few km/s off drives the predicted Doppler past
  +-10 kHz (w = +-14 316 558); a filter position moved 150 km away from the started channels drives u to
  CODE_STEP_MIN and CODE_STEP_MAX, the code error through the +M/2 wrap and the code residual through the -511.5-chip
  wrap.
- Seeds whose channel 0 starts at llround(phi 2^32) mod M = 0, 1 and M - 1 (within 0.1 unit on the model).
- Full-scale int8 streams planted on the open-loop NCO trajectory at N = 100: P and |cross| near their bounds.
- The `-s now` week-roll scenario seeded 3 s before 604 800 s: the model's predicted code phases stay on the
  scenario's on both sides of the roll (t runs past 604 800 s without a fold).
- A repeated PRN is refused by the seed."""

import mpmath
import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import scenario
import track_model as T
import track_truth as TT
import vtrack_model as V
from scenario import gps
from test_acquire import golden_rows
from test_scenario import LOC
from test_track import START_SOW
from test_vtrack import chans_of, seed_x

W_CLAMP = 14316558                     # llround(10 kHz 2^32 / FS)
FULL = 1.85e16                         # the header's bound of one period's squared prompt (and early, late)
JUMP_M = 150e3                         # the filter's position moved off the started channels (m)
SPEED_MPS = 4000.0                     # the seed's velocity error (m/s)
WRAP_TARGETS = (0, 1, V.M - 1)         # llround(phi 2^32) mod M of channel 0 at the seed
WRAP_MARGIN = 0.1                      # units of 2^-32 chip: the model's phi 2^32 this close to the target


def sky12_chans(tmp_path):
    g = scenario.load_golden("sky12_static_35s_i8")
    prns = [int(p) for p in golden_rows(g, range(1))[0]["prn"] if p > 0]
    return prns, chans_of(tmp_path, 12, prns)


@pytest.fixture(scope="module")
def sky12(tmp_path_factory):
    return sky12_chans(tmp_path_factory.mktemp("nav12"))


# ---- 50-digit references ---------------------------------------------------------------------------------------------
def t_rx_exact(st, fix):
    """t0 + (t_f - s0) / FS - b / C of a fix record at 50 digits, from the record's own sample and clock."""
    with mpmath.workdps(50):
        t = (mpmath.mpf(float(st["t0"])) + mpmath.mpf(int(fix["sample"]) - int(st["s0"])) / mpmath.mpf(3000000)
             - mpmath.mpf(float(fix["clock_m"])) / mpmath.mpf(V.C))
        return float(t)


def geodetic_exact(x):
    """WGS-84 latitude, longitude (degrees) and height of an ECEF point, iterated at 50 digits until it converges."""
    with mpmath.workdps(50):
        a, e2 = mpmath.mpf(PM.WGS_A), mpmath.mpf(PM.WGS_E) ** 2
        X, Y, Z = (mpmath.mpf(float(v)) for v in x[:3])
        p = mpmath.sqrt(X * X + Y * Y)
        lat = mpmath.atan2(Z, p * (1 - e2))
        for _ in range(100):
            sl = mpmath.sin(lat)
            nxt = mpmath.atan2(Z + e2 * a / mpmath.sqrt(1 - e2 * sl * sl) * sl, p)
            done = abs(nxt - lat) < mpmath.mpf(10) ** -45
            lat = nxt
            if done:
                break
        else:
            raise AssertionError("no convergence")
        sl, cl = mpmath.sin(lat), mpmath.cos(lat)
        h = p * cl + Z * sl - a * mpmath.sqrt(1 - e2 * sl * sl)
        return float(mpmath.degrees(lat)), float(mpmath.degrees(mpmath.atan2(Y, X))), float(h)


def test_references_at_50_digits():
    """The model's six fixed-point steps (pvt_model.ecef_llh) and its t_rx against the 50-digit references, at the
    Tokyo site, near the poles and the equator and 20 km up: within the bounds test_vtrack_edges_gpu holds the kernel
    to (1e-10 deg, 1e-5 m, 1.2e-10 s)."""
    for lat, lon, h in ((LOC[0], LOC[1], LOC[2]), (89.9, -170.0, 10.0), (-0.01, 0.0, 20000.0), (-66.0, 140.0, 0.0)):
        x = PM.llh_ecef(lat, lon, h)
        la, lo, hh = PM.ecef_llh(x)
        ref = geodetic_exact(x)
        assert abs(np.degrees(la) - ref[0]) <= 1e-10 and abs(np.degrees(lo) - ref[1]) <= 1e-10
        assert abs(hh - ref[2]) <= 1e-5 and abs(ref[2] - h) <= 1e-6
    st = np.zeros(1, V.STATE_DTYPE)[0]
    st["t0"], st["s0"] = 604799.123456789, 17
    fix = dict(sample=17 + 5 * 3000000 + 123, clock_m=19.25)
    t = float(st["t0"]) + (fix["sample"] - 17) / V.FS - fix["clock_m"] / V.C
    assert abs(t - t_rx_exact(st, fix)) <= 1.2e-10 and t > 604800.0


# ---- open loop: the command clamps and wraps ---------------------------------------------------------------------------
def speed_direction():
    """A unit vector whose dot product with the LOS of sky12's channels 11 and 10 is about +0.72 and -0.72 at the seed."""
    d = np.array([-0.73, -0.11, -0.67])
    return d / np.linalg.norm(d)


def open_loop_seed(kind, prns, chans, cfg, first=V.first):
    """The state of an open-loop run on zeros. 'speed': the truth-seeded filter SPEED_MPS off along speed_direction,
    so that predicted Dopplers pass +10 kHz on some channels and -10 kHz on others. 'jump': the channels started
    from the seed, then the filter's position moved JUMP_M along that direction (a filter that jumped away from its
    channels), so that the code errors are hundreds of chips either way. first(st) starts the channels (the model's,
    or the kernel's one-sample call)."""
    x8 = seed_x(PM.llh_ecef(*LOC))
    if kind == "speed":
        x8[3:6] += SPEED_MPS * speed_direction()
    st = V.seed(cfg, x8, START_SOW, 0, prns)
    st = first(st)
    if kind == "jump":
        st["x"][:3] += JUMP_M * speed_direction()
    return st


def model_first(chans, cfg):
    def f(st):
        V.first(st, [c["eph"] for c in chans], int(cfg["periods"]))
        return st
    return f


def command_record(monkeypatch):
    """Wrap the model's command: -> list of (phi 2^32 - phi') before the wrap, one per command."""
    errs = []
    real = V.command

    def rec(phi, rr, phi_nco, N):
        errs.append(phi * 2.0 ** 32 - float(phi_nco))
        return real(phi, rr, phi_nco, N)
    monkeypatch.setattr(V, "command", rec)
    return errs


def raw_code_residuals(st, chans, cfg, outs, eps, trace):
    """Every channel's code residual r (chips) before the +-511.5-chip wrap, from the run's records: the NCO phase at
    the interval's end (its last epoch), du n / 2^33 with the interval's u and w, D = 0 (E = L = 0 on zeros) and phi
    predicted at the prior X."""
    N = int(cfg["periods"])
    r = np.zeros(outs.shape)
    for k in range(outs.shape[0]):
        for c in range(outs.shape[1]):
            ep = eps[c][k * N:(k + 1) * N]
            assert ep.size == N and int(ep[-1]["sample"]) < int(outs[k, c]["sample"])
            u, w = int(ep[-1]["code_step"]), int(ep[-1]["carr_step"])
            du = u - int(T.code_step_of(np.int64(w)))
            n = int(outs[k, c]["sample"]) - int(ep[0]["sample"])
            phi, _, _ = V.predict(st, trace[k]["X_prior"], int(outs[k, c]["sample"]), chans[c]["eph"],
                                  int(outs[k, c]["sample"]))
            r[k, c] = int(ep[-1]["code_phase"]) / 2.0 ** 32 - du * n / 2.0 ** 33 - phi
    return r


def open_loop_edges(outs, errs, r_raw):
    """The edges an open-loop run reached: -> dict of booleans."""
    return dict(w_plus=bool((outs["carr_step"] == W_CLAMP).any()), w_minus=bool((outs["carr_step"] == -W_CLAMP).any()),
                u_min=bool((outs["code_step"] == T.CODE_STEP_MIN).any()),
                u_max=bool((outs["code_step"] == T.CODE_STEP_MAX).any()),
                err_wrap=bool((np.asarray(errs) >= V.M / 2).any()), r_wrap=bool((r_raw < -511.5).any()))


@pytest.mark.parametrize("kind,N", [("speed", 20), ("jump", 1), ("jump", 20)])
def test_open_loop_reaches_the_command_edges(sky12, kind, N, monkeypatch):
    """0.5 s of zeros. The code error err = phi 2^32 - phi' takes the +M/2 branch of its wrap (phi' < CODE_STEP_MAX at a
    period start, so the -M/2 branch cannot run), and r the -511.5 one (|phi'| < 0.35 chip, |du n / 2^33| <= 17 chips
    and phi >= 0, so r >= 511.5 cannot occur). Every channel is unused, so X runs on F alone."""
    prns, chans = sky12
    cfg = V.config(periods=N)
    st = open_loop_seed(kind, prns, chans, cfg, model_first(chans, cfg))
    errs = command_record(monkeypatch)
    trace = []
    fixes, outs, eps, _ = V.run(np.zeros(2 * 1500000, np.int8), 1, 0, st, chans, cfg, 10000, trace=trace)
    assert len(fixes) >= 450 // N and (outs["used"] == 0).all() and all(f["nused"] == 0 for f in fixes)
    e = open_loop_edges(outs, errs, raw_code_residuals(st, chans, cfg, outs, eps, trace))
    print(kind, N, e)
    if kind == "speed":
        assert e["w_plus"] and e["w_minus"] and e["err_wrap"]
    else:
        assert e["u_min"] and e["u_max"] and e["err_wrap"] and e["r_wrap"]


# ---- the first period at the code wrap --------------------------------------------------------------------------------
def wrap_seed(prns, chans, cfg, target):
    """A seed near the truth whose channel 0 starts at llround(phi 2^32) mod M = target: the seed sample s0 where
    channel 0's code is about to wrap, then the position moved along channel 0's line of sight (Newton's method on the
    model's predict) until the model's phi 2^32 lies within WRAP_MARGIN of target."""
    x8 = seed_x(PM.llh_ecef(*LOC))
    eph = chans[0]["eph"]

    def state(s0, d, e):
        x = x8.copy()
        x[:3] += d * e
        return V.seed(cfg, x, START_SOW + s0 / V.FS, s0, prns)

    def off(s0, d, e):
        st = state(s0, d, e)
        phi, _, _ = V.predict(st, st["x"], s0, eph, s0)
        err = phi * 2.0 ** 32 - target
        return err - V.M * np.floor(err / V.M + 0.5)
    st = V.seed(cfg, x8, START_SOW, 0, prns)
    phi, e, _ = V.predict(st, st["x"], 0, eph, 0)
    s0 = int(round((1023.0 - phi) / 1023.0 * 3000.0)) % 3000
    d = 0.0
    for _ in range(20):
        g = off(s0, d, e)
        if abs(g) <= WRAP_MARGIN / 2:
            break
        slope = (off(s0, d + 1e-3, e) - off(s0, d - 1e-3, e)) / 2e-3
        d -= g / slope
    g = off(s0, d, e)
    assert abs(g) <= WRAP_MARGIN, (target, g)
    return state(s0, d, e), s0, d, g


@pytest.mark.parametrize("target", WRAP_TARGETS)
def test_seeds_land_on_the_code_wrap(sky12, target):
    prns, chans = sky12
    cfg = V.config()
    st, s0, d, g = wrap_seed(prns, chans, cfg, target)
    assert abs(d) <= 200.0
    V.first(st, [c["eph"] for c in chans], int(cfg["periods"]))
    n = st["ch"][0]["nco"]
    print("target %d: s0 %d, %.3f m along the LOS, phi 2^32 - target %.4f unit; first period at s0 + %d" % (
        target, s0, d, g, int(n["sample"]) - s0))
    if target == 0:
        assert int(n["sample"]) == s0 and int(n["code_phase"]) == 0
    elif target == V.M - 1:
        assert int(n["sample"]) == s0 + 1 and int(n["code_phase"]) == int(n["code_step"]) - 1
    else:
        L = -(-(V.M - 1) // int(n["code_step"]))
        assert int(n["sample"]) == s0 + L and int(n["code_phase"]) == 1 + L * int(n["code_step"]) - V.M


# ---- full-scale sums at N = 100 -------------------------------------------------------------------------------------
def full_scale_plant(st, chans, cfg, nsamples, rotate):
    """An int8 stream at the corners that maximise channel 0's prompt wipe-off on the NCO trajectory the model runs on
    zeros from st (open loop: the trajectory does not depend on the samples): I = 127 or -128 by the sign of c_p cos
    theta, Q by that of c_p sin theta; rotate: the carrier turned by 45 degrees more in every period. Zeros outside the
    periods. -> (iq int8, the trajectory's epochs of channel 0)."""
    _, _, eps, _ = V.run(np.zeros(2 * nsamples, np.int8), 1, 0, st, chans, cfg, 10000)
    ep = eps[0]
    cos, sin = A.tables()
    code = T.code_pm(int(st["ch"][0]["nco"]["prn"]))
    I, Q = np.zeros(nsamples, np.int64), np.zeros(nsamples, np.int64)
    n0 = st["ch"][0]["nco"]
    theta, phi = int(n0["carr_phase"]), int(n0["code_phase"])
    for k in range(ep.size):
        s, u, w = int(ep[k]["sample"]), int(ep[k]["code_step"]), int(ep[k]["carr_step"]) & 0xFFFFFFFF
        L = (V.M - phi + u - 1) // u
        m = np.arange(L, dtype=np.int64)
        th = (theta + m * w + (k << 29 if rotate else 0)) & 0xFFFFFFFF
        cp = code[(phi + m * u) >> 32]
        I[s:s + L] = np.where(cp * cos[th >> 23] >= 0, 127, -128)
        Q[s:s + L] = np.where(cp * sin[th >> 23] >= 0, 127, -128)
        theta, phi = int(ep[k]["carr_phase"]), int(ep[k]["code_phase"])
    iq = np.empty(2 * nsamples, np.int8)
    iq[0::2], iq[1::2] = I, Q
    return iq, ep


def full_scale_config():
    return V.config(periods=100, q_min=1e300)


def check_full_scale(outs, rotate):
    """P near the header's bound; dot near its bound on the replica's carrier, dot ~ |cross| when rotated."""
    p, dot, cross = outs["p"][:, 0].astype(float), outs["dot"][:, 0].astype(float), outs["cross"][:, 0].astype(float)
    assert (p >= 0.4 * 100 * FULL).all(), p.min() / (100 * FULL)
    if rotate:
        assert (np.abs(cross) >= 0.4 * 99 * FULL).all() and (np.abs(np.abs(cross) / dot - 1) < 0.05).all()
    else:
        assert (dot >= 0.4 * 99 * FULL).all() and (np.abs(cross) <= 0.01 * dot).all()
    print("P %.3f, dot %.3f, |cross| %.3f of their bounds" % (
        p.max() / (100 * FULL), dot.max() / (99 * FULL), np.abs(cross).max() / (99 * FULL)))


def interval_power(iq, outs, eps):
    """S of every interval of channel 0 as the direct int64 sum of I^2 + Q^2 from its first period's start."""
    x = iq.astype(np.int64)
    c = np.concatenate([[0], np.cumsum(x[0::2] ** 2 + x[1::2] ** 2)])
    starts = eps[0]["sample"][0::100][:outs.shape[0]].astype(np.int64)
    return c[outs["sample"][:, 0].astype(np.int64)] - c[starts]


@pytest.mark.parametrize("rotate", [False, True])
def test_full_scale_plant_reaches_the_bounds(sky12, rotate):
    """0.31 s (3 updates) on the model: the sums reach the bounds the kernel's test asserts, and S is the direct sum."""
    prns, chans = sky12
    cfg = full_scale_config()
    st = V.seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, 0, prns[:1])
    V.first(st, [chans[0]["eph"]], 100)
    n = 930000
    iq, _ = full_scale_plant(st, chans[:1], cfg, n, rotate)
    fixes, outs, eps, _ = V.run(iq, 1, 0, st, chans[:1], cfg, 10000)
    assert len(fixes) == 3 and (outs["used"] == 0).all()
    check_full_scale(outs, rotate)
    assert np.array_equal(outs["s"][:, 0], interval_power(iq, outs, eps))


# ---- across the GPS week roll ---------------------------------------------------------------------------------------
WEEK_S = 604800.0
WEEKROLL_LEAD = 3.0                    # s from the seed to the roll
WEEKROLL_BLOCKS = 60                   # 6 s of 0.1 s blocks
BLOCK = 300000


def weekroll_case(tmp_path):
    """sky12_now_weekroll_300s (`-s now` at 23:58 on a Saturday) from the scenario engine, seeded WEEKROLL_LEAD before
    604 800 s. -> (rows of every block, NAV frames, PRNs, chans from the NAV frames of the seed's block, the seed's
    block, true t_rx at its first sample, receiver ECEF)."""
    import test_time_overwrite as TO
    g, kw = TO.now_case("sky12_now_weekroll_300s_i8", tmp_path)
    ch, nav = gps.scenario(**kw, time_overwrite=True)
    _, sow = TO.gps_time(kw["start"])
    b0 = int(round((WEEK_S - WEEKROLL_LEAD - sow) * V.FS / BLOCK))
    rows = ch[b0:b0 + WEEKROLL_BLOCKS]
    prns = [int(p) for p in rows[0]["prn"] if p > 0]
    assert all((rows["prn"] == p).any(1).all() for p in prns)
    chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    for c, p in enumerate(prns):
        slot = int(np.nonzero(rows[0]["prn"] == p)[0][0])
        chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(nav[int(rows[0]["nav_frame"][0])][slot]))[0]
        chans[c]["prn"] = p
    return ch, nav, prns, chans, b0, sow + b0 * BLOCK / V.FS, PM.llh_ecef(kw["lat"], kw["lon"], kw["height"])


def test_weekroll_seed_lands_before_the_roll(tmp_path):
    """The seed's t_rx is 604 797 s and the roll lies 3 s into the 6 s run; from the true position (clock 0) the
    model's predicted code phase of every channel is within 0.1 chip of the scenario's (the unmodelled ionosphere)
    at the seed, one sample either side of the roll and at the run's end: predict takes t past 604 800 s unfolded."""
    ch, nav, prns, chans, b0, t_rx0, x0 = weekroll_case(tmp_path)
    s0 = b0 * BLOCK
    roll = s0 + int(WEEKROLL_LEAD * V.FS)
    assert t_rx0 == WEEK_S - WEEKROLL_LEAD and t_rx0 + (roll - s0) / V.FS == WEEK_S
    st = V.seed(V.config(), np.concatenate([x0, np.zeros(5)]), t_rx0, s0, prns)
    worst = 0.0
    for s in (s0, roll - 1, roll + 1, s0 + WEEKROLL_BLOCKS * BLOCK - 3001):
        for c, p in enumerate(prns):
            phi, _, _ = V.predict(st, st["x"], s0, chans[c]["eph"], s)
            _, _, _, cp = TT.at(ch, p, s)
            d = (cp % 1023.0 - phi + 511.5) % 1023.0 - 511.5
            worst = max(worst, abs(d))
    print("%d channels, worst predicted code phase off the scenario's %.4f chip" % (len(prns), worst))
    assert len(prns) >= 8 and worst <= 0.1


# ---- arguments ------------------------------------------------------------------------------------------------------
def test_seed_refuses_a_repeated_prn():
    """Two channels on one PRN would enter the filter as independent satellites and make the PDOP's normal matrix
    singular: the seed refuses them; distinct PRNs in any order are accepted."""
    cfg = gps.vtrack_config()
    x8 = seed_x(PM.llh_ecef(*LOC))
    for prns in ([5, 5, 6, 7], [1, 2, 3, 1], [32] * 2, list(range(1, 32)) + [1]):
        with pytest.raises(gps.GpsB200Error):
            gps.vtrack_seed(cfg, x8, START_SOW, 0, prns)
    for prns in ([5, 6, 7, 8], list(range(32, 0, -1)), [9]):
        st = gps.vtrack_seed(cfg, x8, START_SOW, 0, prns)
        assert list(st["ch"]["nco"]["prn"][:len(prns)]) == prns
