"""RAIM on the CPU: the chi^2 tables of gpsb200_raim_thresholds against scipy, and the numpy model of the RAIM stage
(tests/raim_model.py) on ideal epochs with and without injected faults.

The faults are edits of the host-side inputs: a code-phase bias on a channel's epochs, a satellite clock (af0) error in
a channel's ephemeris, a whole-ms error in a channel's time anchor. Found with the model at sigma = 1 m on ideal epochs:
the largest stat / T of a fault-free fix is LARGEST_FREE (sky12_static_35s, sky32_static_10s, the 310 s run at 60 deg N)."""
import numpy as np
import pytest

import pvt_model as PM
import raim_model as RM
from scenario import gps
import scenario
from test_pvt import IDEAL, TRACKED, check_truth, ideal_inputs, rinex, tracked_fixes
from test_scenario import LOC, START
from test_track import ACQ, START_SOW, starts

LARGEST_FREE = 1e-3                          # stat / T at sigma = 1 m, p_fa = 1e-5, on ideal epochs (6.0e-4 seen)
EXCLUDED_VEL = 0.015                         # m/s: the velocity error bound of a fix with a channel excluded
CHIP = 2.0 ** 32                             # code_phase units per chip


def tables(rcfg):
    return gps.raim_thresholds(float(rcfg["p_fa"]), float(rcfg["p_md"]))


def run(chans, eps, cfg, rcfg):
    return RM.raim(chans, eps, cfg, rcfg, *tables(rcfg))


def code_bias(eps, c, chips):
    """Add `chips` to the code phase of every epoch of channel c: its pseudorange drops by chips x 293 m. -> bias (m)."""
    add = int(round(chips * CHIP))
    assert int(eps[c]["code_phase"].max()) + add < 2 ** 32
    eps[c] = eps[c].copy()
    eps[c]["code_phase"] += np.uint32(add)
    return -add / PM.CODE_MOD * PM.C_MS


def sky(name, nchan=None):
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    prns = None if nchan is None else [int(p) for p in ch[0]["prn"] if p > 0][:nchan]
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"], prns)
    return g, ch, chans, eps


def fault_free_check(chans, eps, cfg):
    rcfg = gps.raim_config(1.0)
    fix, res, rec, _ = run(chans, eps, cfg, rcfg)
    want, wres, _ = PM.pvt(chans, eps, cfg)
    few = want["nused"] < 5
    assert (rec["verdict"][few] == RM.UNAVAILABLE).all() and (rec["verdict"][~few] == RM.PASS).all()
    for k in want:
        assert np.array_equal(fix[k], want[k], equal_nan=True), k
    assert np.array_equal(res, wres, equal_nan=True)
    worst = float(np.nanmax(rec["stat"] / rec["threshold"]))
    assert worst <= LARGEST_FREE, worst
    return worst


# ---- the tables ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p_fa", [1e-2, 1e-5, 1e-8])
@pytest.mark.parametrize("p_md", [1e-3, 1e-6])
def test_thresholds_against_scipy(p_fa, p_md):
    """T_d = chi2.isf(p_fa, d) to 1e-9 relative; lambda_d to 1e-9 relative: the noncentral CDF at T_d crosses p_md
    between lambda_d (1 - 1e-9) and lambda_d (1 + 1e-9)."""
    stats = pytest.importorskip("scipy.stats")
    T, lam = gps.raim_thresholds(p_fa, p_md)
    for d in range(1, 29):
        assert abs(T[d - 1] / stats.chi2.isf(p_fa, d) - 1.0) <= 1e-9, d
        assert stats.ncx2.cdf(T[d - 1], d, lam[d - 1] * (1 - 1e-9)) >= p_md >= \
            stats.ncx2.cdf(T[d - 1], d, lam[d - 1] * (1 + 1e-9)), d
    assert np.all(np.diff(T) > 0) and np.all(lam > T[0] * 0)


def test_thresholds_refuse_bad_arguments():
    for p_fa, p_md in ((0.0, 1e-3), (1e-13, 1e-3), (0.6, 1e-3), (1e-5, 0.0), (1e-5, 0.51), (float("nan"), 1e-3),
                       (1e-5, float("inf"))):
        with pytest.raises(gps.GpsB200Error):
            gps.raim_thresholds(p_fa, p_md)
    T, lam = gps.raim_thresholds(1e-12, 0.5)        # the ends of the range are accepted
    assert np.isfinite(T).all() and np.isfinite(lam).all()


# ---- the model on ideal epochs ---------------------------------------------------------------------------------------
def test_dof_1_alerts_and_never_excludes(tmp_path):
    """5 channels: every normalized residual is equal, so a detected fault cannot be identified: ALERT, nothing
    excluded, and the fix is gpsb200_pvt's."""
    g, _, chans, eps = sky("sky12_static_35s_i8", 5)
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 2999993, 11, iono)
    code_bias(eps, 2, 0.3)
    fix, _, rec, tests = run(chans, eps, cfg, gps.raim_config(1.0, max_exclude=4))
    assert (rec["verdict"] == RM.ALERT).all() and (rec["excluded"] == 0).all() and (rec["dof"] == 1).all()
    for t in tests:
        key = t[-1][2]
        assert len(t) == 1 and np.allclose(key, key[0], rtol=1e-6)
    want, _, _ = PM.pvt(chans, eps, cfg)
    assert np.array_equal(fix["x"], want["x"])


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8"])
def test_no_false_alarm_on_ideal_epochs(name, tmp_path):
    _, ch, chans, eps = sky(name)
    _, _, iono = rinex(tmp_path, len(eps))
    n = ch.shape[0]
    fault_free_check(chans, eps, gps.pvt_config(30000, 99991, (n * 300000 - 330000) // 99991, iono))


def test_no_false_alarm_while_satellites_rise_and_set(tmp_path):
    from test_scenario import LOC60
    nav_file, _, iono = rinex(tmp_path, 32)
    ch, nav = gps.scenario(nav_file, *LOC60, seconds=310, max_chan=32, start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    fault_free_check(chans, eps, gps.pvt_config(30000, 14999993, 61, iono))


def sky12_faults():
    """(label, channel, edit) of the injected single faults on sky12: a +0.1 chip code bias on each channel, af0 + 1e-7 s
    on channel 3, anchor_ms + 1 on channel 7. edit(chans, eps) -> the expected residual of the channel (m)."""
    out = [("code%d" % c, c, (lambda c: lambda ch, ep: code_bias(ep, c, 0.1))(c)) for c in range(12)]

    def clock(ch, ep):
        ch[3]["eph"]["af0"] += 1e-7
        return 1e-7 * PM.C

    def anchor(ch, ep):
        ch[7]["anchor_ms"] += 1
        return -PM.C_MS
    return out + [("af0", 3, clock), ("anchor", 7, anchor)]


def sky12_fault_case(edit, tmp_path):
    g, ch, chans, eps = sky("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    chans = chans.copy()
    bias = edit(chans, eps)
    cfg = gps.pvt_config(30000, 1999993, 17, iono)
    return ch, chans, eps, cfg, bias


def assert_excluded(ch, fix, res, rec, chans_excl, biases, start_sow=START_SOW):
    assert (rec["verdict"] == RM.EXCLUDED).all(), rec["verdict"]
    assert (rec["excluded"] == sum(1 << c for c in chans_excl)).all()
    for c, b in zip(chans_excl, biases):
        assert np.all(np.abs(res[:, c] - b) < 1.0), (c, b, res[:, c])
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    # position and time within the ideal bounds; the velocity, which no fault here touches, from one channel fewer
    # (0.011 m/s seen)
    check_truth(fix, xyz, start_sow, IDEAL["pos"], IDEAL["time"], EXCLUDED_VEL)


@pytest.mark.parametrize("label", [f[0] for f in sky12_faults()])
def test_single_fault_is_excluded(label, tmp_path):
    """Every fix excludes exactly the faulty channel; the final fix is within the ideal bounds; the excluded channel's
    residual against it is the fault within 1 m."""
    _, c, edit = next(f for f in sky12_faults() if f[0] == label)
    ch, chans, eps, cfg, bias = sky12_fault_case(edit, tmp_path)
    fix, res, rec, _ = run(chans, eps, cfg, gps.raim_config(1.0))
    assert_excluded(ch, fix, res, rec, [c], [bias])


def sky32_two_faults(tmp_path):
    _, ch, chans, eps = sky("sky32_static_10s_i8")
    _, _, iono = rinex(tmp_path, 32)
    b = [code_bias(eps, 5, 0.1), code_bias(eps, 20, 0.15)]
    return ch, chans, eps, gps.pvt_config(30000, 999991, 8, iono), b


def test_two_faults_on_32_channels(tmp_path):
    """Two biased channels: both excluded with max_exclude 2; ALERT with max_exclude 1 (the larger one out)."""
    ch, chans, eps, cfg, b = sky32_two_faults(tmp_path)
    fix, res, rec, _ = run(chans, eps, cfg, gps.raim_config(1.0, max_exclude=2))
    assert_excluded(ch, fix, res, rec, [5, 20], b)
    fix, res, rec, _ = run(chans, eps, cfg, gps.raim_config(1.0, max_exclude=1))
    assert (rec["verdict"] == RM.ALERT).all() and (rec["excluded"] == 1 << 20).all()


def test_hpl_is_the_error_of_the_worst_undetectable_bias(tmp_path):
    """A bias of noncentrality lambda on the channel of the largest horizontal slope (detection only) moves the fix
    horizontally by HPL within 1 % (and vertically, on the channel of the largest vertical slope, by VPL)."""
    g, ch, chans, eps = sky("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(4500017, 1, 1, iono)
    rcfg = gps.raim_config(1.0, max_exclude=0)
    T, lam = tables(rcfg)
    fix, _, rec, _ = run(chans, eps, cfg, rcfg)
    assert rec["verdict"][0] == RM.PASS
    _, _, ms = RM.solve(chans, eps, cfg)
    _, x, omh = RM.loo(ms, 0)
    lat, lon = np.radians(fix["lat_deg"][0]), np.radians(fix["lon_deg"][0])
    enu = np.array([[-np.sin(lon), np.cos(lon), 0.0],
                    [-np.sin(lat) * np.cos(lon), -np.sin(lat) * np.sin(lon), np.cos(lat)],
                    [np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)]])
    xe = x[:, :3] @ enu.T
    k = np.sqrt(lam[rec["dof"][0] - 1])
    for axis, level, slope in (("h", rec["hpl"][0], np.hypot(xe[:, 0], xe[:, 1]) / np.sqrt(omh)),
                               ("v", rec["vpl"][0], np.abs(xe[:, 2]) / np.sqrt(omh))):
        c = int(np.argmax(slope))
        assert abs(slope[c] * k - level) <= 1e-9 * level
        bad = [e.copy() for e in eps]
        code_bias(bad, c, k / np.sqrt(omh[c]) / (PM.C_MS / 1023.0))   # sigma sqrt(lambda / (1 - h_cc)) metres
        bfix, _, brec, _ = run(chans, bad, cfg, rcfg)
        assert brec["verdict"][0] == RM.ALERT
        d = (np.array([bfix[f][0] - fix[f][0] for f in ("x", "y", "z")]) @ enu.T)
        err = np.hypot(d[0], d[1]) if axis == "h" else abs(d[2])
        assert abs(err / level - 1.0) <= 0.01, (axis, err, level)


# ---- tracked on the CPU: a stream whose broadcast clock of one PRN is wrong ---------------------------------------------
TRACKED_SIGMA = 8.0          # m: no fault-free tracked fix of sky12_static_35s alarms (stat <= T / 2)
AF0_ERROR = 1e-6             # s: the broadcast af0 error of the faulty PRN, ~300 m of pseudorange
FAULT_SLOT = 4               # its channel slot in sky12_static_35s


def rinex_with_af0(nav, out, prn, add):
    """A copy of the RINEX file `nav` with af0 + add in every record of prn."""
    lines = open(nav).read().splitlines()
    i = next(k for k, ln in enumerate(lines) if "END OF HEADER" in ln) + 1
    for i in range(i, len(lines), 8):
        if int(lines[i][0:2]) == prn:
            v = float(lines[i][22:41].replace("D", "E")) + add
            lines[i] = lines[i][:22] + ("%19.12E" % v).replace("E", "D") + lines[i][41:]
    open(out, "w").write("\n".join(lines) + "\n")


def faulty_frames(g, tmp_path, seconds):
    """The scenario's NAV frames with FAULT_SLOT's PRN broadcasting af0 + AF0_ERROR (the records, and so the signal's
    timing, stay those of the RINEX file). -> (frames, prn)"""
    nav, _, _ = rinex(tmp_path, 12)
    prn = int(g["chans"][0]["prn"][FAULT_SLOT])
    bad = tmp_path / "bad.nav"
    rinex_with_af0(nav, bad, prn, AF0_ERROR)
    _, good_frames = gps.scenario(nav, *LOC, seconds=seconds, max_chan=12, start=START)
    ch2, bad_frames = gps.scenario(str(bad), *LOC, seconds=seconds, max_chan=12, start=START)
    frames = np.array(g["nav_frames"], copy=True)
    n = min(len(frames), len(bad_frames))
    assert np.array_equal(good_frames[:n], frames[:n])
    assert (ch2["prn"][:, FAULT_SLOT] == prn).all()
    frames[:n, FAULT_SLOT] = bad_frames[:n, FAULT_SLOT]
    assert not np.array_equal(frames[0, FAULT_SLOT], g["nav_frames"][0, FAULT_SLOT])
    return frames, prn


def cpu_tracked(g, frames, nblk):
    """model_run of tests/test_track.py on the golden records with these NAV frames."""
    import acq_model as A
    import track_model as T
    from test_acquire import golden_rows
    ch = golden_rows(g, range(nblk))
    ss = int(g["sample_size"])
    iq, _ = scenario.oracle_run(ch, frames, ss)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    res = A.search(iq[:2 * A.CODE * 13], ss, 0, ACQ["ms"], prns, ACQ["f_lo"], ACQ["step"], ACQ["nbins"])
    eps, _ = T.track(iq, ss, 0, starts(res))
    return ch, prns, eps


def test_tracked_fault_is_excluded_on_the_cpu(tmp_path):
    """12.1 s of sky12_static_35s through the CPU acquisition and tracking models. Fault-free, at sigma TRACKED_SIGMA no
    fix alarms (stat <= T / 2). With one PRN broadcasting a clock 1 us off, every fix excludes that PRN and the final
    fixes are within the tracked bounds."""
    g = scenario.load_golden("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    rcfg = gps.raim_config(TRACKED_SIGMA)
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], g["chans"].shape[0] + 1, 0)
    ch, prns, eps = cpu_tracked(g, g["nav_frames"], 121)
    chans, cfg = tracked_fixes(eps, prns, g, ch, iono)
    _, _, rec, _ = run(chans, eps, cfg, rcfg)
    assert (rec["verdict"] == RM.PASS).all() and np.all(rec["stat"] <= rec["threshold"] / 2), \
        float(np.max(rec["stat"] / rec["threshold"]))
    frames, prn = faulty_frames(g, tmp_path, 35)
    ch, prns, eps = cpu_tracked(g, frames, 121)
    chans, cfg = tracked_fixes(eps, prns, dict(nav_frames=frames), ch, iono)
    c = prns.index(prn)
    assert chans[c]["eph"]["af0"] - g_af0(g, FAULT_SLOT) > 0.99 * AF0_ERROR
    fix, res, rec, _ = run(chans, eps, cfg, rcfg)
    assert (rec["verdict"] == RM.EXCLUDED).all() and (rec["excluded"] == 1 << c).all()
    assert np.all(np.abs(res[:, c] - AF0_ERROR * PM.C) < 30.0), res[:, c]
    check_truth(fix, xyz, START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])


def g_af0(g, slot):
    return float(gps.nav_ephemeris(gps.nav_words_of_frame(g["nav_frames"][0][slot]))[0]["af0"])
