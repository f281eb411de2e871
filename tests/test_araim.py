"""ARAIM on the CPU: K_fa of gpsb200_araim_kfa against scipy, and the numpy model of the ARAIM stage
(tests/araim_model.py): its subset solutions against least squares on the reduced rows, its protection levels against
their equation, and its verdicts on ideal epochs with and without an injected code bias."""
import numpy as np
import pytest

import araim_model as AM
import pvt_model as PM
from scenario import gps
from test_pvt import IDEAL, check_truth, ideal_inputs, rinex, tracked_fixes
from test_raim import AF0_ERROR, code_bias, cpu_tracked, faulty_frames, g_af0, sky, FAULT_SLOT
from test_scenario import LOC, LOC60, START
from test_track import START_SOW

stats = pytest.importorskip("scipy.stats")


def kfa(acfg):
    return gps.araim_kfa(float(acfg["p_fa_vert"]), float(acfg["p_fa_horz"]))


def run(chans, eps, cfg, acfg, trace=None):
    return AM.araim(chans, eps, cfg, acfg, *kfa(acfg), trace=trace)


def new_trace():
    return dict(mask=[], test=[], argmax=[])


def assert_margin(trace):
    """No decision within 1e-9 relative of its threshold: the mask, the test, the exclusion argmax (where an exclusion
    can run: a failed test on 6 or more channels)."""
    for v in trace["mask"] + trace["test"]:
        assert np.all(np.abs(np.asarray(v) - 1.0) > 1e-9)
    for key in trace["argmax"]:
        k = np.sort(key)
        if k.size >= 6 and k[-1] > 1.0:
            assert k[-1] - k[-2] > 1e-9 * k[-1]


@pytest.mark.parametrize("p", [1e-12, 9e-8, 3.9e-6, 1e-3, 0.5])
def test_kfa_against_scipy(p):
    kh, kv = gps.araim_kfa(p, p)
    n = np.arange(5, 33)
    assert np.all(np.abs(kh / stats.norm.isf(p / (4 * n)) - 1.0) <= 1e-12)
    assert np.all(np.abs(kv / stats.norm.isf(p / (2 * n)) - 1.0) <= 1e-12)
    for bad in ((0.0, p), (p, 0.6), (float("nan"), p)):
        with pytest.raises(gps.GpsB200Error):
            gps.araim_kfa(*bad)


def ideal(name, tmp_path, nchan=None, nfix=6):
    _, ch, chans, eps = sky(name, nchan)
    _, _, iono = rinex(tmp_path, len(eps) if nchan is None else 12)
    return ch, chans, eps, gps.pvt_config(30000, 999983, nfix, iono)


def test_subset_solutions_are_least_squares_on_the_reduced_rows(tmp_path):
    """S(k) y is the weighted least-squares step of the rows without k, rotated to east / north / up."""
    _, chans, eps, cfg = ideal("sky12_static_35s_i8", tmp_path, 8, 2)
    acfg = gps.araim_config()
    inp = AM.Inputs(chans, eps, cfg)
    S = inp.use[0].copy()
    ok, X, _, last = AM.gauss_newton(inp, acfg, 0, S, np.zeros(4))
    assert ok
    o = AM.mhss(last, S, X, int(S.sum()), acfg, *kfa(acfg))
    idx = o["idx"]
    sw = 1.0 / np.sqrt(last["int2"][idx])
    G, y = last["g"][idx] * sw[:, None], last["r"][idx] * sw
    E = AM.enu(X)
    x0 = np.linalg.lstsq(G, y, rcond=None)[0]
    for kk in range(idx.size):
        keep = np.arange(idx.size) != kk
        xk = np.linalg.lstsq(G[keep], y[keep], rcond=None)[0]
        assert np.allclose(o["dx"][kk], E @ (xk - x0)[:3], rtol=1e-9, atol=1e-9)


def ideal_case(name, tmp_path):
    """(scenario records, chans, epochs, fix config, location) of the ideal-epoch cases."""
    if name == "lat60":
        nav_file, _, iono = rinex(tmp_path, 32)
        ch, nav = gps.scenario(nav_file, *LOC60, seconds=310, max_chan=32, start=START)
        chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
        return ch, chans, eps, gps.pvt_config(30000, 14999993, 21, iono), LOC60
    ch, chans, eps, cfg = ideal(name, tmp_path)
    return ch, chans, eps, cfg, LOC


def truth_elevations(chans, eps, cfg, xyz):
    """[F, C] elevation (rad) of each channel's satellite (rotated for its flight time) seen from the truth position."""
    inp = AM.Inputs(chans, eps, cfg)
    tau = np.linalg.norm(inp.P - xyz, axis=-1) / PM.C
    sth, cth = np.sin(PM.OMEGA_E * tau), np.cos(PM.OMEGA_E * tau)
    P = inp.P
    los = np.stack([P[..., 0] * cth + P[..., 1] * sth, P[..., 1] * cth - P[..., 0] * sth, P[..., 2]], -1) - xyz
    up = los @ AM.enu(xyz)[2]
    return np.arcsin(up / np.linalg.norm(los, axis=-1)), inp.use


@pytest.mark.parametrize("mask", [5.0, 10.0])
@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8", "lat60"])
def test_ideal_epochs_pass_and_bound_the_truth(name, mask, tmp_path):
    """Every fault-free fix with 5 or more channels above the mask passes; the truth errors stay below HPL and VPL; each
    PL satisfies its equation; the masked channels are exactly those whose truth elevation is below the mask."""
    ch, chans, eps, cfg, loc = ideal_case(name, tmp_path)
    acfg = gps.araim_config(mask_deg=mask)
    tr = new_trace()
    fix, _, rec, extra = run(chans, eps, cfg, acfg, tr)
    assert_margin(tr)
    ok = rec["n"] >= 5
    assert ok.all() and (rec["verdict"] == AM.PASS).all(), rec["verdict"]
    xyz = PM.llh_ecef(*loc)
    E = AM.enu(xyz)
    err = (np.stack([fix["x"], fix["y"], fix["z"]], 1) - xyz) @ E.T
    assert np.all(np.hypot(err[:, 0], err[:, 1]) < rec["hpl"]) and np.all(np.abs(err[:, 2]) < rec["vpl"])
    for f, (o, rhs, pl) in enumerate(extra):
        for q, L, r in zip((2, 0, 1), pl, rhs):
            args = (o["b0"][q], o["s0"][q], o["T"][:, q], o["b"][:, q], o["s"][:, q], float(acfg["p_sat"]))
            assert AM.pl_lhs(L, *args) <= r < AM.pl_lhs(L - 1e-3, *args)
    el, use = truth_elevations(chans, eps, cfg, xyz)
    low = use & (el < np.radians(mask))
    want = (low * (1 << np.arange(len(eps), dtype=np.int64))).sum(1)
    assert np.array_equal(rec["masked"].astype(np.int64), want)
    if name == "lat60":
        assert want.any()                                    # satellites rise and set there: the mask acts
    check_truth(fix, np.repeat(xyz[None], ch.shape[0] + 1, 0), START_SOW, IDEAL["pos"], IDEAL["time"], 1.0)


def test_single_code_bias_is_excluded(tmp_path):
    """A code bias of at least twice the channel's largest T gives EXCLUDED with exactly that channel, and ALERT with
    max_exclude 0."""
    _, ch, chans, eps = sky("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 1999993, 3, iono)
    acfg = gps.araim_config()
    _, _, rec0, extra = run(chans, eps, cfg, acfg)
    for c in (0, 5, 11):
        o = extra[0][0]
        kk = int(np.nonzero(o["idx"] == c)[0][0])
        bias_m = 2.0 * float(o["T"][kk].max()) + 10.0
        bad = list(eps)
        code_bias(bad, c, bias_m / (PM.C_MS / 1023.0))
        tr = new_trace()
        fix, _, rec, _ = run(chans, bad, cfg, acfg, tr)
        assert_margin(tr)
        assert (rec["verdict"] == AM.EXCLUDED).all() and (rec["excluded"] == 1 << c).all(), (c, rec["verdict"])
        xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
        check_truth(fix, xyz, START_SOW, IDEAL["pos"], IDEAL["time"], 1.0)
        _, _, rec, _ = run(chans, bad, cfg, gps.araim_config(max_exclude=0))
        assert (rec["verdict"] == AM.ALERT).all() and (rec["excluded"] == 0).all()


def test_ura_index_15_is_never_used_and_a_large_ura_deweights(tmp_path):
    _, ch, chans, eps = sky("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 1999993, 2, iono)
    acfg = gps.araim_config(max_exclude=0)
    bad = list(eps)
    code_bias(bad, 3, 0.02)
    xyz = PM.llh_ecef(*LOC)
    moved = []
    for ura in (0, 8, 15):
        c2 = chans.copy()
        c2[3]["eph"]["ura"] = ura
        fix, _, rec, _ = run(c2, bad, cfg, acfg)
        assert ((fix["mask"] >> 3) & 1 == (ura < 15)).all()
        moved.append(np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - xyz, axis=1).max())
    assert moved[1] < moved[0]


ARAIM_TRACKED = dict(sigma_ura=8.0, sigma_ure=16.0 / 3.0)   # as tests/test_raim.py's sigma for the tracked stream


def test_tracked_streams_on_the_cpu(tmp_path):
    """12.1 s of sky12_static_35s through the CPU acquisition and tracking models, sigma_ura 8 m: no fault-free fix
    alarms; with one PRN broadcasting af0 + 1 us, every fix excludes exactly that PRN."""
    g = scenario_golden()
    _, _, iono = rinex(tmp_path, 12)
    acfg = gps.araim_config(**ARAIM_TRACKED)
    ch, prns, eps = cpu_tracked(g, g["nav_frames"], 121)
    chans, cfg = tracked_fixes(eps, prns, g, ch, iono)
    _, _, rec, _ = run(chans, eps, cfg, acfg)
    assert np.isin(rec["verdict"], (AM.PASS, AM.UNAVAILABLE)).all() and (rec["verdict"] == AM.PASS).mean() > 0.9, \
        rec["verdict"]
    frames, prn = faulty_frames(g, tmp_path, 35)
    ch, prns, eps = cpu_tracked(g, frames, 121)
    chans, cfg = tracked_fixes(eps, prns, dict(nav_frames=frames), ch, iono)
    c = prns.index(prn)
    assert chans[c]["eph"]["af0"] - g_af0(g, FAULT_SLOT) > 0.99 * AF0_ERROR
    _, _, rec, _ = run(chans, eps, cfg, acfg)
    assert (rec["verdict"] == AM.EXCLUDED).all() and (rec["excluded"] == 1 << c).all(), rec["verdict"]


def scenario_golden():
    import scenario
    return scenario.load_golden("sky12_static_35s_i8")
