"""Coarse-time fixes on the CPU: the numpy model of gpsb200_pvt_coarse (tests/coarse_model.py) on ideal and tracked
epochs against the scenario's truth, with the time anchors dropped and an a-priori position and time in their place.

The bounds below were fixed from the model; they are shared with the GPU tests. K is each fix's common integer: the
HOW-anchored whole ms (what gpsb200_pvt reads from the words) less the resolved ones; the satellites then sit at the
anchored transmit times when delta = K ms.
- Ideal epochs (sky12_static_35s, sky32_static_10s, the 60 s circle, 310 s at 60 deg N; a-priori offsets 0, 50 km east +
  1 km up with +10 s, 35 km west with -10 s; every offset gives the same fixes): 3D error at most 0.199 m (0.041 m with
  32 channels), receive time and |1000 delta - K| 35.2 us, velocity 4.6 mm/s static and 6.9 mm/s on the circle; on the
  `-s now` week-roll run of tests/test_coarse_gpu.py receive time and |1000 delta - K| reach 118 us and on its gapped
  channel 51 us. delta is weakly observable: a 35 us error moves the ranges by at most 3 cm (range rates below 800 m/s), the
  size of the quantisation of the broadcast terms and of the scenario's own range model, so the fit trades the two.
  Every post-fit residual is below 0.08 m. No rounding argument lies within 0.3 ms of a half.
- What the fifth state costs: the 5-state PDOP is 1.3 % (32 channels) to 2.8 % (12 channels) above gpsb200_pvt's on the
  same epochs; the mean 3D error is 0.95 (sky12) to 1.32 (sky32) times gpsb200_pvt's.
- Tracked on the CPU (track_model on 12.1 s of sky12_static_35s; a fix every 10 ms from 0.5 s): 3D error at most 22.4 m,
  mean 6.1 m (gpsb200_pvt: 20.2 m, 5.7 m), velocity 1.13 m/s, receive time and |1000 delta - K| at most 8.3 ms. With
  code noise of metres, delta is known to milliseconds only: 8 ms moves the ranges by at most 6.6 m.
The limits leave a margin of about a third over those figures."""
import numpy as np
import pytest

import coarse_model as CM
import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_pvt import check_truth, ideal_inputs, rinex, tracked_fixes
from test_scenario import LOC, LOC60, START, make_nav, motion_file
from test_track import START_SOW, model_run

WEEK = 2296
# ideal epochs: 3D error (m), receive time (s), velocity (m/s), |1000 delta - K| (ms)
IDEAL = dict(pos=0.27, time=1.6e-4, vel=0.0095, k=0.16)
# tracked epochs: per-fix and mean 3D error (m), receive time (s), velocity (m/s), |1000 delta - K| (ms)
TRACKED = dict(pos=30.0, pos_mean=8.1, time=0.011, vel=1.5, k=11.0)


def enu(x):
    lat, lon, _ = PM.ecef_llh(np.asarray(x, np.float64))
    return (np.array([-np.sin(lon), np.cos(lon), 0.0]),
            np.array([-np.sin(lat) * np.cos(lon), -np.sin(lat) * np.sin(lon), np.cos(lat)]),
            np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)]))


def offsets(x0):
    """The a-priori offsets: (position offset, time offset s)."""
    e, _, u = enu(x0)
    return [(np.zeros(3), 0.0), (50e3 * e + 1e3 * u, 10.0), (-35e3 * e, -10.0)]


def apriori(x0, sow, off=(np.zeros(3), 0.0), week=WEEK):
    """The a-priori config at sample 0: x0 + off[0], the true time of sample 0 + off[1]."""
    t = sow + off[1]
    return gps.coarse_config(np.asarray(x0) + off[0], t % 604800.0, 0, week + int(np.floor(t / 604800.0)))


def common_k(ms, anchored):
    """Per fix: the anchored less the resolved whole ms (wrapped into half a week) of the used channels, which must be
    one integer; -> K [F] (0 where no channel is used)."""
    d = np.where(ms >= 0, (anchored - ms + PT.WEEK_MS // 2) % PT.WEEK_MS - PT.WEEK_MS // 2, 0)
    k = np.zeros(len(ms), np.int64)
    for i in range(len(ms)):
        u = np.unique(d[i][ms[i] >= 0])
        assert u.size <= 1, (i, u)
        k[i] = u[0] if u.size else 0
    return k


def unanchored(chans):
    """The channels with their anchors dropped (the coarse-time call never reads them)."""
    c = chans.copy()
    c["anchor_epoch"], c["anchor_ms"] = -1, -1
    return c


def check_coarse(chans, eps, cfg, ap, rows, sow, bounds, nused_min=5, pos_mean=None):
    """Every fix OK, one common K per fix, |1000 delta - K| and the truth errors within the bounds; no rounding within
    1e-6 ms of a half and no residual near the ambiguity bound. -> (figures, fix, coarse record, ms)."""
    tr = {"half": [], "residual": [], "step": [], "runaway": []}
    fix, co, _, ms = CM.coarse(unanchored(chans), eps, cfg, ap, trace=tr)
    assert (fix["nused"] >= nused_min).all()
    anchored = PM.measure(chans, eps, fix["sample"])["T"]
    K = common_k(ms, anchored)
    dk = np.abs(1000.0 * co["delta"] - K)
    fig = check_truth(fix, rows, sow, bounds["pos"], bounds["time"], bounds["vel"], pos_mean)
    fig["k"] = float(dk.max())
    assert fig["k"] <= bounds["k"], fig
    assert np.concatenate(tr["half"]).min() > 1e-6
    assert np.concatenate(tr["residual"]).max() < CM.MAX_RESIDUAL / 10
    return fig, fix, co, ms


def static_rows(ch, loc):
    return np.repeat(PM.llh_ecef(*loc)[None], ch.shape[0] + 1, 0)


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8"])
def test_ideal_coarse_fixes_on_the_fixtures(name, tmp_path):
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, int(g["max_chan"]))
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    rows = static_rows(ch, LOC)
    cfg = gps.pvt_config(30000, 99991, (ch.shape[0] * PT.BLOCK - 30000 - PT.BLOCK) // 99991, iono)
    plain, _, _ = PM.pvt(chans, eps, cfg)
    for off in offsets(rows[0]):
        _, fix, co, _ = check_coarse(chans, eps, cfg, apriori(rows[0], START_SOW, off), rows, START_SOW, IDEAL)
        # the fifth state's cost in geometry (docstring)
        ratio = co["pdop"] / plain["pdop"]
        assert (ratio > 1.0).all() and (ratio < 1.04).all(), (ratio.min(), ratio.max())
        assert np.array_equal(fix["pdop"], co["pdop"])


def test_ideal_coarse_fixes_on_the_circle(tmp_path):
    g = scenario.load_golden("sky12_circle_60s_i16")
    nav_file, _, iono = rinex(tmp_path, 12)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    rows = g["motion_rows"][:, 1:4]
    cfg = gps.pvt_config(30000, 199999, (ch.shape[0] * PT.BLOCK - 30000 - PT.BLOCK) // 199999, iono)
    for off in offsets(rows[0]):
        check_coarse(chans, eps, cfg, apriori(rows[0], START_SOW, off), rows, START_SOW, IDEAL)


def test_ideal_coarse_fixes_while_satellites_rise_and_set(tmp_path):
    nav_file, _, iono = rinex(tmp_path, 32)
    ch, nav = gps.scenario(nav_file, *LOC60, seconds=310, max_chan=32, start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    rows = static_rows(ch, LOC60)
    cfg = gps.pvt_config(30000, 14999993, 61, iono)
    for off in offsets(rows[0]):
        _, fix, _, _ = check_coarse(chans, eps, cfg, apriori(rows[0], START_SOW, off), rows, START_SOW, IDEAL)
        assert len(set(fix["nused"])) > 1


def test_tracked_coarse_fixes_on_the_cpu(tmp_path):
    """12.1 s of sky12_static_35s through the acquisition and tracking models, the ephemeris from the scenario's frame,
    no anchors: sets the tracked bounds the GPU tests share."""
    g, ch, prns, eps = model_run("sky12_static_35s_i8", 121)
    _, _, iono = rinex(tmp_path, 12)
    chans, cfg = tracked_fixes(eps, prns, g, ch, iono, step=30000)
    rows = static_rows(ch, LOC)
    for off in offsets(rows[0]):
        check_coarse(chans, eps, cfg, apriori(rows[0], START_SOW, off), rows, START_SOW, TRACKED,
                     pos_mean=TRACKED["pos_mean"])


def ambiguity_case(tmp_path, nchan):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    chans, eps = chans[:nchan], eps[:nchan]
    x0 = PM.llh_ecef(*LOC)
    _, n, _ = enu(x0)
    cfg = gps.pvt_config(30000, 299993, 100, iono)
    fix, co, res, ms = CM.coarse(unanchored(chans), eps, cfg, apriori(x0, START_SOW, (400e3 * n, 30.0)))
    anchored = PM.measure(chans, eps, fix["sample"])["T"]
    d = np.where(ms >= 0, (anchored - ms + PT.WEEK_MS // 2) % PT.WEEK_MS - PT.WEEK_MS // 2, 0)
    wrong = np.array([np.unique(d[i][ms[i] >= 0]).size > 1 for i in range(len(d))])
    return fix, co, res, wrong


@pytest.mark.parametrize("nchan", [6, 12])
def test_wrong_integers_are_reported_ambiguous(nchan, tmp_path):
    """400 km north and 30 s off: the 0.5 ms condition breaks and some integers come out wrong in every fix. The status
    is then AMBIGUOUS, never OK. Here the wrong position fits the wrong integers well enough that re-resolving at it
    gives them back (no bit of `changed`); the residual bound sees them (kilometres of residual)."""
    fix, co, res, wrong = ambiguity_case(tmp_path, nchan)
    assert wrong.all()
    assert (fix["status"] == CM.FIX_AMBIGUOUS).all()
    assert np.isnan(fix["x"]).all() and np.isnan(co["delta"]).all() and np.isnan(res).all()
    assert (co["changed"] == 0).all()


def test_a_wrong_integer_cannot_be_seen_with_five_channels(tmp_path):
    """With exactly 5 channels the five unknowns fit any integers exactly: the same offset gives OK fixes whose
    integers are wrong, at the wrong place, with residuals of zero."""
    fix, co, res, wrong = ambiguity_case(tmp_path, 5)
    assert wrong.all() and (fix["status"] == PM.FIX_OK).all()
    err = np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - PM.llh_ecef(*LOC), axis=1)
    assert err.min() > 1e3 and np.nanmax(np.abs(res)) < 1e-3


def test_rinex_ephemeris_equals_the_file(tmp_path):
    """gpsb200_rinex_ephemeris on gen_rinex's file: every field of each PRN's record is read_rinex's value, toc the
    second of week of the record's epoch line and toe the orbit field; the RINEX-3 file of the same sky gives the same
    records; PRNs the file lacks, and times more than 2 h from every toe, give valid 0. (tests/test_ephemeris_terms.py
    reads files whose toc and toe differ.)"""
    nav = make_nav(tmp_path, 12)
    recs, _, _ = PT.read_rinex(nav)
    toe = next(iter(recs.values()))["toe"]
    eph = gps.rinex_ephemeris(nav, WEEK, toe + 1800.0)
    for prn in range(1, 33):
        e = eph[prn - 1]
        if prn not in recs:
            assert e["valid"] == 0
            continue
        r = recs[prn]
        assert e["valid"] == 1 and e["week"] == int(r["week"]) % 1024 and e["iode"] == int(r["iode"])
        assert e["iodc"] == int(r["iodc"]) and e["health"] == int(r["svh"])
        for f in ("toc", "toe", "af0", "af1", "af2", "tgd", "m0", "deltan", "ecc", "sqrta", "omg0", "inc0", "aop",
                  "omgdot", "idot", "cuc", "cus", "crc", "crs", "cic", "cis"):
            assert e[f] == r[f], (prn, f)
    (tmp_path / "v3").mkdir()
    nav3 = make_nav(tmp_path / "v3", 12, v3=True)
    assert gps.rinex_ephemeris(nav3, WEEK, toe + 1800.0, rinex3=True).tobytes() == eph.tobytes()
    assert (gps.rinex_ephemeris(nav, WEEK, toe + 7300.0)["valid"] == 0).all()
    assert (gps.rinex_ephemeris(nav, WEEK + 1, toe)["valid"] == 0).all()
    for bad in (dict(week=-1, sow=toe), dict(week=WEEK, sow=604800.0), dict(week=WEEK, sow=-1.0)):
        with pytest.raises(gps.GpsB200Error):
            gps.rinex_ephemeris(nav, **bad)
    with pytest.raises(gps.GpsB200Error):
        gps.rinex_ephemeris(tmp_path / "missing.nav", WEEK, toe)
