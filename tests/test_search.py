"""Position search on the CPU: the grid of gpsb200_pvt_search and its covering radius, and the numpy model
(tests/search_model.py) on ideal and tracked epochs against the scenario's truth, with no a-priori position.

Model figures (DESIGN §11.4), sky12_static_35s at 7 200.1 s with the default grid and the a-priori time 0 / +10 s off:
12 channels search 48 800 nodes of 262 144 and find 66-67 OK ones, all within 1 m of the winner; the 7 channels of its
first PRNs search 73 000 and find 145-147, all within 1 m; its first 6 channels find about 1 200, of which about 1 000
are wrong-integer fixes 2 300 km and more away with rms from 8.9 m (the winner: 3 mm). 32 channels (sky32_static_10s)
search 8 470 and find 31-32."""
import numpy as np
import pytest
from scipy.spatial import ConvexHull

import pvt_model as PM
import pvt_truth as PT
import search_model as SM
import scenario
import test_sites as TS
from scenario import gps
from test_coarse import IDEAL, TRACKED, WEEK, unanchored
from test_pvt import check_truth, ideal_inputs, rinex, tracked_fixes
from test_scenario import LOC, LOC60, START, motion_file
from test_track import START_SOW, model_run


def circumradii(p, simplices):
    """Circumradius of each triangle p[simplices] in 3D."""
    a, b, c = (p[simplices[:, k]] for k in range(3))
    ab, ac = b - a, c - a
    n = np.cross(ab, ac)
    num = np.linalg.norm(np.cross(n, ab) * (ac * ac).sum(1, keepdims=True)
                         + np.cross(ac, n) * (ab * ab).sum(1, keepdims=True), axis=1)
    return num / (2.0 * (n * n).sum(1))


def test_default_grid_covering_radius():
    """The largest circumradius of the convex hull's facets: 33.99 km on a sphere of the WGS-84 equatorial radius, at
    most 35 km on the nodes themselves; 131 072 nodes give 48.06 km. The library's nodes equal the model's to 1 mm."""
    lat, lon = SM.grid_llh(SM.NODES_DEFAULT)
    u = np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], 1)
    r = circumradii(u, ConvexHull(u).simplices).max() * PM.WGS_A
    assert abs(r - 33.99e3) < 10.0, r
    x = SM.nodes(SM.NODES_DEFAULT)
    assert circumradii(x, ConvexHull(x).simplices).max() <= 35e3
    lat, lon = SM.grid_llh(131072)
    u = np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], 1)
    assert abs(circumradii(u, ConvexHull(u).simplices).max() * PM.WGS_A - 48.06e3) < 10.0
    for n in (64, 4096, SM.NODES_DEFAULT):
        assert np.abs(gps.search_nodes(n) - SM.nodes(n)).max() < 1e-3
    for n in (63, (1 << 22) + 1):
        with pytest.raises(gps.GpsB200Error):
            gps.search_nodes(n)


def search_cfg(sow, dt, week=WEEK):
    t = sow + dt
    return gps.search_config(t % 604800.0, 0, week + int(np.floor(t / 604800.0)))


def check_search(chans, eps, cfg, sow, week, rows, bounds, instants):
    """At each of `instants` (indices into cfg's instants), with the a-priori time 0, +10 and -10 s off in turn: OK,
    support >= 1, no distinct solution, within the bounds. -> the last (fix, record)."""
    ch = unanchored(chans)
    for k, i in enumerate(instants):
        one = gps.pvt_config(int(cfg["s0"]) + int(i) * int(cfg["step"]), 1, 1, (cfg["alpha"], cfg["beta"]))
        fix, rec, _, _ = SM.search(ch, eps, one, search_cfg(sow, (0.0, 10.0, -10.0)[k % 3], week))
        assert (fix["status"] == PM.FIX_OK).all() and (rec["support"] >= 1).all(), (fix["status"], rec)
        assert np.isnan(rec["alt_rms"]).all() and (rec["support"] == rec["ok"]).all()
        check_truth(fix, rows, sow, bounds["pos"], bounds["time"], bounds["vel"])
    return fix, rec


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8"])
def test_ideal_searches_on_the_fixtures(name, tmp_path):
    """Three instants, the a-priori time 0 and +-10 s off."""
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, int(g["max_chan"]))
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    rows = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    check_search(chans, eps, gps.pvt_config(30000, 2999993, 3, iono), START_SOW, WEEK, rows, IDEAL, [0, 1, 2])


def test_ideal_searches_on_the_circle(tmp_path):
    """The 60 s circle: the truth moves along the motion file's rows."""
    g = scenario.load_golden("sky12_circle_60s_i16")
    nav_file, _, iono = rinex(tmp_path, 12)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    cfg = gps.pvt_config(30000, 199999, (ch.shape[0] * PT.BLOCK - 30000 - PT.BLOCK) // 199999, iono)
    n = int(cfg["nfix"])
    check_search(chans, eps, cfg, START_SOW, WEEK, g["motion_rows"][:, 1:4], IDEAL, [0, n // 2, n - 1])


def test_ideal_searches_at_60_north(tmp_path):
    """310 s at 60 deg N with 32 channels, at the start, middle and end of the run while satellites rise and set."""
    nav_file, _, iono = rinex(tmp_path, 32)
    ch, nav = gps.scenario(nav_file, *LOC60, seconds=310, max_chan=32, start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    rows = np.repeat(PM.llh_ecef(*LOC60)[None], ch.shape[0] + 1, 0)
    check_search(chans, eps, gps.pvt_config(30000, 14999993, 21, iono), START_SOW, WEEK, rows, IDEAL, [0, 10, 20])


@pytest.mark.parametrize("name", TS.SITES)
def test_ideal_searches_at_the_sites(name, tmp_path):
    """66 deg N 100 deg W, 66 deg S 140 deg E and 34 deg S 58 deg W: every search OK and unique."""
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    chans, eps, cfg, _, (xyz, sow), _ = TS.fix_inputs(name, tmp_path / "a")
    week, _ = TS.gps_time(TS.site_case(name, tmp_path / "b")[1]["start"])
    check_search(chans, eps, cfg, sow, week, xyz, IDEAL, [0, 4, 8])


def test_five_channels_are_too_few(tmp_path):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    fix, rec, res, ms = SM.search(unanchored(chans[:5]), eps[:5], gps.pvt_config(30000, 299993, 2),
                                  search_cfg(START_SOW, 10.0))
    assert (fix["status"] == PM.FIX_FEW).all() and (rec["searched"] == 0).all() and (rec["winner"] == -1).all()
    assert np.isnan(fix["x"]).all() and np.isnan(res).all() and (ms == -1).all()


def test_tracked_searches_on_the_cpu(tmp_path):
    """12.1 s of sky12_static_35s through the acquisition and tracking models: searches at three instants are OK and
    within coarse-time's tracked bounds."""
    g, ch, prns, eps = model_run("sky12_static_35s_i8", 121)
    _, _, iono = rinex(tmp_path, 12)
    chans, cfg = tracked_fixes(eps, prns, g, ch, iono, step=30000)
    rows = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    n = int(cfg["nfix"])
    check_search(chans, eps, cfg, START_SOW, WEEK, rows, TRACKED, [0, n // 2, n - 1])
