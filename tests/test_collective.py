"""Collective detection's numpy model (tests/collective_model.py) on the CPU oracle's streams against the scenario's
truth, and the snapshot chain it seeds (snapshot_model's measurement and coarse_model's fix).

The figures below were taken from the model, K = 10 coherent ms from sample 1000 of a block, the standard grid of
32 PRNs x 41 bins, a lattice of +-3.5 km at 250 m east and north and +-1.5 s at 0.5 s (5 887 hypotheses):
- sky12_static_35s blocks 0 and 50, a-priori offsets 0, (2 km east, +0.5 s), (-3 km north, -1 s): the winner lies on
  the lattice point nearest the truth (within 1.5 m: the lattice holds the truth up to the conversion's rounding), the
  time offset is the true one, and every seed is the truth's sample and bin. The runner-up beyond 1 km reaches at most
  0.74 of the winner's score.
- The weakened stream (block 0 with the gain of PRNs 1-8 scaled by 0.12): only PRNs 9-12 pass ratio 2.5, so the plain
  snapshot chain has 4 OK records and its fix is FEW. The winner is again the truth's lattice point, the eight weak
  PRNs' seeds are their true cells, and the seeded measurement gives 12 OK records and a fix 48.3 m from the truth
  (bound WEAK_POS; receive time and velocity within test_snapshot's bounds). The runner-up reaches 0.84 of the winner (DESIGN §11.7 gives the figures at other caps on q).
The position bound is the lattice's half cell diagonal plus a margin of 5 m."""
import numpy as np
import pytest

import acq_model as A
import collective_model as CM
import pvt_model as PM
import pvt_truth as PT
import scenario
import snapshot_model as S
from scenario import gps
from test_acquire import golden_rows
from test_coarse import WEEK, enu, static_rows, unanchored
from test_pvt import check_truth, rinex
from test_scenario import LOC
from test_snapshot import BOUNDS, S0, K, block_stream
from test_track import START_SOW

PRNS = list(range(1, 33))
FLO = np.full(32, -5000.0)
WEAK_PRNS, WEAK_GAIN = (1, 2, 3, 4, 5, 6, 7, 8), 0.12
MARGIN = 5.0
WEAK_POS = 65.0   # m: the weakened stream's fix, 48.3 m on the model (its eight weak PRNs measure their codes less well)


def lattice():
    return gps.collective_config(3500.0, 250.0, 1.5, 0.5, mask_deg=5.0, distinct_m=1000.0)


def bound(cfg):
    return 0.5 * np.sqrt(float(cfg["step"][0]) ** 2 + float(cfg["step"][1]) ** 2) + MARGIN


def ephemeris(tmp_path, nsat, sow):
    nav, _, iono = rinex(tmp_path, nsat)
    return gps.rinex_ephemeris(nav, WEEK, sow), iono


def pvt_chans(eph, prns):
    ch = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    for c, p in enumerate(prns):
        ch[c]["eph"], ch[c]["prn"] = eph[p - 1], p
    return unanchored(ch)


def run(iq, ss, eph, ap, cfg=None):
    res, P = A.search(iq, ss, S0, K, PRNS, want_grid=True)
    cfg = lattice() if cfg is None else cfg
    rec, seed, Sc, b, cells = CM.collective(P, res, eph, PRNS, ap, S0, cfg, FLO, 250.0)
    return res, P, rec, seed, cfg


def check_seeds(seed, ch, rec):
    held = {int(r["prn"]): r for r in ch[0] if r["prn"] > 0}
    for p, s in enumerate(seed):
        if not (int(rec["used"]) >> p) & 1:
            assert s["ratio"] == -1.0
            continue
        if int(s["prn"]) not in held:
            continue
        f, tau = A.truth(held[int(s["prn"])], S0)
        assert A.circ_dist(s["delay"], int(np.rint(tau)) % A.CODE) <= 2, (s["prn"], s["delay"], tau)
        assert abs(s["doppler_hz"] - f) <= 125.0 + 1e-9, (s["prn"], s["doppler_hz"], f)


def fix_from(seed, iq, ss, b, eph, iono, rec, ap, prns):
    """The seeded measurement and the coarse fix from the winner, in stream samples."""
    m = S.measure(iq, ss, S0, K, seed, min_ratio=0.0)
    sel = [int(np.nonzero(m["prn"] == p)[0][0]) for p in prns]
    mm = m[sel]
    mm["sample"] += b * PT.BLOCK
    apw = gps.coarse_config(rec["x"], float(ap["t_a"]) + float(rec["o_t"]) - 0.1 * b, 0, WEEK)
    fix, _, _, _ = S.coarse(pvt_chans(eph, prns), mm[None], gps.pvt_config(0, 1, 1, iono), apw)
    return m, fix


@pytest.mark.parametrize("block", [0, 50])
def test_model_truth_on_sky12_static(block, tmp_path):
    g, ch, iq = block_stream("sky12_static_35s_i8", block)
    sow = START_SOW + 0.1 * block
    eph, iono = ephemeris(tmp_path, 12, sow)
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    rows = static_rows(ch, LOC)
    prns = sorted(int(p) for p in ch[0]["prn"] if p > 0)
    for dx, dt in ((np.zeros(3), 0.0), (2000.0 * e, 0.5), (-3000.0 * n, -1.0)):
        ap = gps.coarse_config(x0 + dx, sow + dt, 0, WEEK)
        res, P, rec, seed, cfg = run(iq, 1, eph, ap)
        assert rec["status"] == CM.OK and rec["nused"] == 12, rec
        assert np.linalg.norm(rec["x"] - x0) <= bound(cfg), rec
        assert abs(rec["o_t"] + dt) <= float(cfg["step"][3]), rec
        check_seeds(seed, ch, rec)
        _, fix = fix_from(seed, iq, 1, block, eph, iono, rec, ap, prns)
        assert fix["status"][0] == gps.FIX_OK
        check_truth(fix, rows, START_SOW, BOUNDS["pos"], BOUNDS["time"], BOUNDS["vel"])


def weak_block(g, b=0):
    ch = golden_rows(g, [b])
    for c in range(ch.shape[1]):
        if int(ch[0, c]["prn"]) in WEAK_PRNS:
            ch[0, c]["gain"] *= WEAK_GAIN
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], int(g["sample_size"]))
    return ch, iq


def test_model_finds_the_weakened_stream(tmp_path):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, iq = weak_block(g)
    eph, iono = ephemeris(tmp_path, 12, START_SOW)
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    prns = sorted(int(p) for p in ch[0]["prn"] if p > 0)
    ap = gps.coarse_config(x0 + 1500.0 * e + 750.0 * n, START_SOW + 0.5, 0, WEEK)
    res, P, rec, seed, cfg = run(iq, 1, eph, ap)
    # alone, at most 4 PRNs pass: the plain chain is FEW
    assert (res["ratio"] >= 2.5).sum() <= 4
    plain = S.measure(iq, 1, S0, K, res)
    sel = [int(np.nonzero(plain["prn"] == p)[0][0]) for p in prns]
    pf, _, _, _ = S.coarse(pvt_chans(eph, prns), plain[sel][None], gps.pvt_config(0, 1, 1, iono), ap)
    assert pf["status"][0] == gps.FIX_FEW
    # collectively: the truth, its cells, and a fix
    assert rec["status"] == CM.OK and rec["nused"] == 12, rec
    assert np.linalg.norm(rec["x"] - x0) <= bound(cfg) and abs(rec["o_t"] + 0.5) <= float(cfg["step"][3]), rec
    check_seeds(seed, ch, rec)
    m, fix = fix_from(seed, iq, 1, 0, eph, iono, rec, ap, prns)
    assert (m["status"][:12] == S.OK).all()
    assert fix["status"][0] == gps.FIX_OK and fix["nused"][0] == 12
    check_truth(fix, static_rows(ch, LOC), START_SOW, WEAK_POS, BOUNDS["time"], BOUNDS["vel"])


def test_model_on_sky32_static(tmp_path):
    g, ch, iq = block_stream("sky32_static_10s_i8", 0)
    eph, _ = ephemeris(tmp_path, 32, START_SOW)
    x0 = PM.llh_ecef(*LOC)
    e, _, _ = enu(x0)
    ap = gps.coarse_config(x0 + 1000.0 * e, START_SOW + 0.5, 0, WEEK)
    cfg = gps.collective_config(1500.0, 250.0, 0.5, 0.5, mask_deg=5.0, distinct_m=1000.0)
    res, P, rec, seed, cfg = run(iq, 1, eph, ap, cfg)
    assert rec["status"] == CM.OK and rec["nused"] >= 8, rec
    assert np.linalg.norm(rec["x"] - x0) <= bound(cfg) and abs(rec["o_t"] + 0.5) <= 0.5, rec
    check_seeds(seed, ch, rec)


def test_few_with_three_used_prns(tmp_path):
    _, ch, iq = block_stream("sky12_static_35s_i8", 0)
    eph, _ = ephemeris(tmp_path, 12, START_SOW)
    eph["valid"][3:] = 0
    ap = gps.coarse_config(PM.llh_ecef(*LOC), START_SOW, 0, WEEK)
    res, P, rec, seed, cfg = run(iq, 1, eph, ap, gps.collective_config(500.0, 250.0, mask_deg=-90.0))
    assert rec["status"] == CM.FEW and rec["nused"] == 3 and rec["used"] == 0b111 and rec["winner"] == -1
    assert np.isnan(rec["x"]).all() and (seed["ratio"] == -1.0).all()
    assert np.array_equal(seed[["prn", "bin", "delay", "p1", "p2"]], res[["prn", "bin", "delay", "p1", "p2"]])


def test_one_point_lattice(tmp_path):
    _, ch, iq = block_stream("sky12_static_35s_i8", 0)
    eph, _ = ephemeris(tmp_path, 12, START_SOW)
    x0 = PM.llh_ecef(*LOC)
    ap = gps.coarse_config(x0, START_SOW, 0, WEEK)
    cfg = gps.collective_config(0.0, 250.0)
    cfg["step"] = np.nan   # not read where n is 1
    assert (cfg["n"] == 1).all()
    res, P, rec, seed, _ = run(iq, 1, eph, ap, cfg)
    assert rec["status"] == CM.OK and rec["winner"] == 0 and rec["runner"] == -1 and np.isnan(rec["runner_dist"])
    assert np.array_equal(rec["x"], ap["x_a"]) and rec["o_t"] == 0.0
    check_seeds(seed, ch, rec)


def test_tie_rules(tmp_path):
    """A flat grid: every q is 2^8, every hypothesis and shift scores alike. The winner is hypothesis 0 at shift 0, the
    runner-up the lowest hypothesis beyond distinct_m, and the call AMBIGUOUS."""
    eph, _ = ephemeris(tmp_path, 12, START_SOW)
    prns = list(range(1, 13))
    P = np.ones((12, 5, A.CODE), np.uint64)
    res = A.reduce(P, prns, -500.0, 250.0)
    ap = gps.coarse_config(PM.llh_ecef(*LOC), START_SOW, 0, WEEK)
    cfg = gps.collective_config(1000.0, 500.0, 0.0, 1.0, mask_deg=-90.0, distinct_m=600.0)
    rec, seed, Sc, b, cells = CM.collective(P, res, eph, prns, ap, S0, cfg, np.full(12, -5000.0), 2500.0)
    on = (cells[..., 0] >= 0).sum(1)
    assert (Sc == 256 * on).all() and (b == 0).all()
    w = int(np.argmax(on))
    assert rec["winner"] == w and rec["shift"] == 0
    o = CM.offsets(cfg, np.arange(Sc.size))
    far = np.sqrt(((o[:, :3] - o[w, :3]) ** 2).sum(1)) > 600.0
    assert rec["runner"] == int(np.argmax(np.where(far, Sc.astype(np.int64), -1)))
    assert rec["status"] == CM.AMBIGUOUS


def test_model_on_the_int16_site(tmp_path):
    from test_snapshot import scene
    sc = scene("site_34s_58w_10s_i16", tmp_path)
    iq, r = sc["stream"](0)
    eph = np.zeros(32, gps.EPHEMERIS_DTYPE)
    for c in sc["chans"]:
        eph[int(c["prn"]) - 1] = c["eph"]
    x0 = sc["rows"][0]
    e, n, _ = enu(x0)
    ap = gps.coarse_config(x0 - 2000.0 * n, sc["sow"] + 0.5, 0, WEEK)
    res, P, rec, seed, cfg = run(iq, sc["ss"], eph, ap)
    assert rec["status"] == CM.OK and rec["nused"] >= 8, rec
    assert np.linalg.norm(rec["x"] - x0) <= bound(cfg) and abs(rec["o_t"] + 0.5) <= 0.5, rec
    check_seeds(seed, r, rec)
