"""Pooled collective detection on the numpy model (tests/collective_pool_model.py; DESIGN §11.8): one
lattice scored over several 10 ms windows of one static receiver, with one clock shift common to every window.

The stream is sky12_static_35s with the gain of PRNs 1-8 scaled by g in every block; window w starts at sample 1 000
of block w (K = 10, the standard grid of 32 PRNs x 41 bins), the lattice and a-priori are test_collective's weakened
ones. The figures below are the model's (DESIGN §11.8 has them for g from 0.03 to 0.12 and W up to 16):
- g = 0.12: the single window and the pool of 4 are OK at the truth's lattice point with the true time offset;
  runner-up / winner 0.8200 and 0.8352.
- g = 0.07: both are AMBIGUOUS, 0.9227 and 0.9280. Pooling does not separate the truth from its runner-up on these
  noise-free streams: the runner-up's score per window hardly changes from window to window, so it grows with W as the
  winner's does."""
import numpy as np
import pytest

import acq_model as A
import collective_model as CM
import collective_pool_model as CP
import pvt_model as PM
import scenario
from scenario import gps
from test_acquire import golden_rows
from test_coarse import WEEK, enu
from test_collective import FLO, PRNS, WEAK_PRNS, bound, ephemeris, lattice
from test_scenario import LOC
from test_snapshot import S0, K
from test_track import START_SOW

NWIN = 4
BLOCK = 300000
RATIO = {0.12: (0.8200, 0.8352), 0.07: (0.9227, 0.9280)}   # runner-up / winner at W = 1 and W = NWIN


def pooled_stream(g, nwin, gain):
    ch = golden_rows(g, list(range(nwin)))
    for b in range(nwin):
        for c in range(ch.shape[1]):
            if int(ch[b, c]["prn"]) in WEAK_PRNS:
                ch[b, c]["gain"] *= gain
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], int(g["sample_size"]))
    return ch, iq


@pytest.fixture(scope="module", params=sorted(RATIO))
def windows(request, tmp_path_factory):
    gain = request.param
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, iq = pooled_stream(g, NWIN, gain)
    s0 = [S0 + w * BLOCK for w in range(NWIN)]
    found = [A.search(iq, 1, s, K, PRNS, want_grid=True) for s in s0]
    eph, iono = ephemeris(tmp_path_factory.mktemp("nav"), 12, START_SOW)
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    ap = gps.coarse_config(x0 + 1500.0 * e + 750.0 * n, START_SOW + 0.5, 0, WEEK)
    return dict(gain=gain, ch=ch, s0=s0, res=[f[0] for f in found], P=[f[1] for f in found], eph=eph, ap=ap, x0=x0,
                memo={})


def pool(wd, order):
    """The pooled call on the windows in `order` (memoised per fixture: each pool scores 5 887 hypotheses per window)."""
    key = tuple(order)
    if key not in wd["memo"]:
        wd["memo"][key] = _pool(wd, key)
    return wd["memo"][key]


def _pool(wd, order):
    return CP.collective_pool([wd["P"][w] for w in order], [wd["res"][w] for w in order], wd["eph"], PRNS, wd["ap"],
                              [wd["s0"][w] for w in order], lattice(), FLO, 250.0)


def ratio(rec):
    return float(rec["runner_score"]) / float(rec["score"])


def test_one_window_is_the_single_call(windows):
    wd = windows
    rec, seed, S, b, cells = pool(wd, [0])
    r1, s1, S1, b1, c1 = CM.collective(wd["P"][0], wd["res"][0], wd["eph"], PRNS, wd["ap"], wd["s0"][0], lattice(), FLO,
                                       250.0)
    assert rec.tobytes() == r1.tobytes()
    assert seed.shape == (1, len(PRNS)) and seed[0].tobytes() == s1.tobytes()
    assert np.array_equal(S, S1) and np.array_equal(b, b1) and np.array_equal(cells[0], c1)


def test_pooled_scores_are_the_sum_of_the_windows(windows):
    """S(h, b) adds over the windows at one common b: S_h of the pool is at least each window's S(h, b_h)."""
    wd = windows
    rec, _, S, b, cells = pool(wd, range(NWIN))
    qs = [CM.normalise(P)[1] for P in wd["P"]]
    h = np.array([int(rec["winner"]), int(rec["runner"])])
    total = np.zeros(2, np.int64)
    for w in range(NWIN):
        one, _ = CP.score_pool([qs[w]], cells[w:w + 1, h])
        Sw = np.zeros(2, np.int64)
        for p in range(len(PRNS)):
            j, d = cells[w, h, p, 0], cells[w, h, p, 1]
            on = j >= 0
            Sw[on] += qs[w][p][j[on], (d[on] + b[h][on]) % CM.CODE]
        assert (Sw <= one).all()
        total += Sw
    assert np.array_equal(total, S[h].astype(np.int64))


def test_the_truth_and_the_runner_up(windows):
    wd = windows
    cfg = lattice()
    single, _, _, _, _ = pool(wd, [0])
    rec, seed, _, _, _ = pool(wd, range(NWIN))
    want1, want = RATIO[wd["gain"]]
    assert abs(ratio(single) - want1) < 5e-5 and abs(ratio(rec) - want) < 5e-5, (ratio(single), ratio(rec))
    assert ratio(rec) >= ratio(single)
    status = CM.OK if want < CM.AMBIGUOUS_PCT / 100.0 else CM.AMBIGUOUS
    assert single["status"] == status and rec["status"] == status
    for r in (single, rec):
        assert r["nused"] == 12 and abs(r["o_t"] + 0.5) < 1e-12
        assert np.linalg.norm(r["x"] - wd["x0"]) <= bound(cfg), r
    # every window's seeds: the truth's sample and bin
    for w in range(NWIN):
        held = {int(c["prn"]): c for c in wd["ch"][w] if c["prn"] > 0}
        for p, s in enumerate(seed[w]):
            if not (int(rec["used"]) >> p) & 1:
                assert s["ratio"] == -1.0
                continue
            if int(s["prn"]) not in held:
                continue
            f, tau = A.truth(held[int(s["prn"])], S0)
            assert A.circ_dist(s["delay"], int(np.rint(tau)) % A.CODE) <= 2, (w, s["prn"], s["delay"], tau)
            assert abs(s["doppler_hz"] - f) <= 125.0 + 1e-9, (w, s["prn"], s["doppler_hz"], f)


def test_window_order_does_not_matter(windows):
    wd = windows
    rec, seed, S, b, _ = pool(wd, range(NWIN))
    rev, rseed, rS, rb, _ = pool(wd, list(reversed(range(NWIN))))
    assert rev.tobytes() == rec.tobytes() and np.array_equal(rS, S) and np.array_equal(rb, b)
    assert rseed[::-1].tobytes() == seed.tobytes()
    # a repeated window counts twice, and the winner stays
    rep, _, _, _, _ = pool(wd, [0, 1, 1, 2, 3])
    assert rep["winner"] == rec["winner"] and rep["shift"] == rec["shift"]


def test_few_over_every_window(windows):
    wd = windows
    eph = wd["eph"].copy()
    eph["valid"][3:] = 0
    rec, seed, S, b, cells = CP.collective_pool(wd["P"], wd["res"], eph, PRNS, wd["ap"], wd["s0"],
                                                gps.collective_config(500.0, 250.0, mask_deg=-90.0), FLO, 250.0)
    assert rec["status"] == CM.FEW and rec["nused"] == 3 and rec["used"] == 0b111 and rec["winner"] == -1
    assert (seed["ratio"] == -1.0).all() and (S == 0).all() and (cells == -1).all()
    for w in range(NWIN):
        assert np.array_equal(seed[w][["prn", "bin", "delay", "p1", "p2"]], wd["res"][w][["prn", "bin", "delay", "p1", "p2"]])
