"""Collective detection, the snapshot measurement, snapshot batches and tracking on the GPU at the edges of their
contracts. Every call is compared with its numpy model byte for byte (collective detection through test_collective_gpu's
check_against_model, the measurement against snapshot_model.measure, batches against the single calls, tracking against
track_model.track), and each test asserts that its run reached the edge it is about: lattices collective_config never
builds (even sizes, n_e != n_n, up offsets, 1 to 1025 hypotheses), one Doppler bin, all-zero scores (the tie rules on
the device), per-PRN power sums above 2^64, the used-PRN rules at their limits, 0 and 16 code iterations, +-10 kHz,
ratios at min_ratio, code phases that wrap, data-bit flips, full-scale windows at K = 100, windows of zeros, one window
per batch pass, and a tracking loop coasting through zeros."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import acq_model as A
import collective_model as CM
import pvt_model as PM
import scenario
import snapshot_model as S
import track_model as T
from scenario import gps
from test_coarse import WEEK
from test_collective import ephemeris
from test_collective_gpu import check_against_model
from test_receiver_edges import full_scale, planted
from test_scenario import LOC
from test_snapshot import S0, K, block_stream
from test_stage_edges import FREQ_BOUND, flipped, max_e_plus_l, phase_trace, result, true_step
from test_track import START_SOW

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    with gps.Context(12, 4) as c:
        yield c


@pytest.fixture(scope="module")
def sky(tmp_path_factory):
    eph, _ = ephemeris(tmp_path_factory.mktemp("nav"), 12, START_SOW)
    eph32, _ = ephemeris(tmp_path_factory.mktemp("nav32"), 32, START_SOW)
    return eph, eph32


@pytest.fixture(scope="module")
def block0():
    return block_stream("sky12_static_35s_i8", 0)[2]


def raw_config(n, step=(150.0, 150.0, 100.0, 0.5), mask_deg=-90.0, distinct_m=300.0):
    """A COLLECTIVE_CONFIG record as it stands, not collective_config's odd square lattices."""
    c = np.zeros(1, gps.COLLECTIVE_CONFIG_DTYPE)[0]
    c["n"], c["step"], c["mask_deg"], c["distinct_m"] = n, step, mask_deg, distinct_m
    return c


def apriori(t_a=START_SOW):
    """The a-priori at the receiver, at s_a = S0: the window's time t0 is t_a exactly."""
    return gps.coarse_config(PM.llh_ecef(*LOC), t_a, S0, WEEK)


# ---- collective detection -------------------------------------------------------------------------------------------
LATTICES = [[1, 1, 1, 1], [3, 5, 1, 1], [4, 4, 1, 1], [17, 1, 1, 1], [11, 31, 3, 1], [8, 8, 4, 4], [5, 5, 1, 41],
            [2, 6, 4, 2]]


@pytest.mark.parametrize("n", LATTICES, ids=lambda n: "x".join(map(str, n)))
def test_raw_lattices_equal_the_model(ctx, sky, block0, n):
    """nhyp 1, 15, 16, 17, 1023, 1024, 1025 and 96: half-step offsets (even n), n_e != n_n (the axis order of the
    decomposition of h), up offsets (n_u 3 and 4: the U term of the position and du of runner_dist), partial tiles."""
    cfg = raw_config(n)
    _, _, rec = check_against_model(ctx, block0, gps.SC08, list(range(1, 33)), sky[0], apriori(), cfg)
    nhyp = int(np.prod(n))
    assert rec["nused"] == 12 and 0 <= rec["winner"] < nhyp
    o = CM.offsets(cfg, np.arange(nhyp))
    if n[0] % 2 == 0:
        assert (o[:, 0] % 150.0 != 0).all()                       # every east offset a half step
    if n[2] > 1:
        assert np.unique(o[:, 2]).size == n[2]


def test_one_bin_puts_every_prn_in_bin_0(ctx, sky, block0):
    cfg = raw_config([5, 3, 1, 3])
    _, _, rec = check_against_model(ctx, block0, gps.SC08, list(range(1, 33)), sky[0], apriori(), cfg, nbins=1,
                                    f_lo=2000.0)
    tb = ctx.collective(sky[0], apriori(), cfg, iq=block0, ms=K, s0=S0, nbins=1, f_lo=2000.0, want_table=True)[3]
    used = (int(rec["used"]) >> np.arange(32)) & 1 == 1
    assert rec["nused"] == 12 and (tb["bin"][:, used] == 0).all() and (tb["bin"][:, ~used] == -1).all()


def test_all_zero_scores_follow_the_tie_rules(ctx, sky, block0):
    """Every PRN's window 9-10 kHz, far above every prediction: every cell is off the grid and every score 0. The
    device's shuffle keeps the lowest shift (0) and the pick the lowest h: winner 0, runner-up the first h beyond
    distinct_m, AMBIGUOUS at 0 >= 0, every seed ratio -1."""
    cfg = raw_config([4, 4, 1, 1])
    flo = np.full(32, 9000.0)
    _, seed, rec = check_against_model(ctx, block0, gps.SC08, list(range(1, 33)), sky[0], apriori(), cfg, f_lo_prn=flo,
                                       nbins=5)
    sc = ctx.collective(sky[0], apriori(), cfg, iq=block0, ms=K, s0=S0, f_lo_prn=flo, nbins=5, want_scores=True)[3]
    assert rec["nused"] == 12 and (sc["score"] == 0).all() and (sc["shift"] == 0).all()
    o = CM.offsets(cfg, np.arange(16))
    far = np.nonzero(np.sqrt(((o[:, :3] - o[0, :3]) ** 2).sum(1)) > 300.0)[0]
    assert rec["winner"] == 0 and rec["shift"] == 0 and rec["runner"] == far[0] and rec["status"] == gps.CD_AMBIGUOUS
    assert (seed["ratio"] == -1.0).all()


def prn_sums(P):
    """Each PRN's exact power sum (Python ints) over its grid, from its low and high 32-bit halves."""
    m = np.uint64(0xffffffff)
    return [int((P[p] & m).sum(dtype=np.uint64)) + (int((P[p] >> np.uint64(32)).sum(dtype=np.uint64)) << 32)
            for p in range(P.shape[0])]


@pytest.mark.parametrize("nbins", [41, 1024])
def test_normalisation_sums_beyond_64_bits(ctx, sky, nbins):
    """Saturating int16 at K = 100: every PRN's power sum exceeds 2^64 (measured: about 7e19 at 41 bins, 1.6e21 at
    1024), so the 128-bit carry of the sums and the 128-bit division of mu decide the q rows and the scores."""
    ms = 100
    rng = np.random.default_rng(nbins)
    n = S0 + gps.acq_window_samples(ms) + 10
    iq = rng.integers(-32768, 32768, 2 * n, dtype=np.int16)
    prns = [3, 11, 19, 24, 30]
    cfg = raw_config([3, 4, 1, 1])
    _, P = ctx.acquire(iq, gps.SC16, prns, ms=ms, s0=S0, nbins=nbins, want_grid=True)
    sums = prn_sums(P)
    assert min(sums) > 2 ** 64, [float(s) for s in sums]
    _, _, rec = check_against_model(ctx, iq, gps.SC16, prns, sky[1], apriori(), cfg, nbins=nbins, ms=ms)
    assert rec["nused"] == 5 and rec["score"] > 0


def test_used_prn_rules_at_their_limits(ctx, sky, block0):
    """t0 = 7200 s exactly. PRN 1 invalid, PRN 2 unhealthy, PRN 3 at toe 0 (|t0 - toe| exactly 7200: used), PRN 4 at
    toe 14400 (exactly 7200 ahead: used), PRN 5 at toe 14400.001 (just past: not used). Then t0 = 1800 s with PRN 6's
    toe 601200 (5400 s back across the week wrap: used) and PRN 7's 593000 (13600 s: not used)."""
    eph = sky[0].copy()
    eph[0]["valid"] = 0
    eph[1]["health"] = 1
    eph[2]["toe"], eph[3]["toe"], eph[4]["toe"] = 0.0, 14400.0, 14400.001
    cfg = raw_config([3, 3, 1, 1])
    _, _, rec = check_against_model(ctx, block0, gps.SC08, list(range(1, 33)), eph, apriori(), cfg)
    used = [(int(rec["used"]) >> p) & 1 for p in range(12)]
    assert used[:5] == [0, 0, 1, 1, 0] and all(used[5:])
    eph = sky[0].copy()
    eph[5]["toe"], eph[6]["toe"] = 601200.0, 593000.0
    _, _, rec = check_against_model(ctx, block0, gps.SC08, list(range(1, 33)), eph, apriori(1800.0), cfg)
    used = [(int(rec["used"]) >> p) & 1 for p in range(12)]
    assert used[5] == 1 and used[6] == 0


def test_largest_lattice_against_sampled_model_scores(ctx, sky, block0):
    """2^24 hypotheses (GPSB200_CD_MAX_HYP), 12 used PRNs, scores without a table: the model scores about 4 000 h
    (every tile edge of the first tiles, the last h, the winner, the runner-up, random h) on its own table, and the
    pick is recomputed from the device's whole score array in chunks."""
    cfg = raw_config([256, 256, 16, 16], step=(40.0, 40.0, 60.0, 0.1), distinct_m=300.0)
    nhyp = gps.CD_MAX_HYP
    assert int(np.prod(cfg["n"])) == nhyp
    prns = list(range(1, 33))
    res, P = ctx.acquire(block0, gps.SC08, prns, ms=K, s0=S0, want_grid=True)
    _, _, rec, sc = ctx.collective(sky[0], apriori(), cfg, iq=block0, ms=K, s0=S0, want_scores=True)
    assert rec["nused"] == 12 and sc.size == nhyp
    mu, q = CM.normalise(P)
    use = CM.used(sky[0], prns, apriori(), S0, cfg["mask_deg"], mu)
    rng = np.random.default_rng(24)
    edges = np.concatenate([np.arange(0, 2048, 16), np.arange(15, 2048, 16)])
    h = np.unique(np.concatenate([edges, [nhyp - 1, nhyp - 16, rec["winner"], rec["runner"]],
                                  rng.integers(0, nhyp, 3700)]))
    cells, dc, jc = CM.table(sky[0], prns, use, apriori(), S0, cfg, np.full(32, -5000.0), 250.0, 41, h)
    near = ((np.abs(dc - np.floor(dc) - 0.5) < 1e-6) | (np.abs(jc - np.floor(jc) - 0.5) < 1e-6)).any(1)
    Sm, bm = CM.score(q, cells)
    ok = ~near
    assert ok.sum() > 3900
    assert np.array_equal(sc["score"][h][ok], Sm[ok]) and np.array_equal(sc["shift"][h][ok], bm[ok])
    # the pick from the whole array, in chunks of 2^20
    best, win = -1, -1
    for c in range(0, nhyp, 1 << 20):
        s = sc["score"][c:c + (1 << 20)]
        k = int(np.argmax(s))
        if int(s[k]) > best:
            best, win = int(s[k]), c + k
    wo = CM.offsets(cfg, [win])[0]
    rbest, run = -1, -1
    for c in range(0, nhyp, 1 << 20):
        o = CM.offsets(cfg, np.arange(c, min(nhyp, c + (1 << 20))))
        far = np.sqrt(((o[:, :3] - wo[:3]) ** 2).sum(1)) > 300.0
        s = np.where(far, sc["score"][c:c + (1 << 20)].astype(np.int64), -1)
        k = int(np.argmax(s))
        if s[k] > rbest:
            rbest, run = int(s[k]), c + k
    assert (rec["winner"], rec["score"], rec["runner"], rec["runner_score"]) == (win, best, run, rbest)
    assert rec["shift"] == sc["shift"][win]


# ---- snapshot measurement -------------------------------------------------------------------------------------------
def measure_both(ctx, iq, ss, K_, res, min_ratio=2.5, iterations=gps.SNAP_ITERATIONS):
    """The device's records of res over the window of K_ chunks from sample 0, equal to the model's; -> records."""
    got = ctx.snapshot_measure(res, iq, ss, ms=K_, s0=0, cfg=gps.snapshot_config(min_ratio, iterations))
    want = S.measure(iq, ss, 0, K_, res, min_ratio=min_ratio, iterations=iterations)
    assert got.tobytes() == want.tobytes()
    return got


def window(K_, sigs, ss=gps.SC08):
    return planted(gps.acq_window_samples(K_), sigs, ss)


SIGS = [(7, 1234.5, 1234, 40), (13, -3100.0, 17, 30), (22, 4020.0, 2950, 30)]


def results(sigs, off=(0.0, 125.0, -240.0), ratio=10.0):
    r = np.concatenate([result(p, f + o, d, ratio) for (p, f, d, _), o in zip(sigs, off)])
    return r


@pytest.mark.parametrize("iterations", [0, 16])
def test_zero_and_sixteen_iterations(ctx, iterations):
    rec = measure_both(ctx, window(10, SIGS), gps.SC08, 10, results(SIGS), iterations=iterations)
    assert (rec["iterations"] == iterations).all() and (rec["status"] == gps.SNAP_OK).all()
    if iterations == 0:
        assert (rec["last_step"] == 0).all() and (rec["power"] > 0).all()


@pytest.mark.parametrize("f", [10000.0, -10000.0])
def test_doppler_at_the_accepted_limit(ctx, f):
    sigs = [(5, f, 321, 60)]
    rec = measure_both(ctx, window(10, sigs), gps.SC08, 10, results(sigs, off=(0.0,)))
    assert rec["status"][0] == gps.SNAP_OK and abs(int(rec["carr_step"][0]) - true_step(f)) <= FREQ_BOUND[10]


def test_ratios_at_the_threshold(ctx):
    """Ratios min_ratio, the next double below it, NaN, -1 and infinity: OK, WEAK, WEAK, WEAK, OK."""
    sigs = [(p, 1000.0 * i - 2000.0, 300 * i + 5, 30) for i, p in enumerate((2, 9, 16, 23, 31))]
    res = results(sigs, off=(0.0,) * 5)
    res["ratio"] = [2.5, np.nextafter(2.5, 0.0), np.nan, -1.0, np.inf]
    rec = measure_both(ctx, window(2, sigs), gps.SC08, 2, res)
    assert list(rec["status"]) == [gps.SNAP_OK, gps.SNAP_WEAK, gps.SNAP_WEAK, gps.SNAP_WEAK, gps.SNAP_OK]


@pytest.mark.parametrize("seed_delay,true_delay,crosses", [(0, 1, "zero"), (1, 0, "M")])
def test_code_phase_wraps(ctx, seed_delay, true_delay, crosses):
    sigs = [(7, 1234.5, true_delay, 60)]
    res = result(7, 1234.5, seed_delay)
    rec = measure_both(ctx, window(10, sigs), gps.SC08, 10, res, iterations=16)
    tr = []
    S.measure(window(10, sigs), gps.SC08, 0, 10, res, iterations=16, trace=tr)
    raw = phase_trace(res[0], tr[0])
    assert (min(raw) < 0) if crosses == "zero" else (max(raw) >= S.M)
    assert rec["status"][0] == gps.SNAP_OK


def test_data_bit_flips(ctx):
    K_ = 10
    iq = window(K_, SIGS)
    body = flipped(iq[:2 * 3000 * K_], K_, np.arange(K_) % 3 == 1)
    iqf = np.concatenate([body, iq[2 * 3000 * K_:]])
    a = measure_both(ctx, iqf, gps.SC08, K_, results(SIGS))
    assert a.tobytes() == measure_both(ctx, iq, gps.SC08, K_, results(SIGS)).tobytes()


@pytest.mark.parametrize("ss", [gps.SC08, gps.SC16])
def test_full_scale_window_at_k_100(ctx, ss):
    """The largest sums the contract allows in practice: E + L above 4.6e17 (int8) and 7.5e17 (int16) on the model's
    trace, power 8.6e17 / 1.39e18 (tests/test_stage_edges.py measured them)."""
    K_ = 100
    iq = full_scale(gps.acq_window_samples(K_), 13, 1750.0, ss, delay=1234)
    res = result(13, 1750.0, 1234)
    rec = measure_both(ctx, iq, ss, K_, res, iterations=16)
    tr = []
    S.measure(iq, ss, 0, K_, res, iterations=16, trace=tr)
    el = max_e_plus_l(iq, ss, K_, res[0], rec[0], tr[0])
    lo = {gps.SC08: (8.5e17, 4.6e17), gps.SC16: (1.38e18, 7.5e17)}[ss]
    assert int(rec["power"][0]) >= lo[0] and el >= lo[1]


def test_window_of_zeros(ctx):
    """Zeros, an infinite ratio: OK records with w, u and the phase of the seed, D = 0 and power 0 (angle(0, 0) = 0)."""
    K_ = 10
    iq = np.zeros(2 * gps.acq_window_samples(K_), np.int8)
    res = results(SIGS, ratio=np.inf)
    rec = measure_both(ctx, iq, gps.SC08, K_, res)
    for r, m in zip(res, rec):
        w, u, phi = S.seed(r, 0)
        assert (int(m["carr_step"]), int(m["code_step"]), int(m["code_phase"])) == (w, u, phi)
    assert (rec["status"] == gps.SNAP_OK).all() and (rec["power"] == 0).all() and (rec["last_step"] == 0).all()


# ---- snapshot batches -----------------------------------------------------------------------------------------------
def batch_vs_singles(ctx, iq, ss, s0, prns, K_, nbins, cfg, step=250.0, device=False):
    """A batch on the standard grid from -5 kHz at `step` against its single calls (every bin within the measurement's
    +-10 kHz); -> the batch's (results, records)."""
    want_res = np.zeros((len(s0), len(prns)), gps.ACQ_RESULT_DTYPE)
    want_out = np.zeros((len(s0), len(prns)), gps.SNAPSHOT_DTYPE)
    for w, s in enumerate(s0):
        want_res[w] = ctx.acquire(iq, ss, prns, ms=K_, s0=int(s), step=step, nbins=nbins)
        want_out[w] = ctx.snapshot_measure(want_res[w], iq, ss, ms=K_, s0=int(s), step=step, nbins=nbins, cfg=cfg)
    src = dict(iq=iq)
    if device:
        d = torch.from_numpy(iq.copy()).cuda()
        torch.cuda.synchronize()
        src = dict(device_ptr=d.data_ptr(), nsamples=iq.size // 2)
    got = ctx.snapshot_batch(s0, sample_size=ss, prns=prns, ms=K_, step=step, nbins=nbins, cfg=cfg, **src)
    assert got[0].tobytes() == want_res.tobytes() and got[1].tobytes() == want_out.tobytes()
    return got


def test_batch_of_one_window_per_pass(ctx):
    """32 PRNs x 1024 bins: one window's scratch exceeds the cap, so each pass holds one window."""
    assert gps.snapshot_batch_pass(32, 1024, 1) == 1
    sigs = [(7, 1234.5, 1234, 40), (13, -3100.0, 17, 30)]
    iq = planted(gps.acq_window_samples(1) + 5000, sigs, gps.SC08, noise=20, seed=1)
    _, out = batch_vs_singles(ctx, iq, gps.SC08, [0, 4321], list(range(1, 33)), 1, 1024, gps.snapshot_config(),
                              step=10.0)
    assert (out["status"] == gps.SNAP_OK).sum() >= 2


@pytest.mark.parametrize("extra", [0, 1])
def test_batch_of_p_and_p_plus_one_windows(ctx, extra):
    p = gps.snapshot_batch_pass(32, 100, 1)
    assert p == 3
    iq = planted(gps.acq_window_samples(1) + 9000, SIGS, gps.SC08, noise=20, seed=2)
    s0 = np.arange(p + extra) * 1999
    batch_vs_singles(ctx, iq, gps.SC08, s0, list(range(1, 33)), 1, 100, gps.snapshot_config(), step=100.0)


@pytest.mark.parametrize("device", [False, True])
def test_batch_of_k_100_int16_windows(ctx, device):
    sigs = [(7, -4500.0, 1234, 40), (13, -4250.0, 17, 30)]    # inside the 5 bins from -5 kHz
    iq = planted(gps.acq_window_samples(100) + 7000, sigs, gps.SC16, noise=40, seed=3)
    _, out = batch_vs_singles(ctx, iq, gps.SC16, [0, 6999, 3000], [7, 13, 20], 100, 5, gps.snapshot_config(),
                              device=device)
    assert (out["status"][:, :2] == gps.SNAP_OK).all()


# ---- tracking through a gap ----------------------------------------------------------------------------------------
def test_track_coasts_through_zeros(ctx):
    """A channel past its FLL epochs tracks 20 periods of a planted signal, then 20 periods of zeros: kernel and model
    agree, and from the second period of zeros on carr_freq, carr_step and code_step stay constant (the PLL term
    angle(0, 0) is 0; before, F drifted by -0.2 Hz per period)."""
    n_sig, n_gap = 20 * 3000, 20 * 3000
    iq = np.concatenate([planted(n_sig, [(7, 1234.5, 1234, 60)], gps.SC08), np.zeros(2 * n_gap, np.int8)])
    st = T.start(7, 1234.5, 1234)
    st["epochs"] = T.FLL_EPOCHS
    eps, after = ctx.track(np.array([st], gps.TRACK_STATE_DTYPE), iq, gps.SC08)
    want, wafter = T.track(iq, gps.SC08, 0, np.array([st], T.STATE_DTYPE))
    assert eps[0].tobytes() == want[0].astype(gps.TRACK_EPOCH_DTYPE).tobytes()
    assert after.tobytes() == wafter.astype(gps.TRACK_STATE_DTYPE).tobytes()
    e = eps[0]
    gap = e["sample"] >= n_sig
    assert gap.sum() >= 18 and (e["p_i"][gap] == 0).all()
    g = np.nonzero(gap)[0][1:]
    assert np.unique(e["carr_step"][g]).size == 1 and np.unique(e["code_step"][g]).size == 1
    assert int(after["carr_freq"][0]) >> 10 == int(e["carr_step"][g[0]])


# ---- memcheck -------------------------------------------------------------------------------------------------------
def sanitizer_run():
    """The small shapes that move indexing: a one-hypothesis lattice, one bin, 16 iterations, K = 100 -> a digest."""
    import hashlib
    import pathlib
    import tempfile
    iq = block_stream("sky12_static_35s_i8", 0)[2]
    eph, _ = ephemeris(pathlib.Path(tempfile.mkdtemp()), 12, START_SOW)
    h = hashlib.sha256()
    with gps.Context(12, 1) as c:
        for a in c.collective(eph, apriori(), raw_config([1, 1, 1, 1]), iq=iq, prns=range(1, 13), nbins=1,
                              want_scores=True, want_table=True):
            h.update(np.asarray(a).tobytes())
        w = full_scale(gps.acq_window_samples(100) + 100, 13, 1750.0, gps.SC16, delay=1234)
        h.update(c.snapshot_measure(result(13, 1750.0, 1234), w, gps.SC16, ms=100, s0=0,
                                    cfg=gps.snapshot_config(2.5, 16)).tobytes())
        for a in c.snapshot_batch([0, 100], w, gps.SC16, [13, 14], ms=100, nbins=1, cfg=gps.snapshot_config(0.0, 16)):
            h.update(a.tobytes())
    return h.hexdigest()


def test_small_shapes_clean_under_compute_sanitizer():
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_stage_edges_gpu as T; "
            "print('ok', T.sanitizer_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0, plain.stderr[-2000:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1200)
    from test_coarse_gpu import _device_not_supported
    if _device_not_supported(r):
        assert sanitizer_run() == plain.stdout.split()[-1]
        torch.cuda.synchronize()
        return
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert r.stdout.split()[-1] == plain.stdout.split()[-1]
