"""Snapshot measurement and fixes on the GPU (gpsb200_snapshot_measure, gpsb200_pvt_snapshot,
gpsb200_pvt_snapshot_search; DESIGN §11.5): bit for bit against the numpy model (tests/snapshot_model.py), the fixes
against the tracked-epoch calls they must equal, and the whole chain from the I/Q stream to a position on
sky12_static_35s against the scenario's truth, with the bounds of tests/test_snapshot.py."""
import ctypes as C

import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import pvt_truth as PT
import scenario
import snapshot_model as S
from scenario import gps
from test_acquire import golden_rows
from test_coarse import apriori, offsets, static_rows, unanchored
from test_pvt import ideal_inputs, rinex
from test_scenario import LOC
from test_search import search_cfg
from test_snapshot import BOUNDS, S0, SCENE_BOUNDS, K as K_CHAIN
from test_track import START_SOW

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    with gps.Context(12, 4) as c:
        yield c


def fake_results(prns, rng, ratio=10.0):
    res = np.zeros(len(prns), gps.ACQ_RESULT_DTYPE)
    res["prn"] = prns
    res["delay"] = rng.integers(0, 3000, len(prns))
    res["doppler_hz"] = rng.uniform(-5000.0, 5000.0, len(prns))
    res["ratio"] = ratio
    return res


@pytest.mark.parametrize("kind", ["int8_random", "int16_saturating"])
@pytest.mark.parametrize("K,nprn", [(1, 12), (2, 32), (10, 12), (100, 1)])
def test_measure_equals_model_on_random_input(ctx, kind, K, nprn):
    rng = np.random.default_rng(K * 100 + nprn)
    n = 3000 * K + 2999 + 17
    if kind == "int8_random":
        iq, ss = rng.integers(-128, 128, 2 * n).astype(np.int8), gps.SC08
    else:
        iq, ss = rng.choice(np.array([-32768, -32767, -2049, 2047, 32767, 0, 5000], np.int16), 2 * n), gps.SC16
    prns = list(rng.choice(np.arange(1, 33), nprn, replace=False))
    res = fake_results(prns, rng)
    res["ratio"][::3] = 2.0   # below the threshold: WEAK, never refined
    got = ctx.snapshot_measure(res, iq, ss, ms=K, s0=17)
    want = S.measure(iq, ss, 17, K, res, iterations=gps.SNAP_ITERATIONS)
    assert got.tobytes() == want.tobytes()
    assert (got["status"][::3] == gps.SNAP_WEAK).all()


@pytest.fixture(scope="module")
def sky12_block():
    g = scenario.load_golden("sky12_static_35s_i8")
    ch = golden_rows(g, [50])
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], 1)
    return g, ch, iq


@pytest.mark.parametrize("K", [1, 2, 10])
def test_measure_equals_model_on_a_signal(ctx, sky12_block, K):
    """All 32 PRNs searched on the GPU, measured by both paths (host buffer, device buffer in place) and the model."""
    _, ch, iq = sky12_block
    res = ctx.acquire(iq, gps.SC08, range(1, 33), ms=K, s0=S0)
    got = ctx.snapshot_measure(res, iq, gps.SC08, ms=K, s0=S0)
    want = S.measure(iq, 1, S0, K, res, iterations=gps.SNAP_ITERATIONS)
    assert got.tobytes() == want.tobytes()
    dev = torch.from_numpy(iq.copy()).cuda()
    torch.cuda.synchronize()
    got_d = ctx.snapshot_measure(res, None, gps.SC08, ms=K, s0=S0, device_ptr=dev.data_ptr(), nsamples=iq.size // 2)
    assert got_d.tobytes() == got.tobytes()
    present = {int(p) for p in ch[0]["prn"] if p > 0}
    assert all((r["status"] == gps.SNAP_WEAK) == (int(r["prn"]) not in present) for r in got)


def snapshots_from_epochs(chans, eps, samples):
    """Snapshot records of ideal epochs at the given instants: the phase at s on the code step of the period holding
    it, and that period's carrier step (gpsb200_pvt_coarse's measurement, as records). The phase is left unreduced
    (phi' + (s - sample) u can pass 1023 * 2^32, outside a measured record's range) on purpose: frac is then the very
    double gpsb200_pvt_coarse forms, so the two calls can agree byte for byte."""
    out = np.zeros((len(samples), len(eps)), gps.SNAPSHOT_DTYPE)
    for c, e in enumerate(eps):
        smp = e["sample"].astype(np.int64)
        for i, s in enumerate(samples):
            k = int(np.searchsorted(smp, s, side="right") - 1)
            r = out[i, c]
            r["prn"], r["sample"], r["status"] = chans[c]["prn"], s, gps.SNAP_OK
            r["code_phase"] = int(e["code_phase"][k - 1]) + (int(s) - int(smp[k])) * int(e["code_step"][k - 1])
            r["code_step"], r["carr_step"] = e["code_step"][k - 1], e["carr_step"][k - 1]
    return out


@pytest.fixture(scope="module")
def ideal(tmp_path_factory):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path_factory.mktemp("nav"), 12)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    return ch, unanchored(chans), eps, iono


def test_snapshot_fixes_equal_the_tracked_calls(ctx, ideal):
    """Records built from the epochs give gpsb200_pvt_coarse's records byte for byte, and gpsb200_pvt_search's."""
    ch, chans, eps, iono = ideal
    rows = static_rows(ch, LOC)
    cfg = gps.pvt_config(30000, 1499993, 20, iono)
    samples = [int(cfg["s0"]) + i * int(cfg["step"]) for i in range(20)]
    meas = snapshots_from_epochs(chans, eps, samples)
    for off in offsets(rows[0]):
        ap = apriori(rows[0], START_SOW, off)
        want = ctx.pvt_coarse(chans, eps, cfg, ap, want_residuals=True, want_ms=True)
        got = ctx.pvt_snapshot(chans, meas, cfg, ap, want_residuals=True, want_ms=True)
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes()
    three = gps.pvt_config(30000, 14999965, 3, iono)
    meas3 = snapshots_from_epochs(chans, eps, [int(three["s0"]) + i * int(three["step"]) for i in range(3)])
    sc = search_cfg(START_SOW, 10.0)
    want = ctx.pvt_search(chans, eps, three, sc, want_residuals=True, want_ms=True)
    got = ctx.pvt_snapshot_search(chans, meas3, three, sc, want_residuals=True, want_ms=True)
    for a, b in zip(got, want):
        assert a.tobytes() == b.tobytes()
    assert (got[0]["status"] == gps.FIX_OK).all()


def test_snapshot_fixes_equal_the_model(ctx, ideal, sky12_block):
    """Fixes from measured records against the model's solve on the same records."""
    ch, chans, eps, iono = ideal
    g, _, iq = sky12_block
    prns = [int(p) for p in chans["prn"]]
    res = ctx.acquire(iq, gps.SC08, prns, ms=K_CHAIN, s0=S0)
    m = ctx.snapshot_measure(res, iq, gps.SC08, ms=K_CHAIN, s0=S0)
    m["sample"] += 50 * PT.BLOCK
    meas = m[None, :]
    rows = static_rows(ch, LOC)
    cfg = gps.pvt_config(0, 1, 1, iono)
    for off in offsets(rows[0]):
        ap = apriori(rows[0], START_SOW, off)
        fix, co, res_, ms = ctx.pvt_snapshot(chans, meas, cfg, ap, want_residuals=True, want_ms=True)
        wfix, wco, wres, wms = S.coarse(chans, meas, cfg, ap)
        assert (fix["status"] == wfix["status"]).all() and np.array_equal(ms, wms)
        for f in ("x", "y", "z", "clock_m"):
            assert np.abs(fix[f] - wfix[f]).max() < 1e-6, f
        for f in ("vx", "vy", "vz"):
            assert np.abs(fix[f] - wfix[f]).max() < 1e-6, f
        assert np.abs(co["delta"] - wco["delta"]).max() < 1e-9


def test_whole_chain_on_sky12_static(ctx, ideal):
    """20 snapshots spread over 34 s: acquire (cold: the whole grid; per-PRN windows: 5 bins around each cold peak,
    as a warm start searches around its predictions), measure both results (the same records: the window holds the
    peak's row), fix from the 50 km / +10 s a-priori, then search with no position. Every fix within the CPU bounds; the
    search is unique and equals the coarse fix from its winning node."""
    ch_all, chans, eps, iono = ideal
    g = scenario.load_golden("sky12_static_35s_i8")
    prns = [int(p) for p in chans["prn"]]
    blocks = list(range(0, 340, 17))
    meas = np.zeros((len(blocks), len(prns)), gps.SNAPSHOT_DTYPE)
    for i, b in enumerate(blocks):
        r = golden_rows(g, [b])
        iq, _ = scenario.oracle_run(r, g["nav_frames"], 1)
        assert scenario.crc_blocks(iq)[0] == g["crcs"][b, 0]
        cold = ctx.acquire(iq, gps.SC08, prns, ms=K_CHAIN, s0=S0)
        warm = ctx.acquire_windows(iq, gps.SC08, prns, cold["doppler_hz"] - 500.0, step=250.0, nbins=5, ms=K_CHAIN,
                                   s0=S0)
        assert np.array_equal(warm["delay"], cold["delay"]) and np.array_equal(warm["doppler_hz"], cold["doppler_hz"])
        m = ctx.snapshot_measure(cold, iq, gps.SC08, ms=K_CHAIN, s0=S0)
        assert ctx.snapshot_measure(warm, iq, gps.SC08, ms=K_CHAIN, s0=S0, nbins=5).tobytes() == m.tobytes()
        assert (m["status"] == gps.SNAP_OK).all()
        m["sample"] += b * PT.BLOCK
        meas[i] = m
    rows = static_rows(ch_all, LOC)
    cfg = gps.pvt_config(0, 1, len(blocks), iono)
    x0 = rows[0]
    ap = apriori(x0, START_SOW, offsets(x0)[1])
    fix, co = ctx.pvt_snapshot(chans, meas, cfg, ap)
    assert (fix["status"] == gps.FIX_OK).all()
    tx, tv = PT.truth_xyz(rows, fix["sample"])
    e3 = np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - tx, axis=1)
    ev = np.linalg.norm(np.stack([fix["vx"], fix["vy"], fix["vz"]], 1) - tv, axis=1)
    et = np.abs((fix["t_rx"] - PT.truth_time(START_SOW, fix["sample"]) + 302400.0) % 604800.0 - 302400.0)
    assert e3.max() <= BOUNDS["pos"] and ev.max() <= BOUNDS["vel"] and et.max() <= BOUNDS["time"], (e3, ev, et)
    sfix, rec = ctx.pvt_snapshot_search(chans, meas[::4], cfg, search_cfg(START_SOW, 10.0))
    assert (sfix["status"] == gps.FIX_OK).all() and np.isnan(rec["alt_rms"]).all() and (rec["support"] >= 1).all()
    nodes = gps.search_nodes()
    for i in range(len(sfix)):
        one = gps.coarse_config(nodes[rec["winner"][i]], (START_SOW + 10.0) % 604800.0, 0, 2296)
        f1, _ = ctx.pvt_snapshot(chans, meas[::4][i:i + 1], cfg, one)
        assert f1.tobytes() == sfix[i:i + 1].tobytes()


def test_refusals_leave_the_context_working(ctx, sky12_block):
    _, _, iq = sky12_block
    res = ctx.acquire(iq, gps.SC08, [1, 2, 3], ms=2, s0=S0)
    with pytest.raises(gps.GpsB200Error):
        ctx.snapshot_measure(res, iq, gps.SC08, ms=101, s0=S0)
    with pytest.raises(gps.GpsB200Error):
        ctx.snapshot_measure(res, iq, gps.SC08, ms=2, s0=S0, prns=[1, 2, 4])
    with pytest.raises(gps.GpsB200Error):
        ctx.snapshot_measure(res, iq, gps.SC08, ms=2, s0=S0, cfg=gps.snapshot_config(iterations=17))
    dev = torch.from_numpy(iq.copy()).cuda()
    with pytest.raises(gps.GpsB200Error):
        ctx.snapshot_measure(res, None, gps.SC08, ms=2, s0=S0, device_ptr=dev.data_ptr() + 2, nsamples=iq.size // 2 - 1)
    meas = np.zeros((1, 3), gps.SNAPSHOT_DTYPE)
    meas["sample"] = [[5, 5, 6]]
    chans = np.zeros(3, gps.PVT_CHAN_DTYPE)
    with pytest.raises(gps.GpsB200Error):
        ctx.pvt_snapshot(chans, meas, gps.pvt_config(0, 1, 1), gps.coarse_config([6.4e6, 0, 0], 100.0))
    good = ctx.snapshot_measure(res, iq, gps.SC08, ms=2, s0=S0)
    assert good.tobytes() == S.measure(iq, 1, S0, 2, res, iterations=gps.SNAP_ITERATIONS).tobytes()


def test_search_equals_the_model(ctx, ideal, sky12_block):
    """One measured snapshot (block 50) searched with no position on the GPU and on the model: the same winner,
    counts and resolved ms, the fixes within the tolerances of test_search_gpu."""
    ch, chans, eps, iono = ideal
    _, _, iq = sky12_block
    res = ctx.acquire(iq, gps.SC08, [int(p) for p in chans["prn"]], ms=K_CHAIN, s0=S0)
    m = ctx.snapshot_measure(res, iq, gps.SC08, ms=K_CHAIN, s0=S0)
    m["sample"] += 50 * PT.BLOCK
    meas = m[None, :]
    cfg = gps.pvt_config(0, 1, 1, iono)
    sc = search_cfg(START_SOW, -10.0)
    fix, rec, r, ms = ctx.pvt_snapshot_search(chans, meas, cfg, sc, want_residuals=True, want_ms=True)
    wfix, wrec, wr, wms = S.search(chans, meas, cfg, sc)
    assert fix["status"][0] == wfix["status"][0] == gps.FIX_OK
    for f in ("winner", "searched", "ok", "support"):
        assert int(rec[f][0]) == int(wrec[f][0]), f
    assert np.array_equal(ms, wms)
    for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz", "rms"):
        assert abs(float(fix[f][0]) - float(wfix[f][0])) < 1e-6, f
    assert np.nanmax(np.abs(r - wr)) < 1e-6


def sanitizer_run():
    """One call of each entry point (host and device measurement at K = 10 with 32 PRNs from s0 = 1001, a snapshot fix
    and a search on a 4 096-node grid) -> a hex digest of the results."""
    import hashlib
    g = scenario.load_golden("sky12_static_35s_i8")
    ch = golden_rows(g, [50])
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], 1)
    chs, frames = scenario.golden_chans(g)
    chans, _ = ideal_inputs(chs, frames, g["nav_frame_of_block"])
    chans = unanchored(chans)
    with gps.Context(1, 1) as c:
        res = c.acquire(iq, gps.SC08, range(1, 33), ms=10, s0=1001)
        m = c.snapshot_measure(res, iq, gps.SC08, ms=10, s0=1001)
        dev = torch.from_numpy(iq.copy()).cuda()
        torch.cuda.synchronize()
        md = c.snapshot_measure(res, None, gps.SC08, ms=10, s0=1001, device_ptr=dev.data_ptr(), nsamples=iq.size // 2)
        assert md.tobytes() == m.tobytes()
        sel = [int(np.nonzero(m["prn"] == p)[0][0]) for p in chans["prn"]]
        meas = m[sel][None, :]
        x0 = PM.llh_ecef(*LOC)
        fix, co = c.pvt_snapshot(chans, meas, gps.pvt_config(0, 1, 1), apriori(x0, START_SOW, offsets(x0)[1]))
        sfix, rec = c.pvt_snapshot_search(chans, meas, gps.pvt_config(0, 1, 1), gps.search_config(START_SOW, 0, 2296, 4096))
    assert (fix["status"] == gps.FIX_OK).all()
    return hashlib.sha256(m.tobytes() + fix.tobytes() + co.tobytes() + sfix.tobytes() + rec.tobytes()).hexdigest()


def test_entry_points_clean_under_compute_sanitizer():
    """memcheck over one call of each entry point. Where the tool reports the device unsupported, the fallback of
    test_sanitizers: CUDA reports no error and repeated runs give the same bytes."""
    import os
    import shutil
    import subprocess
    import sys
    from test_coarse_gpu import _device_not_supported
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_snapshot_gpu as S; "
            "print('ok', S.sanitizer_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1500)
    if _device_not_supported(r):
        for _ in range(3):
            assert sanitizer_run() == plain.stdout.split()[-1]
            torch.cuda.synchronize()                          # raises on an illegal address or any sticky error
        return
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-500:])
    assert plain.stdout.split()[-1] == r.stdout.split()[-1]


def test_cli_snapshot_fixes(tmp_path):
    """gpsb200-sim -d 3 -t 1500.5,33.3,120.25 from 02:00:00, then gpsb200-acq --fix --assist with the same RINEX file
    and the a-priori time 10 s late: a snapshot every 100 ms from 1 ms, from the -l location as a-priori position and
    with no position (search). Every line OK, delta about -10 s, support >= 1 with search, and every position within
    the site's bound of the -t start point: this stream's sky is none of the model's fixtures, and its 25 snapshots
    reach 39.2 m, beyond the 39 m fixed on sky12_static_35s but within the loosest bound the model fixed (45 m, the
    int16 site). --fix without --assist is refused."""
    import os
    import subprocess
    from test_scenario import START, make_nav
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-acq")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav = make_nav(tmp_path, 12)
    iq = tmp_path / "iq.bin"
    loc = "%.6f,%.6f,%.1f" % LOC
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", loc, "-d", "3",
                           "-t", "1500.5,33.3,120.25", "-s", "2024/01/07,02:00:00", "-o", str(iq)])
    with gps.LiveScenario(nav, *LOC, seconds=3, start=START, target=(1500.5, 33.3, 120.25)) as live:
        x_true = np.array(live.state().xyz[:], np.float64)
    acq = [os.path.join(exe_dir, "gpsb200-acq"), str(iq), "--offset-ms", "1", "--fix", "--every", "100", "--count", "25",
           "--assist", nav, "--assist-time", "2024/01/07,02:00:10"]
    for pos in (loc, "search"):
        r = subprocess.run(acq + ["--assist-pos", pos], capture_output=True, text=True, check=True)
        lines = [ln.split() for ln in r.stdout.splitlines() if ln and not ln.startswith("#")]
        assert len(lines) >= 20 and all(ln[1] == "OK" for ln in lines), r.stdout[-2000:]
        rows = np.array([[float(v) for v in ln[2:]] for ln in lines])
        xyz = np.stack([PM.llh_ecef(la, lo, h) for la, lo, h in rows[:, 0:3]])
        err = np.linalg.norm(xyz - x_true, axis=1)
        assert err.max() <= SCENE_BOUNDS["site_34s_58w_10s_i16"]["pos"], err
        delta = rows[:, 9]
        assert np.all(np.abs(delta + 10.0) <= BOUNDS["time"]), delta
        if pos == "search":
            assert np.all(rows[:, 10] >= 1)
    assert subprocess.run(acq[:acq.index("--assist")] + ["--assist-pos", loc, "--assist-time", "2024/01/07,02:00:10"],
                          capture_output=True).returncode == 2
