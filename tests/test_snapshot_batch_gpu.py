"""Snapshot batches on the GPU (gpsb200_snapshot_batch / _device, Context.snapshot_batch, gpsb200-acq --fix; DESIGN
§11.6): every window of a batch against the single calls it stands for (gpsb200_acquire or gpsb200_acquire_windows, then
gpsb200_snapshot_measure) byte for byte, on random input and on sky12_static_35s, through every split of the search
and across passes; one small case against the numpy models; the argument checks; memcheck; and the command-line fixes,
warm started from the almanac, against the cold ones."""
import os
import subprocess

import numpy as np
import pytest

import acq_model as A
import almanac_model as AM
import pvt_truth as PT
import scenario
import snapshot_model as S
from scenario import gps
from test_acquire import golden_rows
from test_acquire_gpu import random_stream
from test_almanac import make_sem
from test_coarse import apriori, offsets, static_rows, unanchored
from test_pvt import ideal_inputs, rinex
from test_scenario import LOC
from test_search import search_cfg
from test_snapshot import BOUNDS, S0, SCENE_BOUNDS, K as K_CHAIN
from test_track import START_SOW

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ERR_ARG = -1
STEP = 250.0


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    with gps.Context(12, 4) as c:
        yield c


def singles(ctx, iq, ss, s0, prns, K, f_lo, cfg, nbins=41):
    """The single calls a batch stands for: per window a search (f_lo None: the standard grid; else its row of first
    bins) and the measurement of its results. -> (ACQ_RESULT[nwin, nprn], SNAPSHOT[nwin, nprn])."""
    res = np.zeros((len(s0), len(prns)), gps.ACQ_RESULT_DTYPE)
    out = np.zeros((len(s0), len(prns)), gps.SNAPSHOT_DTYPE)
    for w, s in enumerate(s0):
        if f_lo is None:
            res[w] = ctx.acquire(iq, ss, prns, ms=K, s0=int(s), nbins=nbins)
        else:
            res[w] = ctx.acquire_windows(iq, ss, prns, f_lo[w], STEP, nbins, ms=K, s0=int(s))
        out[w] = ctx.snapshot_measure(res[w], iq, ss, ms=K, s0=int(s), cfg=cfg)
    return res, out


def window_starts(rng, nwin, K, n):
    """nwin window starts in a buffer of n samples: unsorted, two overlapping, one repeated, one ending on the last
    sample."""
    last = n - gps.acq_window_samples(K)
    s = rng.integers(0, last + 1, nwin)
    if nwin >= 3:
        s[0] = last
        s[1] = max(0, last - 1234)          # overlaps window 0
        s[2] = s[1]                          # repeats window 1
    else:
        s[-1] = last
    return s.astype(np.int64)


CASES = [(1, 10, 32), (3, 1, 12), (3, 2, 1), (17, 2, 12), (17, 10, 1), (3, 10, 32)]


@pytest.mark.parametrize("kind", ["int8", "int16"])
@pytest.mark.parametrize("nwin,K,nprn", CASES)
@pytest.mark.parametrize("warm", [False, True])
def test_batch_equals_single_calls_on_random_input(ctx, kind, nwin, K, nprn, warm):
    """Random int8 and saturating int16 input; windows overlapping, unsorted, repeated and ending on the buffer's last
    sample; a third of the PRNs below min_ratio. Host and device sources give the same bytes."""
    rng = np.random.default_rng(nwin * 1000 + K * 10 + nprn + (7 if warm else 0) + len(kind))
    n = gps.acq_window_samples(K) + 45678
    iq, ss = random_stream(kind, n, seed=int(rng.integers(1 << 30)))
    s0 = window_starts(rng, nwin, K, n)
    prns = [int(p) for p in rng.choice(np.arange(1, 33), nprn, replace=False)]
    f_lo = rng.uniform(-6000.0, 6000.0, (nwin, nprn)).round(1) if warm else None
    nbins = 5 if warm else 41
    first = singles(ctx, iq, ss, s0, prns, K, f_lo, gps.snapshot_config(0.0), nbins)[0]
    r = np.sort(first["ratio"].ravel())     # about a third below min_ratio (repeated windows repeat their ratios)
    cfg = gps.snapshot_config(float(r[len(r) // 3] if r[len(r) // 3] > r[0] else np.nextafter(r[0], np.inf)))
    want_res, want_out = singles(ctx, iq, ss, s0, prns, K, f_lo, cfg, nbins)
    assert (want_out["status"] == gps.SNAP_WEAK).any()
    res, out = ctx.snapshot_batch(s0, iq, ss, prns, ms=K, nbins=nbins, f_lo_prn=f_lo, cfg=cfg)
    assert res.tobytes() == want_res.tobytes()
    assert out.tobytes() == want_out.tobytes()
    dev = torch.from_numpy(iq.copy()).cuda()
    torch.cuda.synchronize()
    res_d, out_d = ctx.snapshot_batch(s0, None, ss, prns, ms=K, nbins=nbins, f_lo_prn=f_lo, cfg=cfg,
                                      device_ptr=dev.data_ptr(), nsamples=n)
    assert res_d.tobytes() == res.tobytes() and out_d.tobytes() == out.tobytes()


def test_batch_equals_the_models(ctx):
    """One small case against acq_model and snapshot_model: 3 windows, K = 2, 2 PRNs, 3 bins from per-window rows."""
    rng = np.random.default_rng(5)
    K, prns = 2, [3, 29]
    n = gps.acq_window_samples(K) + 9001
    iq, ss = random_stream("int8", n, seed=17)
    s0 = window_starts(rng, 3, K, n)
    f_lo = rng.uniform(-4000.0, 4000.0, (3, 2)).round(1)
    cfg = gps.snapshot_config(0.0)
    res, out = ctx.snapshot_batch(s0, iq, ss, prns, ms=K, nbins=3, f_lo_prn=f_lo, cfg=cfg)
    for w, s in enumerate(s0):
        for p, prn in enumerate(prns):
            want = A.reduce(A.grid(iq, ss, int(s), K, [prn], f_lo[w, p], STEP, 3), [prn], f_lo[w, p], STEP)
            assert res[w, p:p + 1].tobytes() == want.tobytes()
        m = S.measure(iq, ss, int(s), K, res[w], min_ratio=0.0, iterations=gps.SNAP_ITERATIONS)
        assert out[w].tobytes() == m.tobytes()


def test_every_split_gives_the_same_bytes(ctx):
    """A batch of 3 windows x 4 PRNs x 5 bins (60 rows, under one wave) with each split forced, host and device."""
    rng = np.random.default_rng(11)
    K, prns = 2, [1, 8, 17, 30]
    n = gps.acq_window_samples(K) + 30000
    iq, ss = random_stream("int16", n, seed=23)
    s0 = window_starts(rng, 3, K, n)
    f_lo = rng.uniform(-5000.0, 5000.0, (3, 4)).round(1)
    cfg = gps.snapshot_config(0.0)
    assert ctx.debug_acq_split(3 * 4, 5) > 1
    want = singles(ctx, iq, ss, s0, prns, K, f_lo, cfg, 5)
    dev = torch.from_numpy(iq.copy()).cuda()
    torch.cuda.synchronize()
    try:
        for split in (1, 2, 3, 4, 6):
            assert ctx.debug_acq_split(3 * 4, 5, force=split) == split
            for src in (dict(iq=iq), dict(device_ptr=dev.data_ptr(), nsamples=n)):
                got = ctx.snapshot_batch(s0, sample_size=ss, prns=prns, ms=K, nbins=5, f_lo_prn=f_lo, cfg=cfg, **src)
                assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), split
    finally:
        ctx.debug_acq_split(1, 1, force=0)


def test_passes_give_the_same_bytes(ctx):
    """700 windows of K = 1, 32 PRNs and one bin: more than two passes under the scratch cap (whose pairs stay under
    the grid's y limit of 65535). Every window equals its single calls, and the same windows submitted as two batches
    give the same bytes."""
    K, prns = 1, list(range(1, 33))
    per = gps.snapshot_batch_pass(32, 1, K, gps.SC08)
    assert 2 * per < 700 and per * 32 < 65535
    rng = np.random.default_rng(3)
    n = 200000
    iq, ss = random_stream("int8", n, seed=99)
    s0 = window_starts(rng, 700, K, n)
    f_lo = rng.uniform(-5000.0, 5000.0, (700, 32)).round(1)
    cfg = gps.snapshot_config(1.2)
    res, out = ctx.snapshot_batch(s0, iq, ss, prns, ms=K, nbins=1, f_lo_prn=f_lo, cfg=cfg)
    want = singles(ctx, iq, ss, s0, prns, K, f_lo, cfg, 1)
    assert res.tobytes() == want[0].tobytes() and out.tobytes() == want[1].tobytes()
    a = ctx.snapshot_batch(s0[:350], iq, ss, prns, ms=K, nbins=1, f_lo_prn=f_lo[:350], cfg=cfg)
    b = ctx.snapshot_batch(s0[350:], iq, ss, prns, ms=K, nbins=1, f_lo_prn=f_lo[350:], cfg=cfg)
    assert np.concatenate([a[0], b[0]]).tobytes() == res.tobytes()
    assert np.concatenate([a[1], b[1]]).tobytes() == out.tobytes()


@pytest.fixture(scope="module")
def chain(tmp_path_factory):
    """sky12_static_35s: 20 blocks spread over 34 s, one after another in one buffer, a window of K = 10 from S0 in
    each; the channels and the SEM almanac of the same orbits."""
    g = scenario.load_golden("sky12_static_35s_i8")
    ch_all, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path_factory.mktemp("nav"), 12)
    chans, _ = ideal_inputs(ch_all, frames, g["nav_frame_of_block"])
    blocks = list(range(0, 340, 17))
    parts = []
    for b in blocks:
        iq, _ = scenario.oracle_run(golden_rows(g, [b]), g["nav_frames"], 1)
        assert scenario.crc_blocks(iq)[0] == g["crcs"][b, 0]
        parts.append(iq)
    sem = make_sem(tmp_path_factory.mktemp("sem"))
    return ch_all, unanchored(chans), iono, blocks, np.concatenate(parts), gps.almanac_read(sem)[1]


def test_chain_on_sky12_static(ctx, chain):
    """20 windows of one batch, cold and warm (each window's rows from almanac_predict at its own time): the records
    equal the single calls', and the fixes and searches from them equal those from the single calls' records, within
    the CPU bounds."""
    ch_all, chans, iono, blocks, iq, alm = chain
    prns = [int(p) for p in chans["prn"]]
    s0 = np.array([i * gps.BLOCK_SAMPLES + S0 for i in range(len(blocks))], np.int64)
    week = 2296
    x_a = AM.llh_to_ecef(*LOC)
    f_lo = np.zeros((len(blocks), len(prns)))
    for w, b in enumerate(blocks):
        sky = gps.almanac_predict(alm, week, START_SOW + 0.1 * b + S0 / 3e6, x_a)
        f_lo[w] = [STEP * round(float(sky[p - 1]["doppler_hz"]) / STEP) - 2 * STEP for p in prns]
    cfg = gps.snapshot_config()
    cold = ctx.snapshot_batch(s0, iq, gps.SC08, prns, ms=K_CHAIN, cfg=cfg)
    single = singles(ctx, iq, gps.SC08, s0, prns, K_CHAIN, None, cfg)
    assert cold[0].tobytes() == single[0].tobytes() and cold[1].tobytes() == single[1].tobytes()
    # the warm windows hold every cold peak: then the warm records are the cold ones
    j = np.rint((cold[0]["doppler_hz"] - f_lo) / STEP)
    assert ((j >= 0) & (j <= 4)).all(), j
    warm = ctx.snapshot_batch(s0, iq, gps.SC08, prns, ms=K_CHAIN, nbins=5, f_lo_prn=f_lo, cfg=cfg)
    wsingle = singles(ctx, iq, gps.SC08, s0, prns, K_CHAIN, f_lo, cfg, 5)
    assert warm[0].tobytes() == wsingle[0].tobytes() and warm[1].tobytes() == wsingle[1].tobytes()
    assert warm[1].tobytes() == cold[1].tobytes()
    assert (cold[1]["status"] == gps.SNAP_OK).all()

    def stream(m):
        m = m.copy()
        m["sample"] += (np.array(blocks)[:, None] * PT.BLOCK - s0[:, None] + S0)
        return m
    meas, meas1 = stream(cold[1]), stream(single[1])
    rows = static_rows(ch_all, LOC)
    pcfg = gps.pvt_config(0, 1, len(blocks), iono)
    ap = apriori(rows[0], START_SOW, offsets(rows[0])[1])
    fix, co = ctx.pvt_snapshot(chans, meas, pcfg, ap)
    fix1, co1 = ctx.pvt_snapshot(chans, meas1, pcfg, ap)
    assert fix.tobytes() == fix1.tobytes() and co.tobytes() == co1.tobytes()
    assert (fix["status"] == gps.FIX_OK).all()
    tx, tv = PT.truth_xyz(rows, fix["sample"])
    e3 = np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - tx, axis=1)
    ev = np.linalg.norm(np.stack([fix["vx"], fix["vy"], fix["vz"]], 1) - tv, axis=1)
    et = np.abs((fix["t_rx"] - PT.truth_time(START_SOW, fix["sample"]) + 302400.0) % 604800.0 - 302400.0)
    assert e3.max() <= BOUNDS["pos"] and ev.max() <= BOUNDS["vel"] and et.max() <= BOUNDS["time"], (e3, ev, et)
    sc = search_cfg(START_SOW, 10.0)
    sfix, rec = ctx.pvt_snapshot_search(chans, meas[::4], pcfg, sc)
    sfix1, rec1 = ctx.pvt_snapshot_search(chans, meas1[::4], pcfg, sc)
    assert sfix.tobytes() == sfix1.tobytes() and rec.tobytes() == rec1.tobytes()
    assert (sfix["status"] == gps.FIX_OK).all() and (rec["support"] >= 1).all()
    tx, _ = PT.truth_xyz(rows, sfix["sample"])
    assert np.linalg.norm(np.stack([sfix["x"], sfix["y"], sfix["z"]], 1) - tx, axis=1).max() <= BOUNDS["pos"]


def test_refusals_leave_the_context_working(ctx):
    """nwin 0, NULL s0, one window outside the buffer, one f_lo row outside +-1.5 MHz, a misaligned device pointer:
    each refused before anything is enqueued (nothing written), and the next batch equals its single calls."""
    import ctypes as C
    rng = np.random.default_rng(8)
    K, prns = 2, [4, 9, 22]
    n = gps.acq_window_samples(K) + 20000
    iq, ss = random_stream("int8", n, seed=5)
    s0 = window_starts(rng, 4, K, n)
    f_lo = rng.uniform(-3000.0, 3000.0, (4, 3)).round(1)
    acq = ctx._acq_config(prns, K, 0, -5000.0, STEP, 5)
    sc = np.array(gps.snapshot_config(), dtype=gps.SNAPSHOT_CONFIG_DTYPE).reshape(1)
    res = np.zeros((4, 3), gps.ACQ_RESULT_DTYPE)
    out = np.zeros((4, 3), gps.SNAPSHOT_DTYPE)

    def call(nwin, s, fl=None, dev_ptr=None):
        L = gps.lib()
        fn, src, extra = ((L.gpsb200_snapshot_batch, iq.ctypes, ()) if dev_ptr is None
                          else (L.gpsb200_snapshot_batch_device, C.c_void_p(dev_ptr), (None,)))
        return fn(ctx._h, src, n, ss, C.byref(acq), nwin, None if s is None else s.ctypes.data,
                  None if fl is None else fl.ctypes.data, sc.ctypes.data, res.ctypes.data, out.ctypes.data, *extra)
    assert call(0, s0) == ERR_ARG
    assert call(4, None) == ERR_ARG
    outside = s0.copy()
    outside[2] = n - gps.acq_window_samples(K) + 1
    assert call(4, outside) == ERR_ARG
    bad = f_lo.copy()
    bad[3, 1] = 1.6e6
    assert call(4, s0, bad) == ERR_ARG
    dev = torch.from_numpy(iq.copy()).cuda()
    torch.cuda.synchronize()
    assert call(4, s0, f_lo, dev.data_ptr() + 2) == ERR_ARG
    assert not res.view(np.uint8).any() and not out.view(np.uint8).any()     # nothing was written
    with pytest.raises(gps.GpsB200Error):
        ctx.snapshot_batch(s0, iq, ss, prns, ms=K, nbins=5, f_lo_prn=f_lo[:3])
    got = ctx.snapshot_batch(s0, iq, ss, prns, ms=K, nbins=5, f_lo_prn=f_lo)
    want = singles(ctx, iq, ss, s0, prns, K, f_lo, gps.snapshot_config(), 5)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


def test_a_doppler_result_beyond_10_khz_is_refused_before_its_measurement(ctx):
    """Bins of 10.5 kHz and up: the search runs, the measurement's check of its results refuses the call, as
    gpsb200_snapshot_measure refuses those results; the context still works."""
    K = 1
    n = gps.acq_window_samples(K) + 100
    iq, ss = random_stream("int8", n, seed=1)
    with pytest.raises(gps.GpsB200Error, match="10 kHz"):
        ctx.snapshot_batch([0, 100], iq, ss, [5], ms=K, f_lo=10500.0, nbins=3)
    got = ctx.snapshot_batch([0, 100], iq, ss, [5], ms=K, nbins=3)
    want = singles(ctx, iq, ss, [0, 100], [5], K, None, gps.snapshot_config(), 3)
    assert got[1].tobytes() == want[1].tobytes()


def sanitizer_run():
    """One host and one device batch (8 windows of K = 10, 12 PRNs, warm rows, from sky12 block 50) -> a hex digest."""
    import hashlib
    g = scenario.load_golden("sky12_static_35s_i8")
    iq, _ = scenario.oracle_run(golden_rows(g, [50]), g["nav_frames"], 1)
    s0 = np.arange(8, dtype=np.int64) * 30000 + 1001
    prns = list(range(1, 13))
    f_lo = np.tile(np.arange(12) * 500.0 - 3000.0, (8, 1))
    with gps.Context(1, 1) as c:
        res, out = c.snapshot_batch(s0, iq, gps.SC08, prns, ms=10, nbins=5, f_lo_prn=f_lo)
        dev = torch.from_numpy(iq.copy()).cuda()
        torch.cuda.synchronize()
        rd, od = c.snapshot_batch(s0, None, gps.SC08, prns, ms=10, nbins=5, f_lo_prn=f_lo, device_ptr=dev.data_ptr(),
                                  nsamples=iq.size // 2)
        assert rd.tobytes() == res.tobytes() and od.tobytes() == out.tobytes()
    return hashlib.sha256(res.tobytes() + out.tobytes()).hexdigest()


def test_batch_clean_under_compute_sanitizer():
    """memcheck over one host and one device batch. Where the tool reports the device unsupported, the fallback of
    test_sanitizers: CUDA reports no error and repeated runs give the same bytes."""
    import shutil
    import sys
    from test_coarse_gpu import _device_not_supported
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_snapshot_batch_gpu as S; "
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


def test_cli_warm_fixes_equal_the_cold_ones(tmp_path):
    """The stream and command of test_snapshot_gpu's test_cli_snapshot_fixes (25 windows every 100 ms from 1 ms, the
    a-priori time 10 s late), with --almanac from the SEM file of the same orbits: first the precondition, every PRN
    the cold run measures is predicted in the warm list with its cold peak inside its window; then every warm line
    equals the cold run's, every line OK within that test's bounds. --almanac with search stays refused."""
    from test_scenario import START, make_nav
    import pvt_model as PM
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-acq")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav, sem = make_nav(tmp_path, 12), make_sem(tmp_path)
    iq = tmp_path / "iq.bin"
    loc = "%.6f,%.6f,%.1f" % LOC
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", loc, "-d", "3",
                           "-t", "1500.5,33.3,120.25", "-s", "2024/01/07,02:00:00", "-o", str(iq)])
    with gps.LiveScenario(nav, *LOC, seconds=3, start=START, target=(1500.5, 33.3, 120.25)) as live:
        x_true = np.array(live.state().xyz[:], np.float64)
    acq = [os.path.join(exe_dir, "gpsb200-acq"), str(iq), "--offset-ms", "1", "--fix", "--every", "100", "--count", "25",
           "--assist", nav, "--assist-time", "2024/01/07,02:00:10"]

    # the precondition, with the library: the cold run's measured PRNs and peaks against each window's prediction
    s = np.fromfile(iq, np.int8)
    s0 = np.array([3000 + i * 300000 for i in range(25) if 3000 + i * 300000 + gps.acq_window_samples(10) <= s.size // 2])
    with gps.Context(1, 1) as c:
        res, meas = c.snapshot_batch(s0, s, gps.SC08, range(1, 33), ms=10)
    rec = gps.almanac_read(sem)[1]
    skies = [gps.almanac_predict(rec, 2296, 7210.0 + (int(v) - int(s0[0])) / 3e6, AM.llh_to_ecef(*LOC)) for v in s0]
    warm = [p for p in range(1, 33) if any(k[p - 1]["valid"] and k[p - 1]["el_deg"] >= -5.0 for k in skies)]
    for w, sky in enumerate(skies):
        for r, m in zip(res[w], meas[w]):
            if m["status"] != gps.SNAP_OK:
                continue
            p = int(r["prn"])
            assert p in warm, p
            j = (float(r["doppler_hz"]) - (STEP * round(float(sky[p - 1]["doppler_hz"]) / STEP) - 2 * STEP)) / STEP
            assert 0 <= j <= 4, (w, p, j)

    def fixes(extra):
        r = subprocess.run(acq + extra, capture_output=True, text=True, check=True)
        return [ln for ln in r.stdout.splitlines() if ln and not ln.startswith("#")]
    cold = fixes(["--assist-pos", loc])
    warm_lines = fixes(["--assist-pos", loc, "--almanac", sem])
    assert warm_lines == cold
    lines = [ln.split() for ln in warm_lines]
    assert len(lines) >= 20 and all(ln[1] == "OK" for ln in lines)
    rows = np.array([[float(v) for v in ln[2:]] for ln in lines])
    xyz = np.stack([PM.llh_ecef(la, lo, h) for la, lo, h in rows[:, 0:3]])
    assert np.linalg.norm(xyz - x_true, axis=1).max() <= SCENE_BOUNDS["site_34s_58w_10s_i16"]["pos"]
    assert np.all(np.abs(rows[:, 9] + 10.0) <= BOUNDS["time"])
    refused = subprocess.run(acq + ["--assist-pos", "search", "--almanac", sem], capture_output=True)
    assert refused.returncode == 2
