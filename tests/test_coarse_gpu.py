"""Coarse-time fixes on the GPU (gpsb200_pvt_coarse, Context.pvt_coarse): the kernel against the numpy model
(tests/coarse_model.py) at every channel count, around tracking events, across the week roll, on a gapped channel and
with the samples shifted past 2^33; and the whole receiver chain, with no time anchor, against the scenario's truth within
the bounds tests/test_coarse.py fixed on the CPU."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import coarse_model as CM
import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_coarse import IDEAL, TRACKED, apriori, check_coarse, common_k, offsets, static_rows, unanchored
from test_pvt import check_truth, ideal_inputs, rinex, tracked_inputs
from test_pvt_gpu import gpu_track
from test_scenario import LOC, START, make_nav
from test_track import START_SOW
from test_track_gpu import signal

pytestmark = pytest.mark.gpu

ERR_ARG = -1
SHIFT = 1 << 33
FIELDS = ("x", "y", "z", "clock_m", "vx", "vy", "vz", "drift", "height")
# The delta tolerance, DELTA_ABS + DELTA_REL |delta|: at |delta| = 10 s it admits 5.1e-10 s, which moves no modelled
# range by more than 0.4 um (range rates stay below 800 m/s), inside the fixes' own 1 um. The largest gaps seen on the
# H100 were 1.1e-10 s at |delta| = 10 s with 5 channels, where delta is worst conditioned, and 3.5e-12 s at |delta| < 1e-5 s.
DELTA_ABS, DELTA_REL = 1e-11, 5e-11


def assert_coarse_equals_model(ctx, chans, eps, cfg, ap):
    """Statuses, masks, iteration counts, reference channels, `changed` and resolved ms equal; fixes within 1 um
    (1 um/s), residuals within 1 um; delta within DELTA_ABS + DELTA_REL |delta|. -> (fixes, records, ms)."""
    ch = unanchored(chans)
    got, rec, res, ms = ctx.pvt_coarse(ch, eps, cfg, ap, want_residuals=True, want_ms=True)
    want, wrec, wres, wms = CM.coarse(ch, eps, cfg, ap)
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(got[f], want[f].astype(got[f].dtype)), f
    for f in ("ref", "week", "changed"):
        assert np.array_equal(rec[f], wrec[f].astype(rec[f].dtype)), f
    assert np.array_equal(ms, wms)
    ok = got["status"] == gps.FIX_OK
    for f in FIELDS:
        assert np.all(np.abs(got[f][ok] - want[f][ok]) < 1e-6), (f, np.abs(got[f][ok] - want[f][ok]).max())
    assert np.all(np.abs(got["t_rx"][ok] - want["t_rx"][ok]) < 1e-14 * 604800 + 1e-12)
    assert np.all(np.abs(got["lat_deg"][ok] - want["lat_deg"][ok]) < 1e-11)
    assert np.all(np.abs(got["pdop"][ok] - want["pdop"][ok]) < 1e-9) and np.all(np.abs(got["rms"][ok] - want["rms"][ok]) < 1e-6)
    d = np.abs(rec["delta"][ok] - wrec["delta"][ok])
    assert np.all(d <= DELTA_ABS + DELTA_REL * np.abs(wrec["delta"][ok])), d.max() if d.size else 0
    both = ~np.isnan(res)
    assert np.array_equal(both, ~np.isnan(wres)) and np.all(np.abs(res[both] - wres[both]) < 1e-6)
    assert np.all(np.isnan(got["x"][~ok])) and np.all(np.isnan(rec["delta"][~ok]))
    return got, rec, ms


def used(fix, c):
    return (fix["mask"].astype(np.int64) >> c) & 1 == 1


def period_of(e, s):
    return int(np.searchsorted(e["sample"], s, side="right")) - 1


@pytest.mark.parametrize("nchan", [1, 4, 5, 6, 12])
def test_kernel_equals_model_on_ideal_epochs(nchan, tmp_path):
    """sky12_static_35s, the first nchan PRNs, with the events of test_pvt_gpu's test of the same name: channel 0 loses
    lock for epochs 5000-5999, the last channel for epoch 20000; with 3 channels and more channel 1's epochs end at 15 s
    and channel 2's start 3 s late. Fixes every 0.1 s over the whole run and past its end, and three per period around
    every event; a-priori 50 km and 10 s off. Fewer than 5 used channels give FIX_FEW."""
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    prns = [int(p) for p in ch[0]["prn"] if p > 0][:nchan]
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"], prns)
    last = nchan - 1
    if nchan > 2:
        eps[1] = eps[1][:15000]
        eps[2] = eps[2][3000:]
    eps[0]["lock"][5000:6000] = 0
    eps[last]["lock"][20000] = 0
    x0 = PM.llh_ecef(*LOC)
    ap = apriori(x0, START_SOW, offsets(x0)[1])

    def around(c, k):
        return gps.pvt_config(int(eps[c]["sample"][k - 2]), 997, 18, iono)
    cfgs = [gps.pvt_config(1000, 299993, 352, iono), around(0, 2), around(0, 5000), around(0, 6000),
            around(last, 20000)]
    if nchan > 2:
        cfgs += [around(1, len(eps[1]) - 3), around(2, 2)]
    fixes = []
    with gps.Context(1, 1) as ctx:
        for cfg in cfgs:
            fixes.append(assert_coarse_equals_model(ctx, chans, eps, cfg, ap)[0])
    fix = np.concatenate(fixes)
    for c, k_off, k_on in [(0, [0], [1, 2]), (0, [5000, 5001, 6000], [4999, 6001]),
                           (last, [20000, 20001], [19999, 20002])] + \
            ([(1, [len(eps[1]) - 1], [len(eps[1]) - 2])] if nchan > 2 else []):
        k = np.array([period_of(eps[c], s) for s in fix["sample"]])
        for kk in k_off:
            assert (k == kk).any() and not used(fix, c)[k == kk].any(), (c, kk)
        for kk in k_on:
            assert (k == kk).any() and used(fix, c)[k == kk].all(), (c, kk)
    st = set(int(v) for v in fix["status"])
    if nchan < 5:
        assert st == {gps.FIX_FEW}, st
    else:
        assert {gps.FIX_OK, gps.FIX_FEW} <= st, st
        assert (fix["nused"][fix["status"] == gps.FIX_FEW] < 5).all()
        assert (fix["status"][fix["nused"] >= 5] == gps.FIX_OK).all()


def test_kernel_equals_model_on_32_channels_and_without_iono(tmp_path):
    g = scenario.load_golden("sky32_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    x0 = PM.llh_ecef(*LOC)
    with gps.Context(1, 1) as ctx:
        for cfg, off in ((gps.pvt_config(12345, 3001, 9000, rinex(tmp_path, 32)[2]), offsets(x0)[2]),
                         (gps.pvt_config(12345, 299999, 90), offsets(x0)[0])):
            got, _, _ = assert_coarse_equals_model(ctx, chans, eps, cfg, apriori(x0, START_SOW, off))
            assert (got["nused"] == 32).all() and (got["status"] == gps.FIX_OK).all()


def test_ambiguous_fixes_equal_the_model(tmp_path):
    """The 400 km / 30 s offset of test_coarse: AMBIGUOUS at 6 and 12 channels, a wrong OK fix at 5, on both sides."""
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    x0 = PM.llh_ecef(*LOC)
    lat, lon, _ = PM.ecef_llh(x0)
    north = np.array([-np.sin(lat) * np.cos(lon), -np.sin(lat) * np.sin(lon), np.cos(lat)])
    ap = apriori(x0, START_SOW, (400e3 * north, 30.0))
    cfg = gps.pvt_config(30000, 299993, 100, iono)
    with gps.Context(1, 1) as ctx:
        for n, status in ((12, CM.FIX_AMBIGUOUS), (6, CM.FIX_AMBIGUOUS), (5, gps.FIX_OK)):
            got, _, _ = assert_coarse_equals_model(ctx, chans[:n], eps[:n], cfg, ap)
            assert (got["status"] == status).all(), n


def shifted(eps, cfg, ap):
    e2 = []
    for e in eps:
        e = e.copy()
        e["sample"] += SHIFT
        e2.append(e)
    c2, a2 = cfg.copy(), ap.copy()
    c2["s0"] += SHIFT
    a2["s_a"] += SHIFT
    return e2, c2, a2


@pytest.mark.parametrize("case", ["weekroll", "gap"])
def test_week_roll_gap_and_shift(case, tmp_path):
    """Across the `-s now` week roll, with the a-priori time given on both sides of 604 800 s (at sample 0, before the
    roll, and at a sample after it, in the next week); and on test_receiver_edges' channel whose epochs resume after a
    2.2 s gap. The kernel equals the model, the fixes are within the ideal bounds, and with every sample shifted by
    2^33 the results are byte-equal apart from `sample`."""
    import test_receiver_edges_gpu as RE
    chans, eps, cfg, (xyz, sow) = (RE.weekroll_case if case == "weekroll" else RE.gap_case)(tmp_path)
    if case == "weekroll":
        import test_time_overwrite as TO
        (tmp_path / "week").mkdir()
        week, _ = TO.gps_time(TO.now_case("sky12_now_weekroll_300s_i8", tmp_path / "week")[1]["start"])
    else:
        week = 2296
    x0 = xyz[0]
    aps = [apriori(x0, sow, offsets(x0)[1], week)]
    if case == "weekroll":
        s_a = 290 * 3000000                                   # after the roll
        t = sow + s_a / 3e6 + 10.0
        assert t >= 604800.0
        a = gps.coarse_config(x0 + offsets(x0)[1][0], t - 604800.0, s_a, week + 1)
        aps.append(a)
    with gps.Context(1, 1) as ctx:
        for ap in aps:
            fix, rec, ms = assert_coarse_equals_model(ctx, chans, eps, cfg, ap)
            check_coarse(chans, eps, cfg, ap, xyz, sow, IDEAL)
            e2, c2, a2 = shifted(eps, cfg, ap)
            fix2, rec2, res2, ms2 = ctx.pvt_coarse(unanchored(chans), e2, c2, a2, want_residuals=True, want_ms=True)
            _, _, res, _ = ctx.pvt_coarse(unanchored(chans), eps, cfg, ap, want_residuals=True, want_ms=True)
            assert np.array_equal(fix2["sample"], fix["sample"] + SHIFT)
            fix2["sample"] -= SHIFT
            assert fix.tobytes() == fix2.tobytes() and rec.tobytes() == rec2.tobytes()
            assert res.tobytes() == res2.tobytes() and ms.tobytes() == ms2.tobytes()
            if case == "weekroll":
                t = fix["t_rx"]
                assert (t < 100.0).any() and (t > 604700.0).any()
                assert set(rec["week"]) == {week, week + 1}
                assert np.array_equal(rec["week"] == week + 1, t < 302400.0)


def test_bad_configs_are_refused_before_anything_runs(tmp_path):
    g = scenario.load_golden("sky12_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch[:5], frames, g["nav_frame_of_block"])
    chans = unanchored(chans)
    x0 = PM.llh_ecef(*LOC)
    good = gps.coarse_config(x0, START_SOW, 0, 2296)
    cfg = gps.pvt_config(30000, 3000, 10)

    def ap(f, v):
        a = good.copy()
        a[f] = v
        return a
    nanx = good.copy()
    nanx["x_a"][1] = np.nan
    infx = good.copy()
    infx["x_a"][2] = np.inf
    cases = [dict(apriori=nanx), dict(apriori=infx), dict(apriori=ap("t_a", -1e-9)), dict(apriori=ap("t_a", 604800.0)),
             dict(apriori=ap("t_a", np.nan)), dict(apriori=ap("s_a", -1)), dict(apriori=ap("s_a", (1 << 62) + 1)),
             dict(apriori=ap("week", -1)), dict(apriori=ap("reserved", 1)), dict(cfg=gps.pvt_config(30000, 3000, 0)),
             dict(cfg=gps.pvt_config(30000, 0, 10)), dict(chans=np.repeat(chans[:1], 33), epochs=[eps[0]] * 33)]
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(frames)
        for kw in cases:
            a = dict(chans=chans, epochs=eps, cfg=cfg, apriori=good)
            a.update(kw)
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.pvt_coarse(**a)
            assert e.value.code == ERR_ARG, kw
        fix, rec = ctx.pvt_coarse(chans, eps, cfg, good)
        assert (fix["status"] == gps.FIX_OK).all()
        ctx.pvt_replay()                                      # re-runs the coarse call
        out, _ = ctx.synth_blocks(ch[:1], gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]


def _device_not_supported(r):
    return any(ln.startswith("========= Error: Device not supported") for ln in (r.stdout + r.stderr).splitlines())


def sanitizer_run():
    """One 32-channel coarse call -> a hex digest of its results."""
    import hashlib
    g = scenario.load_golden("sky32_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    x0 = PM.llh_ecef(*LOC)
    with gps.Context(1, 1) as ctx:
        fix, rec, res, ms = ctx.pvt_coarse(unanchored(chans), eps, gps.pvt_config(12345, 29989, 900),
                                           apriori(x0, START_SOW, offsets(x0)[1]), want_residuals=True, want_ms=True)
    assert (fix["status"] == gps.FIX_OK).all() and (fix["nused"] == 32).all()
    return hashlib.sha256(fix.tobytes() + rec.tobytes() + res.tobytes() + ms.tobytes()).hexdigest()


def test_coarse_kernel_clean_under_compute_sanitizer():
    """memcheck over one 32-channel call. Where the tool reports the device unsupported, the fallback of
    test_sanitizers: CUDA reports no error and repeated runs give the same bytes."""
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_coarse_gpu as S; "
            "print('ok', S.sanitizer_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1500)
    if _device_not_supported(r):
        import torch
        for _ in range(3):
            assert sanitizer_run() == plain.stdout.split()[-1]
            torch.cuda.synchronize()                          # raises on an illegal address or any sticky error
        return
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-500:])
    assert plain.stdout.split()[-1] == r.stdout.split()[-1]


# ---- the whole chain, with no time anchor ----------------------------------------------------------------------------
CHAIN = {"sky12_target_3s_i8": dict(target=(1500.5, 33.3, 120.25)), "sky12_pluto_3s_i16": dict(pluto_gain=True),
         "sky12_rinex3_3s_i8": dict(rinex3=True), "sky12_static_35s_i8": dict()}


@pytest.mark.parametrize("name", list(CHAIN))
def test_chain_without_anchors(name, tmp_path):
    """Synthesized on the GPU (block CRCs equal to the reference's), acquired, tracked; the ephemeris from the
    scenario's frames, the a-priori position and time 50 km and 10 s off; coarse fixes every 10 ms from 0.5 s. Every
    fix is OK and within the tracked per-fix bounds; the truth of the -t run is the start point the scenario engine
    computes. On sky12_static_35s (12.1 s, the window the CPU figures come from) the mean error is within the tracked
    mean bound too (the 3 s runs average over 2.3 s, where the slow tracking error does not average out: 8.5 m seen on
    sky12_target_3s), and the resolved ms equal the decoded anchors' up to one K per fix."""
    kw = CHAIN[name]
    nblk = 121 if name == "sky12_static_35s_i8" else int(scenario.load_golden(name)["crcs"].shape[0])
    g, ch, out, ss = signal(nblk, name)
    if "target" in kw:
        nav = make_nav(tmp_path, 12)
        with gps.LiveScenario(nav, *LOC, seconds=3, start=START, target=kw["target"]) as live:
            x_true = np.array(live.state().xyz[:], np.float64)
        assert np.linalg.norm(x_true - PM.llh_ecef(*LOC)) > 1000.0
    else:
        x_true = PM.llh_ecef(*LOC)
    rows = np.repeat(x_true[None], ch.shape[0] + 1, 0)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    slot_of_prn = {p: k for k, p in enumerate(int(x) for x in ch[0]["prn"]) if p > 0}
    _, _, iono = rinex(tmp_path, 12)
    with gps.Context(12, 1) as ctx:
        eps = gpu_track(ctx, out, ss, prns)
        if name == "sky12_static_35s_i8":
            chans = tracked_inputs(eps, prns, g["nav_frames"], slot_of_prn)
        else:
            chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
            for c, prn in enumerate(prns):
                chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(g["nav_frames"][0][slot_of_prn[prn]]))[0]
                chans[c]["prn"] = prn
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        ap = apriori(x_true, START_SOW, offsets(x_true)[1])
        fix, rec, ms = assert_coarse_equals_model(ctx, chans, eps, cfg, ap)
    assert fix.size >= 100 and (fix["nused"] == 12).all()
    long = name == "sky12_static_35s_i8"
    check_truth(fix, rows, START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"] if long else None)
    if long:
        K = common_k(ms, PM.measure(chans, eps, fix["sample"])["T"])
        assert np.all(np.abs(1000.0 * rec["delta"] - K) <= TRACKED["k"])


def test_cli_assisted_fixes(tmp_path):
    """gpsb200-sim -d 3 -t 1500.5,33.3,120.25 from 02:00:00, then gpsb200-track --fix --assist with the same RINEX file,
    the a-priori position at the -l point (1.5 km off) and the a-priori time 10 s late: nothing is decoded in 3 s, yet
    every 10 ms from 0.5 s a fix is printed, within the tracked bounds of the -t start point; delta is about -10 s.
    Without --assist the same file gives no fix at all."""
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-track")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav = make_nav(tmp_path, 12)
    iq = tmp_path / "iq.bin"
    loc = "%.6f,%.6f,%.1f" % LOC
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", loc, "-d", "3",
                           "-t", "1500.5,33.3,120.25", "-s", "2024/01/07,02:00:00", "-o", str(iq)])
    with gps.LiveScenario(nav, *LOC, seconds=3, start=START, target=(1500.5, 33.3, 120.25)) as live:
        x_true = np.array(live.state().xyz[:], np.float64)
    track = [os.path.join(exe_dir, "gpsb200-track"), str(iq), "--fix", "--fix-every", "10"]
    r = subprocess.run(track + ["--assist", nav, "--assist-pos", loc, "--assist-time", "2024/01/07,02:00:10"],
                       capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    head = next(i for i, ln in enumerate(lines) if ln.startswith("# sample"))
    assert lines[head].endswith("delta_s")
    rows = np.array([[float(v) for v in ln.split()] for ln in lines[head + 1:] if ln and not ln.startswith("#")])
    assert len(rows) >= 200
    xyz = np.stack([PM.llh_ecef(la, lo, h) for la, lo, h in rows[:, 2:5]])
    err = np.linalg.norm(xyz - x_true, axis=1)
    assert err.max() <= TRACKED["pos"] and err.mean() <= TRACKED["pos_mean"], (err.max(), err.mean())
    assert np.all(np.abs(rows[:, -1] + 10.0) < 0.02)
    plain = subprocess.run(track, capture_output=True, text=True, check=True).stdout.splitlines()
    assert not [ln for ln in plain if ln and not ln.startswith("#") and len(ln.split()) > 7]
    for bad in (["--raim", "1"], ["--araim", "5"]):
        assert subprocess.run(track + ["--assist", nav, "--assist-pos", loc, "--assist-time", "2024/01/07,02:00:10"] + bad,
                              capture_output=True).returncode == 2
