"""Position fixes on the GPU (gpsb200_pvt, Context.pvt, gpsb200-track --fix): the kernel against the numpy model on ideal
and tracked epochs, and the whole receiver chain (synthesis with the reference's block CRCs, acquisition, tracking,
decoding, fix) against the scenario's truth within the bounds tests/test_pvt.py fixed on the CPU."""
import os
import subprocess

import numpy as np
import pytest

import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_pvt import TRACKED, check_truth, ideal_inputs, rinex, tracked_inputs
from test_scenario import LOC, START, motion_file
from test_track import ACQ, START_SOW, starts
from test_track_gpu import signal

pytestmark = pytest.mark.gpu

ERR_ARG = -1
FIELDS = ("x", "y", "z", "clock_m", "vx", "vy", "vz", "drift", "height")


def assert_kernel_equals_model(ctx, chans, eps, cfg):
    """Statuses, channel masks and Gauss-Newton iteration counts equal; fixes within 1 um (1 um/s), residuals within
    1 um."""
    got, res = ctx.pvt(chans, eps, cfg, want_residuals=True)
    want, wres, _ = PM.pvt(chans, eps, cfg)
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(got[f], want[f].astype(got[f].dtype)), f
    ok = got["status"] == gps.FIX_OK
    for f in FIELDS:
        assert np.all(np.abs(got[f][ok] - want[f][ok]) < 1e-6), (f, np.abs(got[f][ok] - want[f][ok]).max())
    assert np.all(np.abs(got["t_rx"][ok] - want["t_rx"][ok]) < 1e-14 * 604800 + 1e-12)
    assert np.all(np.abs(got["lat_deg"][ok] - want["lat_deg"][ok]) < 1e-11)
    assert np.all(np.abs(got["pdop"][ok] - want["pdop"][ok]) < 1e-9) and np.all(np.abs(got["rms"][ok] - want["rms"][ok]) < 1e-6)
    both = ~np.isnan(res)
    assert np.array_equal(both, ~np.isnan(wres)) and np.all(np.abs(res[both] - wres[both]) < 1e-6)
    assert np.all(np.isnan(got["x"][~ok]))
    return got


def period_of(e, s):
    """Index k of the epoch whose period holds sample s (-1 before the first)."""
    return int(np.searchsorted(e["sample"], s, side="right")) - 1


def used(fix, c):
    return (fix["mask"].astype(np.int64) >> c) & 1 == 1


@pytest.mark.parametrize("nchan", [1, 3, 4, 7, 12])
def test_kernel_equals_model_on_ideal_epochs(nchan, tmp_path):
    """sky12_static_35s, the first nchan PRNs. Channel 0 loses lock for epochs 5000-5999 and the last channel for its
    single epoch 20000; with 3 channels and more, channel 1's epochs end at 15 s and channel 2's start 3 s late. Fixes
    every 0.1 s over the whole run and past its end, and three per period around every event. The kernel equals the
    model, and the masks show each channel leave and rejoin exactly where the contract says: a period k is used only
    when epochs k - 1 and k are both locked, and only for 1 <= k <= n - 2 of its n epochs."""
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    prns = [int(p) for p in ch[0]["prn"] if p > 0][:nchan]
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"], prns)
    last = nchan - 1
    if nchan > 2:
        eps[1] = eps[1][:15000]
        eps[2] = eps[2][3000:]
        chans[2]["anchor_epoch"] = 0
        chans[2]["anchor_ms"] = (chans[2]["anchor_ms"] + 3000) % PT.WEEK_MS
    eps[0]["lock"][5000:6000] = 0
    eps[last]["lock"][20000] = 0

    def around(c, k):                      # three fix instants per period, periods k - 2 .. k + 3 of channel c
        return gps.pvt_config(int(eps[c]["sample"][k - 2]), 997, 18, iono)
    cfgs = [gps.pvt_config(1000, 299993, 352, iono), around(0, 2), around(0, 5000), around(0, 6000),
            around(last, 20000)]
    if nchan > 2:
        cfgs += [around(1, len(eps[1]) - 3), around(2, 2)]
    fixes = []
    with gps.Context(1, 1) as ctx:
        for cfg in cfgs:
            fixes.append(assert_kernel_equals_model(ctx, chans, eps, cfg))
    fix = np.concatenate(fixes)
    # every event is reached, on both sides
    for c, k_off, k_on in [(0, [0], [1, 2]), (0, [5000, 5001, 6000], [4999, 6001]),
                           (last, [20000, 20001], [19999, 20002])] + \
            ([(1, [len(eps[1]) - 1], [len(eps[1]) - 2])] if nchan > 2 else []):
        k = np.array([period_of(eps[c], s) for s in fix["sample"]])
        for kk in k_off:
            assert (k == kk).any() and not used(fix, c)[k == kk].any(), (c, kk)
        for kk in k_on:
            assert (k == kk).any() and used(fix, c)[k == kk].all(), (c, kk)
    if nchan > 2:
        assert not used(fix, 1)[fix["sample"] >= eps[1]["sample"][-1]].any()
        assert not used(fix, 2)[fix["sample"] < eps[2]["sample"][1]].any()
    assert (fix["sample"] > max(int(e["sample"][-1]) for e in eps)).any() and \
        (fix["nused"][fix["sample"] >= max(int(e["sample"][-1]) for e in eps)] == 0).all()
    st = set(int(v) for v in fix["status"])
    if nchan < 4:
        assert st == {gps.FIX_FEW}, st
    else:
        assert {gps.FIX_OK, gps.FIX_FEW} <= st, st
        # from the Earth's centre, Gauss-Newton on exactly four satellites can diverge (channels 3-6 alone, in channel 0's
        # first period at 7 channels); the kernel reports it as the model does, and only there
        assert (fix["nused"][fix["status"] == gps.FIX_NO_CONVERGENCE] == 4).all()
    if nchan >= 4:                         # channel 0's lock loss alone takes one channel out (at 4: a fix becomes none)
        k0 = np.array([period_of(eps[0], s) for s in fix["sample"]])
        assert (fix["nused"][(k0 >= 5000) & (k0 <= 6000)] == nchan - 1).all()
        assert (fix["status"][(k0 >= 5000) & (k0 <= 6000)] == (gps.FIX_FEW if nchan == 4 else gps.FIX_OK)).all()


def test_kernel_equals_model_on_32_channels_and_without_iono(tmp_path):
    g = scenario.load_golden("sky32_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    assert len(eps) == 32
    with gps.Context(1, 1) as ctx:
        for cfg in (gps.pvt_config(12345, 3001, 9000, rinex(tmp_path, 32)[2]), gps.pvt_config(12345, 299999, 90)):
            got = assert_kernel_equals_model(ctx, chans, eps, cfg)
    assert (got["nused"] == 32).all()


def gpu_track(ctx, out, ss, prns):
    res = ctx.acquire(out, ss, prns, **ACQ)
    eps, _ = ctx.track(starts(res), out, ss)
    return eps


def tracked_case(name, nblk, tmp_path):
    g, ch, out, ss = signal(nblk, name)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(ch.shape[1], 1) as ctx:
        eps = gpu_track(ctx, out, ss, prns)
        slot_of_prn = {p: k for k, p in enumerate(int(x) for x in ch[0]["prn"]) if p > 0}
        chans = tracked_inputs(eps, prns, g["nav_frames"], slot_of_prn)
        _, _, iono = rinex(tmp_path, ch.shape[1])
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        fix = assert_kernel_equals_model(ctx, chans, eps, cfg)
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    return check_truth(fix, xyz, START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])


@pytest.mark.parametrize("name,nblk", [("sky12_static_35s_i8", 349), ("sky32_static_10s_i8", 99)])
def test_end_to_end_with_scenario_ephemeris(name, nblk, tmp_path):
    """Synthesized on the GPU (block CRCs equal to the reference's), acquired, tracked, the TOW anchor from the tracked
    words, the ephemeris from the scenario's frames; the kernel equals the model on these epochs; the fixes (every 10 ms
    from 0.5 s) are within the tracked bounds, receive time of sample 0 included."""
    tracked_case(name, nblk, tmp_path)


def test_unassisted_circle_60s(tmp_path):
    """The receiver on circle.csv, int16, 60 s: the ephemeris is read from the tracked words themselves (subframes 1-3
    of the second frame, 30-48 s) and so is the time anchor; only the Klobuchar terms come from the configuration.
    Fixes every 10 ms from 0.5 s to the end, along the whole circle."""
    g = scenario.load_golden("sky12_circle_60s_i16")
    nav_file, _, iono = rinex(tmp_path, 12)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
    with gps.Context(12, ch.shape[0], max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        out, _ = ctx.synth_blocks(ch, gps.SC16)
        assert np.array_equal(scenario.crc_blocks(out), g["crcs"][:, 0])
        prns = [int(p) for p in ch[0]["prn"] if p > 0]
        eps = gpu_track(ctx, out, gps.SC16, prns)
        chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
        for c, (prn, e) in enumerate(zip(prns, eps)):
            _, words, sy = gps.nav_decode(e)
            chans[c]["eph"], _ = gps.nav_ephemeris(words)
            assert chans[c]["eph"]["valid"] == 1, prn
            chans[c]["prn"] = prn
            chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = gps.nav_time_anchor(words, sy)
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        fix = assert_kernel_equals_model(ctx, chans, eps, cfg)
    fig = check_truth(fix, g["motion_rows"][:, 1:4], START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"],
                      TRACKED["pos_mean"])
    assert fix["sample"][-1] > 58 * 3000000, fig


def test_bad_arguments_are_rejected_and_the_context_still_synthesizes(tmp_path):
    g = scenario.load_golden("sky12_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch[:5], frames, g["nav_frame_of_block"])
    good = gps.pvt_config(10000, 3000, 10)
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(frames)

        def cfg(f, v):
            c = good.copy()
            c[f] = v
            return c

        def chan(f, v):
            c = chans.copy()
            c[0][f] = v
            return c
        bad_eph = chans.copy()
        bad_eph[1]["eph"]["valid"] = 2
        cases = [dict(cfg=cfg("nfix", 0)), dict(cfg=cfg("step", 0)), dict(cfg=cfg("iono", 2)), dict(cfg=cfg("s0", -1)),
                 dict(chans=chan("anchor_epoch", -1)), dict(chans=chan("anchor_epoch", len(eps[0]))),
                 dict(chans=chan("anchor_ms", PT.WEEK_MS)), dict(chans=bad_eph),
                 dict(chans=np.repeat(chans[:1], 33), epochs=[eps[0]] * 33), dict(chans=chans[:0], epochs=[])]
        for kw in cases:
            a = dict(chans=chans, epochs=eps, cfg=good)
            a.update(kw)
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.pvt(**a)
            assert e.value.code == ERR_ARG, kw
        with pytest.raises(gps.GpsB200Error), gps.Context(1, 1) as fresh:
            fresh.pvt_replay()
        fix = ctx.pvt(chans, eps, good)
        assert (fix["status"] == gps.FIX_OK).all()
        # a channel without an ephemeris keeps its slot whatever its anchor holds, and is never used
        idle = chans.copy()
        idle[1]["eph"]["valid"] = 0
        idle[1]["anchor_epoch"], idle[1]["anchor_ms"] = -1, -1
        fix = ctx.pvt(idle, eps, good)
        assert (fix["status"] == gps.FIX_OK).all() and (fix["mask"] == (1 << len(chans)) - 1 - 0b10).all()
        out, _ = ctx.synth_blocks(ch[:1], gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]


def test_cli_prints_what_the_api_returns(tmp_path):
    """gpsb200-sim from 02:00:24 for 33 s (a full subframe 1-3 set, 02:00:30-02:00:48, after pull-in), then
    gpsb200-track --fix: each row is what nav_decode, nav_ephemeris, nav_time_anchor and Context.pvt return for the
    API's own acquisition and tracking of the file."""
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-track")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav, _, (alpha, beta) = rinex(tmp_path, 12, sets=2)     # a second set, so that 02:00:24 is inside the span
    iq = tmp_path / "iq.bin"
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", "35.681298,139.766247,10.0", "-d", "33",
                           "-s", "2024/01/07,02:00:24", "-o", str(iq)])
    iono = ",".join("%.17g" % v for v in list(alpha) + list(beta))
    r = subprocess.run([os.path.join(exe_dir, "gpsb200-track"), str(iq), "--fix", "--fix-every", "500", "--iono", iono],
                       capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    head = next(i for i, ln in enumerate(lines) if ln.startswith("# sample"))   # the fix table follows the PRN table
    rows = [ln.split() for ln in lines[head + 1:] if ln and not ln.startswith("#")]
    s = np.fromfile(iq, dtype=np.int8)
    with gps.Context(1, 1) as ctx:
        res = ctx.acquire(s, gps.SC08, range(1, 33), **ACQ)
        res = res[res["ratio"] >= 2.5]
        eps, _ = ctx.track(starts(res), s, gps.SC08)
        chans = np.zeros(len(res), gps.PVT_CHAN_DTYPE)
        for c, e in enumerate(eps):
            _, words, sy = gps.nav_decode(e)
            chans[c]["eph"], _ = gps.nav_ephemeris(words)
            chans[c]["prn"] = res[c]["prn"]
            chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = gps.nav_time_anchor(words, sy)
        keep = (chans["anchor_epoch"] >= 0) & (chans["eph"]["valid"] == 1)
        chans, eps = chans[keep], [e for e, k in zip(eps, keep) if k]
        end = max(int(e["sample"][-1]) for e in eps)
        fix = ctx.pvt(chans, eps, gps.pvt_config(1500000, 1500000, (end - 1500000) // 1500000 + 1, (alpha, beta)))
    fix = fix[fix["status"] == gps.FIX_OK]
    assert len(rows) == fix.size >= 40
    for row, f in zip(rows, fix):
        assert row[0] == str(f["sample"])
        assert row[1:7] == ["%.9f" % f["t_rx"], "%.8f" % f["lat_deg"], "%.8f" % f["lon_deg"], "%.3f" % f["height"],
                            "%.3f" % f["clock_m"], "%.3f" % f["vx"]]
        assert row[7:] == ["%.3f" % f["vy"], "%.3f" % f["vz"], str(f["nused"]), "%.2f" % f["pdop"]]
    xyz = PM.llh_ecef(*LOC)
    assert np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - xyz, axis=1).max() <= TRACKED["pos"]
