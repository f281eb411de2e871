"""RAIM on the GPU (gpsb200_pvt_raim, Context.pvt_raim, gpsb200-track --fix --raim): the kernel against the numpy model
(tests/raim_model.py) on the cases of tests/test_raim.py, fault-free fixes bit for bit those of gpsb200_pvt, and the
whole receiver chain on a stream whose broadcast clock of one PRN is wrong."""
import os
import subprocess

import numpy as np
import pytest

import pvt_model as PM
import raim_model as RM
import scenario
from scenario import gps
from test_pvt import TRACKED, check_truth, rinex
from test_pvt_gpu import FIELDS, gpu_track
from pvt_truth import truth_xyz
from test_raim import (AF0_ERROR, FAULT_SLOT, TRACKED_SIGMA, code_bias, rinex_with_af0, sky, sky12_fault_case,
                       sky12_faults, sky32_two_faults, tables)
from test_scenario import LOC
from test_track import ACQ, START_SOW, starts

pytestmark = pytest.mark.gpu

ERR_ARG = -1
REC_EXACT = ("verdict", "excluded", "dof")


def rel_close(a, b, tol=1e-9):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same = (np.isnan(a) & np.isnan(b)) | (a == b)
    return bool(np.all(same | (np.abs(a - b) <= tol * np.abs(b))))


def assert_margin(tests):
    """The model's decisions are not knife-edge: no stat within 1e-9 relative of its T (nor within what the residual
    tolerance allows, 1e-6 relative), and where a channel was chosen for exclusion, the two largest normalized
    residuals more than 1e-9 relative apart."""
    for t in tests:
        for stat, T, key in t:
            assert abs(stat / T - 1.0) > 1e-6
            cand = np.sort(key[key >= 0.0])
            if stat > T and cand.size >= 2 and not np.allclose(cand, cand[-1], rtol=1e-6):
                assert cand[-1] - cand[-2] > 1e-9 * cand[-1]


def assert_kernel_equals_model(ctx, chans, eps, cfg, rcfg):
    got, grec, gres = ctx.pvt_raim(chans, eps, cfg, rcfg, want_residuals=True)
    want, wres, wrec, tests = RM.raim(chans, eps, cfg, rcfg, *tables(rcfg))
    assert_margin(tests)
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(got[f], want[f].astype(got[f].dtype)), f
    for f in REC_EXACT:
        assert np.array_equal(grec[f], wrec[f].astype(grec[f].dtype)), f
    for f in ("threshold", "hpl", "vpl"):
        assert rel_close(grec[f], wrec[f]), (f, grec[f], wrec[f])
    # stat sums squared residuals of a few cm that agree to the 1 um below, not to 1e-9 relative: within 1e-9 relative
    # plus what residuals 1 um apart allow, |sum (e + d)^2 - sum e^2| <= 2 |e| |d| + |d|^2 with |d| <= sqrt(n) 1 um
    sig, n = float(rcfg["sigma"]), grec["dof"] + 4.0
    tol = 1e-9 * wrec["stat"] + 2.0 * np.sqrt(wrec["stat"] * n) * 1e-6 / sig + n * 1e-12 / sig ** 2
    ran = ~np.isnan(wrec["stat"])
    assert np.array_equal(ran, ~np.isnan(grec["stat"])) and np.all(np.abs(grec["stat"] - wrec["stat"])[ran] <= tol[ran])
    ok = got["status"] == gps.FIX_OK
    for f in FIELDS:
        assert np.all(np.abs(got[f][ok] - want[f][ok]) < 1e-6), (f, np.abs(got[f][ok] - want[f][ok]).max())
    assert np.all(np.abs(got["rms"][ok] - want["rms"][ok]) < 1e-6)
    both = ~np.isnan(gres)
    assert np.array_equal(both, ~np.isnan(wres)) and np.all(np.abs(gres[both] - wres[both]) < 1e-6)
    return got, grec, gres


@pytest.mark.parametrize("nchan", [5, 6, 12])
def test_kernel_equals_model_on_sky12(nchan, tmp_path):
    """The first nchan channels of sky12_static_35s, fault-free and with a code bias on channel 2; 5 channels give dof
    1 (ALERT), 6 and more exclude; detection only, one and four exclusions allowed."""
    _, _, chans, eps = sky("sky12_static_35s_i8", nchan)
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 999983, 34, iono)
    bad = list(eps)
    code_bias(bad, 2, 0.3 if nchan == 5 else 0.1)
    verdicts = set()
    with gps.Context(1, 1) as ctx:
        for e in (eps, bad):
            for mx in (0, 1, 4):
                _, rec, _ = assert_kernel_equals_model(ctx, chans, e, cfg, gps.raim_config(1.0, max_exclude=mx))
                verdicts |= set(int(v) for v in rec["verdict"])
    assert verdicts == ({RM.PASS, RM.ALERT} if nchan == 5 else {RM.PASS, RM.ALERT, RM.EXCLUDED})


@pytest.mark.parametrize("label", [f[0] for f in sky12_faults()])
def test_kernel_equals_model_on_single_faults(label, tmp_path):
    _, c, edit = next(f for f in sky12_faults() if f[0] == label)
    _, chans, eps, cfg, _ = sky12_fault_case(edit, tmp_path)
    with gps.Context(1, 1) as ctx:
        _, rec, _ = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.raim_config(1.0))
    assert (rec["verdict"] == RM.EXCLUDED).all() and (rec["excluded"] == 1 << c).all()


def test_kernel_equals_model_on_32_channels(tmp_path):
    _, chans, eps, cfg, _ = sky32_two_faults(tmp_path)
    with gps.Context(1, 1) as ctx:
        for mx, verdict in ((2, RM.EXCLUDED), (1, RM.ALERT), (4, RM.EXCLUDED)):
            _, rec, _ = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.raim_config(1.0, max_exclude=mx))
            assert (rec["verdict"] == verdict).all()


def test_kernel_equals_model_as_channels_come_and_go(tmp_path):
    """Six channels, channel 5 tracked from 4 s to 6 s and channel 4 to 5 s: fixes with 6, 5 and 4 channels used;
    UNAVAILABLE (and NaN protection levels) below 5."""
    _, _, chans, eps = sky("sky12_static_35s_i8", 6)
    _, _, iono = rinex(tmp_path, 12)
    eps[5] = eps[5][4000:6000]
    chans[5]["anchor_epoch"] = 0
    chans[5]["anchor_ms"] = (chans[5]["anchor_ms"] + 4000) % 604800000
    eps[4] = eps[4][:5000]
    cfg = gps.pvt_config(30000, 299993, 100, iono)
    with gps.Context(1, 1) as ctx:
        got, rec, _ = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.raim_config(1.0))
    assert {int(n) for n in got["nused"]} >= {4, 5, 6}
    assert (rec["verdict"][got["nused"] < 5] == RM.UNAVAILABLE).all()
    assert np.isnan(rec["hpl"][got["nused"] < 5]).all() and np.isfinite(rec["hpl"][got["nused"] >= 5]).all()


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8"])
def test_fault_free_fixes_are_those_of_pvt(name, tmp_path):
    """RAIM on, no fault: fixes and residuals bit for bit those of gpsb200_pvt; replay runs whichever call ran last."""
    _, ch, chans, eps = sky(name)
    _, _, iono = rinex(tmp_path, len(eps))
    cfg = gps.pvt_config(12345, 3001, 9000, iono)
    with gps.Context(1, 1) as ctx:
        fix, res = ctx.pvt(chans, eps, cfg, want_residuals=True)
        rfix, rec, rres = ctx.pvt_raim(chans, eps, cfg, gps.raim_config(1.0), want_residuals=True)
        ctx.pvt_replay()
        ctx.pvt(chans, eps, cfg)
        ctx.pvt_replay()
    assert (rec["verdict"] == RM.PASS).all()
    assert fix.tobytes() == rfix.tobytes() and res.tobytes() == rres.tobytes()


def test_end_to_end_faulty_clock(tmp_path):
    """02:00:24 + 33 s of sky12 with one PRN broadcasting af0 + 1 us, synthesized, acquired, tracked and decoded on the
    GPU, the ephemeris and time anchor read from the tracked words: every fix from 0.5 s excludes exactly that PRN and
    lands within the tracked bounds; without RAIM the same fixes are more than 100 m off."""
    nav, _, iono = rinex(tmp_path, 12, sets=2)     # a second set, so that 02:00:24 is inside the span
    start = (2024, 1, 7, 2, 0, 24.0)
    ch, frames = gps.scenario(nav, *LOC, seconds=33, max_chan=12, start=start)
    prn = int(ch[0]["prn"][FAULT_SLOT])
    rinex_with_af0(nav, tmp_path / "bad.nav", prn, AF0_ERROR)
    ch2, bad = gps.scenario(str(tmp_path / "bad.nav"), *LOC, seconds=33, max_chan=12, start=start)
    assert np.array_equal(ch2["prn"], ch["prn"]) and (ch["prn"][:, FAULT_SLOT] == prn).all()
    frames = np.array(frames, copy=True)
    frames[:, FAULT_SLOT] = bad[:, FAULT_SLOT]
    with gps.Context(12, ch.shape[0], max_nav_frames=len(frames)) as ctx:
        ctx.set_nav_frames(frames)
        out, _ = ctx.synth_blocks(ch, gps.SC08)
        prns = [int(p) for p in ch[0]["prn"] if p > 0]
        eps = gpu_track(ctx, out, gps.SC08, prns)
        chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
        for c, (p, e) in enumerate(zip(prns, eps)):
            _, words, sy = gps.nav_decode(e)
            chans[c]["eph"], _ = gps.nav_ephemeris(words)
            assert chans[c]["eph"]["valid"] == 1, p
            chans[c]["prn"] = p
            chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = gps.nav_time_anchor(words, sy)
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        fix, rec, _ = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.raim_config(TRACKED_SIGMA))
        plain = ctx.pvt(chans, eps, cfg)
    c = prns.index(prn)
    assert (rec["verdict"] == RM.EXCLUDED).all() and (rec["excluded"] == 1 << c).all()
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    sow = START_SOW + 24.0
    check_truth(fix, xyz, sow, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])
    tx, _ = truth_xyz(xyz, plain["sample"])
    off = np.linalg.norm(np.stack([plain["x"], plain["y"], plain["z"]], 1) - tx, axis=1)
    assert off.min() > 100.0, off.min()


def test_bad_raim_configs_are_rejected_and_the_context_still_synthesizes(tmp_path):
    g = scenario.load_golden("sky12_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, chans, eps = sky("sky12_static_35s_i8", 6)
    cfg = gps.pvt_config(30000, 3000, 10)
    good = gps.raim_config(1.0)

    def bad(f, v):
        r = good.copy()
        r[f] = v
        return r
    cases = [bad("sigma", 0.0), bad("sigma", -1.0), bad("sigma", np.inf), bad("sigma", np.nan), bad("p_fa", 0.6),
             bad("p_fa", 1e-13), bad("p_md", 0.0), bad("p_md", np.nan), bad("max_exclude", -1), bad("max_exclude", 5),
             bad("reserved", 1)]
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(frames)
        for r in cases:
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.pvt_raim(chans, eps, cfg, r)
            assert e.value.code == ERR_ARG, r
        with pytest.raises(gps.GpsB200Error) as e:             # the checks of gpsb200_pvt apply too
            ctx.pvt_raim(chans, eps, gps.pvt_config(30000, 0, 10), good)
        assert e.value.code == ERR_ARG
        fix, rec = ctx.pvt_raim(chans, eps, cfg, good)
        assert (fix["status"] == gps.FIX_OK).all() and (rec["verdict"] == RM.PASS).all()
        out, _ = ctx.synth_blocks(ch[:1], gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]


VERDICT = {RM.PASS: "PASS", RM.EXCLUDED: "EXCLUDED", RM.ALERT: "ALERT", RM.UNAVAILABLE: "UNAVAILABLE"}


def test_cli_raim_prints_what_the_api_returns(tmp_path):
    """gpsb200-track --fix --raim on the CLI test's file: each fix row carries pvt_raim's verdict, excluded PRNs and
    HPL / VPL after the columns it has without --raim, which stay as they are."""
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-track")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav, _, (alpha, beta) = rinex(tmp_path, 12, sets=2)
    iq = tmp_path / "iq.bin"
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", "35.681298,139.766247,10.0", "-d", "33",
                           "-s", "2024/01/07,02:00:24", "-o", str(iq)])
    iono = ",".join("%.17g" % v for v in list(alpha) + list(beta))
    base = [os.path.join(exe_dir, "gpsb200-track"), str(iq), "--fix", "--fix-every", "500", "--iono", iono]
    plain = subprocess.run(base, capture_output=True, text=True, check=True).stdout.splitlines()
    raim = subprocess.run(base + ["--raim", "8,1e-5,1e-3,1"], capture_output=True, text=True, check=True).stdout.splitlines()
    rows = lambda lines: [ln.split() for ln in lines[next(i for i, ln in enumerate(lines) if ln.startswith("# sample")) + 1:]
                          if ln and not ln.startswith("#")]
    prow, rrow = rows(plain), rows(raim)
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
        cfg = gps.pvt_config(1500000, 1500000, (end - 1500000) // 1500000 + 1, (alpha, beta))
        fix, rec = ctx.pvt_raim(chans, eps, cfg, gps.raim_config(8.0, 1e-5, 1e-3, 1))
    ok = fix["status"] == gps.FIX_OK
    fix, rec = fix[ok], rec[ok]
    assert len(rrow) == fix.size >= 40 and len(prow) >= 40
    for r, f, q in zip(rrow, fix, rec):
        assert r[0] == str(f["sample"])
        assert r[1:7] == ["%.9f" % f["t_rx"], "%.8f" % f["lat_deg"], "%.8f" % f["lon_deg"], "%.3f" % f["height"],
                          "%.3f" % f["clock_m"], "%.3f" % f["vx"]]
        assert r[7:11] == ["%.3f" % f["vy"], "%.3f" % f["vz"], str(f["nused"]), "%.2f" % f["pdop"]]
        excl = [str(int(chans[c]["prn"])) for c in range(len(chans)) if int(q["excluded"]) >> c & 1]
        assert r[11:] == [VERDICT[int(q["verdict"])], ",".join(excl) or "-", "%.2f/%.2f" % (q["hpl"], q["vpl"])]
    # a fix that excluded nothing is the fix printed without --raim
    plain_of = {r[0]: r for r in prow}
    for r, q in zip(rrow, rec):
        if q["excluded"] == 0:
            assert r[:11] == plain_of[r[0]]
