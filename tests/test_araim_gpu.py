"""ARAIM on the GPU (gpsb200_pvt_araim, Context.pvt_araim, gpsb200-track --fix --araim): the kernel against the numpy
model (tests/araim_model.py) at 5, 6, 12 and 32 channels, fault-free and with an injected code bias, across the week
roll, at 60 deg N, on a gapped channel and shifted by 2^33; the whole receiver chain on the GPU with and without a PRN
whose broadcast clock is wrong; bad configurations refused; the CLI; an exclusion under compute-sanitizer."""
import os
import subprocess
import sys

import numpy as np
import pytest

import araim_model as AM
import pvt_model as PM
from scenario import gps
from test_araim import kfa, new_trace, assert_margin
from test_pvt import rinex
from test_pvt_gpu import FIELDS
from test_raim import code_bias, sky

pytestmark = pytest.mark.gpu

ERR_ARG = -1
EXACT = ("verdict", "excluded", "masked", "n")


def rel_close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same = (np.isnan(a) & np.isnan(b)) | (a == b)
    return bool(np.all(same | (np.abs(a - b) <= tol * np.abs(b))))


def assert_kernel_equals_model(ctx, chans, eps, cfg, acfg):
    got, grec, gres = ctx.pvt_araim(chans, eps, cfg, acfg, want_residuals=True)
    tr = new_trace()
    want, wres, wrec, _ = AM.araim(chans, eps, cfg, acfg, *kfa(acfg), trace=tr)
    assert_margin(tr)
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(got[f], want[f].astype(got[f].dtype)), (f, got[f], want[f])
    for f in EXACT:
        assert np.array_equal(grec[f], wrec[f].astype(grec[f].dtype)), (f, grec[f], wrec[f])
    ok = got["status"] == gps.FIX_OK
    for f in FIELDS:
        assert np.all(np.abs(got[f][ok] - want[f][ok]) < 1e-6), (f, np.abs(got[f][ok] - want[f][ok]).max())
    both = ~np.isnan(gres)
    assert np.array_equal(both, ~np.isnan(wres)) and np.all(np.abs(gres[both] - wres[both]) < 1e-6)
    # sigmas and thresholds come from rows that agree to ~1 um over ranges of 2e7 m; the test ratio |dx| / T also from
    # residuals 1 um apart, so it may differ by what 1 um over thresholds of metres allows
    for f in ("emt", "sigma_acc_v", "p_nm"):
        assert rel_close(grec[f], wrec[f], 1e-9), (f, grec[f], wrec[f])
    a, b = grec["test_ratio"], wrec["test_ratio"]
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.all(np.abs(a - b)[~np.isnan(b)] <= 1e-7 * b[~np.isnan(b)] + 1e-6)
    for f in ("hpl", "vpl"):
        a, b = grec[f], wrec[f]
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.all(np.abs(a - b)[~np.isnan(b)] <= 1e-3 + 1e-9 * b[~np.isnan(b)]), \
            (f, a, b)
    return got, grec


@pytest.mark.parametrize("nchan", [5, 6, 12])
def test_kernel_equals_model_on_sky12(nchan, tmp_path):
    _, _, chans, eps = sky("sky12_static_35s_i8", nchan)
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 1999993, 6, iono)
    bad = list(eps)
    code_bias(bad, 2, 0.3)
    verdicts = set()
    with gps.Context(1, 1) as ctx:
        for e in (eps, bad):
            for mx in (0, 1):
                for mask in (5.0, 10.0):
                    _, rec = assert_kernel_equals_model(ctx, chans, e, cfg, gps.araim_config(mask_deg=mask,
                                                                                             max_exclude=mx))
                    verdicts |= set(int(v) for v in rec["verdict"])
    assert AM.PASS in verdicts and AM.ALERT in verdicts
    if nchan >= 6:
        assert AM.EXCLUDED in verdicts


def test_kernel_equals_model_on_32_channels(tmp_path):
    _, _, chans, eps = sky("sky32_static_10s_i8")
    _, _, iono = rinex(tmp_path, 32)
    cfg = gps.pvt_config(30000, 999991, 8, iono)
    bad = list(eps)
    code_bias(bad, 20, 0.3)
    with gps.Context(1, 1) as ctx:
        _, rec = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.araim_config(mask_deg=10.0))
        assert (rec["verdict"] == AM.PASS).all()
        _, rec = assert_kernel_equals_model(ctx, chans, bad, cfg, gps.araim_config(mask_deg=10.0))
        assert (rec["verdict"] == AM.EXCLUDED).all() and (rec["excluded"] == 1 << 20).all()


def test_ura_index_15_is_never_used(tmp_path):
    _, _, chans, eps = sky("sky12_static_35s_i8")
    _, _, iono = rinex(tmp_path, 12)
    cfg = gps.pvt_config(30000, 1999993, 3, iono)
    chans = chans.copy()
    chans[3]["eph"]["ura"] = 15
    chans[4]["eph"]["ura"] = 8
    with gps.Context(1, 1) as ctx:
        got, _ = assert_kernel_equals_model(ctx, chans, eps, cfg, gps.araim_config())
    assert not ((got["mask"] >> 3) & 1).any()


def test_bad_araim_configs_are_rejected(tmp_path):
    _, _, chans, eps = sky("sky12_static_35s_i8", 6)
    cfg = gps.pvt_config(30000, 3000, 10)
    good = gps.araim_config()

    def bad(f, v):
        r = good.copy()
        r[f] = v
        return r
    cases = [bad("mask_deg", -1.0), bad("mask_deg", 91.0), bad("sigma_ura", 0.0), bad("sigma_ura", np.nan),
             bad("sigma_ure", 2.0), bad("sigma_ure", 0.0), bad("sigma_noise", -1.0), bad("b_nom", np.inf),
             bad("p_sat", 0.0), bad("p_sat", 0.1), bad("p_hmi_vert", 0.6), bad("p_hmi_horz", 0.0),
             bad("p_fa_vert", np.nan), bad("p_fa_horz", 1e-13), bad("max_exclude", 2), bad("max_exclude", -1)]
    r = good.copy()
    r["reserved"][1] = 1
    cases.append(r)
    with gps.Context(1, 1) as ctx:
        for r in cases:
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.pvt_araim(chans, eps, cfg, r)
            assert e.value.code == ERR_ARG, r
        c2 = chans.copy()
        c2[0]["eph"]["ura"] = 16
        with pytest.raises(gps.GpsB200Error):
            ctx.pvt_araim(c2, eps, cfg, good)
        fix, rec = ctx.pvt_araim(chans, eps, cfg, good)
        assert (fix["status"] == gps.FIX_OK).all()


@pytest.mark.parametrize("case", ["weekroll", "lat60", "gap"])
def test_kernel_equals_model_on_the_edge_cases(case, tmp_path):
    """The fix cases of tests/test_receiver_edges_gpu.py (Klobuchar on): across the week roll, at 60 deg N while
    satellites rise and set, and on a channel resuming after a 2.2 s gap; masks 5 and 10 deg. Shifted by 2^33 the
    fixes, records and residuals are byte-equal apart from `sample`."""
    from test_receiver_edges_gpu import CASES, SHIFT, shifted
    chans, eps, cfg, _ = CASES[case](tmp_path)
    with gps.Context(1, 1) as ctx:
        for mask in (5.0, 10.0):
            acfg = gps.araim_config(mask_deg=mask)
            fix, rec = assert_kernel_equals_model(ctx, chans, eps, cfg, acfg)
            _, _, res = ctx.pvt_araim(chans, eps, cfg, acfg, want_residuals=True)
            e2, c2 = shifted(eps, cfg)
            fix2, rec2, res2 = ctx.pvt_araim(chans, e2, c2, acfg, want_residuals=True)
            assert np.array_equal(fix2["sample"], fix["sample"] + SHIFT)
            fix2["sample"] -= SHIFT
            assert fix.tobytes() == fix2.tobytes() and rec.tobytes() == rec2.tobytes() and res.tobytes() == res2.tobytes()
            assert np.isin(rec["verdict"], (AM.PASS, AM.UNAVAILABLE)).all()
            if case == "lat60":
                assert rec["masked"].any()


def gpu_chain(tmp_path, faulty):
    """02:00:24 + 33 s of sky12 synthesized, acquired, tracked and decoded on the GPU (tests/test_raim_gpu.py's chain),
    with or without FAULT_SLOT's PRN broadcasting af0 + 1 us. -> (chans, eps, fix config, prns, prn of the slot, ch)"""
    from test_pvt_gpu import gpu_track
    from test_raim import FAULT_SLOT, rinex_with_af0, AF0_ERROR
    from test_scenario import LOC
    nav, _, iono = rinex(tmp_path, 12, sets=2)
    start = (2024, 1, 7, 2, 0, 24.0)
    ch, frames = gps.scenario(nav, *LOC, seconds=33, max_chan=12, start=start)
    prn = int(ch[0]["prn"][FAULT_SLOT])
    if faulty:
        rinex_with_af0(nav, tmp_path / "bad.nav", prn, AF0_ERROR)
        _, bad = gps.scenario(str(tmp_path / "bad.nav"), *LOC, seconds=33, max_chan=12, start=start)
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
    return chans, eps, gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono), prns, prn, ch


def test_end_to_end_chain(tmp_path):
    """The whole chain on the GPU, sigma_ura 8 m: the fault-free stream passes with the truth errors below the
    protection levels along the run; with one PRN broadcasting af0 + 1 us every fix from 0.5 s excludes that PRN."""
    from pvt_truth import truth_xyz
    from test_araim import ARAIM_TRACKED
    from test_scenario import LOC
    acfg = gps.araim_config(**ARAIM_TRACKED)
    chans, eps, cfg, prns, prn, ch = gpu_chain(tmp_path, False)
    with gps.Context(1, 1) as ctx:
        fix, rec = assert_kernel_equals_model(ctx, chans, eps, cfg, acfg)
    assert (rec["verdict"] == AM.PASS).all(), rec["verdict"]
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    tx, _ = truth_xyz(xyz, fix["sample"])
    err = (np.stack([fix["x"], fix["y"], fix["z"]], 1) - tx) @ AM.enu(PM.llh_ecef(*LOC)).T
    assert np.all(np.hypot(err[:, 0], err[:, 1]) < rec["hpl"]) and np.all(np.abs(err[:, 2]) < rec["vpl"])
    chans, eps, cfg, prns, prn, _ = gpu_chain(tmp_path, True)
    with gps.Context(1, 1) as ctx:
        _, rec = assert_kernel_equals_model(ctx, chans, eps, cfg, acfg)
    assert (rec["verdict"] == AM.EXCLUDED).all() and (rec["excluded"] == 1 << prns.index(prn)).all(), rec["verdict"]


VERDICT = {AM.PASS: "PASS", AM.EXCLUDED: "EXCLUDED", AM.ALERT: "ALERT", AM.UNAVAILABLE: "UNAVAILABLE"}


def test_cli_araim_prints_what_the_api_returns(tmp_path):
    """gpsb200-track --fix --araim on the CLI test's file: each fix row carries pvt_araim's verdict, excluded PRN,
    masked PRNs, HPL / VPL and EMT after the columns it has without --araim."""
    import scenario
    from test_track import ACQ, starts
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-track")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav, _, (alpha, beta) = rinex(tmp_path, 12, sets=2)
    iq = tmp_path / "iq.bin"
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav, "-l", "35.681298,139.766247,10.0", "-d", "33",
                           "-s", "2024/01/07,02:00:24", "-o", str(iq)])
    iono = ",".join("%.17g" % v for v in list(alpha) + list(beta))
    base = [os.path.join(exe_dir, "gpsb200-track"), str(iq), "--fix", "--fix-every", "500", "--iono", iono]
    lines = subprocess.run(base + ["--araim", "5,8,5.3333333333333333,0.75,1e-5"], capture_output=True, text=True,
                           check=True).stdout.splitlines()
    rows = [ln.split() for ln in lines[next(i for i, ln in enumerate(lines) if ln.startswith("# sample")) + 1:]
            if ln and not ln.startswith("#")]
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
        acfg = gps.araim_config(mask_deg=5.0, sigma_ura=8.0, sigma_ure=5.3333333333333333, b_nom=0.75, p_sat=1e-5)
        fix, rec = ctx.pvt_araim(chans, eps, cfg, acfg)
    ok = fix["status"] == gps.FIX_OK
    fix, rec = fix[ok], rec[ok]
    assert len(rows) == fix.size >= 40
    prn_list = lambda bits: ",".join(str(int(chans[c]["prn"])) for c in range(len(chans)) if int(bits) >> c & 1) or "-"
    for r, f, q in zip(rows, fix, rec):
        assert r[0] == str(f["sample"])
        assert r[1:11] == ["%.9f" % f["t_rx"], "%.8f" % f["lat_deg"], "%.8f" % f["lon_deg"], "%.3f" % f["height"],
                           "%.3f" % f["clock_m"], "%.3f" % f["vx"], "%.3f" % f["vy"], "%.3f" % f["vz"],
                           str(f["nused"]), "%.2f" % f["pdop"]]
        assert r[11:] == [VERDICT[int(q["verdict"])], prn_list(q["excluded"]), prn_list(q["masked"]),
                          "%.2f/%.2f" % (q["hpl"], q["vpl"]), "%.2f" % q["emt"]]


def araim_exclusion_run():
    """One ARAIM call on 12 sky12 channels with a code bias on channel 2 that every fix excludes -> its bytes (hex)."""
    import hashlib
    _, _, chans, eps = sky("sky12_static_35s_i8")
    code_bias(eps, 2, 0.3)
    with gps.Context(1, 1) as ctx:
        fix, rec, res = ctx.pvt_araim(chans, eps, gps.pvt_config(30000, 999983, 34), gps.araim_config(),
                                      want_residuals=True)
    assert (rec["verdict"] == AM.EXCLUDED).all() and (rec["excluded"] == 1 << 2).all(), rec["verdict"]
    return hashlib.sha256(fix.tobytes() + rec.tobytes() + res.tobytes()).hexdigest()


def test_araim_exclusion_clean_under_compute_sanitizer():
    """An ARAIM call that excludes a channel under compute-sanitizer memcheck; where the tool reports the device
    unsupported, the fallback of tests/test_sanitizers.py: CUDA reports no error and repeated runs are equal."""
    import shutil
    import scenario
    from test_sanitizers import _device_not_supported
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_araim_gpu as A; "
            "print('ok', A.araim_exclusion_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1500)
    if _device_not_supported(r):
        import torch
        want = araim_exclusion_run()
        for _ in range(3):
            assert araim_exclusion_run() == want
        torch.cuda.synchronize()                                  # raises on an illegal address or any sticky error
        return
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-500:])
    assert plain.stdout.split()[-1] == r.stdout.split()[-1]
