"""Position search on the GPU (gpsb200_pvt_search, Context.pvt_search): the kernels against the numpy model
(tests/search_model.py) at every channel count, on small grids node by node and on the default grid at a few instants,
with the samples shifted past 2^33; argument checks, memcheck, repeatability; and the whole receiver chain with no
position and no time anchor against the scenario's truth."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import pvt_model as PM
import scenario
import search_model as SM
from scenario import gps
from test_coarse import TRACKED, WEEK, unanchored
from test_coarse_gpu import DELTA_ABS, DELTA_REL, ERR_ARG, FIELDS, SHIFT, _device_not_supported
from test_pvt import check_truth, ideal_inputs, rinex
from test_pvt_gpu import gpu_track
from test_scenario import LOC, START, make_nav
from test_track import START_SOW
from test_track_gpu import signal

pytestmark = pytest.mark.gpu


def search_cfg(dt=10.0, nodes=SM.NODES_DEFAULT, s_a=0):
    t = START_SOW + dt
    return gps.search_config(t % 604800.0, s_a, WEEK + int(np.floor(t / 604800.0)), nodes)


def assert_search_equals_model(ctx, chans, eps, cfg, sc, node_rms=True):
    """Counts, winner, statuses, masks, iterations, ref, week, changed and ms equal; node_rms with the same NaN pattern
    and within 1 um; fixes, residuals and delta within test_coarse_gpu's tolerances. -> (fixes, records)."""
    ch = unanchored(chans)
    got = ctx.pvt_search(ch, eps, cfg, sc, want_residuals=True, want_ms=True, want_node_rms=node_rms)
    want = SM.search(ch, eps, cfg, sc, want_node_rms=node_rms)
    fix, rec, res, ms = got[:4]
    wfix, wrec, wres, wms = want[:4]
    if node_rms:
        nr, wnr = got[4], want[4]
        assert np.array_equal(np.isnan(nr), np.isnan(wnr))
        ok = ~np.isnan(nr)
        assert np.all(np.abs(nr[ok] - wnr[ok]) < 1e-6)
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(fix[f], wfix[f].astype(fix[f].dtype)), f
    for f in ("winner", "searched", "ok", "support", "ref", "week", "changed"):
        assert np.array_equal(rec[f], wrec[f].astype(rec[f].dtype)), (f, rec[f], wrec[f])
    assert np.array_equal(ms, wms)
    has = rec["winner"] >= 0
    for f in FIELDS:
        assert np.all(np.abs(fix[f][has] - wfix[f][has]) < 1e-6), f
    assert np.all(np.abs(fix["rms"][has] - wfix["rms"][has]) < 1e-6)
    d = np.abs(rec["delta"][has] - wrec["delta"][has])
    assert np.all(d <= DELTA_ABS + DELTA_REL * np.abs(wrec["delta"][has]))
    alt = ~np.isnan(wrec["alt_rms"])
    assert np.array_equal(alt, ~np.isnan(rec["alt_rms"]))
    assert np.all(np.abs(rec["alt_rms"][alt] - wrec["alt_rms"][alt]) < 1e-6)
    assert np.all(np.abs(rec["alt_dist"][alt] - wrec["alt_dist"][alt]) < 1e-3)
    both = ~np.isnan(res)
    assert np.array_equal(both, ~np.isnan(wres)) and np.all(np.abs(res[both] - wres[both]) < 1e-6)
    assert np.all(np.isnan(fix["x"][~has]))
    return fix, rec


def sky12(tmp_path, nchan=12):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    prns = [int(p) for p in ch[0]["prn"] if p > 0][:nchan]
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"], prns)
    return chans, eps, iono


@pytest.mark.parametrize("nchan", [1, 5, 6, 12])
def test_kernel_equals_model_on_small_grids(nchan, tmp_path):
    """sky12_static_35s, the first nchan PRNs, 1 024 and 4 096 nodes, three instants 10 s apart, the a-priori time 10 s
    late. Fewer than 6 used channels give FIX_FEW with nothing searched."""
    chans, eps, iono = sky12(tmp_path, nchan)
    cfg = gps.pvt_config(30000, 29999993, 3, iono)
    with gps.Context(1, 1) as ctx:
        for nodes in (1024, 4096):
            fix, rec = assert_search_equals_model(ctx, chans, eps, cfg, search_cfg(10.0, nodes))
            if nchan < SM.MIN_CHANNELS:
                assert (fix["status"] == gps.FIX_FEW).all() and (rec["searched"] == 0).all()
            else:
                assert (rec["searched"] > 0).all()


def test_kernel_equals_model_on_32_channels(tmp_path):
    g = scenario.load_golden("sky32_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    iono = rinex(tmp_path, 32)[2]
    with gps.Context(1, 1) as ctx:
        fix, rec = assert_search_equals_model(ctx, chans, eps, gps.pvt_config(12345, 3000001, 3, iono),
                                              search_cfg(-10.0, 4096))
        assert (fix["nused"] == 32).all()


@pytest.mark.parametrize("nchan", [12, 32])
def test_kernel_equals_model_on_the_default_grid(nchan, tmp_path):
    """The full 262 144-node grid at two instants: every fix OK, unique, and within 0.27 m of the truth."""
    if nchan == 12:
        chans, eps, iono = sky12(tmp_path)
    else:
        g = scenario.load_golden("sky32_static_10s_i8")
        ch, frames = scenario.golden_chans(g)
        chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
        iono = rinex(tmp_path, 32)[2]
    cfg = gps.pvt_config(30000, 12000007, 2, iono)
    with gps.Context(1, 1) as ctx:
        fix, rec = assert_search_equals_model(ctx, chans, eps, cfg, search_cfg(10.0), node_rms=False)
    assert (fix["status"] == gps.FIX_OK).all() and (rec["support"] == rec["ok"]).all()
    err = np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - PM.llh_ecef(*LOC), axis=1)
    assert err.max() < 0.27


def test_shift_and_repeat_are_byte_equal(tmp_path):
    """Samples shifted by 2^33 give the same bytes apart from `sample`; repeated calls, and a replay, give the same
    bytes."""
    chans, eps, iono = sky12(tmp_path)
    cfg = gps.pvt_config(30000, 2999993, 4, iono)
    sc = search_cfg(-10.0, 65536)
    ch = unanchored(chans)
    with gps.Context(1, 1) as ctx:
        a = ctx.pvt_search(ch, eps, cfg, sc, want_residuals=True, want_ms=True, want_node_rms=True)
        b = ctx.pvt_search(ch, eps, cfg, sc, want_residuals=True, want_ms=True, want_node_rms=True)
        ctx.pvt_replay()
        e2 = []
        for e in eps:
            e = e.copy()
            e["sample"] += SHIFT
            e2.append(e)
        c2, s2 = cfg.copy(), sc.copy()
        c2["s0"] += SHIFT
        s2["s_a"] += SHIFT
        c = ctx.pvt_search(ch, e2, c2, s2, want_residuals=True, want_ms=True, want_node_rms=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert (a[0]["status"] == gps.FIX_OK).all()
    assert np.array_equal(c[0]["sample"], a[0]["sample"] + SHIFT)
    c[0]["sample"] -= SHIFT
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, c))


def test_bad_configs_are_refused_before_anything_runs(tmp_path):
    g = scenario.load_golden("sky12_static_10s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch[:6], frames, g["nav_frame_of_block"])
    chans = unanchored(chans)
    good = gps.search_config(START_SOW, 0, WEEK, 1024)
    cfg = gps.pvt_config(30000, 3000, 10)

    def sc(f, v):
        a = good.copy()
        a[f] = v
        return a
    cases = [dict(search=sc("t_a", -1e-9)), dict(search=sc("t_a", 604800.0)), dict(search=sc("t_a", np.nan)),
             dict(search=sc("s_a", -1)), dict(search=sc("s_a", (1 << 62) + 1)), dict(search=sc("week", -1)),
             dict(search=sc("nodes", 63)), dict(search=sc("nodes", (1 << 22) + 1)), dict(search=sc("reserved", 1)),
             dict(cfg=gps.pvt_config(30000, 3000, 0)), dict(cfg=gps.pvt_config(30000, 0, 10)),
             dict(chans=np.repeat(chans[:1], 33), epochs=[eps[0]] * 33)]
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(frames)
        for kw in cases:
            a = dict(chans=chans, epochs=eps, cfg=cfg, search=good)
            a.update(kw)
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.pvt_search(**a)
            assert e.value.code == ERR_ARG, kw
        fix, rec = ctx.pvt_search(chans, eps, cfg, good)
        assert (rec["searched"] > 0).all()
        ctx.pvt_replay()                                      # re-runs the search
        out, _ = ctx.synth_blocks(ch[:1], gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]


def test_winner_equals_the_coarse_kernel_from_its_node(tmp_path):
    """The search runs k_pvt_coarse's solve (coarse_solve): from the winner node, gpsb200_pvt_coarse gives the same
    bytes."""
    chans, eps, iono = sky12(tmp_path)
    ch = unanchored(chans)
    cfg = gps.pvt_config(30000, 2999993, 3, iono)
    sc = search_cfg(10.0)
    with gps.Context(1, 1) as ctx:
        fix, rec, res, ms = ctx.pvt_search(ch, eps, cfg, sc, want_residuals=True, want_ms=True)
        assert (fix["status"] == gps.FIX_OK).all()
        x = gps.search_nodes(SM.NODES_DEFAULT)
        for i in range(3):
            one = gps.pvt_config(int(cfg["s0"]) + i * int(cfg["step"]), 1, 1, iono)
            ap = gps.coarse_config(x[rec["winner"][i]], sc["t_a"], sc["s_a"], sc["week"])
            f1, c1, r1, m1 = ctx.pvt_coarse(ch, eps, one, ap, want_residuals=True, want_ms=True)
            assert f1.tobytes() == fix[i:i + 1].tobytes() and r1.tobytes() == res[i:i + 1].tobytes()
            assert np.array_equal(m1, ms[i:i + 1])
            for f in ("delta", "pdop", "ref", "week", "changed"):
                assert c1[f][0] == rec[f][i], f


def test_six_channels_overflow_the_ok_list(tmp_path):
    """6 channels on the default grid: about 1 200 OK nodes, more than the list's 1 024. The status is AMBIGUOUS with no
    winner and the exact count, as in the model."""
    chans, eps, iono = sky12(tmp_path, 6)
    with gps.Context(1, 1) as ctx:
        fix, rec = assert_search_equals_model(ctx, chans, eps, gps.pvt_config(30000, 2999993, 1, iono), search_cfg(10.0),
                                              node_rms=False)
    assert (rec["ok"] > SM.max_ok(SM.NODES_DEFAULT)).all() and (rec["winner"] == -1).all()
    assert (fix["status"] == gps.FIX_AMBIGUOUS).all() and np.isnan(fix["x"]).all()


def test_week_roll(tmp_path):
    """The `-s now` run across the week roll, 4 096 nodes, the a-priori time given before the roll (at sample 0) and
    after it (in the next week): the kernels equal the model on both sides."""
    import test_receiver_edges_gpu as RE
    import test_time_overwrite as TO
    chans, eps, cfg, (xyz, sow) = RE.weekroll_case(tmp_path)
    (tmp_path / "week").mkdir()
    week, _ = TO.gps_time(TO.now_case("sky12_now_weekroll_300s_i8", tmp_path / "week")[1]["start"])
    s_a = 290 * 3000000
    t = sow + s_a / 3e6 + 10.0
    assert t >= 604800.0
    scs = [gps.search_config(sow + 10.0, 0, week, 4096), gps.search_config(t - 604800.0, s_a, week + 1, 4096)]
    with gps.Context(1, 1) as ctx:
        for sc in scs:
            fix, rec = assert_search_equals_model(ctx, chans, eps, cfg, sc)
            ok = fix["status"] == gps.FIX_OK
            assert np.array_equal(rec["week"][ok] == week + 1, fix["t_rx"][ok] < 302400.0)


def test_more_instants_than_one_pass(tmp_path):
    """65 540 instants on 64 nodes run in two passes (65 535 per pass): the instants around the seam equal a call of
    their own."""
    chans, eps, iono = sky12(tmp_path)
    ch = unanchored(chans)
    cfg = gps.pvt_config(30000, 1499, 65540, iono)
    sc = search_cfg(10.0, 64)
    with gps.Context(1, 1) as ctx:
        fix, rec, res = ctx.pvt_search(ch, eps, cfg, sc, want_residuals=True)
        one = gps.pvt_config(int(cfg["s0"]) + 65530 * 1499, 1499, 10, iono)
        f2, r2, res2 = ctx.pvt_search(ch, eps, one, sc, want_residuals=True)
    assert f2.tobytes() == fix[65530:].tobytes() and r2.tobytes() == rec[65530:].tobytes()
    assert res2.tobytes() == res[65530:].tobytes()
    assert rec["searched"].max() > 0


def sanitizer_run():
    """One 12-channel search on a 16 384-node grid -> a hex digest of its results."""
    import hashlib
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    with gps.Context(1, 1) as ctx:
        r = ctx.pvt_search(unanchored(chans), eps, gps.pvt_config(30000, 2999993, 3), search_cfg(10.0, 16384),
                           want_residuals=True, want_ms=True, want_node_rms=True)
    assert (r[0]["status"] == gps.FIX_OK).all()
    return hashlib.sha256(b"".join(x.tobytes() for x in r)).hexdigest()


def test_search_kernels_clean_under_compute_sanitizer():
    """memcheck over one call. Where the tool reports the device unsupported, the fallback of test_sanitizers: CUDA
    reports no error and repeated runs give the same bytes."""
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_search_gpu as S; "
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


# ---- the whole chain, with no position and no time anchor -------------------------------------------------------------
CHAIN = {"sky12_target_3s_i8": dict(target=(1500.5, 33.3, 120.25)), "sky12_static_35s_i8": dict()}
SITE_CHAIN = ["site_66n_100w_10s_i8", "site_66s_140e_10s_i8", "site_34s_58w_10s_i16"]


@pytest.mark.parametrize("name", list(CHAIN))
def test_chain_without_position(name, tmp_path):
    """Synthesized on the GPU (block CRCs equal to the reference's), acquired, tracked; the ephemeris from the
    scenario's frames, the a-priori time 10 s late and no position; search fixes every 10 ms from 0.5 s on the default
    grid. Every fix is OK, unique, and within the tracked per-fix bounds of test_coarse_gpu.test_chain_without_anchors."""
    kw = CHAIN[name]
    nblk = 121 if name == "sky12_static_35s_i8" else int(scenario.load_golden(name)["crcs"].shape[0])
    g, ch, out, ss = signal(nblk, name)
    if "target" in kw:
        nav = make_nav(tmp_path, 12)
        with gps.LiveScenario(nav, *LOC, seconds=3, start=START, target=kw["target"]) as live:
            x_true = np.array(live.state().xyz[:], np.float64)
    else:
        x_true = PM.llh_ecef(*LOC)
    rows = np.repeat(x_true[None], ch.shape[0] + 1, 0)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    slot_of_prn = {p: k for k, p in enumerate(int(x) for x in ch[0]["prn"]) if p > 0}
    _, _, iono = rinex(tmp_path, 12)
    with gps.Context(12, 1) as ctx:
        eps = gpu_track(ctx, out, ss, prns)
        chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
        for c, prn in enumerate(prns):
            chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(g["nav_frames"][0][slot_of_prn[prn]]))[0]
            chans[c]["prn"] = prn
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        fix, rec = ctx.pvt_search(unanchored(chans), eps, cfg, search_cfg(10.0))
    assert fix.size >= 100 and (fix["nused"] == 12).all()
    assert (fix["status"] == gps.FIX_OK).all() and (rec["support"] == rec["ok"]).all()
    check_truth(fix, rows, START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"])


@pytest.mark.parametrize("name", SITE_CHAIN)
def test_chain_without_position_at_the_sites(name, tmp_path):
    """The three site fixtures (66 deg N 100 deg W, 66 deg S 140 deg E, 34 deg S 58 deg W), synthesized with the
    reference's block CRCs, acquired and tracked; the ephemeris from the first frames, the a-priori time 10 s late;
    search fixes every 10 ms from 0.5 s, each OK and unique. Each equals gpsb200_pvt_coarse's fix from an a-priori
    position on the truth to 1 mm, so the search adds no error of its own. At the 66 deg sites the fixes are within the
    tracked per-fix bounds; on the 12-channel int16 stream at 34 deg S the coarse-time fix itself reaches 31.9 m once
    (tracking noise, the same from the truth; DESIGN §11.4), so there it is held to 35 m per fix and to the tracked mean
    bound."""
    import test_sites as TS
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    ss = int(g["sample_size"])
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    _, _, _, iono, (xyz, sow), _ = TS.fix_inputs(name, tmp_path / "a")
    week, _ = TS.gps_time(TS.site_case(name, tmp_path / "b")[1]["start"])
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    slot_of_prn = {p: k for k, p in enumerate(int(x) for x in ch[0]["prn"]) if p > 0}
    with gps.Context(ch.shape[1], ch.shape[0], max_nav_frames=len(frames)) as ctx:
        ctx.set_nav_frames(frames)
        out, _ = ctx.synth_blocks(ch, ss)
        assert np.array_equal(scenario.crc_blocks(out), g["block_crcs"])
        eps = gpu_track(ctx, out, ss, prns)
        chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
        for c, prn in enumerate(prns):
            chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(frames[0][slot_of_prn[prn]]))[0]
            chans[c]["prn"] = prn
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        t = sow + 10.0
        wk = week + int(np.floor(t / 604800.0))
        fix, rec = ctx.pvt_search(unanchored(chans), eps, cfg, gps.search_config(t % 604800.0, 0, wk))
        ref, _ = ctx.pvt_coarse(unanchored(chans), eps, cfg, gps.coarse_config(xyz[0], t % 604800.0, 0, wk))
    assert fix.size >= 100 and (fix["nused"] == len(prns)).all()
    assert (fix["status"] == gps.FIX_OK).all() and (rec["support"] == rec["ok"]).all()
    assert (ref["status"] == gps.FIX_OK).all()
    d = np.linalg.norm(np.stack([fix[f] - ref[f] for f in ("x", "y", "z")], 1), axis=1)
    assert d.max() < 1e-3, d.max()
    if name.startswith("site_66"):
        check_truth(fix, xyz, sow, TRACKED["pos"], TRACKED["time"], TRACKED["vel"])
    else:
        check_truth(fix, xyz, sow, 35.0, TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])


def test_cli_search_fixes(tmp_path):
    """gpsb200-sim -d 3 -t 1500.5,33.3,120.25 from 02:00:00, then gpsb200-track --fix --assist with the same RINEX file,
    --assist-pos search and the a-priori time 10 s late: every 10 ms from 0.5 s a fix is printed, within the tracked
    bounds of the -t start point, with delta about -10 s and support >= 1. --raim and --araim are refused with it."""
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
    track = [os.path.join(exe_dir, "gpsb200-track"), str(iq), "--fix", "--fix-every", "10", "--assist", nav,
             "--assist-pos", "search", "--assist-time", "2024/01/07,02:00:10"]
    r = subprocess.run(track, capture_output=True, text=True, check=True)
    lines = r.stdout.splitlines()
    head = next(i for i, ln in enumerate(lines) if ln.startswith("# sample"))
    assert lines[head].endswith("delta_s  support")
    rows = np.array([[float(v) for v in ln.split()] for ln in lines[head + 1:] if ln and not ln.startswith("#")])
    assert len(rows) >= 200
    xyz = np.stack([PM.llh_ecef(la, lo, h) for la, lo, h in rows[:, 2:5]])
    err = np.linalg.norm(xyz - x_true, axis=1)
    assert err.max() <= TRACKED["pos"], err.max()
    assert np.all(np.abs(rows[:, -2] + 10.0) < 0.02) and np.all(rows[:, -1] >= 1)
    for bad in (["--raim", "1"], ["--araim", "5"]):
        assert subprocess.run(track + bad, capture_output=True).returncode == 2
