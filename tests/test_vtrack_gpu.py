"""gpsb200_vtrack on the H100 against its numpy model (tests/vtrack_model.py) and the scenario's truth.

- Correlators bit for bit: with the kernel's commands replayed, the model's epochs and interval sums equal the
  kernel's on signal (int8 and int16) and on random int8; the filter's fixes agree within 1e-6 m.
- Determinism: any cut of a run into calls, any cluster size, and repeated calls give the same bytes.
- Truth: the clean 12-channel stream (10 s) and the 32-channel one (3 s), with test_vtrack's bounds.
- A device source gives the host source's results; bad arguments are refused and the context still works."""
import numpy as np
import pytest

import pvt_model as PM
import vtrack_model as V
from scenario import gps
from test_scenario import LOC
from test_track import START_SOW
import pvt_truth as PT
from test_vtrack import (SETTLE, WEAK_GAIN, WEAK_PRNS, check_truth, check_weak, chans_of, scalar_lost, seed_x,
                         stream)

pytestmark = pytest.mark.gpu
MAX_COMMAND_DIFF = 0.01


def setup(tmp_path, name, nblk, nsat):
    g, ch, iq = stream(name, nblk)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    return g, ch, iq, prns, chans_of(tmp_path, nsat, prns)


@pytest.fixture(scope="module")
def ctx():
    with gps.Context(32, 1) as c:
        yield c


@pytest.fixture(scope="module")
def sky12(tmp_path_factory):
    return setup(tmp_path_factory.mktemp("nav12"), "sky12_static_35s_i8", 100, 12)


def state0(prns, cfg):
    return gps.vtrack_seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, 0, prns)


def seeded(ctx, chans, cfg, st):
    """The state after the device's first call on one sample: the channels started (header 'first'), no period run.
    Its code phases come from rounded doubles, so the model starts from these integers as it replays the commands."""
    f, _, _, s = ctx.vtrack(chans, cfg, st, 1, iq=np.zeros(2, np.int8))
    assert len(f) == 0 and s["seeded"] == 1
    return s


def check_model(iq, ss, chans, cfg, st, fixes, outs, eps, st_after, base=0, max_updates=None):
    """max_updates: that of a kernel call that stopped by it (None: the call ran to its buffer's end)."""
    mu = len(fixes) + 1 if max_updates is None else max_updates
    mf, mo, me, mst = V.run(iq, ss, base, st, chans, cfg, mu, replay=outs)
    assert len(mf) == len(fixes)
    for f in ("sample", "e", "l", "p", "s", "dot", "cross", "prn", "used", "q"):
        assert np.array_equal(mo[f], outs[f]), f
    # the commands: the model's own against the kernel's. Both round doubles from CUDA's and numpy's transcendental
    # functions, which differ by ulps, so a command may differ by one unit where its double lies within ulps of a
    # rounding or division boundary; no more often than MAX_COMMAND_DIFF of the commands.
    for f in ("code_step", "carr_step"):
        d = np.abs(mo[f].astype(np.int64) - outs[f].astype(np.int64))
        assert d.max() <= 1, (f, d.max())
        assert np.count_nonzero(d) <= MAX_COMMAND_DIFF * d.size, (f, np.count_nonzero(d), d.size)
        print("%s: %d of %d commands differ by one unit" % (f, np.count_nonzero(d), d.size))
    for c in range(len(eps)):
        assert eps[c].size == me[c].size, c
        for f in eps[c].dtype.names:
            bad = np.nonzero(eps[c][f] != me[c][f])[0]
            assert bad.size == 0, (c, f, bad[:5], eps[c][f][bad[:3]], me[c][f][bad[:3]])
    kx = np.stack([fixes["x"], fixes["y"], fixes["z"], fixes["vx"], fixes["vy"], fixes["vz"], fixes["clock_m"],
                   fixes["drift"]], 1)
    assert np.abs(kx - np.array([f["x"] for f in mf])).max() <= 1e-6
    assert np.abs(mo["code_res_m"] - outs["code_res_m"]).max() <= 1e-6
    assert np.abs(mo["rate_res_mps"] - outs["rate_res_mps"]).max() <= 1e-6
    assert np.array_equal(fixes["mask"], [f["mask"] for f in mf])
    assert mst["ch"].tobytes() == st_after["ch"].tobytes()
    check_fix_fields(fixes, outs, mf, mo, st, mst, st_after)


FIX_REFS_MAX = 200        # fixes checked against the 50-digit references per call (evenly spaced)


def check_fix_fields(fixes, outs, mf, mo, st, mst, st_after):
    """The rest of the fix record, the channel records and the state after the call against the model's, and t_rx and
    the geodetic coordinates against 50-digit references computed from the kernel's own outputs."""
    from test_vtrack_edges import geodetic_exact, t_rx_exact
    for f in ("sample", "status", "nused"):
        assert np.array_equal(fixes[f], [m[f] for m in mf]), f
    assert (fixes["iterations"] == 1).all()
    rms = np.array([m["rms"] for m in mf])
    assert np.array_equal(np.isnan(fixes["rms"]), np.isnan(rms)) and np.array_equal(np.isnan(rms), fixes["nused"] == 0)
    assert np.nan_to_num(np.abs(fixes["rms"] - rms)).max(initial=0.0) <= 1e-6
    pdop = np.array([m["pdop"] for m in mf])
    few = fixes["status"] == gps.FIX_FEW
    assert np.array_equal(np.isnan(fixes["pdop"]), few) and np.array_equal(np.isnan(pdop), few)
    # X agrees within 1e-6 m, so the lines of sight differ by ~5e-14 and the inverse of G by its condition number
    # (about nused PDOP^2) times that: 1e-9 on a good geometry, more on the near-singular ones of a few channels on noise
    tol = 1e-9 + 1e-12 * fixes["nused"] * np.nan_to_num(pdop) ** 2
    rel = np.nan_to_num(np.abs(fixes["pdop"] / pdop - 1))
    assert (rel <= tol).all(), (rel.max(), pdop[np.argmax(rel / tol)], fixes["nused"][np.argmax(rel / tol)])
    for f in ("sigma_code_m", "sigma_rate_mps"):
        assert np.array_equal(outs[f], mo[f]), f
        assert np.array_equal(np.isinf(outs[f]), outs["used"] == 0), f
    for f in ("t_f", "updates", "seeded"):
        assert int(st_after[f]) == int(mst[f]), (f, st_after[f], mst[f])
    assert np.abs(st_after["x"] - mst["x"]).max() <= 1e-6
    P, Pm = st_after["P"], mst["P"]
    d = np.sqrt(np.abs(np.diag(Pm)))
    assert (np.abs(P - Pm) <= 1e-9 * np.outer(d, d)).all(), np.abs(P - Pm).max()
    for k in np.unique(np.linspace(0, len(fixes) - 1, min(len(fixes), FIX_REFS_MAX)).astype(int)):
        f = fixes[k]
        assert abs(f["t_rx"] - t_rx_exact(st, f)) <= 1.2e-10, (k, f["t_rx"] - t_rx_exact(st, f))
        lat, lon, h = geodetic_exact([f["x"], f["y"], f["z"]])
        assert abs(f["lat_deg"] - lat) <= 1e-10 and abs(f["lon_deg"] - lon) <= 1e-10 and abs(f["height"] - h) <= 1e-5, k


def check_covariance(st):
    """The filter's P after a long run: symmetric within 1e-9 relative and positive definite (a Cholesky factor)."""
    P = st["P"]
    d = np.sqrt(np.diag(P))
    assert (np.abs(P - P.T) <= 1e-9 * np.outer(d, d)).all()
    np.linalg.cholesky(P)


def test_correlators_and_filter_equal_the_model(ctx, sky12):
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config()
    st = seeded(ctx, chans, cfg, state0(prns, cfg))
    n = 2 * 3000000
    fixes, outs, eps, st2 = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], want_epochs=True)
    assert len(fixes) >= 95 and (fixes["status"] == gps.FIX_OK).all()
    check_model(iq[:2 * n], 1, chans, cfg, st, fixes, outs, eps, st2)


def test_random_int8_and_int16_equal_the_model(ctx, sky12, tmp_path):
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config(periods=7)
    st = seeded(ctx, chans, cfg, state0(prns, cfg))
    rng = np.random.default_rng(5)
    noise = rng.integers(-128, 128, 2 * 300000, dtype=np.int64).astype(np.int8)
    fixes, outs, eps, st2 = ctx.vtrack(chans, cfg, st, 1000, iq=noise, want_epochs=True)
    assert len(fixes) >= 10
    check_model(noise, 1, chans, cfg, st, fixes, outs, eps, st2)
    # int16 at full scale (the reduction saturates)
    n16 = (rng.integers(-32768, 32768, 2 * 200000, dtype=np.int64)).astype(np.int16)
    fixes, outs, eps, st2 = ctx.vtrack(chans, cfg, st, 1000, iq=n16, sample_size=gps.SC16, want_epochs=True)
    check_model(n16, 2, chans, cfg, st, fixes, outs, eps, st2)


def test_any_cut_and_cluster_is_one_call(ctx, sky12):
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config(periods=13)
    st = state0(prns, cfg)
    n = 3000000
    ref = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], want_epochs=True)
    again = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], want_epochs=True)
    for a, b in zip(ref[:2], again[:2]):
        assert a.tobytes() == b.tobytes()
    for K in (1, 5, 12):
        ctx.debug_vtrack_cluster(K)
        got = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], want_epochs=True)
        assert got[0].tobytes() == ref[0].tobytes() and got[1].tobytes() == ref[1].tobytes(), K
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got[2], ref[2])), K
        assert got[3].tobytes() == ref[3].tobytes(), K
    ctx.debug_vtrack_cluster(0)
    # odd chunk lengths and update counts
    s = st
    fx, ou = [], []
    eps = [[] for _ in prns]
    base = 0
    for chunk, mu in ((123457, 1000), (700001, 3), (1, 5), (999999, 1), (n, 1000)):
        hi = min(n, base + chunk)
        while True:
            f, o, e, s = ctx.vtrack(chans, cfg, s, mu, iq=iq[2 * base:2 * hi], base=base, want_epochs=True)
            fx.append(f)
            ou.append(o)
            for c in range(len(prns)):
                eps[c].append(e[c])
            if len(f) < mu:
                break
        base = min(int(s["ch"]["nco"]["sample"][:len(prns)].min()), hi)
        if hi == n:
            break
    assert np.concatenate(fx).tobytes() == ref[0].tobytes()
    assert np.concatenate(ou).tobytes() == ref[1].tobytes()
    for c in range(len(prns)):
        assert np.concatenate(eps[c]).tobytes() == ref[2][c].tobytes(), c
    assert s.tobytes() == ref[3].tobytes()


@pytest.mark.parametrize("name,nblk,nsat", [("sky12_static_35s_i8", 100, 12), ("sky32_static_10s_i8", 30, 32)])
def test_truth(ctx, name, nblk, nsat, tmp_path, sky12):
    g, ch, iq, prns, chans = sky12 if name.startswith("sky12") else setup(tmp_path, name, nblk, nsat)
    x0 = PM.llh_ecef(*LOC)
    cfg = gps.vtrack_config()
    fixes, outs, eps, _ = ctx.vtrack(chans, cfg, state0(prns, cfg), 100000, iq=iq, want_epochs=True)
    assert len(fixes) >= nblk * 5 - 5
    late = fixes["sample"] >= SETTLE * 3e6
    assert (fixes["status"][late] == gps.FIX_OK).all()
    if nsat == 12:
        assert (fixes["nused"][late] == len(prns)).all()
    xyz = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
    check_truth(ch, prns, eps, xyz, fixes["sample"], lambda s: np.broadcast_to(x0, (s.size, 3)))


def test_weakened_stream(ctx, tmp_path):
    """PRNs 1-8 at WEAK_GAIN for 10 s: the kernel holds all eight and uses them in every fix after SETTLE, where the
    scalar loops of the model lose at least half (on the first 5 s)."""
    g, ch, iq = stream("sky12_static_35s_i8", 100, weak=WEAK_GAIN)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    lost = scalar_lost(ch[:50], prns, iq[:2 * 50 * PT.BLOCK], 1)
    assert len(set(lost) & set(WEAK_PRNS)) >= 4, lost
    chans = chans_of(tmp_path, 12, prns)
    cfg = gps.vtrack_config()
    fixes, outs, eps, _ = ctx.vtrack(chans, cfg, state0(prns, cfg), 100000, iq=iq, want_epochs=True)
    assert len(fixes) >= 495
    xyz = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
    check_weak(ch, prns, xyz, fixes["sample"], fixes["mask"], eps, PM.llh_ecef(*LOC))


def test_30s_across_the_frame_roll(ctx, tmp_path):
    """30 s of sky12_static_35s (the NAV frame rolls at 30 s of transmit time inside the run): every channel within
    the bounds after SETTLE, every fix OK with all 12 channels."""
    g, ch, iq = stream("sky12_static_35s_i8", 300)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    chans = chans_of(tmp_path, 12, prns)
    cfg = gps.vtrack_config()
    fixes, outs, eps, st = ctx.vtrack(chans, cfg, state0(prns, cfg), 100000, iq=iq, want_epochs=True)
    assert len(fixes) >= 1495
    late = fixes["sample"] >= SETTLE * 3e6
    assert (fixes["nused"][late] == 12).all()
    check_covariance(st)
    xyz = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
    x0 = PM.llh_ecef(*LOC)
    check_truth(ch, prns, eps, xyz, fixes["sample"], lambda s: np.broadcast_to(x0, (s.size, 3)))


CIRCLE_POS = 30.0         # m: test_coarse's TRACKED position bound
CIRCLE_VEL = 1.5          # m/s: test_coarse's TRACKED velocity bound


def test_moving_receiver_on_the_circle(ctx, tmp_path):
    """60 s of the int16 circle (records from the scenario engine): seeded 100 m / 1 m/s / 30 ns off the truth, every
    channel within the bounds and every fix within CIRCLE_POS and CIRCLE_VEL of pvt_truth after SETTLE. A vehicle
    accelerates, so the process noise is that of a moving receiver (accel_psd 10 m^2/s^3), not the static default."""
    import scenario
    from test_pvt import rinex
    from test_scenario import START, motion_file
    g = scenario.load_golden("sky12_circle_60s_i16")
    nav_file, _, _ = rinex(tmp_path, 12)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
    iq, _ = scenario.oracle_run(ch, nav, 2)
    rows = g["motion_rows"][:, 1:4]
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    assert all((ch["prn"] == p).any(1).all() for p in prns)
    (tmp_path / "eph").mkdir()
    chans = chans_of(tmp_path / "eph", 12, prns)
    cfg = gps.vtrack_config(accel_psd=10.0)
    x_true, v_true = PT.truth_xyz(rows, np.array([0]))
    st = gps.vtrack_seed(cfg, seed_x(x_true[0], v_true[0]), START_SOW, 0, prns)
    fixes, outs, eps, st = ctx.vtrack(chans, cfg, st, 100000, iq=iq, sample_size=gps.SC16, want_epochs=True)
    assert len(fixes) >= 2990
    check_covariance(st)
    late = fixes["sample"] >= SETTLE * 3e6
    assert (fixes["status"][late] == gps.FIX_OK).all()
    xyz = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
    check_truth(ch, prns, eps, xyz, fixes["sample"], lambda s: PT.truth_xyz(rows, s)[0], pos_max=CIRCLE_POS)
    vel = np.stack([fixes["vx"], fixes["vy"], fixes["vz"]], 1)[late]
    verr = np.linalg.norm(vel - PT.truth_xyz(rows, fixes["sample"][late])[1], axis=1)
    print("circle: max position error after 1 s %.2f m, max velocity error %.3f m/s" % (
        np.linalg.norm(xyz[late] - PT.truth_xyz(rows, fixes["sample"][late])[0], axis=1).max(), verr.max()))
    assert verr.max() <= CIRCLE_VEL, verr.max()


def test_device_window_past_2_31_of_a_4_gib_buffer(ctx, sky12):
    """1 s of sky12 written across sample 2^31 of an int8 buffer of 2^31 + 2^22 samples (4.3 GB), tracked in place from
    base 0: the fixes, records and epochs equal the host call on the region alone (its base the offset)."""
    import torch
    g, ch, iq, prns, chans = sky12
    total, off, n = (1 << 31) + (1 << 22), (1 << 31) - 1000003, 3000000
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * total + (1 << 30):
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % ((2 * total + (1 << 30)) / 1e9, free / 1e9))
    cfg = gps.vtrack_config()
    st = gps.vtrack_seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, off, prns)
    ref = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], base=off, want_epochs=True)
    buf = torch.zeros(2 * total, dtype=torch.int8, device="cuda")
    buf[2 * off:2 * (off + n)] = torch.from_numpy(iq[:2 * n].copy()).cuda()
    torch.cuda.synchronize()
    got = ctx.vtrack(chans, cfg, st, len(ref[0]), device_ptr=buf.data_ptr(), nsamples=total, want_epochs=True)
    del buf
    assert len(ref[0]) >= 45 and ref[0]["sample"][-1] > 1 << 31
    assert len(got[0]) == len(ref[0])
    for k, (a, b) in enumerate(((got[0], ref[0]), (got[1], ref[1]))):
        for f in a.dtype.names:
            bad = np.nonzero((a[f] != b[f]) & ~(np.isnan(a[f]) & np.isnan(b[f])) if a[f].dtype.kind == "f" else a[f] != b[f])
            assert bad[0].size == 0, (k, f, [x[:3] for x in bad], a[f][bad][:3], b[f][bad][:3])
    # the device call stops at the host call's last update; the host call ran on into its buffer's end
    for a, b in zip(got[2], ref[2]):
        assert a.size == len(ref[0]) * int(cfg["periods"]) - int(st["ch"][0]["k"])
        assert a.tobytes() == b[:a.size].tobytes()


def test_device_source_equals_host(ctx, sky12):
    import torch
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config()
    st = state0(prns, cfg)
    n = 1500000
    ref = ctx.vtrack(chans, cfg, st, 1000, iq=iq[:2 * n], want_epochs=True)
    d = torch.from_numpy(iq[:2 * n].copy()).cuda()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50000000)
        d2 = d.clone()
    got = ctx.vtrack(chans, cfg, st, 1000, device_ptr=d2.data_ptr(), nsamples=n, stream=s.cuda_stream, want_epochs=True)
    torch.cuda.synchronize()
    assert got[0].tobytes() == ref[0].tobytes() and got[1].tobytes() == ref[1].tobytes()
    assert got[3].tobytes() == ref[3].tobytes()


def test_bad_arguments_are_refused(ctx, sky12):
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config()
    st = state0(prns, cfg)
    bad_cfgs = [gps.vtrack_config(periods=0), gps.vtrack_config(periods=101), gps.vtrack_config(q_min=1.0),
                gps.vtrack_config(sigma_code_m=0.0), gps.vtrack_config(accel_psd=-1.0)]
    for bc in bad_cfgs:
        with pytest.raises(gps.GpsB200Error):
            ctx.vtrack(chans, bc, st, 10, iq=iq[:600000])
    wrong = chans.copy()
    wrong[0]["prn"] += 1
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(wrong, cfg, st, 10, iq=iq[:600000])
    noeph = chans.copy()
    noeph[1]["eph"]["valid"] = 0
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(noeph, cfg, st, 10, iq=iq[:600000])
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(chans, cfg, st, 0, iq=iq[:600000])
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(chans, cfg, st, 10, iq=iq[:600000], base=1)
    late = st.copy()
    late["nchan"] = 33
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(chans, cfg, late, 10, iq=iq[:600000])
    with pytest.raises(gps.GpsB200Error):
        ctx.debug_vtrack_cluster(17)
    # a repeated PRN: refused by the seed, and in a state edited to hold one
    with pytest.raises(gps.GpsB200Error):
        gps.vtrack_seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, 0, [5, 5, 6, 7])
    twice = np.array([st], st.dtype)[0]
    twice["ch"][3]["nco"]["prn"] = twice["ch"][1]["nco"]["prn"]
    twice_chans = chans.copy()
    twice_chans[3] = chans[1]
    with pytest.raises(gps.GpsB200Error):
        ctx.vtrack(twice_chans, cfg, twice, 10, iq=iq[:600000])
    f, o, _, _ = ctx.vtrack(chans, cfg, st, 10, iq=iq[:600000])
    assert len(f) == 4 and (f["status"] == gps.FIX_OK).all()
