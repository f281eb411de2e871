"""gpsb200_vtrack on the H100 at the edges of its contract. Every run goes through test_vtrack_gpu's check_model
(epochs, sums, channel states bit for bit with the kernel's commands replayed; every fix field, the filter's x and P
against the model; t_rx and the geodetic coordinates against 50-digit references), and each test asserts that its run
reached the edge it is about (the constructions are shown to reach them on the model in test_vtrack_edges):

- one-update calls on a device source against the matrix-form restatement of the filter (test_vtrack);
- 1 to 32 channels at cluster sizes 1, automatic and 16: FEW fixes with a NaN PDOP below 4 channels, mask bit 31,
  CTAs holding 2 channels next to CTAs holding 1;
- N = 1 (no prompt pairs), N = 100 and no process noise, on signal and on full-scale int16 noise;
- q_min at a channel's q and the next double above it, and at the 4th-largest q (OK with 4, FEW with 3);
- open loop on zeros: w at +-14 316 558, u at CODE_STEP_MIN and MAX, the code error and residual wraps;
- the first period at llround(phi 2^32) mod M = 0, 1 and M - 1;
- full-scale int8 sums at N = 100 (P and |cross| near their bounds), and the same stream as int16 two ways;
- across the GPS week roll: t_rx runs on past 604 800 s, the channels and fixes stay within test_vtrack's bounds,
  and the call spanning the roll equals the model;
- compute-sanitizer memcheck on one channel at K = 1 and 17 channels at K = 16."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import pvt_model as PM
import scenario
import track_model as T
import vtrack_model as V
from scenario import gps
from test_scenario import LOC
from test_track import START_SOW
from test_vtrack import SETTLE, batch_update, chans_of, check_truth, restated_rows, seed_x
from test_vtrack_edges import (BLOCK, W_CLAMP, WEEK_S, WEEKROLL_BLOCKS, WEEKROLL_LEAD, WRAP_TARGETS, check_full_scale,
                               command_record, full_scale_config, full_scale_plant, interval_power, open_loop_edges,
                               open_loop_seed, raw_code_residuals, weekroll_case, wrap_seed)
from test_vtrack_gpu import check_model, seeded, setup, state0

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    with gps.Context(32, 1) as c:
        yield c


@pytest.fixture(scope="module")
def sky12(tmp_path_factory):
    return setup(tmp_path_factory.mktemp("nav12"), "sky12_static_35s_i8", 10, 12)


@pytest.fixture(scope="module")
def sky32(tmp_path_factory):
    return setup(tmp_path_factory.mktemp("nav32"), "sky32_static_10s_i8", 3, 32)


def kernel_first(ctx, chans, cfg):
    return lambda st: seeded(ctx, chans, cfg, st)


def most_updates(iq, cfg):
    """The most updates a buffer of interleaved I,Q can hold (every period at least 2999 samples): the calls size
    their outputs and epoch buffers to the run, not to a fixed bound."""
    return iq.size // 2 // (2999 * int(cfg["periods"])) + 1


def run_checked(ctx, chans, cfg, st, iq, sample_size=gps.SC08, max_updates=None, base=0):
    mu = most_updates(iq, cfg) if max_updates is None else max_updates
    fixes, outs, eps, st2 = ctx.vtrack(chans, cfg, st, mu, iq=iq, sample_size=sample_size, base=base, want_epochs=True)
    check_model(iq, 1 if sample_size == gps.SC08 else 2, chans, cfg, st, fixes, outs, eps, st2, base=base,
                max_updates=max_updates)
    return fixes, outs, eps, st2


def test_one_update_calls_against_the_matrix_form(ctx, sky12):
    """The first second of sky12 as one-update calls on a device source: each call's x equals restated_rows and
    batch_update on the state before it (the kernel against the independent statement, not the replaying model)."""
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config()
    n = 3000000
    d = torch.from_numpy(iq[:2 * n].copy()).cuda()
    st = seeded(ctx, chans, cfg, state0(prns, cfg))
    calls = 0
    while True:
        f, o, _, after = ctx.vtrack(chans, cfg, st, 1, device_ptr=d.data_ptr(), nsamples=n)
        if len(f) == 0:
            break
        t_new = int(f[0]["sample"])
        Xp, Pp = V.time_update(st["x"].astype(np.float64), st["P"].astype(np.float64), (t_new - int(st["t_f"])) / V.FS,
                               cfg)
        rows, ys = restated_rows(st, after, o[0], chans, cfg, Xp, t_new)
        assert len(rows) == 2 * int(o[0]["used"].sum())
        for (yc, yr), oc in zip(ys, o[0]):
            assert abs(yc - oc["code_res_m"]) <= 1e-6 and abs(yr - oc["rate_res_mps"]) <= 1e-6
        X, _ = batch_update(Xp, Pp, rows)
        assert np.abs(X[:6] - after["x"][:6]).max() <= 1e-6, X - after["x"]
        assert np.abs(X[6:] - after["x"][6:]).max() <= 1e-9 * V.C
        st = after
        calls += 1
    assert calls >= 49 and int(st["updates"]) == calls
    del d


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 17, 31, 32])
def test_channel_counts_and_cluster_shapes(ctx, sky32, n):
    """The first n of sky32's PRNs for 0.3 s at clusters of 1, min(n, 8) and min(n, 16) CTAs (channel c on CTA
    c mod K; at n = 17 and 31 and K = 16 some CTAs hold 2 channels and others 1): the first run against the model, the
    others byte for byte equal to it."""
    g, ch, iq, prns, chans = sky32
    cfg = gps.vtrack_config()
    st = seeded(ctx, chans[:n], cfg, state0(prns[:n], cfg))
    runs = []
    try:
        for K in (1, 0, 16):
            ctx.debug_vtrack_cluster(K)
            runs.append(ctx.vtrack(chans[:n], cfg, st, 1000, iq=iq, want_epochs=True))
    finally:
        ctx.debug_vtrack_cluster(0)
    fixes, outs, eps, st2 = runs[0]
    check_model(iq, 1, chans[:n], cfg, st, fixes, outs, eps, st2)
    for r in runs[1:]:
        assert r[0].tobytes() == fixes.tobytes() and r[1].tobytes() == outs.tobytes() and r[3].tobytes() == st2.tobytes()
        assert all(a.tobytes() == b.tobytes() for a, b in zip(r[2], eps))
    assert len(fixes) >= 13
    if n <= 3:
        assert (fixes["status"] == gps.FIX_FEW).all() and np.isnan(fixes["pdop"]).all()
        x = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
        assert (np.linalg.norm(np.diff(x, axis=0), axis=1) > 0).all()
    if n == 32:
        assert (fixes["mask"] >> 31 & 1).any()
    # the shape the K = 16 run had (launch puts channel c on CTA c mod K): this documents it, the byte equality above
    # with the K = 1 run that went through check_model is what covers it
    per_cta = np.bincount(np.arange(n) % min(n, 16))
    print("n %d: %d fixes, nused %d..%d, channels per CTA at K = 16: %s" % (
        n, len(fixes), fixes["nused"].min(), fixes["nused"].max(), sorted(set(per_cta.tolist()))))


def noise16(nsamples):
    return np.random.default_rng(5).integers(-32768, 32768, 2 * nsamples, dtype=np.int64).astype(np.int16)


@pytest.mark.parametrize("edge", ["periods1", "periods100", "no_process_noise"])
def test_config_edges(ctx, sky12, edge):
    """1 s of sky12 (int8) and 0.25 s of full-scale int16 noise under N = 1 (no prompt pairs: dot = cross = 0, so f_m
    comes from w alone), N = 100 and all three process-noise densities 0 (Q = 0). At N = 100 one more call ends by
    max_updates = 3 on a buffer that holds 9, with its epoch buffer at the least the call accepts,
    (max_updates + 1) N = 400: it writes 300 epochs per channel and stops at the third update."""
    g, ch, iq, prns, chans = sky12
    cfg = dict(periods1=gps.vtrack_config(periods=1), periods100=gps.vtrack_config(periods=100),
               no_process_noise=gps.vtrack_config(accel_psd=0.0, bias_psd=0.0, drift_psd=0.0))[edge]
    N = int(cfg["periods"])
    st = seeded(ctx, chans, cfg, state0(prns, cfg))
    for src, ss in ((iq[:2 * 3000000], gps.SC08), (noise16(750000), gps.SC16)):
        fixes, outs, eps, st2 = run_checked(ctx, chans, cfg, st, src, ss)
        assert len(fixes) >= 2
        assert all(e.size == len(fixes) * N + int(k) for e, k in zip(eps, st2["ch"]["k"][:len(prns)]))
        if N == 1:
            assert (outs["dot"] == 0).all() and (outs["cross"] == 0).all()
        if edge == "no_process_noise":
            assert float(cfg["accel_psd"]) == float(cfg["bias_psd"]) == float(cfg["drift_psd"]) == 0.0
        print(edge, ss, "%d fixes, %d used records" % (len(fixes), int(outs["used"].sum())))
    if N == 100:
        src = iq[:2 * 3000000]
        fixes, outs, eps, st2 = run_checked(ctx, chans, cfg, st, src, max_updates=3)
        assert len(fixes) == 3 and all(e.size == 300 for e in eps) and (st2["ch"]["k"] == 0).all()


def test_q_min_at_equality(ctx, sky12):
    """The q of update 0 comes from the seed's commands alone. q_min = a channel's q uses it and the next double does
    not (and the first fix differs); q_min = the 4th-largest q gives an OK fix of 4 channels with a finite PDOP, the
    next double a FEW fix of 3 with a NaN PDOP and the rms of 3."""
    g, ch, iq, prns, chans = sky12
    src = iq[:2 * 300000]
    cfg0 = gps.vtrack_config()
    st = seeded(ctx, chans, cfg0, state0(prns, cfg0))
    q = ctx.vtrack(chans, cfg0, st, 1, iq=src)[1][0]["q"]
    assert np.unique(q).size == q.size and (q > 1.0).all()
    c = int(np.argmin(q))
    first = {}
    for qm, used in ((q[c], 1), (np.nextafter(q[c], np.inf), 0)):
        cfg = gps.vtrack_config(q_min=qm)
        fixes, outs, _, _ = run_checked(ctx, chans, cfg, st, src)
        assert int(outs[0][c]["used"]) == used and int(outs[0]["used"].sum()) == q.size - 1 + used
        first[used] = fixes[0]
    assert first[0].tobytes() != first[1].tobytes()
    q4 = np.sort(q)[::-1][3]
    for qm, nused in ((q4, 4), (np.nextafter(q4, np.inf), 3)):
        cfg = gps.vtrack_config(q_min=qm)
        fixes, outs, _, _ = run_checked(ctx, chans, cfg, st, src)
        f = fixes[0]
        assert int(f["nused"]) == nused and np.isfinite(f["rms"])
        if nused == 4:
            assert int(f["status"]) == gps.FIX_OK and np.isfinite(f["pdop"])
        else:
            assert int(f["status"]) == gps.FIX_FEW and np.isnan(f["pdop"])
        print("q_min %r: fix 0 with %d channels, status %d, pdop %r, rms %.3f m" % (
            qm, nused, int(f["status"]), float(f["pdop"]), float(f["rms"])))


@pytest.mark.parametrize("kind,N", [("speed", 20), ("jump", 1), ("jump", 20)])
def test_command_clamps_and_wraps_open_loop(ctx, sky12, kind, N, monkeypatch):
    """0.5 s of zeros from test_vtrack_edges' open-loop seeds, started by the kernel: the kernel's commands reach the
    clamps (w = +-W_CLAMP, u = CODE_STEP_MIN and MAX), the model's wraps run, the clamped commands equal the model's."""
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config(periods=N)
    st = open_loop_seed(kind, prns, chans, cfg, kernel_first(ctx, chans, cfg))
    zeros = np.zeros(2 * 1500000, np.int8)
    fixes, outs, eps, st2 = ctx.vtrack(chans, cfg, st, most_updates(zeros, cfg), iq=zeros, want_epochs=True)
    assert (outs["used"] == 0).all() and (fixes["nused"] == 0).all()
    errs = command_record(monkeypatch)
    trace = []
    _, mo, _, _ = V.run(zeros, 1, 0, st, chans, cfg, len(fixes), replay=outs, trace=trace)
    e = open_loop_edges(outs, errs, raw_code_residuals(st, chans, cfg, outs, eps, trace))
    print(kind, N, e)
    if kind == "speed":
        assert e["w_plus"] and e["w_minus"] and e["err_wrap"]
    else:
        assert e["u_min"] and e["u_max"] and e["err_wrap"] and e["r_wrap"]
    for f, edges in (("carr_step", (W_CLAMP, -W_CLAMP)), ("code_step", (T.CODE_STEP_MIN, T.CODE_STEP_MAX))):
        at = np.isin(mo[f], edges) | np.isin(outs[f], edges)
        assert np.array_equal(mo[f][at], outs[f][at]), f
    assert (outs["code_step"] >= T.CODE_STEP_MIN).all() and (outs["code_step"] <= T.CODE_STEP_MAX).all()
    assert (np.abs(outs["carr_step"]) <= W_CLAMP).all()
    monkeypatch.undo()
    check_model(zeros, 1, chans, cfg, st, fixes, outs, eps, st2)


@pytest.mark.parametrize("target", WRAP_TARGETS)
def test_first_period_at_the_code_wrap(ctx, sky12, target):
    """test_vtrack_edges' seeds with channel 0 at llround(phi 2^32) mod M = target: the kernel's one-sample call starts
    channel 0 as the model's first (at s0 with phase 0 for target 0, at s0 + 1 for M - 1); then 0.2 s."""
    g, ch, iq, prns, chans = sky12
    cfg = gps.vtrack_config()
    st, s0, _, _ = wrap_seed(prns, chans, V.config(), target)
    ks = seeded(ctx, chans, cfg, st)
    ms = np.array([st], V.STATE_DTYPE)[0]
    V.first(ms, [c["eph"] for c in chans], int(cfg["periods"]))
    a, b = ks["ch"][0], ms["ch"][0]
    for f in ("sample", "code_phase", "code_step", "carr_step"):
        assert int(a["nco"][f]) == int(b["nco"][f]), (f, a["nco"][f], b["nco"][f])
    assert int(a["start"]) == int(b["start"])
    if target == 0:
        assert int(a["nco"]["sample"]) == s0 and int(a["nco"]["code_phase"]) == 0
    if target == V.M - 1:
        assert int(a["nco"]["sample"]) == s0 + 1
    print("target %d: first period at s0 + %d, code phase %d" % (target, int(a["nco"]["sample"]) - s0,
                                                                 int(a["nco"]["code_phase"])))
    run_checked(ctx, chans, cfg, ks, iq[:2 * (s0 + 600000)])


@pytest.mark.parametrize("rotate", [False, True])
def test_full_scale_sums_at_100_periods(ctx, sky12, rotate):
    """One channel, open loop (q_min 1e300), 1.01 s at N = 100 of int8 corners on its NCO trajectory: E, L, P, S, dot
    and cross equal the model's Python-integer sums near their bounds, S the direct sum, and the same stream as int16
    (16 v, and saturated to +-32767 / -32768) gives the same records byte for byte."""
    g, ch, iq, prns, chans = sky12
    cfg = full_scale_config()
    st = seeded(ctx, chans[:1], cfg, state0(prns[:1], cfg))
    n = 3030000
    src, _ = full_scale_plant(st, chans[:1], cfg, n, rotate)
    ref = run_checked(ctx, chans[:1], cfg, st, src)
    fixes, outs, eps, _ = ref
    assert len(fixes) == 10 and (outs["used"] == 0).all()
    check_full_scale(outs, rotate)
    assert np.array_equal(outs["s"][:, 0], interval_power(src, outs, eps))
    v = src.astype(np.int16)
    for s16 in (16 * v, np.where(v == 127, 32767, np.where(v == -128, -32768, 16 * v)).astype(np.int16)):
        got = ctx.vtrack(chans[:1], cfg, st, most_updates(s16, cfg), iq=s16, sample_size=gps.SC16, want_epochs=True)
        for a, b in zip(got[:2] + got[3:], ref[:2] + ref[3:]):
            assert a.tobytes() == b.tobytes()
        assert got[2][0].tobytes() == eps[0].tobytes()


def test_across_the_week_roll(ctx, tmp_path):
    """6 s of the `-s now` week-roll stream (re-synthesised from the scenario rows), seeded 3 s before 604 800 s, in
    three calls: to 2.5 s, the second spanning the roll (through check_model), the rest. t_rx runs on past 604 800 s
    without a fold and within 1 us of the truth; every channel within CERR_MAX and every fix within 30 m after
    SETTLE."""
    ch, nav, prns, chans, b0, t_rx0, x0 = weekroll_case(tmp_path)
    s0, n = b0 * BLOCK, WEEKROLL_BLOCKS * BLOCK
    iq, _ = scenario.oracle_run(ch[b0:b0 + WEEKROLL_BLOCKS], nav, 1)
    cfg = gps.vtrack_config()
    st = gps.vtrack_seed(cfg, seed_x(x0), t_rx0, s0, prns)
    roll = s0 + int(WEEKROLL_LEAD * V.FS)
    fixes, eps, base = [], [[] for _ in prns], s0
    for k, hi in enumerate((roll - 1500000, roll + 1500000, s0 + n)):
        buf = iq[2 * (base - s0):2 * (hi - s0)]
        if k == 1:
            f, _, e, st = run_checked(ctx, chans, cfg, st, buf, base=base)
            assert f["t_rx"].min() < WEEK_S < f["t_rx"].max()
        else:
            f, _, e, st = ctx.vtrack(chans, cfg, st, most_updates(buf, cfg), iq=buf, base=base, want_epochs=True)
        fixes.append(f)
        for c in range(len(prns)):
            eps[c].append(e[c])
        base = int(st["ch"]["nco"]["sample"][:len(prns)].min())
    fixes = np.concatenate(fixes)
    eps = [np.concatenate(e) for e in eps]
    assert len(fixes) >= 290 and (np.diff(fixes["sample"]) > 0).all()
    t = fixes["t_rx"]
    assert (np.diff(t) > 0).all() and t.max() > WEEK_S + 2.5
    late = fixes["sample"] >= s0 + SETTLE * V.FS
    terr = np.abs(t - (t_rx0 + (fixes["sample"] - s0) / V.FS))[late]
    assert (fixes["status"][late] == gps.FIX_OK).all() and terr.max() <= 1e-6, terr.max()
    xyz = np.stack([fixes["x"], fixes["y"], fixes["z"]], 1)
    err = check_truth(ch, prns, eps, xyz, fixes["sample"] - s0, lambda s: np.broadcast_to(x0, (s.size, 3)),
                      skip_samples=lambda s: s < s0 + SETTLE * V.FS)
    print("week roll: %d fixes, t_rx %.3f..%.3f s, worst time error %.2e s, worst fix error %.2f m" % (
        len(fixes), t.min(), t.max(), terr.max(), err.max()))


# ---- memcheck -------------------------------------------------------------------------------------------------------
def sanitizer_run():
    """One channel at K = 1 and 17 channels at K = 16, N = 1, 50 ms of zeros each -> a digest."""
    import hashlib
    import pathlib
    import tempfile
    chans = chans_of(pathlib.Path(tempfile.mkdtemp()), 32, list(range(1, 18)))
    cfg = gps.vtrack_config(periods=1)
    h = hashlib.sha256()
    with gps.Context(32, 1) as c:
        for n, K in ((1, 1), (17, 16)):
            c.debug_vtrack_cluster(K)
            st = gps.vtrack_seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, 0, list(range(1, n + 1)))
            for a in c.vtrack(chans[:n], cfg, st, 100, iq=np.zeros(2 * 150000, np.int8), want_epochs=True):
                h.update(b"".join(np.asarray(x).tobytes() for x in a) if isinstance(a, list) else np.asarray(a).tobytes())
    return h.hexdigest()


def test_small_calls_clean_under_compute_sanitizer():
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_vtrack_edges_gpu as T; "
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
