"""The receiver kernels at the edges of their contracts, against the numpy models: the acquisition grid and pick
(k_acq_grid / k_acq_pick) bit for bit at 32 PRNs, 70 and 1024 bins, real ties and full-scale coherent input at K = 100;
the tracking loop (k_track) bit for bit from states at the contract's limits, one period per call, in odd cuts and
uncut, at 1, 7 and 32 channels; the fixes and RAIM (k_pvt) across the week roll, while satellites rise and set, on a
channel whose epochs resume after a gap, and with every stream sample shifted past 2^32. Each test asserts that its
run reached the edge it is about."""
import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import pvt_truth as PT
import raim_model as RM
import scenario
import test_time_overwrite as TO
import track_model as T
from scenario import gps
from test_pvt import IDEAL, check_truth, ideal_inputs, rinex
from test_pvt_gpu import assert_kernel_equals_model as assert_pvt_equals_model
from test_raim_gpu import assert_kernel_equals_model as assert_raim_equals_model
from test_receiver_edges import (GAP_AT, GAP_CHAN, WEEK_S, bracket_misses, full_scale, gapped_case, limit_states,
                                 period_lengths, planted, sign_changes)
from test_scenario import LOC, LOC60, START
from test_track import START_SOW
from test_track_gpu import acquire_and_start, signal

pytestmark = pytest.mark.gpu

SHIFT = 1 << 33                   # stream samples past 2^32
ALL = list(range(1, 33))


# ---- acquisition -----------------------------------------------------------------------------------------------------
def acq_equals_model(ctx, iq, ss, K, prns, f_lo, step, nbins, s0=0):
    res, grid = ctx.acquire(iq, ss, prns, ms=K, s0=s0, f_lo=f_lo, step=step, nbins=nbins, want_grid=True)
    want = A.grid(iq, ss, s0, K, prns, f_lo, step, nbins)
    assert np.array_equal(grid, want)
    assert np.array_equal(res, A.reduce(want, prns, f_lo, step))
    return res, grid


@pytest.mark.parametrize("ss", [gps.SC08, gps.SC16])
def test_acq_all_prns_70_bins(ss):
    """All 32 PRNs in one call over 70 bins, noise plus three planted signals: PRN 3 (511 sign changes) peaks in bin 40,
    PRN 6 (512) in bin 66 and PRN 22 (543) in bin 5, so the pick's lanes see peaks at j >= 32 and j >= 64."""
    f_lo, step, nbins = -8625.0, 250.0, 70
    sigs = [(3, f_lo + 40 * step, 1700, 24), (6, f_lo + 66 * step, 11, 24), (22, f_lo + 5 * step, 2999, 24)]
    iq = planted(A.CODE * 2 + A.CODE - 1, sigs, ss, noise=20, seed=ss)
    with gps.Context(1, 1) as ctx:
        res, _ = acq_equals_model(ctx, iq, ss, 2, ALL, f_lo, step, nbins)
    got = {int(r["prn"]): (int(r["bin"]), int(r["delay"])) for r in res}
    assert got[3] == (40, 1700) and got[6] == (66, 11) and got[22] == (5, 2999)
    assert {sign_changes(p) % 2 for p in ALL} == {0, 1}
    assert (res["bin"] >= 32).sum() > 2 and (res["bin"] >= 64).sum() > 1


def test_acq_1024_bins_peak_in_the_last_bin():
    """The largest grid: 1024 bins over the whole +-1.5 MHz range, two PRNs planted in bin 1023."""
    f_lo, step, nbins = -1.5e6, 2932.0, 1024
    f_hi = f_lo + 1023 * step
    iq = planted(A.CODE * 2 + A.CODE - 1, [(6, f_hi, 777, 30), (7, f_hi, 2222, 30)], gps.SC08, noise=20, seed=3)
    with gps.Context(1, 1) as ctx:
        res, _ = acq_equals_model(ctx, iq, gps.SC08, 2, [6, 7], f_lo, step, nbins)
    assert list(res["bin"]) == [1023, 1023] and list(res["delay"]) == [777, 2222]


def test_acq_zero_input_ties_everywhere():
    """Every row and delay has power 0: bin 0, delay 0, P2 0 and an infinite ratio for every PRN."""
    iq = np.zeros(2 * (A.CODE * 3 + A.CODE - 1), np.int8)
    with gps.Context(1, 1) as ctx:
        res, _ = acq_equals_model(ctx, iq, gps.SC08, 3, ALL, -8625.0, 250.0, 70)
    assert (res["bin"] == 0).all() and (res["delay"] == 0).all() and (res["p1"] == 0).all() and (res["p2"] == 0).all()
    assert np.isinf(res["ratio"]).all()


def tied_bins(prn, iq, ss, f0, first=40):
    """f_lo of a 64-bin search at step 1e-6 Hz whose bins round to one phase step u below `first` and to u + 1 from
    `first` on, with the u + 1 row the stronger one (u is chosen near phase_step(f0) so that it is)."""
    u0 = A.phase_step(f0)
    for u in range(u0 - 8, u0 + 8):
        rows = A.grid(iq, ss, 0, 1, [prn], u * 3e6 / 2 ** 32, 3e6 / 2 ** 32, 2)
        if rows[0, 1].max() > rows[0, 0].max():
            return (u + 0.5) * 3e6 / 2 ** 32 - (first - 0.5) * 1e-6, u
    raise AssertionError("no step pair with a stronger upper row")


@pytest.mark.parametrize("ss", [gps.SC08, gps.SC16])
def test_acq_tied_rows_pick_the_lowest_bin(ss):
    """Bins 1e-6 Hz apart: bins 0-39 share one phase step and 40-63 the next, whose rows are identical and the
    strongest, so the largest P1 is first reached at j = 40, in lane 8's second bin; the pick takes j = 40."""
    iq = planted(A.CODE * 2 - 1, [(9, 1234.0, 321, 20)], ss, noise=12, seed=9)
    f_lo, u = tied_bins(9, iq, ss, 1234.0)
    assert [A.phase_step(f_lo + j * 1e-6) for j in range(64)] == [u] * 40 + [u + 1] * 24
    with gps.Context(1, 1) as ctx:
        res, grid = acq_equals_model(ctx, iq, ss, 1, [9, 16], f_lo, 1e-6, 64)
    g = grid[0]
    assert (g[40:] == g[40]).all() and (g[:40] == g[0]).all() and g[40].max() > g[39].max()
    assert res[0]["bin"] == 40 and res[0]["delay"] == 321


def test_acq_aliased_end_bins_pick_bin_0():
    """f_lo = -1.5 MHz, step 1.5 MHz: both end bins have phase step 2^31, so their rows are identical; a signal on that
    carrier makes them the strongest, and the pick takes j = 0."""
    assert A.phase_step(-1.5e6) == A.phase_step(1.5e6) == 1 << 31
    iq = planted(A.CODE * 4 + A.CODE - 1, [(11, 1.5e6, 100, 40)], gps.SC08, noise=10, seed=11)
    with gps.Context(1, 1) as ctx:
        res, grid = acq_equals_model(ctx, iq, gps.SC08, 4, [11, 28], -1.5e6, 1.5e6, 3)
    assert np.array_equal(grid[:, 0], grid[:, 2]) and grid[0, 0].max() > grid[0, 1].max()
    assert res[0]["bin"] == 0 and res[0]["delay"] == 100


@pytest.mark.parametrize("ss", [gps.SC08, gps.SC16])
def test_acq_full_scale_coherent_k100(ss):
    """A full-scale replica of PRN 13 on bin 1's exact carrier for K = 100: P1 passes 2^53 (|C| near 9.6e7 per period)."""
    f_lo, step = 1500.0, 250.0
    iq = full_scale(A.CODE * 100 + A.CODE - 1, 13, f_lo + step, ss, delay=2468)
    with gps.Context(1, 1) as ctx:
        res, _ = acq_equals_model(ctx, iq, ss, 100, [13, 6], f_lo, step, 3)
    assert res[0]["bin"] == 1 and res[0]["delay"] == 2468 and int(res[0]["p1"]) > 2 ** 53


# ---- tracking --------------------------------------------------------------------------------------------------------
PERIODS = 300
NTRK = PERIODS * 3001 + 8000        # every channel gets at least 300 periods
COHERENT_AT = 1000                  # stream sample where the full-scale input's first code period starts


def track_input(kind):
    """(interleaved I,Q of NTRK samples, sample size, PRNs to cycle over)."""
    rng = np.random.default_rng(len(kind))
    if kind == "int8":
        return rng.integers(-128, 128, 2 * NTRK).astype(np.int8), gps.SC08, ALL
    if kind == "int16":
        vals = np.array([-32768, -32767, -2049, -2048, -17, 0, 15, 2047, 2048, 32767], np.int16)
        return rng.choice(vals, 2 * NTRK), gps.SC16, ALL
    if kind == "full":   # PRN 7 at full scale, 1 kHz, chip 0 at sample COHERENT_AT (coherent_state tracks it)
        return full_scale(NTRK, 7, 1000.0, gps.SC08, delay=COHERENT_AT), gps.SC08, ALL
    g, ch, out, ss = signal(4)
    assert out.size >= 2 * NTRK
    return out[:2 * NTRK], ss, [int(p) for p in ch[0]["prn"] if p > 0]


def assert_track_equal(got, want):
    (ge, gs), (we, ws) = got, want
    assert len(ge) == len(we)
    for a, b in zip(ge, we):
        assert np.array_equal(a, b)
    assert np.array_equal(gs, ws.astype(gps.TRACK_STATE_DTYPE))


def coherent_state(base):
    """A channel on the full-scale input's signal: PRN 7 at its 1 kHz carrier, the code aligned with the signal's, and
    the code step at its lower clamp with phase 0 (a first period of 3001 samples)."""
    st = T.start(7, 1000.0, base + COHERENT_AT)
    st["code_step"], st["code_phase"] = T.CODE_STEP_MIN, 0
    return st


def coherent_reach(eps):
    """(largest bitlen(E + L), largest |P_I|) over a channel's epochs, exactly."""
    E = eps["e_i"].astype(object) ** 2 + eps["e_q"].astype(object) ** 2
    L = eps["l_i"].astype(object) ** 2 + eps["l_q"].astype(object) ** 2
    return max(int(v).bit_length() for v in E + L), int(np.abs(eps["p_i"].astype(np.int64)).max())


def period_len(st):
    return (T.M - st["code_phase"].astype(object) + st["code_step"].astype(object) - 1) // st["code_step"].astype(object)


@pytest.mark.parametrize("nch", [1, 4, 7, 12, 20, 32])
@pytest.mark.parametrize("kind", ["int8", "int16", "full", "signal"])
def test_track_limit_states(kind, nch):
    """States at the limits (tests/test_receiver_edges.py: limit_states) stepped through 300 periods: one uncut call,
    300 calls of max_epochs = 1, and calls of odd max_epochs at odd buffer cuts; every call's epochs and states equal the
    model's, and the cut runs add up to the uncut one. Reached: periods of 2999 and 3001 samples, carr_freq at +-2^34,
    the FLL switching off inside a call, a call ended by max_epochs before the buffer, a period ending exactly on the
    buffer's last sample (and not tracked one sample short), channels past the end with 0 epochs and their state kept.
    On the full-scale input the last channel tracks the signal coherently (coherent_state), which drives bitlen(E + L)
    past 52 and |P_I| past 2^26, towards the int32 bound of the sums; with one channel that is the only channel, and it
    stays near its 1 kHz carrier, so carr_freq reaches its clamp in the other runs only. Channel 3 (kind 3: 199 epochs,
    no previous prompt) runs its last FLL update on cross = dot = 0, whose angle is 0: its first carrier step is the
    PLL's alone (with four channels on the full-scale input that channel is the coherent one instead)."""
    iq, ss, prns = track_input(kind)
    base = 17
    st0 = limit_states([prns[c % len(prns)] for c in range(nch)], base, nch)
    if kind == "full":
        st0[-1] = coherent_state(base)
    n = iq.size // 2
    with gps.Context(1, 1) as ctx:
        one = ctx.track(st0, iq, ss, base=base)
        assert_track_equal(one, T.track(iq, ss, base, st0))
        eps1, st1 = one
        assert min(e.size for e in eps1) >= PERIODS
        if kind == "full":
            bits, p_i = coherent_reach(eps1[-1])
            assert bits >= 52 and p_i > 2 ** 26, (bits, p_i)
        if nch > 4 or (nch == 4 and kind != "full"):
            z, ep = st0[3], eps1[3][0]
            assert z["epochs"] == T.FLL_EPOCHS - 1 and z["prev_i"] == 0 and z["prev_q"] == 0
            pi, pq = int(ep["p_i"]), int(ep["p_q"])
            e = int(T.angle(np.int64(abs(pi)), np.int64(-pq if pi < 0 else pq)))
            F = min(max(int(z["carr_freq"]) + (e >> 12), -T.FREQ_CLAMP), T.FREQ_CLAMP)
            assert int(ep["carr_step"]) == (F >> 10) + (e >> 16)

        def call(s, lo, hi, me):
            buf = iq[2 * (lo - base):2 * (hi - base)]
            got = ctx.track(s, buf, ss, base=lo, max_epochs=me)
            assert_track_equal(got, T.track(buf, ss, lo, s, max_epochs=me))
            return got

        # one period per call
        s, freq_clamped, steps = st0.copy(), False, []
        for i in range(PERIODS):
            lo = int(s["sample"].min())
            eps, s = call(s, lo, int(s["sample"].max()) + 3001, 1)
            assert all(e.size == 1 for e in eps)
            steps.append(eps)
            freq_clamped |= bool((np.abs(s["carr_freq"]) == T.FREQ_CLAMP).any())
            if i == PERIODS // 2:
                # the buffer ends exactly where the earliest-ending period ends: that period is tracked, the channels
                # whose period ends later get 0 epochs and keep their state; one sample short, nobody is tracked
                L = np.array(period_len(s), np.int64)
                end = int((s["sample"] + L).min())
                first = int(np.argmin(s["sample"] + L))
                e_end, s_end = call(s, lo, end, 5)
                assert e_end[first].size == 1 and e_end[first]["sample"][0] + L[first] == end
                late = s["sample"] + L > end
                assert late.any() or nch == 1         # one channel: the call one sample short below covers it
                for c in np.nonzero(late)[0]:
                    assert e_end[c].size == 0 and s_end[c].tobytes() == s[c].tobytes()
                e_short, s_short = call(s, lo, end - 1, 5)
                assert all(e.size == 0 for e in e_short) and s_short.tobytes() == s.tobytes()
        for c in range(nch):
            assert np.array_equal(np.concatenate([st[c] for st in steps]), eps1[c][:PERIODS])
        assert freq_clamped or (kind == "full" and nch == 1)

        # odd max_epochs at odd buffer cuts
        s, parts, fll_off_inside, ended_by_max = st0.copy(), [[] for _ in range(nch)], False, False
        for cut, me in ((123457, 37), (400001, 101), (400001, 7), (650003, 73), (n + base, 89), (n + base, n)):
            lo = int(s["sample"].min())
            eps, s2 = call(s, lo, cut, me)
            L = np.array(period_len(s2), np.int64)
            for c in range(nch):
                parts[c].append(eps[c])
                fll_off_inside |= s[c]["epochs"] <= T.FLL_EPOCHS - 2 and s2[c]["epochs"] >= T.FLL_EPOCHS + 1
                ended_by_max |= eps[c].size == me and s2[c]["sample"] + L[c] <= cut
            s = s2
        for c in range(nch):
            assert np.array_equal(np.concatenate(parts[c]), eps1[c])
        assert s.tobytes() == st1.tobytes()
        assert fll_off_inside and ended_by_max
    lens = set()
    for c in range(nch):
        lens |= set(int(x) for x in period_lengths(eps1[c], st1[c]))
    assert ({2999, 3001} if nch > 1 else {3001}) <= lens <= {2999, 3000, 3001}   # one channel: kind 0 only


def test_track_sky32_one_second_and_shifted_past_2_32():
    """32 channels of sky32_static from their acquisition for 1 s against the model; the same run with `base` and every
    `sample` shifted by 2^33 gives the same epochs and states with only `sample` shifted."""
    g, ch, out, ss = signal(10, "sky32_static_10s_i8")
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    assert len(prns) == 32
    with gps.Context(32, 1) as ctx:
        st = acquire_and_start(ctx, out, ss, prns)
        got = ctx.track(st, out, ss)
        st2 = st.copy()
        st2["sample"] += SHIFT
        eps2, s2 = ctx.track(st2, out, ss, base=SHIFT)
    assert_track_equal(got, T.track(out, ss, 0, st))
    eps, s = got
    assert min(e.size for e in eps) >= 990
    for a, b in zip(eps, eps2):
        assert np.array_equal(b["sample"], a["sample"] + SHIFT)
        b["sample"] -= SHIFT
        assert a.tobytes() == b.tobytes()
    assert np.array_equal(s2["sample"], s["sample"] + SHIFT)
    s2["sample"] -= SHIFT
    assert s.tobytes() == s2.tobytes()


# ---- fixes and RAIM --------------------------------------------------------------------------------------------------
def weekroll_case(tmp_path):
    """`-s now` at 23:58 on a Saturday, ideal epochs, fixes every 10 s: on both sides of 604 800 s. No instant lies
    within 1 ms of the fold, so t_rx is compared directly (a fix on the fold could wrap on one side only)."""
    g, kw = TO.now_case("sky12_now_weekroll_300s_i8", tmp_path)
    recs, alpha, beta = PT.read_rinex(kw["nav_file"])
    ch, nav = gps.scenario(**kw, time_overwrite=True)
    week, sow = TO.gps_time(kw["start"])
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    cfg = gps.pvt_config(30000, 29999993, 30, PT.klobuchar_broadcast(alpha, beta))
    s = int(cfg["s0"]) + np.arange(int(cfg["nfix"])) * int(cfg["step"])
    t = PT.truth_time(sow, s)
    assert t.min() < 100.0 and t.max() > WEEK_S - 100.0             # both sides of the roll
    assert np.minimum(t, WEEK_S - t).min() > 1e-3
    # the channels' transmit times wrap too: some anchor before the roll, measured after it
    assert (chans["anchor_ms"] > PT.WEEK_MS - 300000).any()
    xyz = np.repeat(PM.llh_ecef(kw["lat"], kw["lon"], kw["height"])[None], ch.shape[0] + 1, 0)
    return chans, eps, cfg, (xyz, sow)


def lat60_case(tmp_path):
    """310 s at 60 deg N, 32 channels, satellites rising and setting; the reference channel's anchor moved to the
    middle of its epochs, so that some fixes lie before it and some after."""
    loc = LOC60
    nav_file, _, iono = rinex(tmp_path, 32)
    ch, nav = gps.scenario(nav_file, *loc, seconds=310, max_chan=32, start=START)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    ref = next(c for c in range(len(chans)) if chans[c]["eph"]["valid"] and chans[c]["eph"]["health"] == 0)
    mid = len(eps[ref]) // 2
    chans[ref]["anchor_ms"] = (int(chans[ref]["anchor_ms"]) + mid - int(chans[ref]["anchor_epoch"])) % PT.WEEK_MS
    chans[ref]["anchor_epoch"] = mid
    cfg = gps.pvt_config(30000, 14999993, 61, iono)
    s = int(cfg["s0"]) + np.arange(int(cfg["nfix"])) * int(cfg["step"])
    a = int(eps[ref]["sample"][mid])
    assert (s < a).any() and (s > a).any()
    xyz = np.repeat(PM.llh_ecef(*loc)[None], ch.shape[0] + 1, 0)
    return chans, eps, cfg, (xyz, START_SOW)


def gap_case(tmp_path):
    chans, eps, cfg, resume = gapped_case(tmp_path)
    s = int(cfg["s0"]) + np.arange(int(cfg["nfix"])) * int(cfg["step"])
    miss, _ = bracket_misses(eps[GAP_CHAN], s)
    assert miss[s >= eps[GAP_CHAN]["sample"][GAP_AT + 1]].all() and miss.sum() > 30
    g = scenario.load_golden("sky12_static_35s_i8")
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], g["chans"].shape[0] + 1, 0)
    return chans, eps, cfg, (xyz, START_SOW)


CASES = {"weekroll": weekroll_case, "lat60": lat60_case, "gap": gap_case}


def model_margins(chans, eps, cfg):
    """Run the model with its decisions traced, and assert that none sits within 1e-9 relative of its threshold: the
    convergence step (1e-4 m), the Klobuchar radius (6e6 m), the runaway radius (1e8 m), the Klobuchar |X| < 1.57 branch
    and the 7200 s toe window."""
    trace = {k: [] for k in ("radius", "runaway", "step", "klobuchar_x")}
    fix, _, ms = PM.pvt(chans, eps, cfg, trace=trace)
    for k, thr in (("step", PM.CONVERGED), ("radius", PM.IONO_MIN_RADIUS), ("runaway", PM.RUNAWAY),
                   ("klobuchar_x", 1.57)):
        v = np.abs(np.concatenate(trace[k]))
        assert v.size and np.abs(v / thr - 1.0).min() > 1e-9, k
    toe = np.stack([chans[c]["eph"]["toe"] for c in range(len(chans))])[None, :]
    dt = np.abs(PM.wrap_half_week(ms["tsv"] - toe))[ms["tsv"] != 0]
    assert np.abs(dt / 7200.0 - 1.0).min() > 1e-9
    return fix


def shifted(eps, cfg):
    e2 = []
    for e in eps:
        e = e.copy()
        e["sample"] += SHIFT
        e2.append(e)
    c2 = cfg.copy()
    c2["s0"] += SHIFT
    return e2, c2


@pytest.mark.parametrize("case", list(CASES))
def test_fixes_and_raim_on_the_model_only_paths(case, tmp_path):
    """Context.pvt and Context.pvt_raim against the models, Klobuchar on: across the week roll, with satellites rising
    and setting at 60 deg N, and on a channel whose epochs resume after a 2.2 s gap (the period bracket misses, so
    find_period's full search runs). The fixes are within the ideal-epoch truth bounds. With every epoch sample and s0
    shifted by 2^33 the fixes and RAIM records are byte-equal except `sample`."""
    chans, eps, cfg, (xyz, sow) = CASES[case](tmp_path)
    model_margins(chans, eps, cfg)
    rcfg = gps.raim_config(1.0)
    with gps.Context(1, 1) as ctx:
        fix = assert_pvt_equals_model(ctx, chans, eps, cfg)
        rfix, rec, _ = assert_raim_equals_model(ctx, chans, eps, cfg, rcfg)
        e2, c2 = shifted(eps, cfg)
        fix2, res2 = ctx.pvt(chans, e2, c2, want_residuals=True)
        rfix2, rec2 = ctx.pvt_raim(chans, e2, c2, rcfg)
        _, res = ctx.pvt(chans, eps, cfg, want_residuals=True)
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])
    assert (rec["verdict"] == RM.PASS).all() and fix.tobytes() == rfix.tobytes()
    for a, b in ((fix, fix2), (rfix, rfix2)):
        assert np.array_equal(b["sample"], a["sample"] + SHIFT)
        b["sample"] -= SHIFT
        assert a.tobytes() == b.tobytes()
    assert rec.tobytes() == rec2.tobytes() and res.tobytes() == res2.tobytes()
    if case == "lat60":
        assert len(set(int(m) for m in fix["mask"])) > 1 and len(set(int(n) for n in fix["nused"])) > 1
    if case == "gap":
        used = (fix["mask"].astype(np.int64) >> GAP_CHAN) & 1 == 1
        after = fix["sample"] >= eps[GAP_CHAN]["sample"][GAP_AT + 1]
        assert used[after].all() and not used[~after].any()
