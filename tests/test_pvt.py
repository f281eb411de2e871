"""Position fixes on the CPU: the ephemeris, Klobuchar terms and time anchor the decoder reads from the words, and the
numpy model of the fix (tests/pvt_model.py) on ideal and tracked epochs against the scenario's truth.

The bounds below were fixed from the model; they are shared with the GPU tests.
- Ideal epochs (a perfect loop, tests/pvt_truth.py) leave only the quantisation of the broadcast ephemeris, clock and
  Klobuchar terms (eph2sbf truncates, page 18 rounds) and the scenario's own range model (the satellite clock taken at the
  receive time, the position extrapolated linearly over the flight time, the range interpolated linearly over a block).
  Seen at most: 3D error 0.21 m (0.03-0.07 m with 32 channels), receive time 0.6 ns, velocity 7 mm/s, on the circle too.
- Tracked on the CPU (track_model on 12.1 s of sky12_static_35s, code errors up to 0.094 chips; a fix every 10 ms from
  0.5 s on): 3D error at most 20.2 m, mean 5.7 m, receive time 58 ns, velocity 1.13 m/s.
The limits leave a margin of about a third over those figures."""
import numpy as np
import pytest

import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_scenario import LOC, START, make_nav, motion_file
from test_time_overwrite import now_case
from test_track import START_SOW, model_run, synthetic_epochs

# ideal epochs: per-fix 3D error (m), receive-time error (s), velocity error (m/s), static / moving receiver
IDEAL = dict(pos=0.28, time=1e-9, vel=0.01)
# tracked epochs: per-fix and mean 3D error (m), receive-time error (s), velocity error (m/s)
TRACKED = dict(pos=27.0, pos_mean=7.6, time=7.7e-8, vel=1.5)


def rinex(tmp_path, nsat, sets=1):
    nav = make_nav(tmp_path, nsat, sets=sets)
    recs, alpha, beta = PT.read_rinex(nav)
    return nav, recs, PT.klobuchar_broadcast(alpha, beta)


# ---- decoding ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,nsat", [("sky12_static_35s_i8", 12), ("sky32_static_10s_i8", 32),
                                       ("sky12_circle_60s_i16", 12), ("sky12_alm_static_780s_i8", 12)])
def test_ephemeris_decode_every_slot(name, nsat, tmp_path):
    """Every active slot of every NAV frame: each field equals eph2sbf's integer times its scale, from the RINEX record
    of the slot's PRN; WN is the start week mod 1024; re-encoding the fields gives the frame's subframe 1-3 words."""
    g = scenario.load_golden(name)
    _, recs, _ = rinex(tmp_path, nsat)
    frames = g["nav_frames"]
    prn_of = g["prn_of_block"] if "prn_of_block" in g else g["chans"]["prn"]
    fob = g["nav_frame_of_block"]
    n = 0
    for f in range(len(frames)):
        b = int(np.nonzero(fob == f)[0][0])
        for c in range(frames.shape[1]):
            if not frames[f][c].any() or prn_of[min(b, len(prn_of) - 1)][c] <= 0:
                continue
            prn = int(prn_of[min(b, len(prn_of) - 1)][c])
            eph, _ = gps.nav_ephemeris(gps.nav_words_of_frame(frames[f][c]))
            assert eph["valid"] == 1 and eph["health"] == 0 and eph["ura"] == 0
            assert eph["week"] == 2296 % 1024
            assert eph["iodc"] == eph["iode"] == int(recs[prn]["iodc"])
            for fld in PT.EPH_FIELDS:
                assert eph[fld] == PT.eph2sbf_value(recs[prn], fld), (f, c, fld)
            words = frames[f][c][10:40] & 0x3FFFFFFF
            assert np.array_equal(encode_sf123(eph, words), words)
            n += 1
    assert n >= len(frames) * 12


def encode_sf123(eph, words):
    """Subframes 1-3 with the decoded fields re-encoded into the data bits eph2sbf fills (gps.c:706-740), the TLM, HOW,
    WN and the parity-solving bits of words 2 and 10 taken from `words`, parity recomputed."""
    def ints(f, scale, semi=False):
        return int(np.round(eph[f] / scale / (PM.PI if semi else 1.0)))
    data = [[0] * 10 for _ in range(3)]
    prev = 0
    for k in range(30):
        _, d = gps.nav_word_check(int(words[k]), prev)
        prev = int(words[k])
        data[k // 10][k % 10] = d
    m = lambda v, b: v & ((1 << b) - 1)
    iodc, iode = int(eph["iodc"]), int(eph["iode"])
    s1, s2, s3 = data
    s1[2] = (int(eph["week"]) << 14) | (int(eph["ura"]) << 8) | (int(eph["health"]) << 2) | (iodc >> 8)
    s1[6] = m(ints("tgd", 2.0 ** -31), 8)
    s1[7] = (m(iodc, 8) << 16) | m(ints("toc", 16.0), 16)
    s1[8] = (m(ints("af2", 2.0 ** -55), 8) << 16) | m(ints("af1", 2.0 ** -43), 16)
    s1[9] = (m(ints("af0", 2.0 ** -31), 22) << 2) | (s1[9] & 3)
    M0, E, SA = ints("m0", 2.0 ** -31, True), ints("ecc", 2.0 ** -33), ints("sqrta", 2.0 ** -19)
    s2[2] = (m(iode, 8) << 16) | m(ints("crs", 2.0 ** -5), 16)
    s2[3] = (m(ints("deltan", 2.0 ** -43, True), 16) << 8) | m(M0 >> 24, 8)
    s2[4] = m(M0, 24)
    s2[5] = (m(ints("cuc", 2.0 ** -29), 16) << 8) | m(E >> 24, 8)
    s2[6] = m(E, 24)
    s2[7] = (m(ints("cus", 2.0 ** -29), 16) << 8) | m(SA >> 24, 8)
    s2[8] = m(SA, 24)
    s2[9] = (m(ints("toe", 16.0), 16) << 8) | (s2[9] & 0xFF)
    O0, I0, W = ints("omg0", 2.0 ** -31, True), ints("inc0", 2.0 ** -31, True), ints("aop", 2.0 ** -31, True)
    s3[2] = (m(ints("cic", 2.0 ** -29), 16) << 8) | m(O0 >> 24, 8)
    s3[3] = m(O0, 24)
    s3[4] = (m(ints("cis", 2.0 ** -29), 16) << 8) | m(I0 >> 24, 8)
    s3[5] = m(I0, 24)
    s3[6] = (m(ints("crc", 2.0 ** -5), 16) << 8) | m(W >> 24, 8)
    s3[7] = m(W, 24)
    s3[8] = m(ints("omgdot", 2.0 ** -43, True), 24)
    s3[9] = (m(iode, 8) << 16) | (m(ints("idot", 2.0 ** -43, True), 14) << 2) | (s3[9] & 3)
    out, prev = [], 0
    for k in range(30):
        d = data[k // 10][k % 10]
        p = gps.nav_parity(d, (prev >> 1) & 1, prev & 1)
        w = (((d ^ (0xFFFFFF if prev & 1 else 0)) & 0xFFFFFF) << 6) | p
        out.append(w)
        prev = w
    return np.array(out, np.uint32)


def test_page18_klobuchar_from_the_780s_stream(tmp_path):
    """Subframe 4 page 18 is sent in frame 17 of sky12_alm_static_780s (the page counter starts at 0): its alpha / beta
    equal the RINEX header's, rounded as gps.c:686-693 rounds them; no earlier frame carries it."""
    g = scenario.load_golden("sky12_alm_static_780s_i8")
    _, _, (alpha, beta) = rinex(tmp_path, 12)
    frames = g["nav_frames"]
    seen = []
    for f in range(len(frames)):
        slot = next(s for s in frames[f] if s.any())
        _, iono = gps.nav_ephemeris(gps.nav_words_of_frame(slot))
        if iono["valid"]:
            seen.append(f)
            assert np.array_equal(iono["alpha"], alpha) and np.array_equal(iono["beta"], beta)
    assert seen == [17]


def test_time_anchor_on_synthetic_epochs():
    """The anchor of test_track's synthetic pattern: the first HOW with good parity, at epoch edge + 20 (frame_bit + 30),
    TOW from the frame's HOW."""
    g = scenario.load_golden("sky12_static_35s_i8")
    fr = g["nav_frames"][0]
    from test_track import frame_bits
    for invert, edge in ((False, 3), (True, 11)):
        bits = [0, 1, 1, 0, 1] + frame_bits(fr, 0)
        e = synthetic_epochs(bits, edge, invert=invert)
        _, words, sy = gps.nav_decode(e)
        ep, ms = gps.nav_time_anchor(words, sy)
        assert ep == edge + 20 * (7 + 30) == edge + 20 * (int(sy["frame_bit"]) + 30 * int(words[1]["index"]))
        tow = int(words[1]["tow"])
        assert ms == (6 * tow - 6) * 1000 + 600
        assert ms == PT.frame_ms0(g["nav_frames"], 0) + 11 * 600
    # no HOW with good parity: no anchor
    _, words, sy = gps.nav_decode(synthetic_epochs([0, 1] * 40, 0))
    assert gps.nav_time_anchor(words, sy)[0] == -1


# ---- fixes from ideal epochs -----------------------------------------------------------------------------------------
def ideal_inputs(ch, frames, fob, prns=None):
    """PVT channels and ideal epochs of every PRN of ch (one channel per PRN), ephemeris from the scenario's frames."""
    prns = sorted({int(p) for p in np.unique(ch["prn"]) if p > 0}) if prns is None else prns
    chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    eps = []
    for c, prn in enumerate(prns):
        e, ae, ams = PT.ideal_epochs(ch, prn, frames, fob)
        eps.append(e)
        b = int(np.nonzero((ch["prn"] == prn).any(1))[0][-1])
        slot = int(np.nonzero(ch[b]["prn"] == prn)[0][0])
        chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(frames[int(fob[b])][slot]))[0]
        chans[c]["prn"], chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = prn, ae, ams
    return chans, eps


def check_truth(fix, xyz_rows, start_sow, pos_max, time_max, vel_max, pos_mean_max=None):
    ok = fix["status"] == PM.FIX_OK
    assert ok.all(), np.unique(fix["status"], return_counts=True)
    tx, tv = PT.truth_xyz(xyz_rows, fix["sample"])
    got = np.stack([fix["x"], fix["y"], fix["z"]], 1)
    e3 = np.linalg.norm(got - tx, axis=1)
    et = np.abs((fix["t_rx"] - PT.truth_time(start_sow, fix["sample"]) + 302400.0) % 604800.0 - 302400.0)
    ev = np.linalg.norm(np.stack([fix["vx"], fix["vy"], fix["vz"]], 1) - tv, axis=1)
    fig = dict(pos=float(e3.max()), pos_mean=float(e3.mean()), time=float(et.max()), vel=float(ev.max()))
    assert fig["pos"] <= pos_max and fig["time"] <= time_max and fig["vel"] <= vel_max, fig
    if pos_mean_max is not None:
        assert fig["pos_mean"] <= pos_mean_max, fig
    return fig


def ideal_run(ch, nav, fob, xyz_rows, iono, start_sow, step, vel_max, s0=30000):
    chans, eps = ideal_inputs(ch, nav, fob)
    last = min(int(e["sample"][-2]) for e in eps if e.size > 2)
    cfg = gps.pvt_config(s0, step, (ch.shape[0] * PT.BLOCK - s0 - PT.BLOCK) // step, iono)
    fix, _, _ = PM.pvt(chans, eps, cfg)
    keep = fix["nused"] >= 4
    assert keep.all() or fix["sample"][~keep].min() > last - 2 * step
    return check_truth({k: v[keep] for k, v in fix.items()}, xyz_rows, start_sow, IDEAL["pos"], IDEAL["time"], vel_max)


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8"])
def test_ideal_fixes_on_the_fixtures(name, tmp_path):
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, int(g["max_chan"]))
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    ideal_run(ch, frames, g["nav_frame_of_block"], xyz, iono, START_SOW, 99991, IDEAL["vel"])


def test_ideal_fixes_on_the_circle(tmp_path):
    """60 s of the receiver on circle.csv (records from the scenario engine): along the whole circle."""
    g = scenario.load_golden("sky12_circle_60s_i16")
    nav_file, _, iono = rinex(tmp_path, 12)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
    ideal_run(ch, nav, ch["nav_frame"][:, 0], g["motion_rows"][:, 1:4], iono, START_SOW, 199999, IDEAL["vel"])


def test_ideal_fixes_while_satellites_rise_and_set(tmp_path):
    """310 s at 60 deg N with 32 channels: a satellite rises into a free slot at 240 s and another sets at 300 s; each
    PRN is a channel of its own, used while its epochs last."""
    from test_scenario import LOC60
    nav_file, _, iono = rinex(tmp_path, 32)
    ch, nav = gps.scenario(nav_file, *LOC60, seconds=310, max_chan=32, start=START)
    xyz = np.repeat(PM.llh_ecef(*LOC60)[None], ch.shape[0] + 1, 0)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    cfg = gps.pvt_config(30000, 14999993, 61, iono)
    fix, _, _ = PM.pvt(chans, eps, cfg)
    assert len(set(fix["nused"])) > 1                 # the set of channels in use changes along the run
    check_truth(fix, xyz, START_SOW, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])


def test_ideal_fixes_across_the_week_roll(tmp_path):
    """`-s now` at 23:58 on a Saturday: the transmit times and the receive time wrap at 604 800 s inside the run."""
    g, kw = now_case("sky12_now_weekroll_300s_i8", tmp_path)
    recs, alpha, beta = PT.read_rinex(kw["nav_file"])
    ch, nav = gps.scenario(**kw, time_overwrite=True)
    import test_time_overwrite as TO
    week, sow = TO.gps_time(kw["start"])
    xyz = np.repeat(PM.llh_ecef(kw["lat"], kw["lon"], kw["height"])[None], ch.shape[0] + 1, 0)
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    cfg = gps.pvt_config(30000, 29999993, 30, PT.klobuchar_broadcast(alpha, beta))
    fix, _, _ = PM.pvt(chans, eps, cfg)
    t = PT.truth_time(sow, fix["sample"])
    assert t.min() < 100.0 and t.max() > 604700.0     # both sides of the roll
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])


# ---- fixes from tracked epochs (the CPU tracking model) --------------------------------------------------------------
def tracked_inputs(eps, prns, frames, slot_of_prn):
    """PVT channels of tracked channels: ephemeris from the scenario's frame, anchor from the decoded words."""
    chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    for c, (prn, e) in enumerate(zip(prns, eps)):
        _, words, sy = gps.nav_decode(e)
        ep, ms = gps.nav_time_anchor(words, sy)
        assert ep >= 0, prn
        chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(frames[0][slot_of_prn[prn]]))[0]
        chans[c]["prn"], chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = prn, ep, ms
    return chans


def tracked_fixes(eps, prns, g, ch, iono, step=30000):
    slot_of_prn = {int(p): int(np.nonzero(ch[0]["prn"] == p)[0][0]) for p in prns}
    chans = tracked_inputs(eps, prns, g["nav_frames"], slot_of_prn)
    s0 = 1500000                                      # after the pull-in of every channel (test_track: 400 epochs)
    end = min(int(e["sample"][-2]) for e in eps)
    return chans, gps.pvt_config(s0, step, (end - s0) // step, iono)


def test_tracked_fixes_on_the_cpu(tmp_path):
    """12.1 s of sky12_static_35s through the acquisition and tracking models, the anchor from the decoded words, the
    ephemeris from the scenario's frame: sets the tracked bounds the GPU tests share."""
    g, ch, prns, eps = model_run("sky12_static_35s_i8", 121)
    _, _, iono = rinex(tmp_path, 12)
    chans, cfg = tracked_fixes(eps, prns, g, ch, iono)
    fix, _, _ = PM.pvt(chans, eps, cfg)
    assert (fix["nused"] == 12).all()
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], ch.shape[0] + 1, 0)
    check_truth(fix, xyz, START_SOW, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])
