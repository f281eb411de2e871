"""Tracking on the GPU (gpsb200_track / _device, Context.track, gpsb200-track): the epochs against the numpy model bit for
bit, cut into calls, and the truth checks of tests/test_track.py on the reference's streams as the GPU path synthesizes
them (every block CRC equal to the reference's)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import scenario
import track_model as T
from scenario import gps
from test_acquire import golden_rows
from test_acquire_gpu import synth_checked
from test_scenario import LOC, START, make_nav, motion_file
from test_track import ACQ, starts, truth_figures

pytestmark = pytest.mark.gpu

ERR_ARG = -1


def acquire_and_start(ctx, iq, ss, prns, s0=0):
    res = ctx.acquire(iq, ss, prns, s0=s0, **ACQ)
    for r in res:
        r["delay"] += s0
    return starts(res)


def random_states(nch, base, seed):
    rng = np.random.default_rng(seed)
    return np.array([T.start(int(rng.integers(1, 33)), float(rng.uniform(-4000, 4000)), base + int(rng.integers(0, 4000)))
                     for _ in range(nch)])


@pytest.mark.parametrize("kind", ["int8", "int16"])
def test_epochs_equal_model_on_random_input(kind):
    """Random int8 and saturating int16 input: the loops wander, deterministically. Buffer at base 12345."""
    rng = np.random.default_rng(len(kind))
    n = 150000
    if kind == "int8":
        iq, ss = rng.integers(-128, 128, 2 * n).astype(np.int8), gps.SC08
    else:
        iq, ss = rng.choice(np.array([-32768, -32767, -2049, -2048, -17, 0, 15, 2047, 2048, 32767], np.int16), 2 * n), gps.SC16
    st = random_states(5, 12345, 7)
    with gps.Context(1, 1) as ctx:
        got, gst = ctx.track(st, iq, ss, base=12345)
    want, wst = T.track(iq, ss, 12345, st)
    for g_, w_ in zip(got, want):
        assert g_.size > 40 and np.array_equal(g_, w_)
    assert np.array_equal(gst, wst.astype(gps.TRACK_STATE_DTYPE))


def signal(nblk=5, name="sky12_static_35s_i8"):
    g = scenario.load_golden(name)
    ch, out, ss = synth_checked(g, range(nblk))
    return g, ch, out, ss


def test_epochs_equal_model_on_a_signal_and_across_cuts():
    """0.5 s of sky12_static from its acquisition: one call equals the model; the same run cut into three calls (the
    state carried, each buffer starting at the earliest channel's next period) gives the same epochs and states."""
    g, ch, out, ss = signal()
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(12, 1) as ctx:
        st = acquire_and_start(ctx, out, ss, prns)
        one, st1 = ctx.track(st, out, ss)
        parts = [[] for _ in prns]
        s = st.copy()
        for cut in (400000, 1000000, out.size // 2):
            base = int(s["sample"].min())
            eps, s = ctx.track(s, out[2 * base:2 * cut], ss, base=base)
            for k, e in enumerate(eps):
                parts[k].append(e)
    want, wst = T.track(out, ss, 0, st)
    for k in range(len(prns)):
        assert np.array_equal(one[k], want[k])
        assert np.array_equal(np.concatenate(parts[k]), one[k])
    assert np.array_equal(s, st1) and np.array_equal(st1, wst.astype(gps.TRACK_STATE_DTYPE))


def track_truth(ch, out, ss, g, frames, frame_of_block, **kw):
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(ch.shape[1], 1) as ctx:
        st = acquire_and_start(ctx, out, ss, prns)
        eps, _ = ctx.track(st, out, ss)
    return truth_figures(ch, eps, prns, frames, frame_of_block, **kw)


def test_truth_sky12_static_35s():
    """35 s, 12 channels, a frame roll at block 300: lock, Doppler, code, bit edges, every word equal to the scenario's
    across the roll with good parity, TOW."""
    g, ch, out, ss = signal(349)
    fig = truth_figures_and_words(ch, out, ss, g)
    assert all(v[3] >= 50 for v in fig.values()), fig


def truth_figures_and_words(ch, out, ss, g, **kw):
    return track_truth(ch, out, ss, g, g["nav_frames"], g["nav_frame_of_block"], **kw)


def test_truth_sky32_static_10s():
    """32 channels, the int8 stream wrapping under 31 interferers."""
    g, ch, out, ss = signal(99, "sky32_static_10s_i8")
    fig = truth_figures_and_words(ch, out, ss, g)
    assert all(v[3] >= 12 for v in fig.values()), fig


def test_truth_sky12_circle_60s_int16(tmp_path):
    """The receiver on the circle, int16; records from the scenario engine (its first two blocks are the reference's,
    all of them pinned by the block CRCs of the reference's stream)."""
    g = scenario.load_golden("sky12_circle_60s_i16")
    ch, nav = gps.scenario(make_nav(tmp_path, 12), *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path),
                           start=START)
    with gps.Context(12, ch.shape[0], max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        out, _ = ctx.synth_blocks(ch, gps.SC16)
    assert np.array_equal(scenario.crc_blocks(out), g["crcs"][:, 0])
    fig = track_truth(ch, out, gps.SC16, g, nav, ch["nav_frame"][:, 0])
    assert all(v[3] >= 90 for v in fig.values()), fig


def test_device_source_in_place_equals_host_source():
    torch = pytest.importorskip("torch")
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, range(4))
    nblk, nchan = ch.shape
    dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    stream = torch.cuda.Stream()
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(nchan, nblk) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        with torch.cuda.stream(stream):
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
            st = starts(ctx.acquire(device_ptr=dev.data_ptr(), nsamples=nblk * gps.BLOCK_SAMPLES, sample_size=gps.SC08,
                                    prns=prns, stream=stream.cuda_stream, **ACQ))
            got, gst = ctx.track(st, device_ptr=dev.data_ptr(), nsamples=nblk * gps.BLOCK_SAMPLES, sample_size=gps.SC08,
                                 stream=stream.cuda_stream)
        stream.synchronize()
        host = dev.cpu().numpy()
        want, wst = ctx.track(st, host, gps.SC08)
    assert np.array_equal(scenario.crc_blocks(host), g["crcs"][:nblk, 0])
    assert all(np.array_equal(a, b) for a, b in zip(got, want)) and np.array_equal(gst, wst)


def test_bad_arguments_are_rejected_and_the_context_still_synthesizes():
    torch = pytest.importorskip("torch")
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, [0])
    iq = np.zeros(2 * 20000, np.int8)
    dev = torch.zeros(2 * 20000 + 64, dtype=torch.int8, device="cuda")
    good = np.array([T.start(3, 100.0, 10)])
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(g["nav_frames"])

        def bad(f, v):
            s = good.copy()
            s[f] = v
            return s
        cases = [dict(states=bad("prn", 0)), dict(states=bad("prn", 33)), dict(states=bad("code_step", 5)),
                 dict(states=bad("code_phase", 1 << 33)), dict(states=bad("carr_freq", (1 << 34) + 1)),
                 dict(states=bad("lock", 2)), dict(states=good, base=11), dict(states=good, sample_size=3),
                 dict(states=good, max_epochs=0), dict(states=np.repeat(good, 33))]
        for kw in cases:
            a = dict(iq=iq, sample_size=gps.SC08)
            a.update(kw)
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.track(**a)
            assert e.value.code == ERR_ARG, kw
        for kw in (dict(device_ptr=dev.data_ptr() + 2), dict(device_ptr=dev.data_ptr(), base=11)):
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.track(good, nsamples=20000, sample_size=gps.SC08, **kw)
            assert e.value.code == ERR_ARG, kw
        eps, _ = ctx.track(good, iq, gps.SC08)
        assert eps[0].size == 6
        out, _ = ctx.synth_blocks(ch, gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]
    with pytest.raises(gps.GpsB200Error):
        gps.track_start(0, 0.0, 0)


def test_cli_prints_what_the_api_returns(tmp_path):
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-track")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav = tmp_path / "sky12.nav"
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat", "12", "--out",
                           str(nav)])
    iq = tmp_path / "iq.bin"
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", str(nav), "-l", "35.681298,139.766247,10.0", "-d", "9",
                           "-s", "2024/01/07,02:00:00", "-o", str(iq)])
    r = subprocess.run([os.path.join(exe_dir, "gpsb200-track"), str(iq), "--block", "1", "--offset-ms", "2",
                        "--prn", "1-20,32"], capture_output=True, text=True, check=True)
    rows = [ln.split() for ln in r.stdout.splitlines() if ln and not ln.startswith("#")]
    s = np.fromfile(iq, dtype=np.int8)
    s0 = gps.BLOCK_SAMPLES + 2 * 3000
    prns = list(range(1, 21)) + [32]
    with gps.Context(1, 1) as ctx:
        res = ctx.acquire(s, gps.SC08, prns, s0=s0, **ACQ)
        res = res[res["ratio"] >= 2.5]
        for r_ in res:
            r_["delay"] += s0
        eps, _ = ctx.track(starts(res), s, gps.SC08)
    assert len(rows) == res.size and res.size >= 8
    for row, r_, e in zip(rows, res, eps):
        _, _, sy = gps.nav_decode(e)
        assert row[0] == str(r_["prn"])
        assert row[1] == ("yes" if e["lock"][-1] else "no") == "yes"
        assert row[2] == "%.1f" % (e["carr_step"][-1] * 3e6 / 2 ** 32)
        assert row[3:] == [str(sy["subframes"]), str(sy["words_ok"]), str(sy["nwords"]), str(sy["first_tow"])]
        assert sy["subframes"] >= 1
