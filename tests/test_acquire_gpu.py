"""The acquisition search on the GPU (gpsb200_acquire / _device, Context.acquire, gpsb200-acq): its grid against the numpy
model bit for bit, and the truth checks on the reference's streams as the GPU path synthesizes them."""
import os
import subprocess
import sys

import numpy as np
import pytest

import acq_model as M
import scenario
from scenario import gps
from test_acquire import ALL, F_LO, K, NBINS, R_ABSENT, R_PRESENT, STEP, golden_rows

pytestmark = pytest.mark.gpu

ERR_ARG = -1


def random_stream(kind, nsamples, seed):
    rng = np.random.default_rng(seed)
    if kind == "int8":
        return rng.integers(-128, 128, 2 * nsamples).astype(np.int8), gps.SC08
    vals = np.array([-32768, -32767, -2049, -2048, -17, 0, 15, 2047, 2048, 32767], np.int16)
    return rng.choice(vals, 2 * nsamples), gps.SC16


@pytest.mark.parametrize("kind", ["int8", "int16"])
@pytest.mark.parametrize("ms", [1, 3])
def test_grid_equals_model_bit_for_bit(kind, ms):
    """Random int8 and saturating int16 input, a window at an odd s0 that ends exactly at the buffer's last sample."""
    s0 = 1237
    n = s0 + gps.acq_window_samples(ms)
    iq, ss = random_stream(kind, n, seed=ms * 10 + len(kind))
    prns, f_lo, step, nbins = [1, 13, 32], -2437.5, 1625.0, 4
    with gps.Context(1, 1) as ctx:
        res, grid = ctx.acquire(iq, ss, prns, ms=ms, s0=s0, f_lo=f_lo, step=step, nbins=nbins, want_grid=True)
    want = M.grid(iq, ss, s0, ms, prns, f_lo, step, nbins)
    assert np.array_equal(grid, want)
    assert np.array_equal(res, M.reduce(want, prns, f_lo, step))


def test_grid_equals_model_on_a_signal_and_wide_bins():
    """A stream with satellites in it (peaks, ties of zero rows absent) over the full 41-bin search of three PRNs."""
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, [0])
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        iq, _ = ctx.synth_blocks(ch, gps.SC08)
        prns = [int(ch[0]["prn"][0]), int(ch[0]["prn"][5]), 31]
        res, grid = ctx.acquire(iq, gps.SC08, prns, ms=2, s0=3001, want_grid=True)
    want = M.grid(iq, 1, 3001, 2, prns, F_LO, STEP, NBINS)
    assert np.array_equal(grid, want)
    assert np.array_equal(res, M.reduce(want, prns, F_LO, STEP))


def synth_checked(g, blocks, ctx=None):
    """GPU synthesis of the fixture's consecutive blocks from their records; every block CRC equals the reference's."""
    ch = golden_rows(g, blocks)
    ss = int(g["sample_size"])
    with gps.Context(ch.shape[1], len(blocks), max_nav_frames=len(g["nav_frames"])) as c:
        c.set_nav_frames(g["nav_frames"])
        out, _ = c.synth_blocks(ch, ss)
    crc = scenario.crc_blocks(out)
    assert np.array_equal(crc, g["crcs"][list(blocks), 0]), np.nonzero(crc != g["crcs"][list(blocks), 0])[0]
    return ch, out, ss


def truth_on(name, blocks, search, edge=None):
    g = scenario.load_golden(name)
    ch, out, ss = synth_checked(g, blocks)
    with gps.Context(1, 1) as ctx:
        for i, b in enumerate(blocks):
            if b not in search:
                continue
            res = ctx.acquire(out, ss, ALL, ms=K, s0=i * gps.BLOCK_SAMPLES, f_lo=F_LO, step=STEP, nbins=NBINS)
            bad = M.truth_failures(res, ch[i], F_LO, STEP, R_PRESENT, R_ABSENT, edge=edge)
            assert bad == [], (name, b, bad)
    return ch


def test_truth_sky12_static_int8():
    ch = truth_on("sky12_static_10s_i8", range(99), {0, 33, 66, 98})
    assert (ch[0]["prn"] > 0).sum() == 12


# Doppler tolerance of the 27-32 channel streams: one bin (|f_j1 - f_carr| <= step) wherever f_carr lies. With 1 ms
# coherent periods the frequency peak is broad (about +-1 kHz), and a NAV bit transition inside one of the K periods
# plus the cross-correlation of 26-31 other signals move it by up to about 65 Hz, so f_carr near a bin edge may land in
# the neighbouring bin. In the model (CPU): PRN 29 of sky32_static block 98 (f_carr 3327.7 Hz, 47 Hz from the edge)
# peaks at 3500 Hz, PRN 4 of sky32_lat60 block 3000 (f_carr -3439.4 Hz, 64 Hz from the edge) at -3250 Hz; a 25 Hz scan of
# PRN 15 of block 2396 peaks at 3354 Hz against f_carr 3404 Hz. The 12-channel streams hold the step/2 rule (step within
# step/10 of an edge).
CROWDED_EDGE = STEP / 2


def test_truth_sky32_static_int8_all_prns_present_wrapped():
    """32 channels: every PRN is present and the int8 stream wraps where the sum of channels exceeds its range."""
    ch = truth_on("sky32_static_10s_i8", range(99), {0, 30, 60, 98}, edge=CROWDED_EDGE)
    assert sorted(ch[0]["prn"]) == ALL


def test_truth_sky32_lat60_prns_come_and_go():
    """27-29 of 32 slots in use, channels reallocated between the two ranges."""
    held = set()
    for rng_ in (range(2396, 2405), range(2996, 3005)):
        ch = truth_on("sky32_lat60_310s_i8", list(rng_), {rng_[0], rng_[4], rng_[8]}, edge=CROWDED_EDGE)
        held |= {frozenset(int(p) for p in row["prn"] if p > 0) for row in ch}
    assert len(held) > 1          # the set of satellites changes


def test_truth_sky12_circle_int16_motion():
    truth_on("sky12_circle_60s_i16", [0, 1], {0, 1})


def test_device_source_in_place_equals_host_source():
    torch = pytest.importorskip("torch")
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, range(3))
    nblk, nchan = ch.shape
    dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    stream = torch.cuda.Stream()
    with gps.Context(nchan, nblk) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        with torch.cuda.stream(stream):
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
            got, ggrid = ctx.acquire(device_ptr=dev.data_ptr(), nsamples=nblk * gps.BLOCK_SAMPLES, sample_size=gps.SC08,
                                     s0=gps.BLOCK_SAMPLES + 7, ms=K, want_grid=True, stream=stream.cuda_stream)
        stream.synchronize()
        host = dev.cpu().numpy()
        want, wgrid = ctx.acquire(host, gps.SC08, s0=gps.BLOCK_SAMPLES + 7, ms=K, want_grid=True)
    assert np.array_equal(scenario.crc_blocks(host), g["crcs"][:nblk, 0])
    assert np.array_equal(got, want) and np.array_equal(ggrid, wgrid)


def test_cli_prints_what_the_api_returns(tmp_path):
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-acq")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav = tmp_path / "sky12.nav"
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat", "12", "--out",
                           str(nav)])
    iq = tmp_path / "iq.bin"
    subprocess.check_call([os.path.join(exe_dir, "gpsb200-sim"), "-e", str(nav), "-l", "35.681298,139.766247,10.0", "-d", "1",
                           "-s", "2024/01/07,02:00:00", "-o", str(iq)])
    r = subprocess.run([os.path.join(exe_dir, "gpsb200-acq"), str(iq), "--block", "4", "--offset-ms", "3", "--ms", "5",
                        "--prn", "1-20,32"], capture_output=True, text=True, check=True)
    rows = [ln.split() for ln in r.stdout.splitlines() if ln and not ln.startswith("#")]
    s = np.fromfile(iq, dtype=np.int8)
    with gps.Context(1, 1) as ctx:
        res = ctx.acquire(s, gps.SC08, list(range(1, 21)) + [32], ms=5, s0=4 * gps.BLOCK_SAMPLES + 3 * 3000)
    assert len(rows) == res.size
    for row, want in zip(rows, res):
        assert row[0] == str(want["prn"])
        assert row[1] == "%.1f" % want["doppler_hz"]
        assert row[2] == str(want["delay"]) and row[3] == "%.3f" % want["delay_chips"]
        assert row[4] == "%.3f" % want["ratio"]
        assert row[5] == ("yes" if want["ratio"] >= 2.5 else "no")
    assert sum(r_[5] == "yes" for r_ in rows) >= 1


def test_bad_arguments_are_rejected_and_the_context_still_synthesizes():
    torch = pytest.importorskip("torch")
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, [0])
    n = gps.acq_window_samples(K) + 100
    iq = np.zeros(2 * n, np.int8)
    dev = torch.zeros(2 * n + 64, dtype=torch.int8, device="cuda")
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        cases = [dict(prns=[0]), dict(prns=[5, 33]), dict(ms=0), dict(ms=101), dict(s0=101),
                 dict(sample_size=3), dict(prns=[]), dict(nbins=0), dict(nbins=1025)]
        for kw in cases:
            a = dict(iq=iq, sample_size=gps.SC08, ms=K)
            a.update(kw)
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.acquire(**a)
            assert e.value.code == ERR_ARG, kw
        ctx.acquire(iq, gps.SC08, ms=K, s0=100)                          # ends exactly at the last sample: fine
        for kw in (dict(device_ptr=dev.data_ptr() + 2), dict(device_ptr=dev.data_ptr(), s0=101)):
            with pytest.raises(gps.GpsB200Error) as e:
                ctx.acquire(nsamples=n, sample_size=gps.SC08, ms=K, **kw)
            assert e.value.code == ERR_ARG, kw
        out, _ = ctx.synth_blocks(ch, gps.SC08)
    assert scenario.crc_blocks(out)[0] == g["crcs"][0, 0]
