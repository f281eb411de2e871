"""Per-PRN Doppler windows on the GPU (gpsb200_acquire_windows / _device, Context.acquire_windows, gpsb200-acq --almanac):
the grid against the numpy model bit for bit, every row against gpsb200_acquire run on that PRN alone, windows on the
cold grid against the standard search, every split of a row's delays against the unsplit search, the argument checks,
memcheck, and the whole chain on the 780 s almanac stream: synthesized, tracked through a page rotation, its almanac
decoded and a warm start made from it."""
import ctypes
import math
import os
import shutil
import subprocess
import sys
import zlib

import numpy as np
import pytest

import acq_model as M
import almanac_model as AM
import scenario
from scenario import gps
from test_acquire import golden_rows
from test_acquire_gpu import random_stream
from test_almanac import LOC, START, make_nav, make_sem
from test_almanac_decode import SOW0, WEEK, slot_words
from test_coarse_gpu import _device_not_supported

pytestmark = pytest.mark.gpu

ERR_ARG = -1
STEP = 250.0


def windows_for(prns, seed):
    """A first bin per PRN, spread over +-6 kHz at odd offsets from the cold grid."""
    rng = np.random.default_rng(seed)
    return rng.uniform(-6000.0, 6000.0, len(prns)).round(1)


@pytest.mark.parametrize("kind", ["int8", "int16"])
@pytest.mark.parametrize("nprn", [1, 12, 32])
def test_windows_equal_the_model_and_each_prn_alone(kind, nprn):
    """Random int8 and saturating int16 input, K = 1..3, at an odd s0 with the window ending at the buffer's end."""
    K = 1 + nprn % 3
    s0 = 1237
    n = s0 + gps.acq_window_samples(K)
    iq, ss = random_stream(kind, n, seed=nprn * 7 + len(kind))
    prns = list(range(32, 32 - nprn, -1))
    f_lo = windows_for(prns, nprn)
    nbins = 3
    with gps.Context(1, 1) as ctx:
        res, grid = ctx.acquire_windows(iq, ss, prns, f_lo, STEP, nbins, ms=K, s0=s0, want_grid=True)
        for p, prn in enumerate(prns):
            one, g1 = ctx.acquire(iq, ss, [prn], ms=K, s0=s0, f_lo=f_lo[p], step=STEP, nbins=nbins, want_grid=True)
            assert res[p].tobytes() == one[0].tobytes(), prn
            assert np.array_equal(grid[p], g1[0]), prn
    for p in ([0, nprn - 1] if nprn > 1 else [0]):     # the model is slow: two rows each
        want = M.grid(iq, ss, s0, K, [prns[p]], f_lo[p], STEP, nbins)
        assert np.array_equal(grid[p:p + 1], want)
        assert res[p:p + 1].tobytes() == M.reduce(want, [prns[p]], f_lo[p], STEP).tobytes()


def test_windows_on_a_signal_equal_the_model_and_the_cold_grid_rows():
    """A stream with satellites in it, K = 2: windows of 5 bins on the cold search's grid around each PRN's f_carr give
    the cold search's rows bit for bit, and the model's."""
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, [0])
    with gps.Context(12, 1) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        iq, _ = ctx.synth_blocks(ch, gps.SC08)
        prns = [int(p) for p in ch[0]["prn"] if p > 0] + [31]
        f_carr = {int(r["prn"]): float(r["f_carr"]) for r in ch[0] if r["prn"] > 0}
        cold, cgrid = ctx.acquire(iq, gps.SC08, prns, ms=2, s0=3001, want_grid=True)
        j0 = [int(round((f_carr.get(p, 0.0) + 5000.0) / STEP)) - 2 for p in prns]
        f_lo = np.array([-5000.0 + j * STEP for j in j0])
        res, grid = ctx.acquire_windows(iq, gps.SC08, prns, f_lo, STEP, 5, ms=2, s0=3001, want_grid=True)
    for p, j in enumerate(j0):
        assert np.array_equal(grid[p], cgrid[p, j:j + 5]), prns[p]
        if p < len(prns) - 1:
            assert res[p]["doppler_hz"] == cold[p]["doppler_hz"] and res[p]["delay"] == cold[p]["delay"]
            assert res[p]["p1"] == cold[p]["p1"] and res[p]["p2"] == cold[p]["p2"]
    for p in (0, len(prns) - 1):                       # a present PRN and the absent PRN 31 against the model
        want = M.grid(iq, 1, 3001, 2, prns[p:p + 1], f_lo[p], STEP, 5)
        assert np.array_equal(grid[p:p + 1], want), prns[p]
        assert res[p:p + 1].tobytes() == M.reduce(want, prns[p:p + 1], f_lo[p], STEP).tobytes()


SPLITS = [1, 2, 3, 4, 6]


def test_the_split_is_chosen_from_the_rows_against_the_sm_count():
    """One side of the selection and the other: the standard search (1312 rows, 3.3 waves) is never split, a warm start
    of 12 x 5 or 12 x 9 rows (under one wave) is; a forced split holds until it is released."""
    with gps.Context(1, 1) as ctx:
        assert ctx.debug_acq_split(32, 41) == 1
        assert ctx.debug_acq_split(12, 5) > 1 and ctx.debug_acq_split(12, 9) > 1
        assert ctx.debug_acq_split(1, 1) > 1
        assert ctx.debug_acq_split(12, 5, force=1) == 1 and ctx.debug_acq_split(32, 41) == 1
        assert ctx.debug_acq_split(32, 41, force=4) == 4
        assert ctx.debug_acq_split(12, 5, force=0) > 1
        for bad in (5, 12, 7, -2):
            with pytest.raises(gps.GpsB200Error):
                ctx.debug_acq_split(12, 5, force=bad)


@pytest.mark.parametrize("kind", ["int8", "int16"])
def test_every_split_gives_the_unsplit_bits(kind):
    """Windows of 12 PRNs (the warm-start shape) and a cold search of 3 PRNs x 41 bins, each with every split forced and
    with the automatic choice: results and grids equal the unsplit search's, bit for bit; random input, K = 2, odd s0."""
    s0 = 777
    iq, ss = random_stream(kind, s0 + gps.acq_window_samples(2) + 3, seed=21 + len(kind))
    prns = list(range(1, 13))
    f_lo = windows_for(prns, 9)
    with gps.Context(1, 1) as ctx:
        got = {}
        for force in SPLITS + [0]:
            assert ctx.debug_acq_split(12, 9, force=force) == (force or ctx.debug_acq_split(12, 9))
            w = ctx.acquire_windows(iq, ss, prns, f_lo, STEP, 9, ms=2, s0=s0, want_grid=True)
            w_nogrid = ctx.acquire_windows(iq, ss, prns, f_lo, STEP, 9, ms=2, s0=s0)
            c = ctx.acquire(iq, ss, [3, 17, 29], ms=2, s0=s0, want_grid=True)
            got[force] = (w, w_nogrid, c)
        ctx.debug_acq_split(1, 1, force=0)
    (w1, g1), w1n, (c1, cg1) = got[1]
    assert w1.tobytes() == w1n.tobytes()
    for force, ((w, g), wn, (c, cg)) in got.items():
        assert w.tobytes() == w1.tobytes() and wn.tobytes() == w1.tobytes() and np.array_equal(g, g1), force
        assert c.tobytes() == c1.tobytes() and np.array_equal(cg, cg1), force
    want = M.grid(iq, ss, s0, 2, prns[:1], f_lo[0], STEP, 9)
    assert np.array_equal(g1[:1], want)


def test_bad_arguments_are_refused_before_anything_is_enqueued():
    iq, ss = random_stream("int8", gps.acq_window_samples(1) + 10, seed=3)
    with gps.Context(1, 1) as ctx:
        good = ctx.acquire_windows(iq, ss, [1, 2], [100.0, -900.0], STEP, 3, ms=1)
        L = gps.lib()
        cfg = gps.AcqConfig()
        cfg.ms, cfg.nprn, cfg.step_hz, cfg.nbins = 1, 2, STEP, 3
        cfg.prn[0], cfg.prn[1] = 1, 2
        res = np.zeros(2, gps.ACQ_RESULT_DTYPE)
        flo = np.array([100.0, -900.0])
        n = iq.size // 2
        assert L.gpsb200_acquire_windows(ctx._h, iq.ctypes.data, n, ss, ctypes.byref(cfg), None, res.ctypes.data, None) == ERR_ARG
        assert "f_lo_prn" in gps.lib().gpsb200_last_error(ctx._h).decode()
        for bad in ([math.nan, 0.0], [1.5e6, 0.0], [0.0, -1.5e6 - 1.0], [1.5e6 - 2 * STEP + 1.0, 0.0]):
            f = np.array(bad)
            assert L.gpsb200_acquire_windows(ctx._h, iq.ctypes.data, n, ss, ctypes.byref(cfg), f.ctypes.data,
                                             res.ctypes.data, None) == ERR_ARG, bad
        for field, val in (("nprn", 0), ("nprn", 33), ("ms", 0), ("ms", 101), ("nbins", 0), ("step_hz", 0.0),
                           ("s0", 11)):
            c2 = gps.AcqConfig.from_buffer_copy(cfg)
            setattr(c2, field, val)
            assert L.gpsb200_acquire_windows(ctx._h, iq.ctypes.data, n, ss, ctypes.byref(c2), flo.ctypes.data,
                                             res.ctypes.data, None) == ERR_ARG, field
        assert L.gpsb200_acquire_windows(ctx._h, None, n, ss, ctypes.byref(cfg), flo.ctypes.data, res.ctypes.data,
                                         None) == ERR_ARG
        assert L.gpsb200_acquire_windows(ctx._h, iq.ctypes.data, n, 3, ctypes.byref(cfg), flo.ctypes.data, res.ctypes.data,
                                         None) == ERR_ARG
        assert L.gpsb200_acquire_windows(None, iq.ctypes.data, n, ss, ctypes.byref(cfg), flo.ctypes.data, res.ctypes.data,
                                         None) == ERR_ARG
        with pytest.raises(gps.GpsB200Error):
            ctx.acquire_windows(iq, ss, [1, 2], [100.0], STEP, 3, ms=1)
        again = ctx.acquire_windows(iq, ss, [1, 2], [100.0, -900.0], STEP, 3, ms=1)   # the context still works
        assert again.tobytes() == good.tobytes()



def sanitizer_run():
    iq, ss = random_stream("int16", gps.acq_window_samples(2) + 5, seed=11)
    prns = list(range(1, 13))
    with gps.Context(1, 1) as ctx:
        res, grid = ctx.acquire_windows(iq, ss, prns, windows_for(prns, 4), STEP, 5, ms=2, s0=5, want_grid=True)
    return zlib.crc32(res.tobytes() + grid.tobytes())


def test_windows_clean_under_compute_sanitizer():
    """memcheck over one windowed call. Where the tool reports the device unsupported, the fallback of
    test_sanitizers: CUDA reports no error and repeated runs give the same bytes."""
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_acquire_windows_gpu as W; "
            "print('ok', W.sanitizer_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1500)
    if _device_not_supported(r):
        import torch
        for _ in range(3):
            assert str(sanitizer_run()) == plain.stdout.split()[-1]
            torch.cuda.synchronize()
        return
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-500:])
    assert plain.stdout.split()[-1] == r.stdout.split()[-1]


# ---- warm start on the 780 s almanac stream ------------------------------------------------------------------------
def offset_apriori(loc):
    lat, lon = math.radians(loc[0]), math.radians(loc[1])
    east = np.array([-math.sin(lon), math.cos(lon), 0.0])
    up = np.array([math.cos(lat) * math.cos(lon), math.cos(lat) * math.sin(lon), math.sin(lat)])
    return AM.llh_to_ecef(*loc) + 50e3 * east + 1e3 * up


def warm_windows(sky, prns, window=500.0):
    h = int(math.ceil(window / STEP))
    return np.array([STEP * round(float(sky[p - 1]["doppler_hz"]) / STEP) - h * STEP for p in prns]), 2 * h + 1


CHUNK = 1000          # blocks synthesized per call (600 MB of int8)
WARM_BLOCK = 6000     # the warm start: 600 s into the run


def test_chain_tracks_a_rotation_decodes_the_almanac_and_warm_starts_from_it(tmp_path):
    """The whole chain on the 780 s almanac stream: synthesized on the GPU in calls of 1000 blocks that continue the
    carrier chain (block CRCs equal to the reference's), slot 0's PRN acquired in block 0 and tracked through all 780 s
    (the state carried across the calls, each buffer starting one block early), its epochs decoded. The almanac of the
    tracked words equals the one decoded from the engine's frames, record for record and bit for bit, all 32 PRNs. A
    warm start from it at 600 s, the a-priori 50 km east, 1 km up and 10 s late: every PRN the engine has allocated is
    predicted above -5 deg, searched, and found within one sample of its code delay and step/2 of its f_carr."""
    nav_file, sem = make_nav(tmp_path, 12), make_sem(tmp_path)
    ch, nav = gps.scenario(nav_file, *LOC, seconds=780, max_chan=12, start=START, almanac_file=sem)
    crcs = scenario.load_golden("sky12_alm_static_780s_i8")["crcs"]
    nblk = ch.shape[0]
    prn = int(ch[0]["prn"][0])
    assert (ch["prn"][:, 0] == prn).all()
    from_frames, wna_frames = gps.nav_almanac(slot_words(nav, 0, range(nav.shape[0])), WEEK)
    assert wna_frames == WEEK % 256 and from_frames["valid"].all()
    epochs, state, carr, tail, warm = [], None, None, None, None
    with gps.Context(12, CHUNK, max_nav_frames=len(nav)) as sctx, gps.Context(1, 1) as rctx:
        sctx.set_nav_frames(nav)
        for lo in range(0, nblk, CHUNK):
            part = ch[lo:lo + CHUNK]
            if lo > 0:
                part = gps.sharding.seed_slice(part, ch[lo - 1], carr)
            out, carr = sctx.synth_blocks(part, 1)
            out = out.reshape(-1)
            assert np.array_equal(scenario.crc_blocks(out), crcs[lo:lo + part.shape[0]])
            if lo <= WARM_BLOCK < lo + part.shape[0]:
                k = WARM_BLOCK - lo
                warm = out[k * gps.BLOCK_ELEMS:(k + 1) * gps.BLOCK_ELEMS].copy()
            if state is None:
                r = rctx.acquire(out, gps.SC08, [prn], ms=10)[0]
                state = gps.track_start(prn, float(r["doppler_hz"]), int(r["delay"]))
                buf, base = out, 0
            else:
                buf, base = np.concatenate([tail, out]), (lo - 1) * gps.BLOCK_SAMPLES
            eps, st = rctx.track([state], buf, gps.SC08, base=base)
            state = st[0]
            epochs.append(eps[0])
            tail = out[-gps.BLOCK_ELEMS:].copy()
            del buf, out
    ep = np.concatenate(epochs)
    assert ep.size >= 779 * 1000 and ep["lock"][2000:].mean() > 0.999
    _, words, sync = gps.nav_decode(ep)
    assert sync["frame_bit"] >= 0 and words["parity_ok"].all()
    rec, wna = gps.nav_almanac(words, WEEK)
    assert wna == wna_frames and rec.tobytes() == from_frames.tobytes()

    b = WARM_BLOCK
    sky = gps.almanac_predict(rec, WEEK, SOW0 + 0.1 * b + 10.0, offset_apriori(LOC))
    held = [int(p) for p in ch[b]["prn"] if p > 0]
    assert all(sky[p - 1]["el_deg"] >= -5.0 for p in held)
    prns = [p for p in range(1, 33) if sky[p - 1]["valid"] and sky[p - 1]["el_deg"] >= -5.0]
    assert set(held) <= set(prns)
    f_lo, nbins = warm_windows(sky, prns)
    with gps.Context(1, 1) as ctx:
        res = ctx.acquire_windows(warm, gps.SC08, prns, f_lo, STEP, nbins, ms=10)
    bad = M.truth_failures([r for r in res if r["prn"] in held], ch[b], f_lo=0.0, step=STEP, r_present=2.5,
                           r_absent=np.inf, edge=0.0)
    assert not bad, bad


def test_cli_almanac_prints_the_warm_start(tmp_path):
    """gpsb200-acq --almanac on a gpsb200-sim --almanac stream: the PRNs predicted above the mask, the results of
    Context.acquire_windows and the predictions beside them; without --almanac the output is the cold search's."""
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-acq")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    nav_file, sem = make_nav(tmp_path, 12), make_sem(tmp_path)
    out = tmp_path / "iq.bin"
    r = subprocess.run([os.path.join(exe_dir, "gpsb200-sim"), "-e", nav_file, "-l", "35.681298,139.766247,10.0", "-d", "3",
                        "-s", "2024/01/07,02:00:00", "--almanac", sem, "-o", str(out)], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-600:]
    B = 10
    args = [os.path.join(exe_dir, "gpsb200-acq"), str(out), "--block", str(B), "--almanac", sem, "--assist-pos",
            "35.9,139.9,1010", "--assist-time", "2024/01/07,02:00:%02d" % (B // 10 + 10)]
    r = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = [l.split() for l in r.stdout.splitlines() if not l.startswith("#")]
    rec = gps.almanac_read(sem)[1]
    sky = gps.almanac_predict(rec, WEEK, SOW0 + B // 10 + 10, AM.llh_to_ecef(35.9, 139.9, 1010.0))
    prns = [p for p in range(1, 33) if sky[p - 1]["valid"] and sky[p - 1]["el_deg"] >= -5.0]
    assert [int(l[0]) for l in lines] == prns
    f_lo, nbins = warm_windows(sky, prns)
    s = np.fromfile(out, np.int8)
    with gps.Context(1, 1) as ctx:
        res = ctx.acquire_windows(s, gps.SC08, prns, f_lo, STEP, nbins, ms=10, s0=B * gps.BLOCK_SAMPLES)
    for l, q in zip(lines, res):
        assert float(l[1]) == round(float(q["doppler_hz"]), 1) and int(l[2]) == q["delay"]
        assert abs(float(l[6]) - sky[q["prn"] - 1]["doppler_hz"]) <= 0.05
        assert abs(float(l[7]) - sky[q["prn"] - 1]["el_deg"]) <= 0.005
    held = {int(p) for p in gps.scenario(nav_file, *LOC, seconds=3, max_chan=12, start=START, almanac_file=sem)[0][B]["prn"]
            if p > 0}
    assert {int(l[0]) for l in lines if l[5] == "yes"} == held
    plain = subprocess.run(args[:4], capture_output=True, text=True, timeout=600)
    assert plain.returncode == 0 and "warm start" not in plain.stdout and "41 bins" in plain.stdout
