"""Device buffers past 2^31 and 2^32 bytes, and device sources behind work pending on the caller's stream.

- Synthesis into one device destination of 4.32 GB: 7200 int8 blocks of the hour-long 32-channel scenario in one call
  (k_synth_lanes and k_synth) and through the three-step slice path (eager and lazy), every block against the CRC of
  the reference's block; 3600 int16 blocks against short calls started from the exact chain.
- Every receiver entry point with a device source, read in place from a 2^31 + 2^22-sample buffer (int8: 4 GiB,
  int16: 8 GiB) of device noise with 1 s of sky12_static_35s written across sample 2^29, 2^30 or 2^31 (byte 2^31, 2^32
  or 2^33) or at the buffer's end: byte for byte the call on a host array holding the region alone, with the region's
  offset added to s0, s_a and the states' samples and taken off the sample fields of the results.
- Each of the six device-source receiver calls issued on a stream still sleeping before the copy (or the synthesis)
  of its source: the results of the true source. Every kernel of the call runs on the caller's stream (torch.profiler's
  trace), and a kernel the caller enqueues after a call cannot change its results.

Before a big buffer a test checks the device's free memory and skips, with the number, when it is short (the device
may be shared). The module prints its run time and the peak device memory in use (device-wide, mem_get_info)."""
import time

import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import scenario
import snapshot_model as SM
import track_model as T
from scenario import gps
from test_acquire import ALL, K, golden_rows
from test_coarse import WEEK
from test_collective import ephemeris
from test_gpu_parity import _nav_file
from test_scenario import LOC
from test_track import ACQ, START_SOW, starts

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GiB = 1 << 30
CTX_MARGIN = 2 * GiB          # a 7200-block context's own buffers and the receiver scratch, with room to spare
_peak = [0]


def note_memory():
    free, total = torch.cuda.mem_get_info()
    _peak[0] = max(_peak[0], total - free)


def need(nbytes):
    """Skip (never run a partial case) unless nbytes of device memory are free now."""
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %.2f GiB of free device memory, %.2f GiB are free" % (nbytes / GiB, free / GiB))


@pytest.fixture(scope="module", autouse=True)
def report():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    t0 = time.perf_counter()
    note_memory()
    yield
    print("\ntest_device_extent_gpu: %.1f s, peak device memory in use %.2f GiB" % (time.perf_counter() - t0,
                                                                                     _peak[0] / GiB))


def release():
    torch.cuda.synchronize()
    note_memory()
    torch.cuda.empty_cache()


def device_crcs(buf, nblk, chunk=1000):
    """CRC-32 of each block of the device buffer (BLOCK_ELEMS elements each), copied down chunk blocks at a time."""
    per = gps.BLOCK_ELEMS
    return np.concatenate([scenario.crc_blocks(buf[b * per:min(nblk, b + chunk) * per].cpu().numpy())
                           for b in range(0, nblk, chunk)])


# ---- synthesis past byte 2^32 -----------------------------------------------------------------------------------------
BIG = 7200                       # int8 blocks: 4.32 GB
I16 = 3600                       # int16 blocks: 4.32 GB


def first_block_past(byte, elem):
    return -(-byte // (gps.BLOCK_ELEMS * elem))


assert (first_block_past(1 << 31, 1), first_block_past(1 << 32, 1)) == (3580, 7159)
assert first_block_past(1 << 32, 2) == 3580 <= I16 and first_block_past(1 << 31, 2) == 1790


@pytest.fixture(scope="module")
def hour(tmp_path_factory):
    """The first 7200 blocks of the 3600 s, 32-channel scenario of sky32_static_3600s_i8, its NAV frames and the
    reference's CRCs of those blocks."""
    g = scenario.load_golden("sky32_static_3600s_i8")
    ch, nav = gps.scenario(_nav_file(tmp_path_factory.mktemp("nav"), 32), 35.681298, 139.766247, 10.0, seconds=3600,
                           max_chan=32, start=(2024, 1, 7, 2, 0, 0.0))
    return ch[:BIG].copy(), nav, g["crcs"][:BIG]


def check_crcs(got, want, what):
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, "%s: %d blocks differ, first %s" % (what, bad.size, bad[:10])


@pytest.mark.parametrize("lanes,kernel", [("1", "k_synth_lanes"), ("0", "k_synth")])
def test_one_int8_call_past_byte_2_32_equals_the_reference(hour, lanes, kernel, monkeypatch):
    """Blocks 0-7199 in one synth_blocks_device call into one buffer: block 3580 is the first past byte 2^31, 7159 the
    first past byte 2^32."""
    ch, nav, want = hour
    need(BIG * gps.BLOCK_ELEMS + CTX_MARGIN)
    monkeypatch.setenv("GPSB200_LANES", lanes)          # read when the context is created
    dev = torch.empty(BIG * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    try:
        with gps.Context(32, BIG, max_nav_frames=len(nav)) as ctx:
            ctx.set_nav_frames(nav)
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr())
            torch.cuda.synchronize()
            assert ctx.synth_kernel_name(32) == kernel
            note_memory()
        check_crcs(device_crcs(dev, BIG), want, kernel)
    finally:
        del dev
        release()


@pytest.mark.parametrize("eager", [False, True])
def test_three_step_int8_slice_past_byte_2_32_equals_the_reference(hour, eager):
    """The same 7200 blocks as one slice of the three-step hand-over (prepare, probe, finish, wait) into one device
    buffer; its exact outgoing state is the host chain's."""
    ch, nav, want = hour
    need(BIG * gps.BLOCK_ELEMS + CTX_MARGIN)
    dev = torch.empty(BIG * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    try:
        with gps.Context(32, BIG, max_nav_frames=len(nav)) as ctx:
            ctx.set_nav_frames(nav)
            ctx.slice_prepare(ch, gps.SC08, dev.data_ptr())
            ctx.slice_probe(eager=eager)
            _, ph = ctx.slice_finish()
            ctx.slice_wait()
            torch.cuda.synchronize()
            note_memory()
            assert np.array_equal(ph, ctx.carrier_chain(ch))
        check_crcs(device_crcs(dev, BIG), want, "eager" if eager else "lazy")
    finally:
        del dev
        release()


@pytest.fixture(scope="module")
def int16_crcs(hour):
    """CRCs of blocks 0-3599 of the hour in int16 from short host-destination calls of at most 900 blocks, each
    started from the exact incoming state of the host chain (the path tests/test_gpu_parity.py holds to the
    reference's streams)."""
    ch, nav, _ = hour
    crcs = []
    with gps.Context(32, 900, max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        for lo in range(0, I16, 900):
            part = ch[lo:lo + 900]
            if lo > 0:
                part = gps.sharding.seed_slice(part, ch[lo - 1], gps.carrier_chain(ch[:lo], threads=16))
            out, _ = ctx.synth_blocks(part, gps.SC16)
            crcs.append(scenario.crc_blocks(out))
    return np.concatenate(crcs)


@pytest.mark.parametrize("lanes,kernel", [("1", "k_synth_lanes"), ("0", "k_synth")])
def test_one_int16_call_past_byte_2_32_equals_short_calls(hour, int16_crcs, lanes, kernel, monkeypatch):
    """Blocks 0-3599 in int16 in one synth_blocks_device call: block 1790 is the first past byte 2^31, 3580 the first
    past byte 2^32."""
    ch, nav, _ = hour
    need(I16 * gps.BLOCK_ELEMS * 2 + CTX_MARGIN)
    monkeypatch.setenv("GPSB200_LANES", lanes)
    dev = torch.empty(I16 * gps.BLOCK_ELEMS, dtype=torch.int16, device="cuda")
    try:
        with gps.Context(32, I16, max_nav_frames=len(nav)) as ctx:
            ctx.set_nav_frames(nav)
            ctx.synth_blocks_device(ch[:I16], gps.SC16, dev.data_ptr())
            torch.cuda.synchronize()
            assert ctx.synth_kernel_name(32) == kernel
            note_memory()
        check_crcs(device_crcs(dev, I16), int16_crcs, kernel)
    finally:
        del dev
        release()


# ---- the six receiver calls -------------------------------------------------------------------------------------------
CALLS = ["acquire", "acquire_windows", "snapshot_measure", "snapshot_batch", "collective", "track"]
LATTICE = gps.collective_config(1000.0, 250.0, 0.5, 0.5)        # tests/test_collective_gpu.py's host/device lattice


def receiver_calls(ctx, ss, region, eph, s0, batch_s0, max_epochs):
    """The receiver calls that take a device source, set up from `region` (a host array of a stream's samples 0 on):
    the search window at region sample s0, the batch windows at batch_s0, the tracking states and the snapshot seeds
    from host searches of the region. -> name -> f(off, base=0, **source) -> tuple of arrays: the call on a source
    whose sample off is the region's sample 0 (its s0, s_a and states' samples moved by off, `base` the tracking
    buffer's first sample), with off taken back off the sample fields of the results, so that every call equals
    f(0, iq=region)."""
    res = ctx.acquire(region, ss, ALL, ms=K, s0=s0)
    sky = res[res["ratio"] >= 2.5]
    assert sky.size >= 8, sky
    sky_prns = [int(p) for p in sky["prn"]]
    f_lo = sky["doppler_hz"] - 2 * 250.0
    states = starts(ctx.acquire(region, ss, sky_prns, s0=0, **ACQ))
    batch_s0 = np.asarray(batch_s0, np.int64)

    def acquire(off, base=0, **src):
        kw = dict(sample_size=ss, ms=K, s0=off + s0)
        return (ctx.acquire(**kw, **src),) + ctx.acquire(want_grid=True, **kw, **src)

    def acquire_windows(off, base=0, **src):
        return ctx.acquire_windows(sample_size=ss, prns=sky_prns, f_lo_prn=f_lo, step=250.0, nbins=5, ms=K,
                                   s0=off + s0, want_grid=True, **src)

    def snapshot_measure(off, base=0, **src):
        out = ctx.snapshot_measure(sky, sample_size=ss, ms=K, s0=off + s0, **src)
        out["sample"] -= off
        return (out,)

    def snapshot_batch(off, base=0, **src):
        r, out = ctx.snapshot_batch(batch_s0 + off, sample_size=ss, prns=ALL, ms=K, **src)
        out["sample"] -= off
        return r, out

    def collective(off, base=0, **src):
        ap = gps.coarse_config(PM.llh_ecef(*LOC), START_SOW, off, WEEK)
        return ctx.collective(eph, ap, LATTICE, sample_size=ss, ms=K, s0=off + s0, want_scores=True, want_table=True,
                              **src)

    def track(off, base=0, **src):
        st = states.copy()
        st["sample"] += off
        eps, st = ctx.track(st, sample_size=ss, base=base, max_epochs=max_epochs, **src)
        for e in eps:
            e["sample"] -= off
        st["sample"] -= off
        return tuple(eps) + (st,)

    calls = dict(acquire=acquire, acquire_windows=acquire_windows, snapshot_measure=snapshot_measure,
                 snapshot_batch=snapshot_batch, collective=collective, track=track)
    assert sorted(calls) == sorted(CALLS)
    return calls, dict(sky=sky, states=states)


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for k, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape, (what, k, a.shape, b.shape)
        assert a.tobytes() == b.tobytes(), (what, k)


# ---- every receiver device source past sample 2^30 and 2^31 ----------------------------------------------------------
N_BIG = (1 << 31) + (1 << 22)                    # samples: int8 4 GiB + 8 MiB, int16 8 GiB + 16 MiB
REGION_BLOCKS = 10
REGION = REGION_BLOCKS * gps.BLOCK_SAMPLES       # 1 s of signal
TRACK_EPOCHS = 900                               # inside the region for every channel (starts within its first 3000)
PLACEMENTS = [("int8", 1 << 30), ("int8", 1 << 31), ("int8", None),
              ("int16", 1 << 29), ("int16", 1 << 30), ("int16", 1 << 31), ("int16", None)]


@pytest.fixture(scope="module")
def sky12(tmp_path_factory):
    """sky12_static_35s: the channel records of blocks 0-9, its NAV frames, the 12-satellite ephemeris, and the
    blocks from the host-destination path in int8 (every CRC the reference's) and int16."""
    g = scenario.load_golden("sky12_static_35s_i8")
    rows = golden_rows(g, range(REGION_BLOCKS))
    eph, _ = ephemeris(tmp_path_factory.mktemp("nav12"), 12, START_SOW)
    with gps.Context(12, REGION_BLOCKS, max_nav_frames=len(g["nav_frames"])) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        i8, _ = ctx.synth_blocks(rows, gps.SC08)
        i16, _ = ctx.synth_blocks(rows, gps.SC16)
    assert np.array_equal(scenario.crc_blocks(i8), g["crcs"][:REGION_BLOCKS, 0])
    return dict(g=g, rows=rows, eph=eph, int8=i8, int16=i16)


def placement_id(p):
    return "%s-%s" % (p[0], "end" if p[1] is None else "sample_2^%d" % (p[1].bit_length() - 1))


@pytest.mark.parametrize("kind,boundary", PLACEMENTS, ids=[placement_id(p) for p in PLACEMENTS])
def test_every_device_source_call_past_the_boundary_equals_the_host_region(sky12, kind, boundary):
    """1 s of signal written into device noise across `boundary` (or ending on the buffer's last sample); each call
    reads the whole buffer in place (base 0) and equals the host call on the region: the search and snapshot window
    straddles the boundary (or ends on the last sample), the batch holds 20 windows on both sides in three passes,
    the tracking states start 1 ms from the region's start. Tracking also runs from a pointer advanced to the region
    with base past 2^32. The host calls equal the numpy models: a small search grid, the measurement and tracking
    (the collective call's host form is held to its model by tests/test_collective_gpu.py)."""
    ss, dt, elem = (gps.SC08, torch.int8, 2) if kind == "int8" else (gps.SC16, torch.int16, 4)
    start = N_BIG - REGION if boundary is None else boundary - REGION // 2
    assert start % 8 == 0 and start * elem % 16 == 0 and start + REGION <= N_BIG
    win = gps.acq_window_samples(K)
    s0 = REGION - win if boundary is None else REGION // 2 - 15000
    assert boundary is None or start + s0 < boundary < start + s0 + win
    batch_s0 = np.sort(np.append(np.linspace(0, REGION - win, 19).astype(np.int64), s0))
    assert gps.snapshot_batch_pass(32, 41, K, ss) * 2 < batch_s0.size <= gps.snapshot_batch_pass(32, 41, K, ss) * 3
    assert boundary is None or (start + batch_s0[-8:] > boundary).all()       # the last pass lies past the boundary
    need(N_BIG * elem + GiB)

    buf = torch.empty(2 * N_BIG, dtype=dt, device="cuda")
    try:
        lim = 128 if kind == "int8" else 2048
        buf.random_(-lim, lim, generator=torch.Generator(device="cuda").manual_seed(N_BIG % 9973 + (boundary or 1)))
        g = sky12["g"]
        with gps.Context(12, REGION_BLOCKS, max_nav_frames=len(g["nav_frames"])) as sctx:
            sctx.set_nav_frames(g["nav_frames"])
            sctx.synth_blocks_device(sky12["rows"], ss, buf.data_ptr() + start * elem)
        torch.cuda.synchronize()
        note_memory()
        region = buf[2 * start:2 * (start + REGION)].cpu().numpy()
        assert np.array_equal(region, sky12[kind]), "the signal is not where it was written"
        dev = dict(device_ptr=buf.data_ptr(), nsamples=N_BIG)
        with gps.Context(12, 1) as ctx:
            calls, aux = receiver_calls(ctx, ss, region, sky12["eph"], s0, batch_s0, TRACK_EPOCHS)
            for name in CALLS:
                want = calls[name](0, iq=region)
                assert_same(calls[name](start, **dev), want, (name, start))
                if name == "acquire_windows":
                    try:
                        for force in (1, 2):
                            assert ctx.debug_acq_split(aux["sky"].size, 5, force=force) == force
                            assert_same(calls[name](start, **dev), want, (name, start, "split", force))
                    finally:
                        ctx.debug_acq_split(1, 1, force=0)
                    assert ctx.debug_acq_split(aux["sky"].size, 5) > 1                 # the unforced split above
                if name == "snapshot_measure":
                    m = SM.measure(region, ss, s0, K, aux["sky"], min_ratio=2.5, iterations=gps.SNAP_ITERATIONS)
                    assert want[0].tobytes() == np.asarray(m).tobytes()
                if name == "track":
                    assert all(e.size == TRACK_EPOCHS for e in want[:-1])             # ended by max_epochs
                    if boundary is None:
                        assert start > 1 << 31                                        # states past sample 2^31
                    else:
                        assert all(e["sample"][-1] > boundary - start for e in want[:-1])   # tracked across it
                    eps, st = T.track(region, ss, 0, aux["states"], max_epochs=TRACK_EPOCHS)
                    for a, b in zip(want[:-1], eps):
                        assert np.array_equal(a, b)
                    assert np.array_equal(want[-1], st.astype(gps.TRACK_STATE_DTYPE))
                    shift = (1 << 32) + start                                         # base past 2^32
                    got = calls[name](shift, base=shift, device_ptr=buf.data_ptr() + start * elem, nsamples=REGION)
                    assert_same(got, want, (name, "advanced pointer, base", shift))
            prns3 = [int(p) for p in aux["sky"]["prn"][:3]]
            small = dict(sample_size=ss, prns=prns3, ms=K, f_lo=-2437.5, step=1625.0, nbins=4, want_grid=True)
            res, grid = ctx.acquire(s0=start + s0, **small, **dev)
            want = A.grid(region, ss, s0, K, prns3, -2437.5, 1625.0, 4)
            assert np.array_equal(grid, want)
            assert np.array_equal(res, A.reduce(want, prns3, -2437.5, 1625.0))
    finally:
        del buf
        release()


# ---- device sources behind work pending on the caller's stream --------------------------------------------------------
SLEEP_CYCLES = 400_000_000        # torch.cuda._sleep: about 0.2 s at the H100's clock, far longer than a call's set-up
SMALL_BLOCKS = 2                  # a call of at most 2 blocks returns with its synthesis still enqueued


@pytest.fixture(scope="module")
def pending(sky12):
    """A context, the 0.2 s source (sky12_static_35s blocks 0-1, int8) on the host, its six calls and their host
    results."""
    g = sky12["g"]
    rows = sky12["rows"][:SMALL_BLOCKS]
    iq = sky12["int8"][:SMALL_BLOCKS * gps.BLOCK_ELEMS].copy()
    s0 = gps.BLOCK_SAMPLES - 15000
    batch_s0 = np.arange(12, dtype=np.int64) * 45000 + 777
    with gps.Context(12, SMALL_BLOCKS, max_nav_frames=len(g["nav_frames"])) as ctx:
        ctx.set_nav_frames(g["nav_frames"])
        calls, _ = receiver_calls(ctx, gps.SC08, iq, sky12["eph"], s0, batch_s0, 150)
        want = {name: calls[name](0, iq=iq) for name in CALLS}
        yield ctx, rows, iq, calls, want


def noise_like(t, seed):
    out = torch.empty_like(t)
    out.random_(-128, 128, generator=torch.Generator(device="cuda").manual_seed(seed))
    return out


def on_stream(stream, iq, dev):
    return dict(device_ptr=dev.data_ptr(), nsamples=iq.size // 2, stream=stream.cuda_stream)


@pytest.mark.parametrize("name", CALLS)
def test_call_waits_for_a_copy_pending_on_the_callers_stream(pending, name):
    """The source holds noise (synchronised); the caller's stream then sleeps and copies the true source in. The call,
    issued on that stream while the copy is still pending, gives the true source's results."""
    ctx, _, iq, calls, want = pending
    true = torch.from_numpy(iq).cuda()
    dev = noise_like(true, 11)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    copied = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        dev.copy_(true)
        copied.record()
    assert not copied.query(), "the copy was done before the call was issued: raise SLEEP_CYCLES"
    got = calls[name](0, **on_stream(s, iq, dev))
    assert copied.query(), "the call returned its results before the caller's stream had copied the source"
    torch.cuda.synchronize()
    assert_same(got, want[name], name)


@pytest.mark.parametrize("name", CALLS)
def test_call_behind_a_synthesis_pending_on_the_callers_stream(pending, name):
    """The source holds noise (synchronised); the caller's stream sleeps, synth_blocks_device writes the true source on
    it (a 2-block call returns with its kernels enqueued) and the call follows on the same stream, nothing
    synchronised in between."""
    ctx, rows, iq, calls, want = pending
    dev = noise_like(torch.empty(iq.size, dtype=torch.int8, device="cuda"), 12)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    ctx.synth_blocks_device(rows, gps.SC08, dev.data_ptr(), stream=s.cuda_stream)
    written = torch.cuda.Event()
    written.record(s)
    assert not written.query(), "the synthesis was done before the call was issued: raise SLEEP_CYCLES"
    got = calls[name](0, **on_stream(s, iq, dev))
    torch.cuda.synchronize()
    assert_same(got, want[name], name)
    assert np.array_equal(dev.cpu().numpy(), iq)


@pytest.mark.parametrize("name", CALLS)
def test_every_kernel_of_the_call_runs_on_the_callers_stream(pending, name, tmp_path):
    """torch.profiler's trace of the call issued behind a short sleep on the caller's stream: every kernel the library
    launched ran on the stream the sleep ran on. A step enqueued on another stream after a host synchronisation gives
    the same results today (the calls above), but no longer orders behind the caller's work."""
    import json
    from torch.profiler import ProfilerActivity, profile
    ctx, _, iq, calls, want = pending
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(s):
            torch.cuda._sleep(1000)
        got = calls[name](0, **on_stream(s, iq, dev))
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        kernels = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ours = [e for e in kernels if "gpsb200" in e["name"]]
    sleep = [e for e in kernels if "gpsb200" not in e["name"]]
    assert len(sleep) == 1 and ours, [e["name"] for e in kernels]
    assert {e["args"]["stream"] for e in ours} == {sleep[0]["args"]["stream"]}, \
        sorted({(e["name"].split("(")[0], e["args"]["stream"]) for e in ours})
    assert_same(got, want[name], name)


@pytest.mark.parametrize("name", CALLS)
def test_a_kernel_after_the_call_on_its_stream_leaves_its_results(pending, name):
    """The call on a stream still sleeping, then a caller kernel on the same stream that overwrites the source: the
    call returned its results on the host, those of the untouched source."""
    ctx, _, iq, calls, want = pending
    dev = torch.from_numpy(iq).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    got = calls[name](0, **on_stream(s, iq, dev))
    with torch.cuda.stream(s):
        dev.random_(-128, 128, generator=torch.Generator(device="cuda").manual_seed(13))
    torch.cuda.synchronize()
    assert not np.array_equal(dev.cpu().numpy(), iq)
    assert_same(got, want[name], name)
