"""Run checkpoints walked in segments: the block probe records its trajectory at the start of every checkpoint segment,
and k_checkpoints starts each segment from that state plus the shift the fix-up found (nco_exact.h:
first_derived_segment). Exact or rejected, never approximate; the walked end of every segment is compared with the
start of the next one on the device."""
import numpy as np
import pytest

from scenario import gps

BLOCK = 300000


def _seg_start(j, nseg, nruns, run_samples):
    return (j * nruns // nseg) * run_samples


@pytest.mark.parametrize("run_samples", [150000, 60000, 2400])       # J = 2, 5, 8 segments
def test_derived_segment_starts_are_exact_or_rejected(run_samples):
    rng = np.random.default_rng(run_samples)
    nruns = BLOCK // run_samples
    nseg = min(8, nruns)
    cases = []
    for _ in range(300):
        f = rng.uniform(-400.0, 400.0) if rng.random() < 0.15 else rng.uniform(-6000.0, 6000.0)
        cases.append((rng.uniform(0.0, 1.0), f))
    # starts just below 1.0 (an immediate wrap for f > 0), and Dopplers so low that the first wrap comes after the start
    # of some segments, or never, of both signs
    below_one = np.nextafter(1.0, 0.0)
    for f in (5.0, -5.0, 30.0, -30.0, 45.0, -45.0, 90.0, -90.0, 3000.0, -3000.0):
        for s in (below_one, 1.0 - 1e-9, 0.05, 0.5, 0.95, 0.0):
            cases.append((s, f))
    accepted = derived = walked = 0
    for s, f in cases:
        err = rng.choice([0.0, 1e-15, 1e-12, 1e-10, 1e-8, 1e-6]) * rng.uniform(-1.0, 1.0)
        g = min(max(s + err, 0.0), below_one)
        ok, starts = gps.checkpoint_segments_host(s, g, f, run_samples)
        assert starts.size == nseg and starts[0] == s
        if not ok:
            assert np.isnan(starts[1:]).all()
            continue
        accepted += 1
        seen_derived = False
        for j in range(1, nseg):
            if np.isnan(starts[j]):
                assert not seen_derived, "only the segments before the first wrap are walked from the block start"
                walked += 1
                continue
            seen_derived = True
            derived += 1
            want = gps.carrier_advance(s, f, _seg_start(j, nseg, nruns, run_samples))
            assert starts[j] == want, (s, g, f, j)
    assert accepted > 0.5 * len(cases)
    assert derived > 0.4 * len(cases) * (nseg - 1)
    assert walked > 0                   # some low-Doppler blocks wrap for the first time after a segment start


def _sequential_checkpoints(ch, run_samples):
    """Carrier phase at every run start, walked sequentially on the host with the pipeline's chaining rule."""
    nblk, nchan = ch.shape
    nruns = BLOCK // run_samples
    x = np.zeros((nblk, nruns, nchan))
    for c in range(nchan):
        prn, ph = 0, 0.0
        for b in range(nblk):
            p, f = int(ch["prn"][b, c]), float(ch["f_carr"][b, c])
            if p <= 0:
                prn = 0
                continue
            if p != prn:
                ph = float(ch["carr_phase"][b, c])
                prn = p
            for r in range(nruns):
                x[b, r, c] = ph
                ph = gps.carrier_advance(ph, f, run_samples)
    return x


def _hard_chans(nblk=64, nchan=32, seed=5):
    ch, nav = gps.synthetic_chans(nblk, nchan, seed=seed)
    # low Dopplers: first wraps late in the block (after some segment starts) or not at all, both signs
    for c, f in zip((1, 2, 3, 4, 5, 6), (40.0, -60.0, 3.0, -2.0, 80.0, -25.0)):
        ch["f_carr"][:, c] = f
    ch["f_code"] = 1.023e6 + ch["f_carr"] / 1540.0
    ch["carr_phase"][0, 7] = np.nextafter(1.0, 0.0)      # an immediate wrap
    ch["carr_phase"][0, 8] = 0.0
    # a reallocation inside the call (the new satellite starts from its own carr_phase) ...
    ch["prn"][30:, 9] = 33 - ch["prn"][0, 9]
    ch["carr_phase"][30, 9] = 0.625
    # ... and idle blocks in two slots
    ch["prn"][10:13, 10] = 0
    ch["prn"][40:, 11] = 0
    ch["carr_phase"][10:, 11] = 0.25
    return ch, nav


@pytest.mark.gpu
def test_device_checkpoints_equal_the_sequential_walk():
    import torch
    ch, nav = _hard_chans()
    nblk, nchan = ch.shape
    want = _sequential_checkpoints(ch, 2400)
    with gps.Context(nchan, nblk) as ctx:
        ctx.set_nav_frames(nav)
        dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        # the device-destination path (one checkpoint launch over the call) ...
        ctx.synth_blocks_device(ch, 1, dev.data_ptr())
        torch.cuda.synchronize()
        got = ctx.debug_run_checkpoints(nblk, nchan)
        assert np.array_equal(got["x"], want)
        # ... the host-destination path (segmented pipeline) and the three-step slice call write the same ones
        out, _ = ctx.synth_blocks(ch, 1)
        assert np.array_equal(ctx.debug_run_checkpoints(nblk, nchan), got)
        ctx.slice_prepare(ch, 1, dev.data_ptr())
        ctx.slice_probe()
        ctx.slice_finish()
        ctx.slice_wait()
        assert np.array_equal(ctx.debug_run_checkpoints(nblk, nchan), got)
        assert np.array_equal(dev.cpu().numpy(), out)


@pytest.mark.gpu
def test_self_check_catches_a_corrupted_segment_state():
    # one recorded segment-start state of the probe, moved by one unit of the rounding grid (gpsb200_debug_corrupt_chain
    # mode 2), must be reported by every path: the walk of the segment before it ends elsewhere
    import torch
    ch, nav = gps.synthetic_chans(12, 32, seed=77)
    ch["f_carr"][:, 0] = 2500.0                         # slot 0: every segment of block 5 starts after the first wrap
    ch["f_code"] = 1.023e6 + ch["f_carr"] / 1540.0
    with gps.Context(32, 12) as ctx:
        ctx.set_nav_frames(nav)
        good, _ = ctx.synth_blocks(ch, 1)
        ctx.debug_corrupt_chain(2)
        with pytest.raises(gps.GpsB200Error) as e:
            ctx.synth_blocks(ch, 1)
        assert e.value.code == -5
        dev = torch.empty(12 * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        with pytest.raises(gps.GpsB200Error) as e:
            ctx.synth_blocks_device(ch, 1, dev.data_ptr())
        assert e.value.code == -5
        ctx.slice_prepare(ch, 1, dev.data_ptr())
        ctx.slice_probe()
        ctx.slice_finish()
        with pytest.raises(gps.GpsB200Error) as e:
            ctx.slice_wait()
        assert e.value.code == -5
        ctx.debug_corrupt_chain(0)
        again, _ = ctx.synth_blocks(ch, 1)
        assert np.array_equal(good, again)
