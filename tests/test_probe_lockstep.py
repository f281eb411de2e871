"""The carrier block probe walks both parity variants in one thread, in lockstep (nco_exact.h: carrier_probe_walk2).
Every record it writes -- first wrap, end states, margins, checkpoint-segment states -- must be bit-identical to the
per-variant walk (carrier_probe_walk), on the host over engineered edge cases and on the device for every (block,
channel) of full-size calls."""
import os
import subprocess
import sys

import numpy as np
import pytest

import scenario
from scenario import gps

BLOCK = 300000
DELT = 1.0 / 3e6
RUN_LENGTHS = [32, 96, 160, 480, 800, 2400, 4000, 12000, 20000, 60000, 100000, 300000]   # every one gpsb200_create accepts
BELOW_ONE = np.nextafter(1.0, 0.0)


def _both(guess, f, run_samples, nsamples=BLOCK):
    p0, s0 = gps.carrier_probe_host(guess, f, nsamples, run_samples, mode=0)
    p1, s1 = gps.carrier_probe_host(guess, f, nsamples, run_samples, mode=1)
    assert p1.tobytes() == p0.tobytes(), (guess, f, run_samples, p0, p1)
    assert s1.tobytes() == s0.tobytes(), (guess, f, run_samples, s0, s1)
    return p0, s0


def _incr(f):
    return float(np.float64(f) * np.float64(DELT))


def _doppler_for(c):
    """A Doppler whose increment fl(f * delt) is exactly c, or None."""
    f = c / DELT
    for k in range(-8, 9):
        g = float(np.float64(f) + k * np.spacing(np.float64(f)))
        if _incr(g) == c:
            return g
    return None


def test_lockstep_probe_equals_per_variant_probe_random():
    rng = np.random.default_rng(11)
    nwrap = 0
    for i in range(2400):
        f = rng.uniform(10.0, 6000.0) * rng.choice([-1.0, 1.0])
        p, _ = _both(rng.uniform(0.0, 1.0), f, RUN_LENGTHS[i % len(RUN_LENGTHS)])
        nwrap += p["n_w"] >= 0
    assert nwrap > 2300


def test_lockstep_probe_without_segments_and_short_walks():
    # the host models walk without segment states; walks shorter than a block
    rng = np.random.default_rng(12)
    for _ in range(300):
        f = rng.uniform(10.0, 6000.0) * rng.choice([-1.0, 1.0])
        n = int(rng.choice([1, 2, 3, 100, 2400, 12345, 299999]))
        _both(rng.uniform(0.0, 1.0), f, 0, nsamples=n)


def test_lockstep_probe_at_the_edge_of_the_fast_range():
    # |c| just above and below 2^-23 (below: no fast walk, the probe reports no wrap), both signs, guesses that wrap
    # early, late and not at all
    base = _doppler_for(2.0 ** -23)
    assert base is not None
    fs = []
    for k in range(-6, 7):
        f = base + k * np.spacing(base)
        fs += [f, -f]
    seen = {"fast": 0, "slow": 0}
    for f in fs:
        c = _incr(f)
        for g in (0.0, 0.5, 1.0 - 200000 * abs(c), 1.0 - 10 * abs(c), BELOW_ONE, 100 * abs(c), 10 * abs(c), 2.0 ** -60):
            for run in (0, 2400, 60000):
                p, _ = _both(g, f, run)
                seen["fast" if abs(c) >= 2.0 ** -23 else "slow"] += 1
                if abs(c) < 2.0 ** -23:
                    assert p["n_w"] == -1
    assert seen["fast"] > 0 and seen["slow"] > 0


def test_lockstep_probe_with_tie_increments():
    # c's lowest set bit half a unit of some binade's grid: round-half-even ties in the walk, where the two variants'
    # mantissa parities matter (per-variant `special`)
    rng = np.random.default_rng(13)
    done = 0
    while done < 400:
        low = int(rng.integers(54, 62))                       # ties in binade [2^(53 - low), 2^(54 - low))
        target = rng.uniform(3e-6, 2e-3)
        m = int(target * 2.0 ** low) | 1
        c = m * 2.0 ** -low * rng.choice([-1.0, 1.0])
        f = _doppler_for(c)
        if f is None:
            continue
        _both(rng.uniform(0.0, 1.0), f, RUN_LENGTHS[done % len(RUN_LENGTHS)])
        done += 1


def test_lockstep_probe_with_an_unusable_partner():
    # c < 0, first wrap onto 1 - 2^-53: x_w + G == 1.0, variant 1 is not walked (margins 0, no segment states)
    rng = np.random.default_rng(14)
    dead = 0
    for _ in range(200):
        f = -rng.uniform(10.0, 6000.0)
        c = _incr(f)
        for g in (-c - 2.0 ** -53, -c - 2.0 ** -55, -c - 2.0 ** -54):
            p, s = _both(g, f, RUN_LENGTHS[dead % len(RUN_LENGTHS)])
            if p["x_end"][1] >= 1.0:
                dead += 1
                assert p["m_pos"][1] == 0.0 and p["m_neg"][1] == 0.0 and np.isnan(s[1]).all()
    assert dead >= 200


def test_lockstep_probe_with_variants_straddling_a_binade_edge():
    # c > 0, first wrap onto 2^e - 2^-52 (and onto exactly 0): x_w and x_w + G in different binades at the start
    rng = np.random.default_rng(15)
    straddle = 0
    for i in range(400):
        f = rng.uniform(10.0, 6000.0)
        c = _incr(f)
        e = int(rng.integers(-45, int(np.floor(np.log2(c))) + 1))
        target = 2.0 ** e - 2.0 ** -52 if i % 8 else 0.0
        g = (1.0 + target) - c
        if not g < 1.0:
            continue
        p, _ = _both(g, f, RUN_LENGTHS[i % len(RUN_LENGTHS)])
        x0, x1 = p["x_w"], p["x_w"] + 2.0 ** -52
        if p["n_w"] >= 0 and (x0 == 0.0 or np.frexp(x0)[1] != np.frexp(x1)[1]):
            straddle += 1
    assert straddle > 300


def test_lockstep_probe_without_a_wrap_and_with_late_wraps():
    # low Dopplers: no wrap in the block, or a first wrap after some segment starts (those are not recorded)
    rng = np.random.default_rng(16)
    nowrap = late = 0
    for i in range(600):
        f = rng.uniform(0.36, 12.0) * rng.choice([-1.0, 1.0])
        run = RUN_LENGTHS[i % len(RUN_LENGTHS)]
        p, s = _both(rng.uniform(0.0, 1.0), f, run)
        if p["n_w"] < 0:
            nowrap += 1
        elif run < BLOCK and np.isnan(s[0, 0]) and not np.isnan(s[0]).all():
            late += 1
    assert nowrap > 100 and late > 20


def test_host_hook_validates_its_arguments():
    with pytest.raises(gps.GpsB200Error):
        gps.carrier_probe_host(0.5, 1000.0, BLOCK, 2400, mode=2)
    with pytest.raises(gps.GpsB200Error):
        gps.carrier_probe_host(0.5, 1000.0, BLOCK, 7000)
    with pytest.raises(gps.GpsB200Error):
        gps.carrier_probe_host(0.5, 1000.0, 2 ** 31, 0)


def _check_device_probes(ctx, ch):
    """Every (block, channel) probe of the context's previous call against the per-variant host walk."""
    nblk, nchan = ch.shape
    probes, seg, guess = ctx.debug_block_probes(nblk, nchan)
    run = ctx.cfg.run_samples or 2400
    n = 0
    for b in range(nblk):
        for c in range(nchan):
            if ch["prn"][b, c] <= 0:
                continue
            want, ws = gps.carrier_probe_host(guess[b, c], ch["f_carr"][b, c], BLOCK, run, mode=0)
            assert probes[b, c].tobytes() == want.tobytes(), (b, c, probes[b, c], want)
            rec = ~np.isnan(ws)
            assert seg[b, c][rec].tobytes() == ws[rec].tobytes(), (b, c)
            n += 1
    return n


@pytest.mark.gpu
def test_device_probes_equal_the_per_variant_walk_32ch():
    import torch
    nblk, nchan = 3000, 32
    ch, nav = gps.synthetic_chans(nblk, nchan, seed=2024)
    with gps.Context(nchan, nblk) as ctx:
        ctx.set_nav_frames(nav)
        dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        ctx.synth_blocks_device(ch, 1, dev.data_ptr())
        torch.cuda.synchronize()
        assert _check_device_probes(ctx, ch) == int((ch["prn"] > 0).sum())


@pytest.mark.gpu
def test_device_probes_equal_the_per_variant_walk_reallocation_310s(tmp_path):
    # the scenario of the sky32_lat60_310s_i8 fixture: a satellite rises into a free slot at 240 s, another sets at 300 s
    nav_file = tmp_path / "sky32.nav"
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat", "32",
                           "--out", str(nav_file)])
    ch, nav = gps.scenario(str(nav_file), 60.0, 140.0, 0.0, seconds=310, max_chan=32, start=(2024, 1, 7, 2, 0, 0.0))
    assert ch.shape[0] == 3099
    with gps.Context(32, ch.shape[0], max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        ctx.synth_blocks(ch, 1)
        assert _check_device_probes(ctx, ch) == int((ch["prn"] > 0).sum())
