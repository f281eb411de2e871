"""GPU tests of the synthesis kernels where they are easiest to get wrong: the exact repair paths of k_synth_lanes hit on
purpose, sums at the full int16 scale the API admits, and device destinations the kernels cannot store to."""
import numpy as np
import pytest

import repair_cases as rc
import scenario
from scenario import gps

pytestmark = pytest.mark.gpu

KERNELS = (("1", "k_synth_lanes"), ("0", "k_synth"))


def _first_diff(got, want):
    bad = np.nonzero(got != want)[0]
    return None if bad.size == 0 else (int(bad[0]) // gps.BLOCK_ELEMS, (int(bad[0]) % gps.BLOCK_ELEMS) // 2, bad.size)


@pytest.mark.parametrize("case", rc.CASES, ids=lambda c: c.name)
def test_engineered_repair_hits_equal_the_oracle(case, monkeypatch):
    """Every hit of repair_cases.CASES (certified on the CPU to reach the exact walk or the exact chip-sign words):
    k_synth_lanes -- warp vote, shuffle of the window state from the half-warp that prepared it, swizzled table patch,
    exact_signs on the channel side, exact_index from the run anchors of k_checkpoints -- and k_synth, int8 and int16,
    one- and four-block calls, bit for bit against the oracle, final carrier phases included."""
    ch, nav, _ = rc.build(case)
    for ss in (1, 2):
        want, carr = scenario.oracle_run(ch, nav, ss)
        for lanes, name in KERNELS:
            monkeypatch.setenv("GPSB200_LANES", lanes)
            with gps.Context(case.nchan, case.nblk) as ctx:
                ctx.set_nav_frames(nav)
                out, cp = ctx.synth_blocks(ch, ss)
                assert ctx.synth_kernel_name(case.nchan) == name
            assert np.array_equal(out, want), (name, ss, _first_diff(out, want))
            assert np.array_equal(cp, carr), (name, ss)


def _api_amplitude(gains):
    amp = 0.0
    for g in gains:                                  # the sum gpsb200 checks, in its order, in double
        amp += abs(float(g)) * 250.0
    return amp


def _coherent_chans(nchan, nblk=3):
    """nchan slots on ONE satellite with identical code phase, carrier phase and Doppler: the table peaks of all slots
    line up. Equal gains with the API's amplitude sum as close to 32767 as it admits."""
    ch = np.zeros((nblk, nchan), gps.CHAN_DTYPE)
    f = 1234.5
    ch["prn"] = 7
    ch["iword"], ch["ibit"], ch["icode"] = 3, 5, 7
    ch["f_carr"] = f
    ch["f_code"] = 1.023e6 + f / 1540.0
    ch["carr_phase"][0] = 0.125
    ch["code_phase"] = 100.5
    g = 32767.0 / (250.0 * nchan)
    while _api_amplitude([g] * nchan) > 32767.0:
        g = np.nextafter(g, 0.0)
    ch["gain"] = g
    row = np.random.default_rng(5150).integers(0, 1 << 30, size=60, dtype=np.uint32)
    nav = np.broadcast_to(row, (1, nchan, 60)).copy()
    return ch, nav


@pytest.mark.parametrize("nchan", [12, 32])
def test_full_scale_coherent_sums_at_the_range_limit(nchan, monkeypatch):
    """Both kernels sum packed I + (Q << 16) words and unpack them; that is exact only while |I|, |Q| <= 32767, which
    the API guarantees by refusing sum(|gain|) * 250 > 32767 (GPSB200_ERR_RANGE). At the largest admitted gains the
    sums reach beyond +-32000 (int8: >> 4 then wraps modulo 256) and must still be exact; one gain raised by the least
    amount that crosses the limit is refused, and the context stays exact afterwards."""
    ch, nav = _coherent_chans(nchan)
    assert _api_amplitude(ch["gain"][0]) <= 32767.0
    over = ch.copy()
    g0 = float(over["gain"][0, 0])
    while _api_amplitude([g0] + list(ch["gain"][0, 1:])) <= 32767.0:
        g0 = np.nextafter(g0, np.inf)
    over["gain"][:, 0] = g0
    wants = {ss: scenario.oracle_run(ch, nav, ss) for ss in (1, 2)}
    iq = wants[2][0].astype(np.int32)
    for part in (iq[0::2], iq[1::2]):                 # I and Q both reach the full scale, with either sign
        assert part.max() >= 32000 and part.min() <= -32000, (part.min(), part.max())
    for lanes, name in KERNELS:
        monkeypatch.setenv("GPSB200_LANES", lanes)
        with gps.Context(nchan, ch.shape[0]) as ctx:
            ctx.set_nav_frames(nav)
            assert ctx.synth_kernel_name(nchan) == name
            for ss in (1, 2):
                want, carr = wants[ss]
                out, cp = ctx.synth_blocks(ch, ss)
                assert np.array_equal(out, want), (name, ss, _first_diff(out, want))
                assert np.array_equal(cp, carr)
                with pytest.raises(gps.GpsB200Error) as e:
                    ctx.synth_blocks(over, ss)
                assert e.value.code == -3
                out, cp = ctx.synth_blocks(ch, ss)
                assert np.array_equal(out, want), (name, ss, "after the refused call")


def test_misaligned_device_destinations_are_refused():
    """k_synth and k_synth_lanes store 2- to 16-byte words: every entry point with a device destination refuses one
    that is not 16-byte aligned (GPSB200_ERR_ARG, before anything is enqueued: the buffer stays untouched) and accepts
    any 16-byte aligned one; the context stays usable."""
    import torch
    nblk, guard = 3, 64
    ch, nav = scenario.synthetic_chans(nblk, 12, seed=1616)
    for ss in (1, 2):
        nbytes = nblk * gps.BLOCK_ELEMS * ss
        with gps.Context(12, nblk) as ctx:
            ctx.set_nav_frames(nav)
            ref = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
            cp_ref = ctx.synth_blocks_device(ch, ss, ref.data_ptr())   # 3 blocks: also what replay_device re-runs
            torch.cuda.synchronize()
            buf = torch.full((nbytes + 2 * guard,), 0xA5, dtype=torch.uint8, device="cuda")
            base = buf.data_ptr() + guard
            assert base % 256 == guard
            for off in (1, 2, 4, 8):
                p = base + off
                calls = (("gpsb200_synth_blocks_device", lambda: ctx.synth_blocks_device(ch, ss, p)),
                         ("gpsb200_slice_prepare", lambda: ctx.slice_prepare(ch, ss, p)),
                         ("gpsb200_replay_device", lambda: ctx.replay_device(p)))
                for fn, call in calls:
                    with pytest.raises(gps.GpsB200Error) as e:
                        call()
                    assert e.value.code == -1 and fn in str(e.value) and "aligned" in str(e.value), (off, str(e.value))
            torch.cuda.synchronize()
            assert bool((buf == 0xA5).all()), "a refused call wrote into the buffer"
            p = base + 16
            region = buf[guard + 16:guard + 16 + nbytes]
            cp = ctx.synth_blocks_device(ch, ss, p)
            torch.cuda.synchronize()
            assert torch.equal(region, ref) and np.array_equal(cp, cp_ref)
            region.zero_()
            ctx.replay_device(p)
            torch.cuda.synchronize()
            assert torch.equal(region, ref)
            region.zero_()
            ctx.slice_prepare(ch, ss, p)
            ctx.slice_probe()
            ctx.slice_finish()
            ctx.slice_wait()
            torch.cuda.synchronize()
            assert torch.equal(region, ref)
            assert bool((buf[:guard + 16] == 0xA5).all()) and bool((buf[guard + 16 + nbytes:] == 0xA5).all())
            host, cp_host = ctx.synth_blocks(ch, ss)
            assert np.array_equal(host.view(np.uint8), ref.cpu().numpy()) and np.array_equal(cp_host, cp_ref)
