"""k_synth_lanes at the edges its repair paths and launch shapes have (hits certified on the CPU in
tests/test_lanes_edges.py): a decisive repair behind every channel slot and every bit of the flagged mask, all 32 bits in
one ballot, lanes with three risky samples, code and wrap hits in the top and padding-adjacent slots; every launch
shape the device gives, with hits at the edges of CTAs, warps and passes; degenerate and extreme carrier steps through
the small-call path and the speculative chain. Bit for bit against the oracle."""
import numpy as np
import pytest

import repair_cases as rc
import scenario
from scenario import gps

pytestmark = pytest.mark.gpu


def _first_diff(got, want):
    bad = np.nonzero(got != want)[0]
    return None if bad.size == 0 else (int(bad[0]) // gps.BLOCK_ELEMS, (int(bad[0]) % gps.BLOCK_ELEMS) // 2, bad.size)


@pytest.mark.parametrize("case", rc.EDGE_CASES, ids=lambda c: c.name)
def test_every_slot_and_flag_bit_equals_the_oracle(case):
    ch, nav, _ = rc.build(case)
    with gps.Context(case.nchan, case.nblk) as ctx:
        ctx.set_nav_frames(nav)
        assert ctx.synth_kernel_name(case.nchan) == "k_synth_lanes"
        for ss in (1, 2):
            want, carr = scenario.oracle_run(ch, nav, ss)
            out, cp = ctx.synth_blocks(ch, ss)
            assert np.array_equal(out, want), (case.name, ss, _first_diff(out, want))
            assert np.array_equal(cp, carr), (case.name, ss)


def _device_shapes(ctx, nchan, limit=40000):
    """{(CTAs per block, runs per CTA): smallest block count >= 3 of one launch with that shape} on this device."""
    shapes = {}
    for nblk in range(3, limit):
        name, per_block, per_cta = ctx.debug_synth_shape(nblk, nchan)
        assert name == "k_synth_lanes"
        shapes.setdefault((per_block, per_cta), nblk)
        if per_block == 1:
            break
    return shapes


def _chunked(ctx, ch, ss, dst, chunk=1024):
    """The call cut into device calls of <= chunk blocks, each continuing the previous one's carr_phase_out (a slot
    whose satellite changes at a cut keeps its own input phase)."""
    import torch
    cp = None
    blk = gps.BLOCK_ELEMS * ss
    for c0 in range(0, ch.shape[0], chunk):
        part = ch[c0:c0 + chunk].copy()
        if cp is not None:
            part["carr_phase"][0] = np.where(ch["prn"][c0] == ch["prn"][c0 - 1], cp, part["carr_phase"][0])
        assert ctx.debug_synth_shape(part.shape[0], ch.shape[1], ss)[2] == 16          # one run per warp
        cp = ctx.synth_blocks_device(part, ss, dst.data_ptr() + c0 * blk)
    torch.cuda.synchronize()
    return cp


def test_every_launch_shape_equals_the_oracle():
    """One eager device-destination call per launch shape the hook reports on this device (on an H100 SXM: 8, 4, 3,
    2 and 1 CTAs per block), at 32 and 12 channels, int8, and int16 at the first multi-pass shape: carrier hits in the
    first and the last run of every CTA, in warp 15's run, in the second and the last pass of a warp; hit blocks against
    the oracle from the exact chained phase, the whole output byte for byte against the same call cut into calls of at
    most 1024 blocks (one run per warp)."""
    import torch
    with gps.Context(32, 8) as probe:
        shapes = _device_shapes(probe, 32)
        assert _device_shapes(probe, 12) == shapes
    assert min(p for p, _ in shapes) == 1 and max(p for p, _ in shapes) == 8, shapes
    multi = min((n, s) for s, n in shapes.items() if s[1] > 16)[1]
    runs = [(s, n, nchan, 1) for s, n in sorted(shapes.items(), key=lambda t: t[1]) for nchan in (32, 12)]
    runs.append((multi, shapes[multi], 32, 2))
    print("launch shapes (CTAs per block, runs per CTA): smallest block count", shapes)
    for (per_block, per_cta), nblk, nchan, ss in runs:
        case = rc.shape_case(nchan, nblk, per_block, per_cta, seed=9300 + nchan)
        ch, nav, decisive = rc.build(case)
        assert all(decisive.values()), case.name
        dt = torch.int8 if ss == 1 else torch.int16
        with gps.Context(nchan, nblk) as ctx:
            ctx.set_nav_frames(nav)
            assert ctx.debug_synth_shape(nblk, nchan, ss) == ("k_synth_lanes", per_block, per_cta)
            dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=dt, device="cuda")
            cp, st = ctx.synth_blocks_device(ch, ss, dev.data_ptr(), want_stats=True)
            torch.cuda.synchronize()
            cut = torch.empty_like(dev)
            cp_cut = _chunked(ctx, ch, ss, cut)
            assert torch.equal(dev, cut), case.name
            del cut
            assert np.array_equal(cp, cp_cut), case.name
            rows = rc.chained_rows(ch, [h.block for h in case.hits])
            for b, row in rows.items():
                want, carr = scenario.oracle_run(row[None], nav, ss)
                got = dev[b * gps.BLOCK_ELEMS:(b + 1) * gps.BLOCK_ELEMS].cpu().numpy()
                assert np.array_equal(got, want), (case.name, b, _first_diff(got, want))
                if b == nblk - 1:
                    assert np.array_equal(cp, carr), case.name
            del dev
        torch.cuda.empty_cache()


@pytest.mark.parametrize("case", rc.DEGEN_CASES, ids=lambda c: c.name)
def test_degenerate_carrier_steps_equal_the_oracle(case):
    """The slots at degenerate and extreme carrier steps, through the small-call path (2 blocks) and the speculative
    chain (3 blocks), int8 and int16, output and final carrier phases against the oracle. The chain falls back to the
    host for every slot with |c| < 2^-23 (nco_exact.h's fast range) and the stats show it."""
    ch, nav, _ = rc.build(case)
    slow = sum(1 for h in case.hits if abs(rc.step_of(h.f_carr)) < 2.0 ** -23)
    with gps.Context(case.nchan, case.nblk) as ctx:
        ctx.set_nav_frames(nav)
        assert ctx.synth_kernel_name(case.nchan) == "k_synth_lanes"
        for ss in (1, 2):
            want, carr = scenario.oracle_run(ch, nav, ss)
            out, cp, st = ctx.synth_blocks(ch, ss, want_stats=True)
            assert np.array_equal(out, want), (case.name, ss, _first_diff(out, want))
            assert np.array_equal(cp, carr), (case.name, ss)
            if case.nblk >= 3:
                assert st.chain_fallbacks >= slow, (case.name, st.chain_fallbacks, slow)


def test_fast_range_edge_falls_back_below_it():
    """c = +-2^-23 and one ulp on either side, one slot each in a 3-block call: the chain falls back to the host for
    |c| < 2^-23, and the output and the final carrier phase equal the oracle either way. (At |c| = 2^-23 itself the
    chain falls back as well; what the kernels compute does not depend on it.)"""
    fallbacks = {}
    for c in rc.EDGE_C:
        f = rc.f_for_step(c)
        assert rc.step_of(f) == c
        case = rc.Case("edge", 1, 3, 9500, [rc.Hit("carr", 0, 2, 40, 7, 33, 256 if c > 0 else 0, f)])
        ch, nav, _ = rc.build(case)
        want, carr = scenario.oracle_run(ch, nav, 1)
        with gps.Context(1, 3) as ctx:
            ctx.set_nav_frames(nav)
            out, cp, st = ctx.synth_blocks(ch, 1, want_stats=True)
        assert np.array_equal(out, want) and np.array_equal(cp, carr), c
        fallbacks[c] = st.chain_fallbacks
    print("chain fallbacks at the edge of the fast range:", fallbacks)
    assert all(n > 0 for c, n in fallbacks.items() if abs(c) < 2.0 ** -23), fallbacks
