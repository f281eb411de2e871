"""CPU certification of the edge cases k_synth_lanes is tested at on the GPU (tests/test_lanes_edges_gpu.py): every hit
of repair_cases.EDGE_CASES, of the launch-shape cases and of the degenerate carrier steps reaches the exact walk (or the
exact chip-sign words) of the host model of the kernel, is decisive where the case claims it, and every block equals the
oracle. Without this, a GPU test that passes could pass because its hits missed the repair paths."""
import numpy as np
import pytest

import repair_cases as rc
import scenario
from scenario import gps


def _flag_bit(case, h):
    return h.slot if case.nchan > 16 else 16 * (h.win % 2) + h.slot


def _certify(case, blocks=None):
    ch, nav, decisive = rc.build(case)
    rows = rc.chained_rows(ch, [h.block for h in case.hits] + list(blocks or []))
    for h in case.hits:
        row = rows[h.block][[h.slot]]
        _, _, counters = gps.lanes_model_block(row, nav[0][[h.slot]])
        assert counters[2 if h.kind in ("code", "wrap") else 3] > 0, (case.name, h, counters)
        assert decisive[h.slot] == (h.slot not in case.plain), (case.name, h)
    return ch, nav, decisive, rows


@pytest.mark.parametrize("case", rc.EDGE_CASES, ids=lambda c: c.name)
def test_edge_cases_are_decisive_and_equal_the_oracle(case):
    ch, nav, decisive, _ = _certify(case)
    want, _ = scenario.oracle_run(ch, nav, 2)
    for b in range(case.nblk):
        iq, _, counters = gps.lanes_model_block(rc.chained_row(ch, b), nav[0])
        assert np.array_equal(iq, want[b * gps.BLOCK_ELEMS:(b + 1) * gps.BLOCK_ELEMS]), (case.name, b, counters)


def test_edge_cases_cover_every_flag_bit():
    """Decisive carrier hits behind all 32 bits of the flagged mask in both variants, all 32 bits in one ballot in
    both, code and wrap hits in the top slots and in the last real slot beside a padding slot."""
    cover = {16: set(), 32: set()}
    kinds = set()
    for case in rc.EDGE_CASES:
        v = 16 if case.nchan <= 16 else 32
        for h in case.hits:
            if h.kind in ("carr", "lat") and h.slot not in case.plain:
                cover[v].add(_flag_bit(case, h))
            if h.slot in (15, 31) or h.slot == case.nchan - 1:
                kinds.add((case.nchan, h.slot, h.kind))
    assert cover[16] == set(range(32)) and cover[32] == set(range(32)), cover
    for nchan, slot in ((16, 15), (15, 14), (32, 31), (31, 30)):
        assert {"code", "wrap"} <= {k for n, s, k in kinds if (n, s) == (nchan, slot)}, (nchan, slot, kinds)
    one = next(c for c in rc.EDGE_CASES if c.name == "v32_one_ballot")
    assert len({(h.block, h.run, h.win) for h in one.hits}) == 1 and len(one.hits) == 32


def test_lattice_lanes_have_three_decisive_samples_and_flag_every_trip():
    """The lattice-step slots: the hit's lane has its three samples (i, 32 + i, 64 + i) decisive in the hit window, and
    in the 16-channel case every window of run 0 is flagged in every slot, so that each ballot of the run has all 32
    bits set (the window certification against its own brute-force test: tests/test_window_band.py)."""
    for case in rc.EDGE_CASES:
        for h in case.hits:
            if h.kind != "lat":
                continue
            x0, dec = rc.place_lattice(h.f_carr, h.win * rc.WIN + h.n, h.target)
            lane = [h.win * rc.WIN + 32 * j + h.n for j in range(3)]           # the hit is the lane's first sample
            assert h.n < 32
            assert set(lane) <= set(dec), (case.name, h, lane)
    case = next(c for c in rc.EDGE_CASES if c.name == "v16_lattice_ballot")
    ch, _, _ = rc.build(case)
    for s in range(case.nchan):
        c = float(np.float64(ch["f_carr"][0, s]) * np.float64(rc.DELT))
        D = rc.carr_step_fix(c)
        P = [(rc.carr_fix(ch["carr_phase"][0, s]) + w * rc.WIN * D) % (1 << 64) for w in range(rc.RUN // rc.WIN)]
        bases = np.array([((p >> 32) - 1) % (1 << 32) for p in P], np.uint32)
        assert gps.lanes_window_band(np.uint32(D >> 32), bases).all(), s


# the H100 SXM's launch shapes (132 SMs): the smallest block count of each
H100_SHAPES = {(8, 16): 3, (4, 32): 1509, (3, 48): 3520, (2, 64): 5280, (1, 128): 10560}


def test_h100_shapes_and_their_runs():
    for (per_block, per_cta), nblk in H100_SHAPES.items():
        assert rc.lanes_shape(nblk) == (per_block, per_cta)
        if nblk > 3:
            assert rc.lanes_shape(nblk - 1) != (per_block, per_cta)
        runs = rc.shape_runs(per_block, per_cta)
        for g in range(per_block):
            lo, hi = g * per_cta, min((g + 1) * per_cta, 125)
            assert lo in runs and hi - 1 in runs
            assert hi - lo < 16 or any((r - lo) % 16 == 15 and lo <= r < hi for r in runs)
            if per_cta > 16:
                assert lo + 16 in runs


@pytest.mark.parametrize("nchan", [12, 32])
@pytest.mark.parametrize("shape", sorted(H100_SHAPES), ids=lambda s: "%dx%d" % s)
def test_shape_hits_are_decisive(shape, nchan):
    """The hits the GPU test places for each launch shape (at the H100 block counts): each reaches the exact walk of the
    model and is decisive."""
    case = rc.shape_case(nchan, H100_SHAPES[shape], shape[0], shape[1], seed=9300 + nchan)
    _certify(case)


@pytest.mark.parametrize("case", rc.DEGEN_CASES, ids=lambda c: c.name)
def test_degenerate_steps_are_repaired_and_equal_the_oracle(case):
    """Each slot's hit reaches the exact walk (counters[3] > 0) and is decisive where the case claims it; every block
    equals the oracle, final carrier phases included."""
    ch, nav, _, _ = _certify(case)
    want, carr = scenario.oracle_run(ch, nav, 2)
    for b in range(case.nblk):
        iq, carr_out, _ = gps.lanes_model_block(rc.chained_row(ch, b), nav[0])
        assert np.array_equal(iq, want[b * gps.BLOCK_ELEMS:(b + 1) * gps.BLOCK_ELEMS]), (case.name, b)
    assert np.array_equal(carr_out, carr)


def test_degenerate_steps_are_the_ones_named():
    """The Dopplers reach the 32-bit steps they stand for (fast_step), and c = +-2^-23 and its neighbours exactly."""
    for name, f in rc.DEGEN_STEPS:
        c = rc.step_of(f)
        if name.startswith("u="):
            assert (rc.carr_step_fix(c) >> 32) == int(name[2:], 16) and rc.carr_step_fix(c) % (1 << 32) == 0, name
        elif name.startswith("k="):
            # no double f gives k 2^-9 exactly: the nearest step is within one unit of the 32-bit step
            assert ((rc.carr_step_fix(c) >> 32) - (int(name[2:]) << 23) + 1) % (1 << 32) <= 2, name
            assert 2.85e6 < abs(f) < 2.9e6, name
        else:
            assert c == float(name[2:]), name
    assert len(rc.DEGEN_STEPS) == 151 and {c.nblk for c in rc.DEGEN_CASES} == {2, 3}
    # every step in the 32-channel variant, and those with a decisive hit in the 16-channel one as well
    for variant, steps in ((32, rc.DEGEN_STEPS), (16, rc._DECISIVE_STEPS)):
        for nblk in (2, 3):
            seen = [f for c in rc.DEGEN_CASES if (c.nchan > 16) == (variant == 32) and c.nblk == nblk for f in
                    (h.f_carr for h in c.hits)]
            assert seen == [f for _, f in steps], (variant, nblk)
    assert len(rc._DECISIVE_STEPS) == 12
