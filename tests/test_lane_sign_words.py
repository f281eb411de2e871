"""The sign words of the lane = sample synthesis (synth_lanes.h sign_pos / sample_words), checked sample by sample against
the reference's own code recurrence: word j of a 96-sample window holds, at bit 11 (i % 3) + i // 3, chip XOR data bit of
sample 32 j + i (gps.c:2789-2817: chip ca[(int) code_phase], the NAV bit of the current code period; a set flag is a
negative product dataBit * codeCA). All three builders of the words are covered: the 32-bit carry-point estimate, its FP64
second opinion (force 8) and the exact walk (force 2)."""
import numpy as np
import pytest

import repair_cases as rc
from scenario import gps

DELT = 1.0 / 3.0e6
WIN = 96
NWIN = gps.BLOCK_SAMPLES // WIN
POS = np.array([11 * (i % 3) + i // 3 for i in range(32)], np.uint32)


def _nav_bit(nav_row, iw, ib):
    return (int(nav_row[min(iw, 59)]) >> (29 - ib)) & 1


def ref_flags(row, nav_row, first, count):
    """Sign flags of samples first .. first + count - 1 of the block, by the reference's recurrence from the block start."""
    ca = gps.codegen(int(row["prn"]))
    d = float(np.float64(row["f_code"]) * np.float64(DELT))
    y = float(row["code_phase"])
    iw, ib, ic = int(row["iword"]), int(row["ibit"]), int(row["icode"])
    dbit = _nav_bit(nav_row, iw, ib)
    out = np.zeros(count, np.uint8)
    for n in range(first + count):
        if n >= first:
            out[n - first] = ca[int(y)] ^ dbit
        y += d
        if y >= 1023.0:
            y -= 1023.0
            ic += 1
            if ic >= 20:
                ic = 0
                ib += 1
                if ib >= 30:
                    ib = 0
                    iw += 1
                dbit = _nav_bit(nav_row, iw, ib)
    return out


def model_flags(words):
    """uint32[..., 3] sign words of windows -> uint8[..., 96] flags in sample order."""
    return ((words[..., :, None] >> POS) & 1).astype(np.uint8).reshape(words.shape[:-1] + (WIN,))


def model_words(row_chans, nav_rows, force=0):
    _, _, counters, signs = gps.lanes_model_block(row_chans, nav_rows, force=force, want_signs=True)
    return signs, counters


def test_sign_words_layout_is_samples_in_order_of_lane():
    """Bit positions: one per lane, a permutation of 0..31, three fields of 11, 11 and 10 bits."""
    assert sorted(POS.tolist()) == list(range(32))
    assert [int(POS[i]) for i in (0, 1, 2, 3, 30, 31)] == [0, 11, 22, 1, 10, 21]


@pytest.mark.parametrize("force", [0, 8, 2])
def test_sign_words_of_random_windows(force):
    """Every window of one block of random channels (Doppler, code phase, NAV position), every builder."""
    ch, nav = gps.synthetic_chans(1, 6, seed=2024 + force)
    signs, counters = model_words(ch[0], nav[0], force)
    for c in range(6):
        want = ref_flags(ch[0][c], nav[0][c], 0, gps.BLOCK_SAMPLES)
        got = model_flags(signs[c]).reshape(-1)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (force, c, bad[:8] // WIN, bad[:8] % WIN)
    if force == 2:
        assert counters[2] == 6 * NWIN
    elif force == 0:
        assert counters[2] < 6 * NWIN // 100                   # nearly every window from the 32-bit estimate


def _window0_case(targets, frac, seed, wrap=False, nav_change=False):
    """One channel per target sample n: its code phase puts sample n of window 0 `frac` chips past a chip boundary
    (wrap: past the 1022 -> 0 wrap; nav_change: in the 20th code period of a NAV bit whose successor differs)."""
    ch, nav = gps.synthetic_chans(1, len(targets), seed=seed)
    nav = nav.copy()
    rng = np.random.default_rng(seed)
    for s, n in enumerate(targets):
        d = float(np.float64(ch["f_code"][0, s]) * np.float64(DELT))
        J = 1023 if wrap else int(rng.integers(40, 980))
        ch["code_phase"][0, s] = (J + frac - n * d) % 1023.0
        if nav_change:
            ch["icode"][0, s] = 19
            iw, ib = int(ch["iword"][0, s]), int(ch["ibit"][0, s])
            nw, nb = (iw, ib + 1) if ib < 29 else (iw + 1, 0)
            w = int(nav[0, s, nw]) & ~(1 << (29 - nb))
            nav[0, s, nw] = w | ((1 - _nav_bit(nav[0, s], iw, ib)) << (29 - nb))
    return ch, nav


def _check_window0(ch, nav, force=0):
    signs, _ = model_words(ch[0], nav[0], force)
    for s in range(ch.shape[1]):
        want = ref_flags(ch[0][s], nav[0][s], 0, WIN)
        got = model_flags(signs[s, 0])
        assert np.array_equal(got, want), (s, np.flatnonzero(got != want))


@pytest.mark.parametrize("frac", [0.004, 0.012])
def test_sign_words_carry_point_at_every_class_position(frac):
    """A sample just past a chip boundary is where its residue class takes its extra chip (the carry point): placed at
    every sample of the window, i.e. at every position q of every class r."""
    for part in range(3):
        targets = list(range(32 * part, 32 * part + 32))
        _check_window0(*_window0_case(targets, frac, seed=700 + part))


def test_sign_words_code_wrap_and_nav_bit_change_inside_the_window():
    """The 1022 -> 0 wrap inside the window, with and without a NAV bit change at that code period, at spread positions;
    every builder."""
    targets = list(range(1, 96, 4))
    for nav_change in (False, True):
        ch, nav = _window0_case(targets, 0.01, seed=810 + nav_change, wrap=True, nav_change=nav_change)
        for force in (0, 8, 2):
            _check_window0(ch, nav, force)


def test_sign_words_engineered_chip_boundary_hits():
    """The code and wrap hits of tests/repair_cases.py (linear code phase on a chip boundary to within the band, in
    later runs and blocks): the hit window's words, rebuilt exactly, against the reference."""
    for case in rc.CASES:
        ch, nav, _ = rc.build(case)
        for h in case.hits:
            if h.kind == "carr":
                continue
            row = ch[h.block][[h.slot]]
            signs, counters = model_words(row, nav[0][[h.slot]])
            assert counters[2] > 0, (case.name, h)
            first = h.run * rc.RUN + h.win * WIN
            want = ref_flags(row[0], nav[0][h.slot], first, WIN)
            got = model_flags(signs[0, first // WIN])
            assert np.array_equal(got, want), (case.name, h, np.flatnonzero(got != want))
