"""Engineered repair hits of the lane = sample synthesis (synth_lanes.h, k_synth_lanes).

The kernel takes a sample's carrier-table index and chip from LINEAR fixed-point phases counted from the exact run
anchor (k_checkpoints), and sends the sample to the exact FP64 walk only when that linear phase lies inside a band
around a boundary: 2^-41 cycles around a table-index boundary (exact_index) or 2^-32 chips around a chip boundary
(window_signs -> exact_signs). Random parameters land there rarely. The helpers below choose a slot's input phase so
that one chosen sample -- (block, run, window, sample in window) -- has its linear phase on a chosen boundary:

  carrier  the anchor of run r of block b is the exact chain of the input phase over b * 300000 + r * 2400 samples
           (gps.carrier_advance); the input phase is corrected until the linear phase from that anchor lands on the
           target, to 2^-48 cycles
  code     the anchor is the reference's own code recurrence (y += d; if y >= 1023: y -= 1023, IEEE double as
           gps.c:2789-2791) from the block's code phase over r * 2400 samples

A hit is DECISIVE when the reference's FP64 phase and the linear phase fall on opposite sides of the boundary, so that
skipping the repair would change the output: the target is then moved by half their difference. Which side each
phase is on is computed exactly (fixed-point linear phase as synth_lanes.h keeps it; exact walk for the FP64 phase)."""
import collections
from fractions import Fraction

import numpy as np

from scenario import gps

DELT = 1.0 / 3.0e6                 # gps.c:2298
BLOCK = gps.BLOCK_SAMPLES
RUN = 2400                         # default run length: the one k_synth_lanes' bands are sized for
WIN = 96                           # samples per window (synth_lanes.h kWindow)
BAND_CARR = 1 << 23                # 2^-41 cycles in units of 2^-64
BAND_CODE = 1 << 22                # 2^-32 chips in units of 2^-54

# kind: "carr" (table-index boundary `target`), "code" (chip boundary near `target`), "wrap" (1022 -> 0 with icode == 19
# and a NAV bit change at that code period); slot, block, run, window, n = sample in the window (lane n // 3, residue n % 3)
Hit = collections.namedtuple("Hit", "kind slot block run win n target f_carr", defaults=(None, None))
Case = collections.namedtuple("Case", "name nchan nblk seed hits")


def carr_fix(x):
    return int(Fraction(x) * (1 << 64))                                  # synth_lanes.h carr_fix (x in [0,1))


def carr_step_fix(c):
    m = int(abs(Fraction(c)) * (1 << 64))
    return (-m) % (1 << 64) if c < 0 else m


def carr_index_exact(x):
    return min(int(Fraction(x) * 512), 511)


def code_walk(y, d, n):
    """The reference's code NCO, n steps (gps.c:2789-2791). -> (phase, code periods completed)"""
    periods = 0
    for _ in range(n):
        y += d
        if y >= 1023.0:
            y -= 1023.0
            periods += 1
    return y, periods


def _centered(v, mod):
    v = v % mod
    return v - mod if v > mod / 2 else v


def _below(v, mod):
    """Largest double below mod that is >= the rational v reduced modulo mod."""
    x = float(v % mod)
    return x if x < mod else float(np.nextafter(mod, 0.0))


def place_carrier(f_carr, T, m, k):
    """Input carrier phase so that the linear phase m samples after the exact anchor T samples on sits on index
    boundary k (or, when the FP64 phase there differs, half their difference off it, on the other side).
    -> (input phase, anchor, decisive)"""
    c = float(np.float64(f_carr) * np.float64(DELT))
    target = Fraction(k, 512)

    def solve(tgt):
        x = _below(tgt - (T + m) * Fraction(c), 1)
        for _ in range(12):
            xr = gps.carrier_advance(x, f_carr, T) if T else x
            err = _centered(Fraction(xr) + m * Fraction(c) - tgt, 1)
            if abs(err) <= Fraction(1, 1 << 48):
                break
            x = _below(Fraction(x) - err, 1)
        return x, xr

    x, xr = solve(target)
    delta = _centered(Fraction(gps.carrier_advance(xr, f_carr, m)) - (Fraction(xr) + m * Fraction(c)), 1)
    if delta != 0:
        x, xr = solve(target - delta / 2)
    lin = (carr_fix(xr) + m * carr_step_fix(c)) % (1 << 64)
    frac = lin & ((1 << 55) - 1)
    assert frac < BAND_CARR or frac > (1 << 55) - BAND_CARR, (f_carr, T, m, k)
    decisive = (lin >> 55) != carr_index_exact(gps.carrier_advance(xr, f_carr, m))
    return x, xr, bool(decisive)


def place_code(d, T, m, J, flags_differ):
    """Block code phase so that the linear code phase m samples after the exact anchor T samples on sits on chip
    boundary J (1023: the wrap), moved off it by half the FP64 difference. flags_differ(chip_lin, chip_exact, wrapped)
    tells whether the two chips give different sign flags. -> (block code phase, decisive)"""
    target = Fraction(J)

    def solve(tgt):
        y = _below(tgt - (T + m) * Fraction(d), 1023)
        for _ in range(12):
            yr = code_walk(y, d, T)[0]
            err = _centered(Fraction(yr) + m * Fraction(d) - tgt, 1023)
            if abs(err) <= Fraction(1, 1 << 40):
                break
            y = _below(Fraction(y) - err, 1023)
        return y, yr

    y, yr = solve(target)
    delta = _centered(Fraction(code_walk(yr, d, m)[0]) - (Fraction(yr) + m * Fraction(d)), 1023)
    if delta != 0:
        y, yr = solve(target - delta / 2)
    one = 1 << 54
    lin = int(Fraction(yr) * one) + m * int(Fraction(d) * one)
    lin_wrapped = lin >= 1023 * one
    lin %= 1023 * one
    frac = lin & (one - 1)
    assert frac < BAND_CODE or frac > one - BAND_CODE, (d, T, m, J)
    ye, periods = code_walk(yr, d, m)
    decisive = flags_differ(lin >> 54, int(ye), (lin_wrapped, periods > 0))
    return y, bool(decisive)


def _nav_bit(nav_row, iw, ib):
    return (int(nav_row[min(iw, 59)]) >> (29 - ib)) & 1


def _set_nav_bit(nav_row, iw, ib, v):
    w = int(nav_row[iw]) & ~(1 << (29 - ib))
    nav_row[iw] = w | (v << (29 - ib))


def build(case):
    """-> (chans[nblk, nchan], nav[1, nchan, 60], {slot: decisive}). Hit slots get gain 1 (adjacent table entries then
    always differ) and, for carrier hits, a constant Doppler over the call."""
    ch, nav = gps.synthetic_chans(case.nblk, case.nchan, seed=case.seed)
    nav = nav.copy()
    decisive = {}
    for h in case.hits:
        s, T, m = h.slot, h.run * RUN, h.win * WIN + h.n
        assert 0 <= h.n < WIN and 0 <= h.win < RUN // WIN and 0 <= h.run < BLOCK // RUN and h.block < case.nblk
        ch["gain"][:, s] = 1.0
        if h.kind == "carr":
            ch["f_carr"][:, s] = h.f_carr
            ch["f_code"][:, s] = 1.023e6 + h.f_carr / 1540.0
            x, _, decisive[s] = place_carrier(h.f_carr, h.block * BLOCK + T, m, h.target)
            ch["carr_phase"][0, s] = x
            continue
        b = h.block
        d = float(np.float64(ch["f_code"][b, s]) * np.float64(DELT))
        if h.kind == "code":
            ca = gps.codegen(int(ch["prn"][b, s]))
            J = h.target
            while ca[J - 1] == ca[J]:                                    # a chip boundary where the chip changes
                J += 1
            y, decisive[s] = place_code(d, T, m, J, lambda jl, je, w: ca[jl] != ca[je])
        else:
            # the code period that ends at the hit is the 20th of its NAV bit, and the next bit differs; the chips
            # 1022 and 0 are equal, so the sign flag of the hit sample is decided by the side of the wrap alone
            assert h.run == 0 and m * 0.342 < 1000.0
            used = set(int(p) for p in ch["prn"][b])
            prn = next(p for p in range(1, 33) if p not in used and gps.codegen(p)[1022] == gps.codegen(p)[0])
            ch["prn"][:, s] = prn
            ch["icode"][b, s] = 19
            iw, ib = int(ch["iword"][b, s]), int(ch["ibit"][b, s])
            nw, nb = (iw, ib + 1) if ib < 29 else (iw + 1, 0)
            assert nw < 60
            old = _nav_bit(nav[0, s], iw, ib)
            _set_nav_bit(nav[0, s], nw, nb, 1 - old)
            y, decisive[s] = place_code(d, 0, m, 1023, lambda jl, je, w: w[0] != w[1])
        ch["code_phase"][b, s] = y
    return ch, nav, decisive


def chained_row(ch, b):
    """Block b of a call with the carrier phases the call chains into it (exact sequential chain)."""
    row = ch[b].copy()
    if b > 0:
        row["carr_phase"] = gps.carrier_chain(ch[:b], threads=4)
    return row


# The placements: every kind of hit in both variants of k_synth_lanes (12 channels: 16-channel variant, whose half-warps
# prepare an even and an odd window per trip; 24 channels: 32-channel variant), at lanes 0 and 31 with every residue,
# in the last window of a run (window 24: the last trip of the 16-channel variant holds one window), in run 0, later
# runs and the last run of a block, in later blocks of a 4-block call (speculative chain path), positive and negative
# Doppler, on the index boundaries 0 (the wrap) and 511.
CASES = [
    Case("v16_one_block", 12, 1, 9101, [
        Hit("carr", 0, 0, 0, 0, 0, 17, 2345.678),           # lane 0 residue 0 of window 0: anchor = input phase
        Hit("carr", 1, 0, 0, 1, 95, 300, -1843.21),         # odd window (second half-warp), lane 31 residue 2
        Hit("carr", 2, 0, 3, 24, 1, 511, 4999.99),          # last window of a run, lane 0 residue 1
        Hit("carr", 3, 0, 7, 13, 93, 0, -4321.5),           # odd window, lane 31 residue 0, the wrap, negative Doppler
        Hit("carr", 4, 0, 124, 24, 94, 256, 3000.25),       # last run, last window, lane 31 residue 1
        Hit("code", 5, 0, 0, 14, 50, 500),                  # even window
        Hit("code", 6, 0, 2, 21, 7, 1000),                  # odd window, run 2
        Hit("wrap", 7, 0, 0, 19, 40),                       # odd window: 1022 -> 0 with a NAV bit change
        Hit("carr", 8, 0, 1, 2, 2, 0, 777.7),               # lane 0 residue 2, the wrap, positive Doppler
        Hit("carr", 9, 0, 5, 5, 93, 511, -2500.125),        # odd window, index boundary 511, negative Doppler
    ]),
    Case("v32_one_block", 24, 1, 9102, [
        Hit("carr", 16, 0, 4, 10, 48, 100, -2999.1),
        Hit("carr", 20, 0, 0, 3, 95, 511, 1500.25),         # lane 31 residue 2
        Hit("carr", 23, 0, 60, 24, 0, 0, -600.5),           # last window, lane 0 residue 0, the wrap
        Hit("code", 17, 0, 1, 12, 10, 3),
        Hit("code", 18, 0, 0, 17, 80, 767),
        Hit("wrap", 19, 0, 0, 20, 61),                      # even window
        Hit("carr", 2, 0, 2, 11, 1, 200, 3456.0),
        Hit("code", 21, 0, 0, 23, 30, 100),                 # odd window
    ]),
    Case("v16_four_blocks", 12, 4, 9103, [
        Hit("carr", 0, 2, 10, 11, 47, 42, 2345.678),        # block 2, odd window
        Hit("carr", 1, 3, 0, 22, 92, 0, -3210.5),           # block 3, run 0
        Hit("carr", 2, 1, 124, 24, 95, 400, 10.0),          # block 1, last run, last window, tiny Doppler
        Hit("code", 3, 2, 3, 9, 20, 222),                   # block 2, run 3, odd window
        Hit("carr", 4, 0, 0, 6, 33, 128, 4500.0),
        Hit("code", 5, 1, 0, 18, 1, 900),
        Hit("wrap", 6, 3, 0, 15, 70),                       # block 3
    ]),
    Case("v32_four_blocks", 24, 4, 9104, [
        Hit("carr", 17, 3, 50, 15, 31, 311, 1234.5),
        Hit("carr", 22, 1, 0, 24, 94, 511, -4999.0),
        Hit("code", 16, 2, 7, 20, 90, 640),
        Hit("carr", 5, 2, 99, 7, 3, 0, 2.5),
        Hit("wrap", 19, 1, 0, 22, 11),
    ]),
]
