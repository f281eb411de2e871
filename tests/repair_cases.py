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
# and a NAV bit change at that code period), "entry" (carrier at a step that is a multiple of 2^-52, run 0 of block 0 or
# of a reallocated block: decisive where the walk enters [1/2, 1), see place_entry), "fcarr" (a "carr" hit placed
# against the fixed-point linear phase: place_carrier(fixed=True)), "lat" (an "entry" hit at a lattice
# step c = j 2^-14: see place_lattice); slot, block, run, window, n = sample in the window (lane n % 32, word n // 32 of k_synth_lanes' sample
# side). realloc: a carrier hit in a later block takes a new satellite in its slot from that block on, so that its
# input phase is placed from the block start (<= 300000 samples of walk) instead of on the chain from block 0.
Hit = collections.namedtuple("Hit", "kind slot block run win n target f_carr realloc", defaults=(None, None, False))
# plain: slots whose hit is certified to reach the exact walk but NOT decisive (the arithmetic admits no straddle there)
Case = collections.namedtuple("Case", "name nchan nblk seed hits plain", defaults=((),))


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


def place_carrier(f_carr, T, m, k, fixed=False):
    """Input carrier phase so that the linear phase m samples after the exact anchor T samples on sits on index
    boundary k (or, when the FP64 phase there differs, half their difference off it, on the other side). fixed: the
    difference is taken to the fixed-point linear phase (synth_lanes.h carr_fix + m carr_step_fix, truncated to 2^-64
    per step) instead of the rational one -- what decides at steps with bits far below 2^-53, where the truncation of
    the step outweighs the rounding of the walk. -> (input phase, anchor, decisive)"""
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
    ref = Fraction(xr) + m * Fraction(c)
    if fixed:
        ref = Fraction((carr_fix(xr) + m * carr_step_fix(c)) % (1 << 64), 1 << 64)
    delta = _centered(Fraction(gps.carrier_advance(xr, f_carr, m)) - ref, 1)
    shift = _centered(ref - (Fraction(xr) + m * Fraction(c)), 1)      # fixed-point - rational linear phase (0 if not fixed)
    if delta != 0:
        x, xr = solve(target - shift - delta / 2)
    lin = (carr_fix(xr) + m * carr_step_fix(c)) % (1 << 64)
    frac = lin & ((1 << 55) - 1)
    assert frac < BAND_CARR or frac > (1 << 55) - BAND_CARR, (f_carr, T, m, k)
    decisive = (lin >> 55) != carr_index_exact(gps.carrier_advance(xr, f_carr, m))
    return x, xr, bool(decisive)


def f_for_step(c):
    """A Doppler f with fl(f * DELT) == c exactly (the nearest reachable step when no double f gives c)."""
    f = float(Fraction(c) / Fraction(DELT))
    best = f
    for _ in range(2):
        for k in range(200):
            got = float(np.float64(f) * np.float64(DELT))
            if got == c:
                return f
            if abs(got - c) < abs(float(np.float64(best) * np.float64(DELT)) - c):
                best = f
            f = float(np.nextafter(f, np.inf if got < c else -np.inf))
    return best


def f_for_fast_step(u):
    """Doppler whose carrier step is u * 2^-32 cycles exactly (u: the 32-bit fast_step, two's complement)."""
    return f_for_step(float(((u ^ 0x80000000) - 0x80000000) * 2.0 ** -32))


def carr_index_lin(x0, c, m):
    return (carr_fix(x0) + m * carr_step_fix(c)) % (1 << 64) >> 55


def entry_boundaries(c, m):
    """Index boundaries b (b / 512 > 1/2) that place_entry can put sample m on at step c."""
    if c == 0.0 or (Fraction(c) * (1 << 52)).denominator != 1:
        return []
    mc = m * Fraction(c)
    return [b for b in range(257, 512) if (Fraction(b, 512) - Fraction(1, 1 << 54) - mc) % 1 < Fraction(1, 2)]


def place_entry(f_carr, m, k):
    """Run 0 from the input phase, at a step c = fl(f_carr * DELT) that is a multiple of 2^-52 (every step a multiple of
    2^-32 is): the input phase x0 < 1/2 is chosen so that x0 + m c = b / 512 - 2^-54 (mod 1) exactly, on a boundary
    b / 512 > 1/2. Below 1/2 the walk is exact (the grid is 2^-54 or finer); it enters [1/2, 1) before sample m -- going
    up, or with c < 0 at the wrap below 0, whose + 1 rounds -- and that sum has its 2^-54 and 2^-53 bits set, so it
    rounds up by 2^-54. From there on the FP64 phase is the linear one + 2^-54 (sums on the 2^-53 grid are exact), and
    sample m is on the other side of boundary b. Of the boundaries that qualify, the one taken is number k modulo their
    count. -> (x0, decisive samples of the run: [sample number in the run]), or None when no boundary qualifies (the
    walk cannot reach a boundary above 1/2 within m samples: |m c| < 2^-9)"""
    c = float(np.float64(f_carr) * np.float64(DELT))
    ok = entry_boundaries(c, m)
    if not ok:
        return None
    mc = m * Fraction(c)
    xf = (Fraction(ok[k % len(ok)], 512) - Fraction(1, 1 << 54) - mc) % 1
    x0 = float(xf)
    assert Fraction(x0) == xf and x0 < 0.5, (f_carr, m, k)
    x, out = x0, []
    for n in range(RUN):
        if carr_index_lin(x0, c, n) != carr_index_exact(x):
            out.append(n)
        x = gps.carrier_advance(x, f_carr, 1)
    return x0, out


def place_lattice(f_carr, m, k):
    """place_entry at a lattice step c = j 2^-14, j odd: n c mod 2^-9 has period 32 in n, so that samples m - 32, m,
    m + 32 of a window share their offset from the index boundaries and are risky -- and past the entry decisive --
    together."""
    c = float(np.float64(f_carr) * np.float64(DELT))
    assert (Fraction(c) * (1 << 14)).denominator == 1 and (int(Fraction(c) * (1 << 14)) & 1), f_carr
    placed = place_entry(f_carr, m, k)
    assert placed is not None, (f_carr, m)
    return placed


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
        if h.kind in ("carr", "fcarr", "lat", "entry"):
            ch["f_carr"][:, s] = h.f_carr
            ch["f_code"][:, s] = 1.023e6 + h.f_carr / 1540.0
            if h.realloc and h.block > 0:
                ch["prn"][h.block:, s] = ch["prn"][h.block - 1, s] % 32 + 1        # a new satellite from this block on
            if h.kind in ("lat", "entry"):
                assert h.run == 0 and (h.block == 0 or h.realloc)
                x, dec = (place_lattice if h.kind == "lat" else place_entry)(h.f_carr, m, h.target)
                decisive[s] = m in dec
            elif h.realloc and h.block > 0:
                x, _, decisive[s] = place_carrier(h.f_carr, T, m, h.target)
            else:
                x, _, decisive[s] = place_carrier(h.f_carr, h.block * BLOCK + T, m, h.target, fixed=h.kind == "fcarr")
            ch["carr_phase"][h.block if h.realloc else 0, s] = x
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
            # an unused PRN when there is one; with every PRN in use (32 channels) one in use: the API allows duplicates
            used = set(int(p) for p in ch["prn"][b])
            fit = [p for p in range(1, 33) if gps.codegen(p)[1022] == gps.codegen(p)[0]]
            prn = next((p for p in fit if p not in used), fit[0])
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
    """Block b of a call with the carrier phases the call chains into it (exact sequential chain); a slot whose
    satellite changes at b keeps its own input phase."""
    row = ch[b].copy()
    if b > 0:
        cont = ch["prn"][b] == ch["prn"][b - 1]
        row["carr_phase"] = np.where(cont, gps.carrier_chain(ch[:b], threads=4), row["carr_phase"])
    return row


def chained_rows(ch, blocks, threads=16):
    """chained_row of each of `blocks`, from ONE incremental pass of the exact chain. -> {block: row}"""
    out, phase, done = {}, None, 0
    for b in sorted(set(blocks)):
        if b > done:
            part = ch[done:b]
            if phase is not None:                      # a slot whose satellite changes at `done` starts afresh
                phase = np.where(ch["prn"][done] == ch["prn"][done - 1], phase, ch["carr_phase"][done])
            phase = gps.carrier_chain(part, phase_in=phase, threads=threads)
            done = b
        row = ch[b].copy()
        if b > 0:
            row["carr_phase"] = np.where(ch["prn"][b] == ch["prn"][b - 1], phase, row["carr_phase"])
        out[b] = row
    return out


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


# ---- every channel slot, every bit of the flagged mask -------------------------------------------------------------
# k_synth_lanes' channel side ballots one bit per (window half, channel): bit c in the 32-channel variant, bit
# 16 h + c in the 16-channel one (h = 1: the odd window of a trip). The cases below put a decisive hit behind every bit,
# all 32 bits into one ballot, code and wrap hits into the top slots (15, 31) and into the last real slot next to a
# padding slot (15 and 31 channels), and lanes with three risky samples in one window (lattice steps).

def _lattice_f(j):
    f = f_for_step(j * 2.0 ** -14)
    assert float(np.float64(f) * np.float64(DELT)) == j * 2.0 ** -14, j      # j = +-15, +-31 have no such f
    return f


def _spread(nchan, seed, parity=0, skip=(), block=0):
    """One carrier hit per slot (but `skip`): random run, sample, boundary and Doppler within +-5 kHz; in the
    16-channel variant slot c's window has parity (c + parity) % 2, so that its hit sits behind bit c or 16 + c."""
    rng = np.random.default_rng(seed)
    hits = []
    for s in range(nchan):
        run, win2, n = int(rng.integers(0, 125)), int(rng.integers(0, 12)), int(rng.integers(0, 96))
        k, f = int(rng.integers(0, 512)), round(float(rng.uniform(-5000.0, 5000.0)), 3)
        if s not in skip:
            hits.append(Hit("carr", s, block, run, 2 * win2 + (s + parity) % 2, n, k, f))
    return hits


EDGE_CASES = [
    Case("v16_bits_even", 16, 1, 9201, _spread(16, 9201, 0)),         # bits 0, 2, .., 14 and 17, 19, .., 31
    Case("v16_bits_odd", 16, 1, 9202, _spread(16, 9202, 1)),          # bits 1, 3, .., 15 and 16, 18, .., 30
    Case("v16_top_code", 16, 1, 9203, _spread(16, 9203, 0, (14, 15)) + [
        Hit("code", 15, 0, 5, 17, 95, 321),                           # top slot, odd window, lane 31 word 2
        Hit("wrap", 14, 0, 0, 20, 1)]),
    Case("v16_top_wrap", 16, 1, 9204, _spread(16, 9204, 1, (14, 15)) + [
        Hit("wrap", 15, 0, 0, 23, 31),                              # top slot, odd window (bit 31's half)
        Hit("code", 14, 0, 124, 24, 64, 1000)]),
    Case("v15_pad_code", 15, 1, 9205, _spread(15, 9205, 1, (14,)) + [
        Hit("code", 14, 0, 77, 9, 33, 600)]),                         # last real slot, padding slot 15 beside it
    Case("v15_pad_wrap", 15, 1, 9206, _spread(15, 9206, 0, (13, 14)) + [
        Hit("wrap", 14, 0, 0, 18, 0),
        Hit("code", 13, 0, 3, 0, 50, 5)]),
    Case("v32_bits", 32, 1, 9207, _spread(32, 9207)),                  # bits 0 .. 31, one window each
    Case("v32_top_code", 32, 1, 9208, _spread(32, 9208, 0, (30, 31)) + [
        Hit("code", 31, 0, 60, 24, 95, 1000),
        Hit("wrap", 30, 0, 0, 11, 48)]),                              # no PRN unused: the wrap PRN is a duplicate
    Case("v32_top_wrap", 32, 1, 9209, _spread(32, 9209, 0, (30, 31)) + [
        Hit("wrap", 31, 0, 0, 5, 95),
        Hit("code", 30, 0, 1, 1, 0, 77)]),
    Case("v31_pad", 31, 1, 9211, _spread(31, 9211, 0, (29, 30)) + [
        Hit("code", 30, 0, 100, 12, 17, 444),
        Hit("wrap", 29, 0, 0, 3, 60)]),
    Case("v31_pad_wrap", 31, 1, 9215, _spread(31, 9215, 0, (0, 1, 30)) + [
        Hit("wrap", 30, 0, 0, 24, 10),
        Hit("lat", 0, 0, 0, 2, 8, 300, _lattice_f(5)),               # lanes with three risky samples, v32 variant
        Hit("lat", 1, 0, 0, 7, 31, 17, _lattice_f(-19))]),
    # every slot's hit in ONE (block, run, window): all 32 bits in one ballot, the repair loop over 32 channels
    Case("v32_one_ballot", 32, 1, 9212,
         [Hit("carr", s, 0, 9, 13, (37 * s + 5) % 96, (97 * s + 3) % 512, round(-4900.0 + 311.7 * s, 3))
          for s in range(32)]),
    # 16 slots at lattice steps: every window of run 0 has a risky lane in every slot, so that both halves of every
    # trip are flagged -- all 32 bits in every ballot -- and each such lane has three risky samples (i, 32 + i,
    # 64 + i), decisive once the walk has entered [1/2, 1)
    Case("v16_lattice_ballot", 16, 1, 9213,
         [Hit("lat", s, 0, 0, 1 + s % 4, (29 * s + 5) % 32, 61 * s + 7, _lattice_f(j))
          for s, j in enumerate((1, -3, 5, -7, 9, -11, 13, -17, 19, -21, 23, -25, 27, -29, 3, -5))]),
]


# ---- every launch shape of k_synth_lanes ---------------------------------------------------------------------------
# A launch splits each block's 125 runs over ctas_per_block CTAs of runs_per_cta runs (the last CTA may have fewer);
# warp w of a CTA takes its runs w, w + 16, w + 32, ... (one run per warp only when runs_per_cta == 16).

def lanes_shape(nblk, sms=132, nruns=BLOCK // RUN):
    """synth_lanes.cu lanes_shape: (CTAs per block, runs per CTA) of one launch over nblk blocks on `sms` SMs."""
    per_block = min(16, max(1, (40 * 2 * sms + nblk - 1) // nblk))
    per_cta = (nruns + per_block - 1) // per_block
    per_cta = (per_cta + 15) // 16 * 16
    return (nruns + per_cta - 1) // per_cta, per_cta


def shape_runs(per_block, per_cta, nruns=BLOCK // RUN):
    """Runs of a block that a launch shape gives to the edges of its CTAs and warps: the first and the last run of every
    CTA, warp 15's first run, the first run of the second pass and of the last pass of a warp."""
    runs = set()
    for g in range(per_block):
        lo, hi = g * per_cta, min((g + 1) * per_cta, nruns)
        runs |= {lo, hi - 1, min(lo + 15, hi - 1)}
        if hi - lo > 16:
            runs |= {lo + 16, lo + 16 * ((hi - 1 - lo) // 16)}
    return sorted(runs)


def shape_case(nchan, nblk, per_block, per_cta, seed):
    """Carrier hits at the shape_runs of a launch shape, each run in block 0 and in the last block (the slot takes a
    new satellite there, so that the placement walks at most one block), as far as the slots go; and one hit in the
    last block on the chain from block 0 (a small Doppler: the placement walks the whole call)."""
    runs = shape_runs(per_block, per_cta)
    last = nblk - 1
    spots = [(0, r) for r in runs] + [(last, r) for r in runs[::-1]]
    hits = [Hit("carr", 0, last, runs[len(runs) // 2], 11, 70, 300, 7.25)]
    for i, (b, r) in enumerate(spots[:nchan - 1]):
        f = (1.0 if i % 2 else -1.0) * (400.0 + (317.3 * i) % 4500.0)
        hits.append(Hit("carr", i + 1, b, r, (7 * i + 3) % 25, (13 * i + 5) % 96, (101 * i + 9) % 512, round(f, 3),
                        b > 0))
    return Case("shape_%dx%d_%dch_%dblk" % (per_block, per_cta, nchan, nblk), nchan, nblk, seed, hits)


# ---- degenerate and extreme carrier steps --------------------------------------------------------------------------
# The 32-bit steps (fast_step) whose residues n u mod 2^23 (n < 96) are degenerate -- all zero, repeating within a
# window, or several inside one 128-unit band (tests/test_window_band.py checks the certification for them on the host)
# -- reached through f_carr; steps k 2^-9 near the API's |f_carr| < 2.9 MHz; and the edge of nco_exact.h's fast range,
# |c| = 2^-23 (f = 0.3576 Hz) and one ulp on either side, below which the speculative chain falls back to the host.
DEGEN_FAST_STEPS = ([0, 1 << 23, 3 << 23, 1 << 31, 1 << 22, 1 << 21, 3 << 20, 1 << 17, 5 << 16, 1 << 16]
                    + list(range(1, 129)) + [0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFF80, 0xFFFFFF81, 0xFFFFF000])
EDGE_C = [s * c for s in (1.0, -1.0) for c in (float(np.nextafter(2.0 ** -23, 0.0)), 2.0 ** -23,
                                               float(np.nextafter(2.0 ** -23, 1.0)))]
DEGEN_STEPS = ([("u=%#x" % u, f_for_fast_step(u)) for u in DEGEN_FAST_STEPS]
               + [("k=%d" % k, f_for_step(k * 2.0 ** -9)) for k in (494, -494)]
               + [("c=%r" % c, f_for_step(c)) for c in EDGE_C])


def step_of(f):
    return float(np.float64(f) * np.float64(DELT))


def degen_hit(s, f, nblk):
    """The hit of slot s at step fl(f * DELT) in an nblk-block call. Where the step is a multiple of 2^-52 and can reach a
    boundary above 1/2 within the run, an "entry" hit (place_entry) in run 0: of block 0 in a 2-block call, of the last
    block, where the slot takes a new satellite, in a 3-block call. Otherwise a carrier hit in the last block on the
    chain from block 0, on a boundary in (1/4, 1/2) for |c| < 2^-9 (a step with bits below 2^-54 rounds at every sum
    there)."""
    c = step_of(f)
    win, n = (3 * s + 1) % 25, (11 * s + 7) % 96
    blk = 0 if nblk <= 2 else nblk - 1
    for w, i in ((win, n), (RUN // WIN - 1, WIN - 1)):
        if entry_boundaries(c, w * WIN + i):
            return Hit("entry", s, blk, 0, w, i, 7 * s, f, blk > 0)
    # the first decisive one of a few positions and boundaries (the default one when none is)
    tries = [((5 * s + 3) % 125, win, n)] + [((5 * s + 3 + 17 * j) % 125, (win + 7 * j) % 25, (n + 29 * j) % 96)
                                              for j in range(1, 4)]
    ks = [205, 150, 230, 100, 60] if abs(c) < 2.0 ** -9 else [(37 * s + 11) % 512, 300, 77]
    for r, w, i in tries:
        for k in ks:
            if c != 0.0 and place_carrier(f, (nblk - 1) * BLOCK + r * RUN, w * WIN + i, k, fixed=True)[2]:
                return Hit("fcarr", s, nblk - 1, r, w, i, k, f)
    return Hit("carr", s, nblk - 1, tries[0][0], win, n, ks[0], f)


# Steps without a decisive hit here (tests/test_lanes_edges.py certifies that these are not decisive and that all other
# steps' hits are); their hits certify that the window is flagged and the sample repaired:
#   c = 0                        no walk at all
#   1 <= u <= 128, -128 <= u < 0 and c = +-2^-23: multiples of 2^-52 too small to reach a boundary above 1/2 within one run
#                                (|c| * 2400 < 2^-9): from an anchor the walk stays exact up to that boundary, and an
#                                anchor on the 2^-53 grid walks exactly forever
#   u = 0xFFFFF000 (c = -2^-20)  the place_entry walk reaches -2^-54 exactly at its wrap, since 2^-20 divides every
#                                boundary; the reference's + 1 then rounds to 1.0, which nco_exact.h clamps to the
#                                largest double below 1 -- a rounding DOWN, so the hit is not decisive, but it runs the
#                                clamp on the device
#   c = +-(2^-23 + 2^-75)        one ulp above 2^-23 in magnitude: carr_step_fix truncates the 2^-75 away, and every sum
#                                of the walk (ulp >= 2^-74 above 2^-22) rounds it away too, so the FP64 phase IS the
#                                fixed-point linear phase
#   k = -494                     none of the positions and boundaries degen_hit tries straddles
DEGEN_PLAIN = ({"u=%#x" % u for u in [0] + list(range(1, 129)) + [0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFF80, 0xFFFFFF81, 0xFFFFF000]}
               | {"k=-494"} | {"c=%r" % (sg * c) for sg in (1.0, -1.0) for c in EDGE_C[1:3]})
assert all(label in dict(DEGEN_STEPS) for label in DEGEN_PLAIN)


def degen_case(name, steps, nblk, seed):
    hits = [degen_hit(s, f, nblk) for s, (_, f) in enumerate(steps)]
    plain = tuple(s for s, (label, _) in enumerate(steps) if label in DEGEN_PLAIN)
    return Case("%s_%dblk" % (name, nblk), len(steps), nblk, seed, hits, plain)


# all steps, 32 per case (32-channel variant), and the steps that admit a decisive hit once more at 16 channels
# (16-channel variant: an even and an odd window per trip)
_DECISIVE_STEPS = [st for st in DEGEN_STEPS if st[0] not in DEGEN_PLAIN]
DEGEN_CASES = ([degen_case("steps%d" % g, DEGEN_STEPS[32 * g:32 * g + 32], nblk, 9400 + g)
                for g in range((len(DEGEN_STEPS) + 31) // 32) for nblk in (2, 3)]
               + [degen_case("steps16_%d" % g, _DECISIVE_STEPS[16 * g:16 * g + 16], nblk, 9410 + g)
                  for g in range((len(_DECISIVE_STEPS) + 15) // 16) for nblk in (2, 3)])
