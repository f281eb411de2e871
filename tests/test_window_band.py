"""The window band certification of the lane = sample synthesis (synth_lanes.h band_residues / window_band_risky), checked
against the per-sample test it replaces: a window with 32-bit carrier phase base `base` and increment `step` has a sample
to repair exactly when some m < 96 gives a phase base + m * step (mod 2^32) whose low 23 bits are 2^23 - 128 or more
(fast_risky). The kernel and the host model decide per (channel, window) with the certification and test samples only in
the windows it flags, so any disagreement here would be a missed or spurious repair."""
import numpy as np

from scenario import gps

WIN = 96
BAND = 128
M23 = 1 << 23
DELT = 1.0 / 3.0e6


def brute(steps, bases):
    """fast_risky of every sample of each window, by brute force over m < 96."""
    steps = np.asarray(steps, np.uint32)
    bases = np.asarray(bases, np.uint32)
    out = np.zeros(steps.size, bool)
    m = np.arange(WIN, dtype=np.uint32)
    for lo in range(0, steps.size, 1 << 16):
        st, bs = steps[lo:lo + (1 << 16)], bases[lo:lo + (1 << 16)]
        p = bs[:, None] + st[:, None] * m[None, :]                   # uint32: modulo 2^32
        out[lo:lo + st.size] = ((p & np.uint32(M23 - 1)) >= np.uint32(M23 - BAND)).any(axis=1)
    return out


def check(steps, bases):
    steps, bases = np.broadcast_arrays(np.asarray(steps, np.uint32), np.asarray(bases, np.uint32))
    got = gps.lanes_window_band(steps, bases)
    want = brute(steps.ravel(), bases.ravel())
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(int(steps.ravel()[i]), int(bases.ravel()[i]), bool(want[i])) for i in bad[:5]]
    return int(want.sum())


def fast_step(f_hz):
    """32-bit carrier increment per sample of a channel at Doppler f_hz (fast_step of carr_step_fix(f * delt))."""
    c = float(np.float64(f_hz) * np.float64(DELT))
    m = int(abs(c) * 2.0 ** 64)
    return (((1 << 64) - m if c < 0 else m) >> 32) & 0xFFFFFFFF


def hitting_bases(steps, ms, offsets):
    """Bases that put sample m of the window at low 23 bits 2^23 - 128 + offset (offset -1: one unit below the band)."""
    out = []
    for st in steps:
        for m in ms:
            for off in offsets:
                out.append((st, (M23 - BAND + off - m * st) & 0xFFFFFFFF))
    a = np.array(out, np.uint64)
    return a[:, 0].astype(np.uint32), a[:, 1].astype(np.uint32)


def test_random_pairs_match_the_per_sample_test():
    rng = np.random.default_rng(20261015)
    n = 1 << 20
    steps = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    bases = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    risky = check(steps, bases)
    assert 500 < risky < 5000                                           # about 96 * 128 / 2^23 = 0.15 % of them
    # the same steps with a random sample put within 64 units of the band: about half of these are risky
    m = rng.integers(0, WIN, n).astype(np.uint32)
    off = rng.integers(-64, 192, n).astype(np.int64)
    near = ((M23 - BAND + off - m.astype(np.int64) * steps.astype(np.int64)) & 0xFFFFFFFF).astype(np.uint32)
    risky = check(steps, near)
    assert n // 4 < risky < 3 * n // 4


def test_degenerate_steps():
    rng = np.random.default_rng(7)
    bases = rng.integers(0, 1 << 32, 4096, dtype=np.uint64).astype(np.uint32)
    edge = np.array([M23 - BAND, M23 - BAND - 1, M23 - 1, 0, 1, M23 - BAND + 127], np.uint32)
    bases = np.concatenate([bases, edge, edge + np.uint32(5 << 23)])
    steps = [0, M23, 1 << 31, 3 << 23,                                   # low 23 bits 0: every sample at the base
             1 << 22, 1 << 21, 3 << 20, 1 << 17, 5 << 16, 1 << 16,      # residues repeat with a period below 96
             0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFF80, 0xFFFFFF81, 0xFFFFF000]  # small negative Doppler
    steps += list(range(1, BAND + 1))                                    # several residues inside one band
    steps += [M23 // k for k in (3, 5, 7, 95, 96, 97)] + [M23 - M23 // 96, (M23 // 96) + 1]
    for st in steps:
        check(np.uint32(st), bases)


def test_doppler_steps_and_hits_at_the_edges():
    dopplers = [5000.0, -5000.0, 1000.0, -1000.0, 0.01, -0.01, 4999.99, -4321.5, 0.0]
    steps = [fast_step(f) for f in dopplers]
    assert steps[-1] == 0 and steps[4] != 0 and steps[5] > 0xFFFF0000
    # sample m exactly at the band's first unit, at its last, and one unit below it, for the first, second and last m
    st, bs = hitting_bases(steps, [0, 1, 2, 47, 94, 95], [-1, 0, 1, 127, 128])
    risky = check(st, bs)
    assert risky >= 3 * 6 * (len(steps) - 1)
    # the interval [t, t + 128) wraps past 2^23 exactly when sample 0 is itself in the band
    low = np.arange(M23 - BAND - 2, M23 + 2, dtype=np.int64) & (M23 - 1)
    for s in steps:
        check(np.uint32(s), (low + (9 << 23)).astype(np.uint32))


def test_every_sample_index_can_be_the_only_hit():
    rng = np.random.default_rng(11)
    steps = rng.integers(0, 1 << 32, 64, dtype=np.uint64).astype(np.uint32).tolist()
    steps += [fast_step(f) for f in rng.uniform(-5000.0, 5000.0, 64)]
    st, bs = hitting_bases(steps, range(WIN), [-1, 0, 63, 127, 128])
    check(st, bs)

