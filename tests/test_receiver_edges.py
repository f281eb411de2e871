"""The receiver kernels' edges on the CPU: the inputs and cases tests/test_receiver_edges_gpu.py runs on the GPU, and the
model-side facts those tests rely on. The replica sign-change counts the acquisition kernel's 8-at-a-time edge loop is
sized for, the acquisition model's FFT path against its direct sum on full-scale coherent input, the period lengths of
tracking states at the code-step limits, and a channel whose epochs resume after a gap, fixed by the model within the
ideal-epoch truth bounds."""
import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import pvt_truth as PT
import scenario
import track_model as T
from scenario import gps
from test_pvt import IDEAL, check_truth, ideal_inputs, rinex
from test_scenario import LOC
from test_track import START_SOW

WEEK_S = 604800.0
AMP = 250                          # amplitude of the carrier tables
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31


# ---- acquisition inputs ----------------------------------------------------------------------------------------------
def sign_changes(prn):
    """Sign changes of the sampled replica within one period (chip c != chip c - 1, c = 1..1022)."""
    ca = A.ca_code(prn)
    return int((ca[1:] != ca[:-1]).sum())


def padded_edges(n):
    """The kernel's edge-list length for n sign changes: an odd count padded with 3000, then (0, 0) pairs up to a
    multiple of 8."""
    n += n & 1
    return (n + 7) // 8 * 8


def carrier_index(n, u):
    """Table index of sample n (from the window start) at phase step u, as the wipe-off reads it."""
    return ((np.asarray(n, np.uint64) * np.uint64(u)) & np.uint64(0xFFFFFFFF)) >> np.uint64(23)


def planted(nsamples, sigs, sample_size, noise=0, seed=0):
    """Interleaved I,Q of `nsamples` samples: each signal (prn, f_hz, delay, amp) is amp x replica(prn) delayed by `delay`
    samples on the table carrier of phase_step(f_hz) from sample 0 (so that the wipe-off of a bin at f_hz removes it
    exactly), plus uniform noise in +-noise; int8, or int16 at 16x that scale."""
    cos, sin = A.tables()
    n = np.arange(nsamples, dtype=np.int64)
    I, Q = np.zeros(nsamples), np.zeros(nsamples)
    for prn, f, delay, amp in sigs:
        c = A.replica(prn)[(n - delay) % A.CODE]
        idx = carrier_index(n, A.phase_step(f)).astype(np.int64)
        I += amp * c * cos[idx] / AMP
        Q += amp * c * sin[idx] / AMP
    if noise:
        rng = np.random.default_rng(seed)
        I += rng.integers(-noise, noise + 1, nsamples)
        Q += rng.integers(-noise, noise + 1, nsamples)
    iq = np.empty(2 * nsamples)
    iq[0::2], iq[1::2] = I, Q
    if sample_size == gps.SC08:
        return np.clip(np.rint(iq), -128, 127).astype(np.int8)
    return np.clip(np.rint(16 * iq), -32768, 32767).astype(np.int16)


def full_scale(nsamples, prn, f_hz, sample_size, delay=0):
    """One PRN at full scale on the exact table carrier of f_hz: int8 -128..127 (floor(127.5 v / 250)), int16
    +-32767 (both reduce to the int8 scale's full range)."""
    cos, sin = A.tables()
    n = np.arange(nsamples, dtype=np.int64)
    c = A.replica(prn)[(n - delay) % A.CODE]
    idx = carrier_index(n, A.phase_step(f_hz)).astype(np.int64)
    iq = np.empty(2 * nsamples, np.int64)
    v = np.stack([c * cos[idx], c * sin[idx]], 1).reshape(-1)
    if sample_size == gps.SC08:
        iq = np.floor(v * 127.5 / AMP).astype(np.int8)
        assert iq.min() == -128 and iq.max() == 127
        return iq
    iq = np.rint(v * 32767.0 / AMP).astype(np.int16)
    assert iq.min() == -32767 and iq.max() == 32767
    return iq


def test_replica_sign_changes_per_prn():
    """The kernel reads each PRN's edge list 8 entries at a time. The sampled replicas have 479, 511, 512 or 543 sign
    changes; the odd counts get one pad entry (3000), and every padded length is then already a multiple of 8, so the
    (0, 0) pair padding never runs with the real codes. Both parities occur, and every list fits the 1024 slots."""
    counts = {p: sign_changes(p) for p in range(1, 33)}
    assert counts == {**{p: 511 for p in range(1, 33)}, 6: 512, 7: 479, 8: 543, 9: 512, 15: 479, 16: 512, 17: 479,
                      21: 479, 22: 543, 24: 479, 28: 512}
    assert {p for p, n in counts.items() if n % 2 == 0} == {6, 9, 16, 28}
    for p, n in counts.items():
        assert padded_edges(n) == n + (n & 1) and padded_edges(n) % 8 == 0 and padded_edges(n) <= 1024
    # the chip boundaries the edges are taken from: chip c starts at ceil(3000 c / 1023), as replica() samples it
    for p in (6, 7, 8):
        r = A.replica(p)
        q = np.nonzero(r[1:] != r[:-1])[0] + 1
        ca = A.ca_code(p)
        c = np.nonzero(ca[1:] != ca[:-1])[0] + 1
        assert np.array_equal(q, (3000 * c + 1022) // 1023)


@pytest.mark.parametrize("sample_size", [gps.SC08, gps.SC16])
def test_acq_model_fft_equals_direct_sum_at_full_scale(sample_size):
    """Full-scale coherent input drives |C| to about 3000 x 127.5 x 250 (9.6e7, below the 2^28 the FFT rounding is
    exact for): the FFT path equals the defining sum, K = 1, on the signal's bin, a neighbour and the aliased 1.5 MHz bin."""
    prn, f = 13, 1750.0
    iq = full_scale(A.CODE + A.CODE - 1, prn, f, sample_size, delay=1234)
    args = (iq, sample_size, 0, 1, [prn, 6], f - 250.0, 250.0, 2)
    P = A.grid(*args)
    assert np.array_equal(P, A.grid(*args, method="direct"))
    peak = int(P[0, 1].max())
    assert int(np.argmax(P[0, 1])) == 1234 and 2 ** 53 < peak < 2 ** 54 and peak < 2 ** 56   # |C| < 2^28
    edge = (iq, sample_size, 0, 1, [prn], -1.5e6, 1.5e6, 3)
    Pe = A.grid(*edge)
    assert np.array_equal(Pe, A.grid(*edge, method="direct")) and np.array_equal(Pe[0, 0], Pe[0, 2])


# ---- tracking states at the contract's limits ------------------------------------------------------------------------
def limit_states(prns, base, seed):
    """Tracking start states with the fields at their limits, cycling over five kinds (channel c gets kind c % 5):
    0: code_step MIN, code_phase 0 (a 3001-sample period), carr_freq +2^34, carr_step 2^31 - 1, carr_phase 2^32 - 1;
    1: code_step MAX, code_phase MAX - 1 (2999 samples), carr_freq -2^34, carr_step -2^31, 190 epochs (the FLL stops
       at the 10th update), prev_i / prev_q at the int32 limits;
    2: 150 epochs, prev_i / prev_q at the opposite limits, lock_i = lock_q = 2^31 - 1, lock 1, carr_freq 2^34 - 1;
    3: 199 epochs (the FLL runs once more), code_step MAX, code_phase 0;
    4: a plain start state from an acquisition within +-4 kHz.
    Each starts within 4000 samples after `base`."""
    rng = np.random.default_rng(seed)
    out = []
    for c, prn in enumerate(prns):
        st = T.start(int(prn), float(rng.uniform(-4000, 4000)), base + int(rng.integers(0, 4000)))
        kind = c % 5
        if kind == 0:
            st["code_step"], st["code_phase"], st["carr_freq"] = T.CODE_STEP_MIN, 0, T.FREQ_CLAMP
            st["carr_step"], st["carr_phase"] = I32_MAX, 0xFFFFFFFF
        elif kind == 1:
            st["code_step"], st["code_phase"], st["carr_freq"] = T.CODE_STEP_MAX, T.CODE_STEP_MAX - 1, -T.FREQ_CLAMP
            st["carr_step"], st["epochs"], st["prev_i"], st["prev_q"] = I32_MIN, 190, I32_MAX, I32_MIN
        elif kind == 2:
            st["epochs"], st["prev_i"], st["prev_q"] = 150, I32_MIN, I32_MAX
            st["lock_i"], st["lock_q"], st["lock"], st["carr_freq"] = I32_MAX, I32_MAX, 1, T.FREQ_CLAMP - 1
        elif kind == 3:
            st["epochs"], st["code_step"], st["code_phase"] = 199, T.CODE_STEP_MAX, 0
        out.append(st)
    return np.array(out, T.STATE_DTYPE)


def period_lengths(eps, st_after):
    """Samples of every period of one channel's epochs, the last one ending at the state's next sample."""
    s = np.append(eps["sample"].astype(np.int64), int(st_after["sample"]))
    return np.diff(s)


def test_period_lengths_at_the_code_step_limits():
    """MIN with phase 0 gives 3001 samples, MAX with phase MAX - 1 gives 2999; the model tracks both states through
    one period of exactly that length."""
    st = limit_states([3, 7], 1000, 1)
    L = (T.M - st["code_phase"].astype(object) + st["code_step"].astype(object) - 1) // st["code_step"].astype(object)
    assert list(L) == [3001, 2999]
    iq = np.zeros(2 * 9000, np.int8)
    eps, after = T.track(iq, gps.SC08, 0, st, max_epochs=1)
    assert [int(period_lengths(e, a)[0]) for e, a in zip(eps, after)] == [3001, 2999]


# ---- fixes ----------------------------------------------------------------------------------------------------------
GAP_CHAN, GAP_AT, GAP_LEN = 4, 6, 2200     # epochs; the gap is 2.2 s


def gapped_case(tmp_path):
    """sky12_static_35s, ideal epochs: channel 4 makes 6 unlocked epochs, nothing is tracked for 2.2 s, and the channel
    resumes with its time anchor after the gap (as a re-acquisition joins its epochs to the earlier ones; the anchor
    counts epochs, so only the part after it tells the time, and the unlocked part is never used). Fixes every 0.3 s
    from 0.01 s to 34.5 s, Klobuchar on.
    -> (channels, epochs, config, stream sample of the first epoch after the gap)."""
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    chans, eps = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    e = eps[GAP_CHAN].copy()
    e["lock"][:GAP_AT] = 0
    eps[GAP_CHAN] = np.concatenate([e[:GAP_AT], e[GAP_AT + GAP_LEN:]])
    anchor = GAP_AT + 10                                       # 10 epochs after the gap, in the joined array
    assert chans[GAP_CHAN]["anchor_epoch"] == 0
    chans[GAP_CHAN]["anchor_epoch"] = anchor
    chans[GAP_CHAN]["anchor_ms"] = (int(chans[GAP_CHAN]["anchor_ms"]) + anchor + GAP_LEN) % PT.WEEK_MS
    cfg = gps.pvt_config(30000, 899993, 115, iono)
    return chans, eps, cfg, int(eps[GAP_CHAN]["sample"][GAP_AT])


def bracket_misses(e, s):
    """For fix instants s, whether the period bracket [d / 3001 - 1, d / 2999 + 1] (d = s - first epoch's sample)
    misses the true period k of the channel's epochs e (only instants inside 1 <= k <= n - 2 count)."""
    smp = e["sample"].astype(np.int64)
    k = np.searchsorted(smp, s, side="right") - 1
    d = np.asarray(s, np.int64) - smp[0]
    lo, hi = np.maximum(1, d // 3001 - 1), np.minimum(len(e) - 2, d // 2999 + 1)
    inside = (k >= 1) & (k <= len(e) - 2)
    return inside & ((k < lo) | (k > hi)), inside


def test_gapped_channel_fixes_within_ideal_truth(tmp_path):
    """The gapped channel is used from its second period after the gap on, and the fixes stay within the ideal-epoch
    truth bounds: the joined epochs describe the same signal. After the gap the period bracket misses the true period."""
    chans, eps, cfg, resume = gapped_case(tmp_path)
    fix, _, _ = PM.pvt(chans, eps, cfg)
    g = scenario.load_golden("sky12_static_35s_i8")
    xyz = np.repeat(PM.llh_ecef(*LOC)[None], g["chans"].shape[0] + 1, 0)
    check_truth(fix, xyz, START_SOW, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])
    used = (fix["mask"].astype(np.int64) >> GAP_CHAN) & 1 == 1
    s = fix["sample"]
    miss, _ = bracket_misses(eps[GAP_CHAN], s)
    after = s >= eps[GAP_CHAN]["sample"][GAP_AT + 1]
    assert 30 < after.sum() < s.size and used[after].all() and not used[~after].any()
    assert miss[after].all()
    assert (fix["nused"][after] == 12).all() and (fix["nused"][~after] == 11).all()
