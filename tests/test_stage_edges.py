"""The models of the snapshot measurement and of the tracking loops' CORDIC angle at the edges of their contracts, on the
CPU, against plain float64 references: track_model.angle against atan2 at every magnitude and in every octant of its
half plane, and snapshot_model.measure on noise-free planted signals against the planted truth (Doppler seeds up to
240 Hz off, code phases that wrap within a pass, data bits that flip between chunks, a window of zeros). The bounds
below were measured on the models and are listed in DESIGN §10 and §11.5; tests/test_stage_edges_gpu.py runs the same
inputs through the kernels."""
import numpy as np
import pytest

import acq_model as A
import snapshot_model as S
import track_model as T
from scenario import gps
from test_receiver_edges import full_scale, planted

TURN = 2.0 ** 32                 # angle units per turn
PRN, F_HZ, DELAY, AMP = 7, 1234.5, 1234, 60
# |w - w_true| in carrier-step units (3e6 / 2^32 Hz = 0.70 mHz) after the frequency pass, seeds within 240 Hz; measured
# on the model at PRN 7, 1234.5 Hz: 154 (K = 2), 32 (K = 10), 3 (K = 100)
FREQ_BOUND = {2: 160, 10: 35, 100: 4}
# |code phase error| in chips at the window's centre after 12 or 16 iterations (the planted code has no code Doppler,
# the measurement's code step is carrier aided, so the error is taken where the fit is centred); measured at most
# 0.0045 (K = 2), 0.0048 (K = 10), 0.0051 (K = 100): the early-late balance on the sampled correlation, not noise
CODE_BOUND = 0.0055
SEED_OFFSETS = (0.0, 50.0, -50.0, 125.0, -125.0, 240.0, -240.0)


def angle_bound(r):
    """The measured error bound of angle() at magnitude r: 1 / r turn plus 90 units (2.1e-8 turn; the 24 steps'
    resolution, reached from r = 2^28 on)."""
    return TURN / r + 90.0


def result(prn, f_hz, delay, ratio=10.0):
    r = np.zeros(1, gps.ACQ_RESULT_DTYPE)
    r["prn"], r["doppler_hz"], r["delay"], r["ratio"] = prn, f_hz, delay, ratio
    return r


def true_step(f_hz):
    w = A.phase_step(f_hz)
    return w - (1 << 32) if w >= 1 << 31 else w


def phase_trace(res_row, ds):
    """The unreduced code phases of a refinement: the seed's, then after each D step."""
    _, _, phi = S.seed(res_row, 0)
    out = [phi]
    for d in ds:
        out.append(out[-1] + d * S.GAIN)
    return out


def code_error_at_centre(rec, delay, K):
    """Chips between the record's replica and the planted code (3000 samples per period) at the window's centre."""
    n = 1500 * K
    got = int(rec["code_phase"]) + n * int(rec["code_step"])
    want = (n - delay) * S.M // 3000
    return float((got - want + S.M // 2) % S.M - S.M // 2) / TURN


def flipped(iq, K, bits):
    """iq (noise-free, no sample at -128) with chunk k negated where bits[k]: a data bit flip at chunk boundaries."""
    v = iq.astype(np.int64).reshape(K, -1).copy()
    v[np.asarray(bits, bool)] *= -1
    return v.reshape(-1).astype(iq.dtype)


# ---- track_model.angle -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", [0, 1, 2, 3, 4, 6, 8, 12, 16, 20, 24, 28, 30, 31, 32, 40, 48, 56, 62])
def test_angle_against_atan2_at_each_magnitude(e):
    """Vectors of magnitude 2^e on 4001 angles over the half plane x >= 0 (every octant, both axes) against atan2."""
    r = 2.0 ** e
    th = np.linspace(-0.25, 0.25, 4001)
    x = np.maximum(np.rint(r * np.cos(2 * np.pi * th)), 0).astype(np.int64)
    y = np.rint(r * np.sin(2 * np.pi * th)).astype(np.int64)
    keep = (x != 0) | (y != 0)
    x, y = x[keep], y[keep]
    octant = np.floor(np.arctan2(y, x) / (np.pi / 4)).astype(int)
    assert set(octant.tolist()) >= {-2, -1, 0, 1}
    got = T.angle(x, y).astype(np.float64)
    err = np.abs(got - np.arctan2(y.astype(np.float64), x.astype(np.float64)) / (2 * np.pi) * TURN)
    assert err.max() <= angle_bound(r), (e, err.max() / TURN)


def test_angle_at_the_int64_corners_and_of_the_zero_vector():
    """The largest inputs the loops can form, the axes, and (0, 0): 0, not the -0.277 turn 24 steps on y = 0 give."""
    big = 2 ** 62
    x = np.array([big, big, big, 1, 0, 0, 1, 1], np.int64)
    y = np.array([big, -big, 0, big, big, -big, 0, -1], np.int64)
    want = np.array([0.125, -0.125, 0.0, 0.25, 0.25, -0.25, 0.0, -0.125]) * TURN
    got = T.angle(x, y).astype(np.float64)
    assert (np.abs(got - want) <= 90.0)[:6].all()
    assert abs(got[6] - 0.0274527 * TURN) < 1e-6 * TURN       # angle(1, 0): the small-vector error, documented
    assert int(T.angle(np.int64(0), np.int64(0))) == 0


# ---- snapshot_model.measure on planted signals ----------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 10, 100])
def test_frequency_pass_pulls_in_seeds_up_to_240_hz_off(K):
    iq = planted(3000 * K, [(PRN, F_HZ, DELAY, AMP)], gps.SC08)
    wt = true_step(F_HZ)
    for off in SEED_OFFSETS:
        m = S.measure(iq, gps.SC08, 0, K, result(PRN, F_HZ + off, DELAY))[0]
        assert m["status"] == S.OK, (K, off, m)
        assert abs(int(m["carr_step"]) - wt) <= FREQ_BOUND[K], (K, off, int(m["carr_step"]) - wt)
        assert abs(code_error_at_centre(m, DELAY, K)) <= CODE_BOUND, (K, off, code_error_at_centre(m, DELAY, K))


@pytest.mark.parametrize("K", [2, 10])
@pytest.mark.parametrize("seed_delay,true_delay,crosses", [(0, 1, "zero"), (1, 0, "M")])
def test_code_phase_wraps_within_the_refinement(K, seed_delay, true_delay, crosses):
    """A seed one sample after the truth walks down through phase 0 (the mod M fold from below), one sample before it
    walks up through M (the fold from above); both end within the code bound of the truth."""
    iq = planted(3000 * K, [(PRN, F_HZ, true_delay, AMP)], gps.SC08)
    r = result(PRN, F_HZ, seed_delay)
    tr = []
    m = S.measure(iq, gps.SC08, 0, K, r, iterations=gps.SNAP_MAX_ITER, trace=tr)[0]
    raw = phase_trace(r[0], tr[0])
    assert (min(raw) < 0) if crosses == "zero" else (max(raw) >= S.M), raw[:4]
    assert 0 <= int(m["code_phase"]) < S.M and m["status"] == S.OK
    assert abs(code_error_at_centre(m, true_delay, K)) <= CODE_BOUND


@pytest.mark.parametrize("K", [2, 10])
def test_data_bit_flips_between_chunks_do_not_change_the_refinement(K):
    """Chunks negated in the pattern of data bits: the FLL pairs straddling a flip have dot < 0 and are negated back,
    the code passes square their sums, so the record is the one without flips byte for byte."""
    iq = planted(3000 * K, [(PRN, F_HZ, DELAY, AMP)], gps.SC08)
    assert iq.min() > -128
    bits = np.arange(K) % 3 == 1
    r = result(PRN, F_HZ + 125.0, DELAY)
    I, Q = A.samples(flipped(iq, K, bits), gps.SC08)
    w, u, phi = S.seed(r[0], 0)
    f = S.sums(I, Q, PRN, K, phi, u, w, code=False)
    dots = f["pi"][:-1] * f["pi"][1:] + f["pq"][:-1] * f["pq"][1:]
    assert (dots < 0).any()
    assert S.measure(flipped(iq, K, bits), gps.SC08, 0, K, r).tobytes() == S.measure(iq, gps.SC08, 0, K, r).tobytes()


def test_a_window_of_zeros_steers_nothing():
    """A window of zeros with an infinite ratio (acquisition's p2 = 0): the PRN is refined and stays OK, but w, u and
    the phase keep their seeds, D = 0 and the power is 0."""
    K = 10
    iq = np.zeros(2 * 3000 * K, np.int8)
    r = result(PRN, 2000.0, 17, ratio=np.inf)
    m = S.measure(iq, gps.SC08, 0, K, r)[0]
    w, u, phi = S.seed(r[0], 0)
    assert m["status"] == S.OK and m["power"] == 0 and m["last_step"] == 0 and m["iterations"] == gps.SNAP_ITERATIONS
    assert (int(m["carr_step"]), int(m["code_step"]), int(m["code_phase"])) == (w, u, phi)


@pytest.mark.parametrize("sample_size", [gps.SC08, gps.SC16])
def test_full_scale_window_reaches_the_sums_the_header_bounds(sample_size):
    """A full-scale coherent PRN at K = 100: power reaches 0.75 of the header's bound of K 1.85e16 (int16) and E + L a
    fifth of its 3.7e18; measured 1.39e18 / 7.57e17 (int16), 8.6e17 / 4.62e17 (int8). The record is OK."""
    K = 100
    iq = full_scale(3000 * K, 13, 1750.0, sample_size, delay=1234)
    r = result(13, 1750.0, 1234)
    tr = []
    m = S.measure(iq, sample_size, 0, K, r, iterations=gps.SNAP_MAX_ITER, trace=tr)[0]
    assert m["status"] == S.OK
    el = max_e_plus_l(iq, sample_size, K, r[0], m, tr[0])
    lo = {gps.SC08: (8.5e17, 4.6e17), gps.SC16: (1.38e18, 7.5e17)}[sample_size]
    assert int(m["power"]) >= lo[0] and el >= lo[1] and el < 3.7e18, (int(m["power"]), el)


def max_e_plus_l(iq, sample_size, K, res_row, rec, ds):
    """The largest E + L over a refinement's code passes, replayed from its D trace at the record's u and w."""
    I, Q = A.samples(iq, sample_size)
    _, _, phi = S.seed(res_row, 0)
    u, w = int(rec["code_step"]), int(rec["carr_step"])
    best = 0
    for d in ds:
        c = S.sums(I, Q, int(res_row["prn"]), K, phi, u, w)
        e = sum(int(a) * int(a) + int(b) * int(b) for a, b in zip(c["ei"], c["eq"]))
        l_ = sum(int(a) * int(a) + int(b) * int(b) for a, b in zip(c["li"], c["lq"]))
        best = max(best, e + l_)
        phi = (phi + d * S.GAIN) % S.M
    return best
