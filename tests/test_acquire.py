"""The acquisition search's numpy model (tests/acq_model.py) on the CPU: its FFT path against the defining sum, its code
generator against the reference's codes, and the truth checks on streams of the CPU oracle.

The thresholds of the truth checks are fixed here from the model and shared with the GPU tests. On every block the
tests search, present PRNs reach P1/P2 >= 3.33 (the 27-32 channel blocks of sky32_static and sky32_lat60; about 14 or
more with 12 channels) and absent PRNs stay at or below 1.63: R_PRESENT = 3.0 and R_ABSENT = 2.0 leave a factor 1.5
between them and at least 10 % to what the model sees on either side."""
import zlib

import numpy as np
import pytest

import acq_model as M
import scenario
from scenario import gps

R_PRESENT = 3.0
R_ABSENT = 2.0
K = 10
F_LO, STEP, NBINS = -5000.0, 250.0, 41
ALL = list(range(1, 33))


def golden_rows(g, blocks):
    """Channel records of the fixture's blocks `blocks` (consecutive) as CHAN_DTYPE rows, with their NAV frame index;
    fixtures that keep only some blocks list them in chans_idx."""
    idx = g["chans_idx"] if "chans_idx" in g.files else np.arange(g["chans"].shape[0])
    pos = [int(np.nonzero(idx == b)[0][0]) for b in blocks]
    rec = g["chans"][pos]
    ch = np.zeros(rec.shape, gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = rec[f]
    ch["nav_frame"] = g["nav_frame_of_block"][list(blocks)][:, None]
    return ch


def test_model_codes_are_the_reference_codes():
    g = scenario.load_golden("sky32_static_10s_i8")
    for i, prn in enumerate(g["code_prns"]):
        assert np.array_equal(M.ca_code(int(prn)), g["codes"][i]), prn


def test_model_phase_step_rounds_half_away_from_zero():
    assert M.phase_step(0.0) == 0
    assert M.phase_step(3e6 / 2 ** 32 * 2.5) == 3            # llround(2.5) = 3
    assert M.phase_step(-3e6 / 2 ** 32 * 2.5) == 2 ** 32 - 3  # llround(-2.5) = -3, modulo 2^32
    assert M.phase_step(-5000.0) == (-7158279) % 2 ** 32     # -5000 * 2^32 / 3e6 = -7158278.83


@pytest.mark.parametrize("kind", ["int8_random", "int16_extremes"])
def test_model_fft_path_equals_direct_sum(kind):
    rng = np.random.default_rng(7)
    K = 2
    n = M.CODE * K + M.CODE - 1 + 5
    if kind == "int8_random":
        iq, ss = rng.integers(-128, 128, 2 * n).astype(np.int8), 1
    else:   # +-32767 and friends: the saturating reduction clamp(x >> 4, -128, 127) at both ends
        iq, ss = rng.choice(np.array([-32768, -32767, -2049, -2048, 2047, 2048, 32767, 0], np.int16), 2 * n), 2
        I, Q = M.samples(iq, ss)
        assert I.min() == -128 and I.max() == 127
    prns, f_lo, step, nbins = [1, 17, 32], -1250.0, 625.0, 3
    a = M.grid(iq, ss, 5, K, prns, f_lo, step, nbins, method="fft")
    b = M.grid(iq, ss, 5, K, prns, f_lo, step, nbins, method="direct")
    assert a.dtype == np.uint64 and np.array_equal(a, b)


@pytest.mark.parametrize("block", [0, 50])
def test_model_truth_on_oracle_stream_sky12_static(block):
    """12 present and 20 absent PRNs: Doppler bin, code delay and P1/P2 of every one from the model on the CPU oracle's
    int8 stream of one block (the block's own record as start state; its CRC is the reference's)."""
    g = scenario.load_golden("sky12_static_10s_i8")
    ch = golden_rows(g, [block])
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], 1)
    assert zlib.crc32(iq.tobytes()) == g["crcs"][block, 0]
    res = M.search(iq, 1, 0, K, ALL, F_LO, STEP, NBINS)
    assert (ch[0]["prn"] > 0).sum() == 12
    assert M.truth_failures(res, ch[0], F_LO, STEP, R_PRESENT, R_ABSENT) == []
