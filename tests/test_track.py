"""The tracking loops' numpy model (tests/track_model.py) and the navigation decoder on the CPU: the decoder's parity and
sync rules on known inputs, and the model's lock, Doppler, code and NAV-word truth on streams of the CPU oracle.

The tolerances of the truth checks are fixed here from the model and shared with the GPU tests. On the first 12.1 s of
sky12_static_35s (12 channels) and the first 3 s of sky32_static_10s (32 channels, the int8 stream wrapping), seeded
from an acquisition with 100 Hz bins, the model shows:
- pull-in: the last unlocked period is epoch 3..260 with 12 channels, 3..274 with 32; every channel stays locked after it;
- Doppler: |carr_step - f_carr| after pull-in at most 4.33 Hz at any period with 12 channels (rms 0.35-0.74 Hz), 12.92 Hz
  with 32 (rms 0.49-1.74 Hz);
- code: |signal - prompt code phase| after pull-in at most 0.094 chips at any period (both streams);
- every bit edge on a scenario bit boundary, every decoded word equal to the scenario's, TOW x 6 s minus the start
  time giving travel times of 67.7-73.0 ms (12 channels) and 67.7-80.8 ms (32).
The limits below leave a margin of about a third over those figures."""
import numpy as np
import pytest

import acq_model as A
import scenario
import track_model as T
import track_truth as TT
from scenario import gps
from test_acquire import golden_rows

PULL_MAX = 400            # epochs (ms) after the start by which every channel is locked for good
FERR_MAX = {12: 6.0, 32: 17.0}   # Hz, by channel count (cross-correlation of 31 other signals and the int8 wrap)
CERR_MAX = 0.125          # chips
ACQ = dict(ms=10, f_lo=-5000.0, step=100.0, nbins=101)  # the seed search: 100 Hz bins keep the FLL within its +-250 Hz
START_SOW = TT.gps_sow(2024, 1, 7, 2, 0, 0.0)          # the fixtures' scenario start, 2024/01/07 02:00:00
TRAVEL = (0.060, 0.090)   # s


def starts(res):
    return np.array([T.start(int(r["prn"]), float(r["doppler_hz"]), int(r["delay"])) for r in res])


def truth_figures(ch, eps, prns, frames, frame_of_block, start_sow=START_SOW, words_exact=True, ferr_max=None):
    """Check every channel's epochs against the scenario records ch (rows of consecutive blocks from sample 0): lock
    within PULL_MAX and kept, Doppler and code within FERR_MAX / CERR_MAX after it, bit edges on the scenario's bit
    boundaries, the decoded words equal to the scenario's (all of them when words_exact), TOW consistent with the
    start time. -> {prn: (pull-in epochs, max |Doppler error|, max |code error|, words, words wrong)}."""
    out = {}
    ferr_max = FERR_MAX[12 if ch.shape[1] <= 12 else 32] if ferr_max is None else ferr_max
    for prn, e in zip(prns, eps):
        assert e.size > 0, prn
        un = np.nonzero(e["lock"] == 0)[0]
        pull = int(un[-1]) + 1 if un.size else 0
        assert pull <= PULL_MAX, (prn, pull)
        cerr, ferr = TT.epoch_errors(ch, prn, e)
        fmax, cmax = float(np.abs(ferr[pull:]).max()), float(np.abs(cerr[pull:]).max())
        assert fmax <= ferr_max and cmax <= CERR_MAX, (prn, fmax, cmax)
        bits, words, sy = gps.nav_decode(e)
        assert sy["bit_edge"] >= 0, prn
        late = bits[bits["sample"] >= e["sample"][pull]]
        edges = [TT.ms_index(ch, prn, int(b["sample"]))[2] % 20 for b in late]
        assert edges.count(0) == len(edges), (prn, edges[:5])
        wrong = TT.word_failures(ch, prn, words, frames, frame_of_block)
        if words_exact:
            assert wrong == [], (prn, wrong[:3])
        for w in words:
            if w["subframe"] and w["parity_ok"]:
                s_sf = int(w["sample"]) - 1800000          # the subframe started 30 bits (0.6 s) before its HOW
                travel = (start_sow + s_sf / 3e6) - (int(w["tow"]) * 6 - 6)
                assert TRAVEL[0] <= travel <= TRAVEL[1], (prn, int(w["tow"]), travel)
        out[prn] = (pull, fmax, cmax, int(sy["nwords"]), len(wrong))
    return out


# ---- the decoder ---------------------------------------------------------------------------------------------------
def test_parity_known_answer():
    """computeChecksum(0x8B0000 << 6, 0) == 0x22C00012: the TLM word with D29* = D30* = 0."""
    assert (0x8B0000 << 6) | gps.nav_parity(0x8B0000, 0, 0) == 0x22C00012
    assert gps.nav_word_check(0x22C00012, 0) == (True, 0x8B0000)
    assert gps.nav_word_check(0x22C00012 ^ 1, 0)[0] is False


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8", "sky12_circle_60s_i16",
                                  "sky12_alm_static_780s_i8"])
def test_every_word_of_the_nav_frames_passes_parity(name):
    """Within each frame of the fixture, words 1-59 pass the decoder's parity check with their predecessor's D29*/D30*,
    and the data it returns is the word with D30* undone."""
    frames = scenario.load_golden(name)["nav_frames"]
    n = 0
    for fr in frames:
        for slot in fr:
            if not slot.any():
                continue
            for w in range(1, 60):
                word, prev = int(slot[w]) & 0x3FFFFFFF, int(slot[w - 1]) & 0x3FFFFFFF
                ok, data = gps.nav_word_check(word, prev)
                assert ok, (w, hex(word))
                assert data == ((word >> 6) ^ (0xFFFFFF if prev & 1 else 0)) & 0xFFFFFF
                n += 1
    assert n >= 59 * 12


def synthetic_epochs(bits, edge, invert=False, lock_from=0):
    """Epochs whose prompt I carries `bits` (0/1, 20 epochs each, the first bit starting at epoch `edge`), the `edge`
    epochs before it carrying the complement of the first bit."""
    n = edge + 20 * len(bits)
    e = np.zeros(n, gps.TRACK_EPOCH_DTYPE)
    v = np.repeat(np.array(bits, np.int64) * 2 - 1, 20)
    v = np.concatenate([np.full(edge, -v[0]), v]) * (-1 if invert else 1)
    e["p_i"] = v * 1000 + np.arange(n) % 7
    e["sample"] = np.arange(n) * 3000
    e["lock"] = (np.arange(n) >= lock_from).astype(np.int32)
    return e


def test_bit_sync_finds_a_known_edge():
    rng = np.random.default_rng(3)
    bits = rng.integers(0, 2, 200)
    for edge in (0, 1, 7, 19):
        _, _, sy = gps.nav_decode(synthetic_epochs(bits, edge))
        assert sy["bit_edge"] == edge
    # sign changes between unlocked epochs do not count
    e = synthetic_epochs(bits, 5, lock_from=0)
    e["lock"][:300] = 0
    e["p_i"][:300:3] *= -1
    _, _, sy = gps.nav_decode(e)
    assert sy["bit_edge"] == 5


def frame_bits(frame, slot):
    """The 300 bits of subframes 1-5 of a NAV frame as transmitted, preceded by the last 2 bits of word 9."""
    words = [int(w) & 0x3FFFFFFF for w in frame[slot]]
    out = [(words[9] >> 1) & 1, words[9] & 1]
    for w in words[10:60]:
        out += [(w >> (29 - i)) & 1 for i in range(30)]
    return out


@pytest.mark.parametrize("invert", [False, True])
def test_frame_sync_resolves_the_polarity(invert):
    g = scenario.load_golden("sky12_static_35s_i8")
    fr = g["nav_frames"][0]
    bits = [0, 1, 1, 0, 1] + frame_bits(fr, 0)
    e = synthetic_epochs(bits, 3, invert=invert)
    b, words, sy = gps.nav_decode(e)
    assert sy["frame_bit"] == 7 and sy["inverted"] == int(invert)
    assert sy["nwords"] == 50 and sy["words_ok"] == 50 and sy["subframes"] == 5
    assert [int(w["raw"]) for w in words] == [int(x) & 0x3FFFFFFF for x in fr[0][10:60]]
    assert list(words["subframe"][1::10]) == [1, 2, 3, 4, 5]
    assert sy["first_tow"] == int(words[1]["tow"])


# ---- the model -----------------------------------------------------------------------------------------------------
def test_model_cordic_table_is_the_formula():
    """The model's atan table is round(atan(2^-i) / 2 pi * 2^32); its angle is within 2^-24 turns of atan2 on inputs of
    24 bits and more (the correlator sums are that large; the contract does not scale smaller inputs up)."""
    assert T.ATAN == T.atan_table()
    rng = np.random.default_rng(5)
    mag = rng.integers(1 << 24, 1 << 58, 2000)
    ang = rng.uniform(-np.pi / 2, np.pi / 2, 2000)
    x = np.maximum((mag * np.cos(ang)).astype(np.int64), 0)
    y = (mag * np.sin(ang)).astype(np.int64)
    keep = np.maximum(x, np.abs(y)) >= 1 << 24
    want = np.arctan2(y[keep], x[keep]) / (2 * np.pi) * 2 ** 32
    assert np.all(np.abs(T.angle(x[keep], y[keep]) - want) < 256)


def test_model_truncating_division():
    assert list(T.tdiv(np.array([7, -7, 7, -7]), np.array([2, 2, -2, -2]))) == [3, -3, -3, 3]


def test_track_start_is_the_model():
    """gpsb200_track_start (the library's start steps, which the snapshot measurement also seeds from) equals the
    model's start state at Dopplers across +-10 kHz: whole and fractional Hz, both signs, the range's ends."""
    rng = np.random.default_rng(11)
    dopplers = np.concatenate([np.linspace(-10000.0, 10000.0, 801), rng.uniform(-10000.0, 10000.0, 400),
                               [-0.4, 0.4, -1e-9, 0.0]])
    for i, f in enumerate(dopplers):
        prn, sample = 1 + i % 32, 7919 * i
        got, want = gps.track_start(prn, f, sample), T.start(prn, f, sample)
        assert all(got[k] == want[k] for k in T.STATE_DTYPE.names), (f, got, want)


def model_run(name, nblk):
    g = scenario.load_golden(name)
    ch = golden_rows(g, range(nblk))
    ss = int(g["sample_size"])
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], ss)
    assert np.array_equal(scenario.crc_blocks(iq), g["crcs"][:nblk, 0])
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    res = A.search(iq[:2 * A.CODE * 13], ss, 0, ACQ["ms"], prns, ACQ["f_lo"], ACQ["step"], ACQ["nbins"])
    eps, _ = T.track(iq, ss, 0, starts(res))
    return g, ch, prns, eps


def test_model_truth_sky12_static_12s():
    """12.1 s, 12 channels: two subframes and more per channel, so frame sync and TOW run on the CPU (20 words each)."""
    g, ch, prns, eps = model_run("sky12_static_35s_i8", 121)
    fig = truth_figures(ch, eps, prns, g["nav_frames"], g["nav_frame_of_block"])
    assert all(v[3] >= 20 for v in fig.values()), fig


def test_model_truth_sky32_static_3s():
    """3 s, 32 channels, the int8 stream wrapping: lock, Doppler, code, and the 4 words each channel decodes."""
    g, ch, prns, eps = model_run("sky32_static_10s_i8", 30)
    fig = truth_figures(ch, eps, prns, g["nav_frames"], g["nav_frame_of_block"])
    assert all(v[3] >= 4 for v in fig.values()), fig
