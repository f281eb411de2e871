"""The almanac read back from the navigation message and the sky predicted from it (host only): gpsb200_nav_almanac on
the scenario engine's frames and on hand-built pages, gpsb200_almanac_predict against tests/almanac_model.py, and the
predicted Doppler and elevation of every allocated channel against the engine's records."""
import math

import numpy as np
import pytest

import almanac_model as AM
from scenario import gps
from test_almanac import LOC, LOC60, START, make_nav, make_sem
from test_ephemeris_terms import word

WEEK, SOW0 = 2296, 7200.0          # START as GPS time
WNA = WEEK % 256
FIELDS = list(AM.FIELDS)


def slot_words(nav, c, frames):
    """The word records of channel slot c over the given frames, one run of indices (a frame's first 10 words repeat
    the previous frame's last subframe, which is harmless: the last page wins)."""
    recs = [gps.nav_words_of_frame(nav[f, c]) for f in frames]
    out = np.concatenate(recs) if recs else np.zeros(0, gps.NAV_WORD_DTYPE)
    out["index"] = np.arange(out.size)
    return out


def active_frames(ch, nav, c):
    """Frames in which slot c holds a satellite, in order."""
    blk = np.searchsorted(ch["nav_frame"][:, 0], np.arange(nav.shape[0]))
    blk = np.minimum(blk, ch.shape[0] - 1)
    return [f for f in range(nav.shape[0]) if ch["prn"][blk[f], c] > 0]


def assert_record_is_engine_integer(got, sem, near=True):
    """Every field of a decoded record is the engine's trunc(SEM / literal) integer x 2^-k and (near) within one LSB of
    SEM."""
    for f in FIELDS:
        lsb = AM.FIELDS[f][2]
        n = got[f] / lsb
        assert n == int(n), (f, got[f])
        assert int(n) == AM.engine_integer(f, float(sem[f])), (f, int(n), float(sem[f]))
        assert not near or abs(got[f] - sem[f]) <= lsb, (f, got[f], sem[f])
    assert got["toa_sec"] == sem["toa_sec"] and got["health"] == 0
    assert got["svn"] == got["ura"] == got["config_code"] == 0 and got["valid"] == 1


RUNS = {"sky12_alm_static_780s": dict(nsat=12, loc=LOC, secs=780), "sky32_alm_lat60_310s": dict(nsat=32, loc=LOC60, secs=310)}


@pytest.mark.parametrize("name", list(RUNS))
def test_engine_frames_decode_to_the_sem_almanac(name, tmp_path):
    cfg = RUNS[name]
    sem_path = make_sem(tmp_path)
    ch, nav = gps.scenario(make_nav(tmp_path, cfg["nsat"]), *cfg["loc"], seconds=cfg["secs"], max_chan=cfg["nsat"],
                           start=START, almanac_file=sem_path)
    _, sem = gps.almanac_read(sem_path)
    covered = []
    for c in range(nav.shape[1]):
        rec, wna = gps.nav_almanac(slot_words(nav, c, active_frames(ch, nav, c)), WEEK)
        got = {int(r["svid"]) for r in rec if r["svid"]}
        for prn in got:
            assert_record_is_engine_integer(rec[prn - 1], sem[prn - 1])
            assert rec[prn - 1]["toa_week"] == (sem[prn - 1]["toa_week"] if wna >= 0 else -1)
        assert wna in (-1, WNA)
        for r in rec:
            if not r["svid"]:
                assert not r.tobytes().strip(b"\0")
        covered.append(got)
    if cfg["secs"] >= 750:
        assert any(g == set(range(1, 33)) for g in covered)      # a whole 25-page rotation in one slot: all 32 PRNs
    else:
        assert set().union(*covered) & set(range(25, 33)) and set().union(*covered) & set(range(1, 25))


def test_literal_scales_round_one_lsb_apart_only_next_to_a_multiple(tmp_path):
    """The quirk the decode tolerates: the engine's literal 2^-23 and 2^-38 scales are 2.6e-15 and 8.7e-16 relative
    below the powers of two, so trunc(SEM / literal) exceeds trunc(SEM / 2^-k) by one LSB only for a value just below
    a multiple of the LSB. No field of the generated SEM file lands there; a constructed one does."""
    _, sem = gps.almanac_read(make_sem(tmp_path))
    for r in sem:
        for f in FIELDS:
            assert AM.engine_integer(f, float(r[f])) == math.trunc(float(r[f]) / AM.FIELDS[f][2]), f
    v = np.nextafter(3_000_000 * 2.0 ** -23, 0.0)
    assert math.trunc(v / 2.0 ** -23) == 2_999_999 and AM.engine_integer("aop", v) == 3_000_000


def test_truncated_record_decodes_as_sent_and_no_almanac_decodes_nothing(tmp_path):
    nav_file = make_nav(tmp_path, 12)
    sem_path = make_sem(tmp_path, ["--truncate", "1"])
    ch, nav = gps.scenario(nav_file, *LOC, seconds=3, max_chan=12, start=START, almanac_file=sem_path)
    _, sem = gps.almanac_read(sem_path)
    assert sem[0]["svid"] == 1 and sem[0]["valid"] == 0
    for c in range(12):
        rec, wna = gps.nav_almanac(slot_words(nav, c, [0]), WEEK)
        assert [int(r["svid"]) for r in rec if r["svid"]] == [1]
        # the cut line's partial number (OMEGA0 8.2235 semicircles, its exponent cut off) is sent modulo 2^24
        assert_record_is_engine_integer(rec[0], sem[0], near=False)
        assert rec[0]["m0"] == rec[0]["af0"] == rec[0]["af1"] == 0.0
        assert wna == -1 and rec[0]["toa_week"] == -1            # page 25 (WNa) is not in the first frame
    _, plain = gps.scenario(nav_file, *LOC, seconds=35, max_chan=12, start=START)
    for c in range(12):
        rec, _ = gps.nav_almanac(slot_words(plain, c, range(plain.shape[0])), WEEK)
        assert not rec["svid"].any()


# ---- hand-built pages (IS-GPS-200 20.3.3.5.1.2, Figure 20-1 sheets 4 and 5), parity computed here ----------------
def m(x, b):
    return x & ((1 << b) - 1)


def page(sf, svid, v, data_id=1):
    """10 words of an almanac page (or with svid 51, the toa / WNa page) from integer fields v."""
    d = [0] * 10
    d[0] = 0x8B << 16
    d[1] = (m(4000 + sf, 17) << 7) | (sf << 2)
    if svid == 51:
        d[2] = (data_id << 22) | (51 << 16) | (v["toa"] << 8) | v["wna"]
    else:
        d[2] = (data_id << 22) | (svid << 16) | m(v["e"], 16)
        d[3] = (v["toa"] << 16) | m(v["delta_i"], 16)
        d[4] = (m(v["omegadot"], 16) << 8) | v["health"]
        d[5] = m(v["sqrta"], 24)
        d[6] = m(v["omega0"], 24)
        d[7] = m(v["aop"], 24)
        d[8] = m(v["m0"], 24)
        af0 = m(v["af0"], 11)
        d[9] = ((af0 >> 3) << 16) | (m(v["af1"], 11) << 5) | ((af0 & 7) << 2)
    return d


def words_of(pages):
    out, prev = [], 0
    for d in [x for p in pages for x in p]:
        w = word(d, prev)
        out.append(w)
        prev = w
    recs = gps.nav_words_of_frame(np.array(out, np.uint32))
    assert recs["parity_ok"].all()
    return recs


BASE = dict(e=12345, toa=147, delta_i=-1000, omegadot=-700, health=0x2A, sqrta=10_555_000, omega0=-4_000_000,
            aop=3_000_000, m0=-123_456, af0=-300, af1=17)
SIGNED = {f: AM.FIELDS[f][0] for f in FIELDS if AM.FIELDS[f][1]}


@pytest.mark.parametrize("field", list(SIGNED))
def test_hand_built_pages_decode_each_signed_field_at_its_limits(field):
    bits = SIGNED[field]
    for x in (-(1 << (bits - 1)), -1, 0, 1, (1 << (bits - 1)) - 1):
        v = dict(BASE, **{field: x})
        rec, wna = gps.nav_almanac(words_of([page(5, 7, v), page(5, 51, dict(toa=147, wna=250))]), 2300)
        r = rec[6]
        assert r["svid"] == 7 and r["valid"] == 1 and wna == 250
        assert r[field] == x * AM.FIELDS[field][2], (field, x)
        for f in FIELDS:
            if f != field:
                assert r[f] == BASE[f] * AM.FIELDS[f][2], f
        assert r["toa_sec"] == 147 * 4096.0 and r["health"] == 0x2A
        assert r["toa_week"] == 2298                   # WNa 250 nearest week 2300 (2300 % 256 = 252)
        assert rec["svid"].tolist().count(0) == 31


def test_hand_built_pages_subframe_4_last_page_wins_week_resolution_and_rejects():
    a, b = dict(BASE), dict(BASE, m0=999)
    pages = [page(4, 25, a), page(4, 32, a), page(4, 25, b), page(5, 0, a), page(5, 3, a, data_id=2),
             page(5, 51, dict(toa=1, wna=3))]
    rec, wna = gps.nav_almanac(words_of(pages), 2300)
    assert sorted(int(s) for s in rec["svid"] if s) == [25, 32]
    assert rec[24]["m0"] == 999 * 2.0 ** -23 and rec[31]["m0"] == BASE["m0"] * 2.0 ** -23
    assert wna == 3 and rec[24]["toa_week"] == 2307            # 3 = 2307 % 256, within +-128 of 2300
    rec, _ = gps.nav_almanac(words_of(pages), 2100)
    assert rec[24]["toa_week"] == 2051                          # 2051 % 256 = 3, 49 weeks before 2100
    rec, _ = gps.nav_almanac(words_of(pages), 2180)
    assert rec[24]["toa_week"] == 2307                          # +127 rather than -129
    w = words_of(pages)
    w["parity_ok"][15] = 0                                      # the second page fails: PRN 32 not decoded
    rec, _ = gps.nav_almanac(w, 2300)
    assert sorted(int(s) for s in rec["svid"] if s) == [25]
    assert not gps.nav_almanac(np.zeros(0, gps.NAV_WORD_DTYPE), 2300)[0]["svid"].any()
    out = np.zeros(32, gps.ALMANAC_RECORD_DTYPE)
    L = gps.lib()
    assert L.gpsb200_nav_almanac(None, 10, 2300, out.ctypes.data, None) == -1          # NULL words with n > 0
    assert L.gpsb200_nav_almanac(w.ctypes.data, w.size, 2300, None, None) == -1        # NULL records
    assert L.gpsb200_nav_almanac(w.ctypes.data, -1, 2300, out.ctypes.data, None) == -1


# ---- prediction ----------------------------------------------------------------------------------------------------
def sem_almanac(tmp_path, args=()):
    return gps.almanac_read(make_sem(tmp_path, args))[1]


def test_predict_equals_the_model(tmp_path):
    rec = sem_almanac(tmp_path)
    rec[3]["valid"] = 0                                         # not predicted
    rng = np.random.default_rng(5)
    for loc, dt in ((LOC, 0.0), (LOC60, 3600.0), ((-34.0, -58.0, 20.0), -86400.0 * 3), ((89.9, 10.0, 0.0), 7.5)):
        x = AM.llh_to_ecef(*loc) + rng.normal(0, 1000, 3)
        sky = gps.almanac_predict(rec, WEEK, SOW0 + dt, x)
        want = AM.predict(rec, WEEK, SOW0 + dt, x)
        assert sorted(want) == [int(s["prn"]) for s in sky if s["valid"]]
        assert (sky["prn"] == np.arange(1, 33)).all() and sky[3]["valid"] == 0
        for s in sky[sky["valid"] == 1]:
            el, az, rng_m, dop = want[int(s["prn"])]
            assert abs(s["doppler_hz"] - dop) <= 1e-6 and abs(s["el_deg"] - el) <= 1e-9
            assert min(abs(s["az_deg"] - az), 360 - abs(s["az_deg"] - az)) <= 1e-9
            assert abs(s["range_m"] - rng_m) <= 1e-3
    with pytest.raises(gps.GpsB200Error):
        gps.almanac_predict(rec, WEEK, float("nan"), x)


# |predicted Doppler - f_carr| over every allocated channel, with the a-priori on the truth and 50 km east + 1 km up and
# 10 s late. The generated SEM file's delta_i is 0.01 semicircles (1.8 deg) off the RINEX orbits' inclination
# (oracle/gen_sem.py gives the field both signs that way), and that dominates. Measured, truth / offset: 60.7 / 79.6 Hz
# on sky12 35 s, 145.9 / 136.2 Hz on sky32 10 s, 129.3 / 118.4 Hz on sky32 at 60 deg N 310 s; lowest predicted
# elevation of an allocated PRN -0.48 / -0.71 deg (60 deg N).
PREDICT_CASES = {"sky12_static_35s": (12, LOC, 35), "sky32_static_10s": (32, LOC, 10), "sky32_lat60_310s": (32, LOC60, 310)}
DOPPLER_BOUND_HZ = 200.0
MASK_DEG = -5.0


def prediction_errors(tmp_path, nsat, loc, secs, offset):
    rec = sem_almanac(tmp_path)
    ch, _ = gps.scenario(make_nav(tmp_path, nsat), *loc, seconds=secs, max_chan=nsat, start=START)
    x = AM.llh_to_ecef(*loc)
    if offset:
        lat, lon = math.radians(loc[0]), math.radians(loc[1])
        east = np.array([-math.sin(lon), math.cos(lon), 0.0])
        up = np.array([math.cos(lat) * math.cos(lon), math.cos(lat) * math.sin(lon), math.sin(lat)])
        x = x + 50e3 * east + 1e3 * up
    worst, low = 0.0, 90.0
    for b in list(range(0, ch.shape[0], 10)) + [ch.shape[0] - 1]:
        sky = gps.almanac_predict(rec, WEEK, SOW0 + 0.1 * b + (10.0 if offset else 0.0), x)
        for r in ch[b]:
            if r["prn"] > 0:
                s = sky[r["prn"] - 1]
                assert s["valid"] == 1
                worst = max(worst, abs(s["doppler_hz"] - float(r["f_carr"])))
                low = min(low, float(s["el_deg"]))
    return worst, low


@pytest.mark.parametrize("offset", [False, True], ids=["on_truth", "50km_10s_off"])
@pytest.mark.parametrize("name", list(PREDICT_CASES))
def test_predicted_doppler_and_elevation_of_every_allocated_channel(name, offset, tmp_path):
    nsat, loc, secs = PREDICT_CASES[name]
    worst, low = prediction_errors(tmp_path, nsat, loc, secs, offset)
    assert worst <= DOPPLER_BOUND_HZ, worst
    assert low >= MASK_DEG, low
