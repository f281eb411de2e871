"""Almanac pages from a SEM file (scenario engine, host only): the SEM reader against the reference's parser for every
edge file, the NAV frames against the reference's dumps with its almanac enabled, the 4-week time check, and the
public interface around it."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import scenario
from scenario import gps

LOC = (35.681298, 139.766247, 10.0)
LOC60 = (60.0, 140.0, 0.0)
START = (2024, 1, 7, 2, 0, 0.0)
# the edge files of tests/golden/sem_edges.npz and the oracle/gen_sem.py options that write them
SEM_EDGES = {"full": [], "truncated": ["--truncate", "1"], "truncated_prn9": ["--truncate", "9"], "malformed": ["--malformed"],
             "bad_ids": ["--bad-ids"], "duplicate": ["--duplicate"], "full_week": ["--full-week"]}
INT_FIELDS = ("svid", "svn", "ura", "health", "config_code", "valid", "toa_week")
DOUBLE_FIELDS = ("e", "delta_i", "omegadot", "sqrta", "omega0", "aop", "m0", "af0", "af1", "toa_sec")


def make_nav(tmp_path, nsat):
    nav = tmp_path / ("sky%d.nav" % nsat)
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nsat),
                           "--out", str(nav)])
    return str(nav)


def make_sem(tmp_path, args=(), name="almanac.sem"):
    sem = tmp_path / name
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_sem.py"), "--out", str(sem)] + list(args))
    return str(sem)


def page_svids(words):
    """SV ids of the subframe 4 and subframe 5 pages in one channel's 60 NAV words (word 3 of each subframe, data bits
    un-complemented by D30* of the word before)."""
    def data(k):
        d = (int(words[k]) >> 6) & 0xFFFFFF
        return d ^ 0xFFFFFF if int(words[k - 1]) & 1 else d
    return (data(42) >> 16) & 0x3F, (data(52) >> 16) & 0x3F


@pytest.mark.parametrize("edge", list(SEM_EDGES))
def test_sem_reader_equals_reference_parser(edge, tmp_path):
    """gpsb200_almanac_read against what the reference's almanac.c read from the same text; doubles bit for bit."""
    g = scenario.load_golden("sem_edges")
    path = tmp_path / "edge.sem"
    path.write_bytes(g["text_" + edge].tobytes())
    valid, rec = gps.almanac_read(str(path))
    assert valid == bool(g["valid_" + edge])
    ints = np.stack([rec[f] for f in INT_FIELDS], axis=1)
    assert np.array_equal(ints, g["ints_" + edge])
    dbl = np.stack([rec[f] for f in DOUBLE_FIELDS], axis=1)
    assert np.array_equal(dbl.view(np.uint64), g["doubles_" + edge].view(np.uint64))


def test_sem_edge_files_cover_what_they_are_for():
    g = scenario.load_golden("sem_edges")
    full, dup, ids = g["ints_full"], g["ints_duplicate"], g["ints_bad_ids"]
    assert (full[:, 5] == 1).all() and (full[:, 0] == np.arange(1, 33)).all()      # all 32 PRNs, all complete
    assert full[4, 1] == 0                                                          # the blank SVN line (PRN 5)
    d = g["doubles_full"]
    for k in (1, 7, 8):                                                             # delta_i, af0, af1: both signs
        assert (d[:, k] < 0).any() and (d[:, k] > 0).any()
    assert (d[:, 2] < 0).all()                                                      # omegadot
    assert g["valid_truncated"] == 0 and g["ints_truncated"][0, 0] == 1 and g["ints_truncated"][0, 5] == 0
    assert g["ints_truncated_prn9"][8, 0] == 9 and g["ints_truncated_prn9"][8, 5] == 0 and g["ints_truncated_prn9"][7, 5] == 1
    assert g["valid_malformed"] == 0 and not g["ints_malformed"].any()              # the whole almanac dropped
    assert not np.array_equal(g["doubles_duplicate"][6], g["doubles_full"][6])     # PRN 7 overwritten
    assert dup[31, 0] == 0                                                          # 33 announced, 32 read
    assert np.array_equal(ids[:, 0], np.arange(1, 33))                              # id 0 -> 1, id 40 -> 32
    assert (g["ints_full_week"][:, 6] == 2296 + 2048).all()


@pytest.mark.parametrize("edge", list(SEM_EDGES))
def test_gen_sem_writes_the_fixture_texts(edge, tmp_path):
    """The GPU tests write their SEM files with oracle/gen_sem.py: it must give the texts the fixtures were made from."""
    g = scenario.load_golden("sem_edges")
    with open(make_sem(tmp_path, SEM_EDGES[edge]), "rb") as f:
        assert f.read() == g["text_" + edge].tobytes()


LONG = {"sky12_alm_static_780s_i8": dict(nsat=12, loc=LOC, secs=780),
        "sky32_alm_lat60_310s_i8": dict(nsat=32, loc=LOC60, secs=310)}


@pytest.mark.parametrize("name", list(LONG))
def test_long_runs_nav_frames_equal_reference_dump(name, tmp_path):
    """Every NAV frame of every slot, slot occupancy of every block and the frame index of every block equal the
    reference's dump with its almanac enabled."""
    cfg = LONG[name]
    g = scenario.load_golden(name)
    info = {}
    ch, nav = gps.scenario(make_nav(tmp_path, cfg["nsat"]), *cfg["loc"], seconds=cfg["secs"], max_chan=cfg["nsat"], start=START,
                           almanac_file=make_sem(tmp_path), info=info)
    assert info["almanac_date"] == "2024/01/07,02:16:32"                # toa 8192 s of week 2296
    assert np.array_equal(ch["prn"], g["prn_of_block"].astype(np.int32))
    assert np.array_equal(ch["nav_frame"][:, 0], g["nav_frame_of_block"])
    frames = g["nav_frames"]
    assert nav.shape == frames.shape
    # slots that hold a satellite in the frame (the dump keeps an idle slot's last words, the engine zeroes them)
    first_block = np.searchsorted(g["nav_frame_of_block"], np.arange(len(frames)))
    act = g["prn_of_block"][first_block] > 0
    assert np.array_equal(nav[act], frames[act])
    # the fixture covers what it is for: a whole 25-page rotation in one slot, almanac pages in subframe 4 and 5
    sv4 = {c: set() for c in range(nav.shape[1])}
    sv5 = {c: set() for c in range(nav.shape[1])}
    for f in range(nav.shape[0]):
        for c in range(nav.shape[1]):
            if act[f, c]:
                a, b = page_svids(frames[f, c])
                sv4[c].add(a)
                sv5[c].add(b)
    assert set().union(*sv4.values()) & set(range(25, 33))              # PRN 25-32 in subframe 4 pages 2-5, 7-10
    if cfg["secs"] >= 750:
        assert any(s5 >= set(range(1, 25)) | {51} for s5 in sv5.values())   # ipage 0-24: PRN 1-24 + page 25
    else:                                                                # slots reused: pages continue across reuse
        prn = g["prn_of_block"]
        assert (prn[1:] != prn[:-1]).any()


def test_truncated_record_3s_matches_reference_dump(tmp_path):
    """The SEM file ends inside PRN 1's record: no complete record (no time check, no almanac date), but the partial
    record goes into subframe 5 page 1 of the first frame and gives page 25 its toa/WNa, as in the reference."""
    g = scenario.load_golden("sky12_alm_trunc_3s_i8")
    want, frames = scenario.golden_chans(g)
    info = {}
    nav_file = make_nav(tmp_path, 12)
    got, nav = gps.scenario(nav_file, *LOC, seconds=3, max_chan=12, start=START,
                            almanac_file=make_sem(tmp_path, ["--truncate", "1"]), info=info)
    assert info["almanac_date"] is None
    act = want["prn"] > 0
    assert np.array_equal(got["prn"], want["prn"])
    for f in ("iword", "ibit", "icode", "f_carr", "f_code", "code_phase", "gain"):
        assert np.array_equal(got[f][act].view(np.uint8), want[f][act].view(np.uint8)), f
    assert np.array_equal(nav, frames)
    assert all(page_svids(nav[0, c])[1] == 1 for c in range(12))
    _, plain = gps.scenario(nav_file, *LOC, seconds=3, max_chan=12, start=START)
    assert not np.array_equal(nav, plain)


def test_malformed_file_and_no_file_give_the_frames_of_a_run_without_almanac(tmp_path):
    g = scenario.load_golden("sky12_static_10s_i8")
    nav_file = make_nav(tmp_path, 12)
    base_ch, base = gps.scenario(nav_file, *LOC, seconds=10, max_chan=12, start=START)
    assert np.array_equal(base, g["nav_frames"])
    for alm in (None, make_sem(tmp_path, ["--malformed"])):
        info = {}
        ch, nav = gps.scenario(nav_file, *LOC, seconds=10, max_chan=12, start=START, almanac_file=alm, info=info)
        assert ch.tobytes() == base_ch.tobytes() and nav.tobytes() == base.tobytes(), alm
        assert info["almanac_date"] is None


@pytest.mark.parametrize("week,toa,ok", [(252, 7200, True), (252, 7201, False), (244, 7200, True), (244, 7199, False)])
def test_almanac_time_must_be_within_4_weeks_of_the_start(week, toa, ok, tmp_path):
    """Start = week 2296, 7200 s; the file's week is read modulo 1024 (+ 2048): 252 -> 2300, 244 -> 2292."""
    nav_file = make_nav(tmp_path, 12)
    sem = make_sem(tmp_path, ["--week", str(week), "--toa", str(toa)])
    if ok:
        gps.scenario(nav_file, *LOC, seconds=2, max_chan=12, start=START, almanac_file=sem)
    else:
        with pytest.raises(gps.GpsB200Error, match="invalid time of almanac"):
            gps.scenario(nav_file, *LOC, seconds=2, max_chan=12, start=START, almanac_file=sem)


def test_full_week_number_in_the_file_is_an_error(tmp_path):
    with pytest.raises(gps.GpsB200Error, match="invalid time of almanac"):
        gps.scenario(make_nav(tmp_path, 12), *LOC, seconds=2, max_chan=12, start=START,
                     almanac_file=make_sem(tmp_path, ["--full-week"]))


def test_missing_almanac_file_is_an_error(tmp_path):
    with pytest.raises(gps.GpsB200Error, match="cannot open almanac file"):
        gps.scenario(make_nav(tmp_path, 12), *LOC, seconds=2, max_chan=12, start=START,
                     almanac_file=str(tmp_path / "missing.sem"))
    with pytest.raises(gps.GpsB200Error):
        gps.almanac_read(str(tmp_path / "missing.sem"))


def test_scenario_config_mirror_matches_the_header():
    """api.ScenarioConfig against gpsb200_scenario_config_t (the C side static_asserts the same offsets): the almanac
    field is appended, no earlier offset moves."""
    S = gps.ScenarioConfig
    want = {"nav_file": 0, "motion_file": 8, "lat_deg": 16, "lon_deg": 24, "height_m": 32, "duration_ds": 40, "max_chan": 44,
            "ionosphere_enable": 48, "pluto_gain": 52, "start_year": 56, "start_month": 60, "start_day": 64,
            "start_hour": 68, "start_min": 72, "rinex3": 76, "start_sec": 80, "target_valid": 88, "reserved": 92,
            "target_distance_m": 96, "target_bearing_deg": 104, "target_height_m": 112, "almanac_file": 120}
    assert {n: getattr(S, n).offset for n, _ in S._fields_} == want
    assert C.sizeof(S) == 128
    assert gps.ALMANAC_RECORD_DTYPE.itemsize == 112
