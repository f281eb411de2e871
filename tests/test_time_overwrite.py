"""`-s now`: the reference's ephemeris and UTC time overwrite (gps.c:2531-2561) in the scenario engine, against runs of
the unmodified reference producer with time_overwrite set (tests/golden/make_golden_now.py): slot occupancy, NAV
position, every double bit for bit, every NAV frame -- subframe 4 page 18 with the overwritten WNt / tot included --
for a start on another date, a week roll and an ephemeris roll; the incremental engine; the errors; the almanac
check against the moved start; the CLI's start options."""
import datetime
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import scenario
from scenario import gps
from test_interactive import assert_params_equal
from test_scenario import make_nav

NOW = ["sky12_now_35s_i8", "sky12_now_weekroll_300s_i8", "sky12_now_ephroll_560s_i8"]
GPS_EPOCH = datetime.datetime(1980, 1, 6)


def parse_start(text):
    d, t = text.split(",")
    y, m, dd = (int(v) for v in d.split("/"))
    hh, mi, sec = t.split(":")
    return (y, m, dd, int(hh), int(mi), float(sec))


def gps_time(start):
    """the start as (week, second of week), UTC taken as GPS time like the reference"""
    dt = datetime.datetime(*start[:5]) + datetime.timedelta(seconds=start[5]) - GPS_EPOCH
    s = dt.days * 86400 + dt.seconds + dt.microseconds * 1e-6
    return int(s // 604800), s % 604800


def now_case(name, tmp_path):
    """fixture -> (golden, scenario kwargs)"""
    g = scenario.load_golden(name)
    d = tmp_path / name
    d.mkdir()
    loc = g["location"]
    kw = dict(nav_file=make_nav(d, 12, sets=int(g["sets"])), lat=loc[0], lon=loc[1], height=loc[2],
              seconds=float(g["seconds"]), max_chan=int(g["max_chan"]), start=parse_start(str(g["start"])))
    return g, kw


def page18(words):
    """(tot / 4096, WNt mod 256) of a channel's NAV words if its subframe 4 is page 18 (SV id 56), else None"""
    def data(k):                     # the 24 data bits of word k, D30* of the previous word undone
        d = (int(words[k]) >> 6) & 0xFFFFFF
        return d ^ 0xFFFFFF if int(words[k - 1]) & 1 else d
    if (data(40 + 1) >> 2) & 0x7 != 4 or (data(40 + 2) >> 16) & 0x3F != 56:
        return None
    w = data(40 + 7)
    return (w >> 8) & 0xFF, w & 0xFF


@pytest.mark.parametrize("name", NOW)
def test_engine_equals_the_reference_time_overwrite(name, tmp_path):
    g, kw = now_case(name, tmp_path)
    info = {}
    got, nav = gps.scenario(**kw, time_overwrite=True, info=info)
    assert info["start_date"] == str(g["start"])
    prn = g["prn_of_block"].astype(np.int32)
    assert got.shape == prn.shape and np.array_equal(got["prn"], prn)
    assert (prn[0] > 0).sum() >= 8
    idx = g["chans_idx"] if "chans_idx" in g else np.arange(prn.shape[0])
    assert_params_equal(got[idx], g["chans"], idx)
    # allocation carrier phase of every slot's first block (allocateChannel, gps.c:2203-2210)
    first = (prn > 0) & np.vstack([np.ones((1, prn.shape[1]), bool), prn[1:] != prn[:-1]])
    for k, b in enumerate(idx):
        assert np.array_equal(got["carr_phase"][b][first[b]].view(np.uint64),
                              g["chans"]["carr_phase"][k][first[b]].view(np.uint64)), b
    frames, fidx = g["nav_frames"], g["nav_frame_of_block"]
    assert np.array_equal(got["nav_frame"][:, 0], fidx) and len(nav) == len(frames)
    for b in range(prn.shape[0]):
        assert np.array_equal(nav[fidx[b]][prn[b] > 0], frames[fidx[b]][prn[b] > 0]), b
    if name == "sky12_now_ephroll_560s_i8":
        # page 18 is transmitted, with WNt / tot of the start's 2-hour epoch rather than the file's (61440 s, 2296)
        week, sow = gps_time(kw["start"])
        want = ((int(sow) // 7200 * 7200 // 4096) & 0xFF, week % 256)
        seen = [page18(frames[f][c]) for f in range(len(frames)) for c in range(frames.shape[1])
                if frames[f][c].any()]
        assert want in seen and (61440 // 4096, 2296 % 256) not in seen


@pytest.mark.parametrize("name", NOW[:2])
def test_incremental_engine_equals_the_batch_engine(name, tmp_path):
    g, kw = now_case(name, tmp_path)
    want, wnav = gps.scenario(**kw, time_overwrite=True)
    args = {k: v for k, v in kw.items() if k not in ("nav_file", "lat", "lon", "height", "seconds")}
    for chunk in (1, 7, 300):
        with gps.LiveScenario(kw["nav_file"], kw["lat"], kw["lon"], kw["height"], kw["seconds"], time_overwrite=True,
                              **args) as s:
            assert s.start_date == str(g["start"])
            got, nav = s.run([], chunk=chunk)
        assert got.tobytes() == want.tobytes() and nav.tobytes() == wnav.tobytes(), chunk


def test_incremental_engine_across_the_ephemeris_roll(tmp_path):
    g, kw = now_case("sky12_now_ephroll_560s_i8", tmp_path)
    want, wnav = gps.scenario(**kw, time_overwrite=True)
    args = {k: v for k, v in kw.items() if k not in ("nav_file", "lat", "lon", "height", "seconds")}
    with gps.LiveScenario(kw["nav_file"], kw["lat"], kw["lon"], kw["height"], kw["seconds"], time_overwrite=True,
                          **args) as s:
        got, nav = s.run([], chunk=300)
    assert got.tobytes() == want.tobytes() and nav.tobytes() == wnav.tobytes()


def test_interactive_run_without_keys_equals_the_static_run(tmp_path):
    _, kw = now_case("sky12_now_35s_i8", tmp_path)
    want, wnav = gps.scenario(**kw, time_overwrite=True)
    got, nav = gps.scenario(**kw, time_overwrite=True, steer=[])
    assert got.tobytes() == want.tobytes() and nav.tobytes() == wnav.tobytes()


def test_without_the_overwrite_a_start_far_from_the_file_is_refused(tmp_path):
    _, kw = now_case("sky12_now_35s_i8", tmp_path)
    with pytest.raises(gps.GpsB200Error, match="outside the ephemeris span"):
        gps.scenario(**kw)


def test_second_hour_start_with_one_set_has_no_current_set(tmp_path):
    nav_file = make_nav(tmp_path, 12)
    with pytest.raises(gps.GpsB200Error, match="no current set of ephemerides") as e:
        gps.scenario(nav_file, 35.681298, -14.586874, 10.0, 2, start=(2026, 10, 15, 13, 34, 56.0), time_overwrite=True)
    assert e.value.code == -1
    # the last second of the first hour still selects the set
    gps.scenario(nav_file, 35.681298, -14.586874, 10.0, 2, start=(2026, 10, 15, 12, 59, 59.0), time_overwrite=True)


@pytest.mark.parametrize("start", [None, (1980, 6, 1, 0, 0, 0.0), (2026, 0, 15, 0, 0, 0.0), (2026, 13, 15, 0, 0, 0.0),
                                   (2026, 10, 0, 0, 0, 0.0), (2026, 10, 32, 0, 0, 0.0), (2026, 10, 15, -1, 0, 0.0),
                                   (2026, 10, 15, 24, 0, 0.0), (2026, 10, 15, 0, -1, 0.0), (2026, 10, 15, 0, 60, 0.0),
                                   (2026, 10, 15, 0, 0, -0.5), (2026, 10, 15, 0, 0, 60.0)])
def test_start_missing_or_out_of_range_is_an_argument_error(start, tmp_path):
    nav_file = make_nav(tmp_path, 12)
    for live in (False, True):
        with pytest.raises(gps.GpsB200Error, match="invalid date and time") as e:
            if live:
                gps.LiveScenario(nav_file, 35.0, 139.0, 10.0, 2, start=start, time_overwrite=True)
            else:
                gps.scenario(nav_file, 35.0, 139.0, 10.0, 2, start=start, time_overwrite=True)
        assert e.value.code == -1


def _sem(tmp_path, *args):
    sem = tmp_path / ("alm%d.sem" % len(list(tmp_path.iterdir())))
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_sem.py"), "--out", str(sem)] +
                          [str(a) for a in args])
    return str(sem)


def test_almanac_time_is_checked_against_the_moved_start(tmp_path):
    _, kw = now_case("sky12_now_35s_i8", tmp_path)
    week, _ = gps_time(kw["start"])
    for dweek, toa in ((0, 389120), (-3, 0), (4, 61440)):        # within 4 weeks of 2026/10/15,12:34:56
        info = {}
        gps.scenario(**kw, almanac_file=_sem(tmp_path, "--week", (week + dweek) % 1024, "--toa", toa),
                     time_overwrite=True, info=info)
        when = GPS_EPOCH + datetime.timedelta(weeks=week + dweek, seconds=toa)
        assert info["almanac_date"] == when.strftime("%Y/%m/%d,%H:%M:%S")
    for dweek, toa in ((-5, 0), (4, 389120 - 2096 + 4096)):      # more than 4 weeks away
        with pytest.raises(gps.GpsB200Error, match="invalid time of almanac"):
            gps.scenario(**kw, almanac_file=_sem(tmp_path, "--week", (week + dweek) % 1024, "--toa", toa),
                         time_overwrite=True)
    # the file's own (2024) almanac is not moved with the ephemerides
    with pytest.raises(gps.GpsB200Error, match="invalid time of almanac"):
        gps.scenario(**kw, almanac_file=_sem(tmp_path), time_overwrite=True)


def test_start_date_is_reported_for_every_start(tmp_path):
    nav_file = make_nav(tmp_path, 12, sets=2)
    for start, want in ((None, "2024/01/07,02:00:00"), ((2024, 1, 7, 2, 30, 15.0), "2024/01/07,02:30:15")):
        info = {}
        gps.scenario(nav_file, 35.681298, 139.766247, 10.0, 2, start=start, info=info)
        assert info["start_date"] == want
        with gps.LiveScenario(nav_file, 35.681298, 139.766247, 10.0, 2, start=start) as s:
            assert s.start_date == want


def _sim():
    exe = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "gpsb200-sim")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "csrc")])
    return exe


def test_cli_start_options(tmp_path):
    """-s checks its date as the reference does, --now needs -s now, and every run reports its start (printed once the
    scenario is open, before any GPU work)"""
    nav_file, out = make_nav(tmp_path, 12), str(tmp_path / "iq.bin")
    base = [_sim(), "-e", nav_file, "-l", "35.681298,-14.586874,10.0", "-d", "1", "-o", out]

    def run(*args):
        return subprocess.run(base + list(args), capture_output=True, text=True)

    for bad in (["-s", "2026/10/15"], ["-s", "yesterday"], ["-s", "1980/01/06,00:00:00"], ["-s", "2026/10/15,24:00:00"],
                ["--now", "2026/10/15,12:34:56"], ["-s", "now", "--now", "2026/10/15"],
                ["-s", "now", "--now", "2026/10/15,12:34:60"]):
        r = run(*bad)
        assert r.returncode == 2 and "gpsb200-sim:" in r.stderr, (bad, r.stderr)
    r = run("-s", "now", "--now", "2026/10/15,12:34:56")
    assert "gpsb200-sim: start time: 2026/10/15,12:34:56 (week 2440, sow 390896)\n" in r.stderr, r.stderr
    r = run("-s", "2024/01/07,02:00:00")
    assert "gpsb200-sim: start time: 2024/01/07,02:00:00 (week 2296, sow 7200)\n" in r.stderr, r.stderr
    r = run()
    assert "gpsb200-sim: start time: 2024/01/07,02:00:00 (week 2296, sow 7200)\n" in r.stderr, r.stderr
    r = run("-s", "now", "--now", "2026/10/15,13:34:56")
    assert r.returncode == 1 and "no current set of ephemerides" in r.stderr, r.stderr
    # the clock: a start within seconds of this process's UTC time (two sets: one is current at any time of day)
    two = tmp_path / "two"
    two.mkdir()
    base[2] = make_nav(two, 12, sets=2)
    t0 = datetime.datetime.now(datetime.timezone.utc).replace(tzinfo=None)
    r = run("-s", "now")
    m = re.search(r"start time: (\S+) \(week (\d+), sow ([\d.]+)\)", r.stderr)
    assert m, r.stderr
    printed = datetime.datetime.strptime(m.group(1), "%Y/%m/%d,%H:%M:%S")
    assert abs((printed - t0).total_seconds()) < 5
    assert (int(m.group(2)), float(m.group(3))) == gps_time(parse_start(m.group(1)))
