"""Interactive mode (-i) on the incremental scenario engine, against the reference's own key handling: the fixtures
are runs of the reference's unmodified main with scripted keys (tests/golden/make_golden_interactive.py). Also: any
cut of a run into advances gives the batch engine's records and frames, and an opened scenario's memory does not
grow with the duration."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import scenario
from scenario import gps
from test_scenario import LOC, LOC60, START, make_nav, motion_file

STEER = ["sky12_steer_60s_i8", "sky12_steer_target_30s_i16", "sky32_lat60_steer_310s_i8"]


def steer_case(name, tmp_path):
    """fixture -> (golden, scenario kwargs, schedule)"""
    g = scenario.load_golden(name)
    opts = str(g["options"]).split()
    target = [float(v) for v in opts[opts.index("-t") + 1].split(",")] if "-t" in opts else None
    C = int(g["max_chan"])
    kw = dict(nav_file=make_nav(tmp_path, C), lat=g["location"][0], lon=g["location"][1], height=g["location"][2],
              seconds=float(g["seconds"]), max_chan=C, start=START, target=target)
    return g, kw, gps.parse_steer(str(g["schedule"]))


def assert_params_equal(got, want, blocks):
    """the comparisons of test_scenario.py: occupancy, NAV position, every double bit for bit"""
    assert np.array_equal(got["prn"], want["prn"])
    act = want["prn"] > 0
    for f in ("iword", "ibit", "icode"):
        assert np.array_equal(got[f][act], want[f][act]), f
    for f in ("f_carr", "f_code", "code_phase", "gain"):
        a, b = got[f][act].view(np.uint64), want[f][act].view(np.uint64)
        bad = np.nonzero(a != b)[0]
        assert bad.size == 0, (f, np.asarray(blocks)[np.nonzero(act)[0][bad[:5]]])


@pytest.mark.parametrize("name", STEER)
def test_steered_run_matches_the_reference_key_handling(name, tmp_path):
    g, kw, sched = steer_case(name, tmp_path)
    got, nav = gps.scenario(**kw, steer=sched)
    prn = g["prn_of_block"].astype(np.int32)
    assert got.shape == prn.shape and np.array_equal(got["prn"], prn)
    idx = g["chans_idx"] if "chans_idx" in g else np.arange(prn.shape[0])
    assert_params_equal(got[idx], g["chans"], idx)
    # allocation carrier phase of every slot's first block (allocateChannel, gps.c:2203-2210)
    first = (prn > 0) & np.vstack([np.ones((1, prn.shape[1]), bool), prn[1:] != prn[:-1]])
    for b in idx:
        k = list(idx).index(b)
        assert np.array_equal(got["carr_phase"][b][first[b]].view(np.uint64), g["chans"]["carr_phase"][k][first[b]].view(np.uint64))
    frames, fidx = g["nav_frames"], g["nav_frame_of_block"]
    assert np.array_equal(got["nav_frame"][:, 0], fidx) and len(nav) == len(frames)
    for b in range(prn.shape[0]):
        assert np.array_equal(nav[fidx[b]][prn[b] > 0], frames[fidx[b]][prn[b] > 0]), b


@pytest.mark.parametrize("name", STEER[:2])
def test_steered_run_is_the_same_for_any_cut_into_advances(name, tmp_path):
    g, kw, sched = steer_case(name, tmp_path)
    want, wnav = gps.scenario(**kw, steer=sched)
    for chunk in (1, 7, 300):
        with gps.LiveScenario(kw["nav_file"], kw["lat"], kw["lon"], kw["height"],
                              kw["seconds"], max_chan=kw["max_chan"], start=START, target=kw["target"], interactive=True) as s:
            got, nav = s.run(sched, chunk=chunk)
        assert got.tobytes() == want.tobytes() and nav.tobytes() == wnav.tobytes(), chunk


def _golden_configs(tmp_path):
    n12, n32 = make_nav(tmp_path, 12), make_nav(tmp_path, 32)
    yield "static12", dict(nav_file=n12, lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=35, start=START)
    yield "static32", dict(nav_file=n32, lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=10, max_chan=32, start=START)
    yield "motion", dict(nav_file=n12, lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=60, start=START,
                         motion_file=motion_file(tmp_path))
    yield "target", dict(nav_file=n12, lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=3, start=START,
                         target=(1500.5, 33.3, 120.25))
    v3 = tmp_path / "v3"
    v3.mkdir()
    yield "rinex3", dict(nav_file=make_nav(v3, 12, v3=True), lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=3, start=START,
                         rinex3=True)
    yield "pluto", dict(nav_file=n12, lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=3, start=START, pluto_gain=True)
    two = tmp_path / "two"
    two.mkdir()
    yield "ephroll", dict(nav_file=make_nav(two, 12, sets=2), lat=LOC[0], lon=LOC[1], height=LOC[2], seconds=400,
                          start=(2024, 1, 7, 2, 55, 0.0))
    yield "lat60", dict(nav_file=n32, lat=LOC60[0], lon=LOC60[1], height=LOC60[2], seconds=310, max_chan=32, start=START)


def test_incremental_equals_batch_for_every_golden_configuration(tmp_path):
    """open + advances of 1, 7 and 300 blocks == gpsb200_scenario_create, records and frames (static 12/32, motion,
    -t, RINEX 3, Pluto, ephemeris roll, 60N reallocation)"""
    for name, kw in _golden_configs(tmp_path):
        want, wnav = gps.scenario(**kw)
        for chunk in (1, 7, 300):
            args = {k: v for k, v in kw.items() if k not in ("nav_file", "lat", "lon", "height", "seconds")}
            with gps.LiveScenario(kw["nav_file"], kw["lat"], kw["lon"], kw["height"], kw["seconds"], **args) as s:
                got, nav = s.run([], chunk=chunk)
            assert got.tobytes() == want.tobytes(), (name, chunk)
            assert nav.tobytes() == wnav.tobytes(), (name, chunk)


def test_interactive_without_keys_is_the_static_run(tmp_path):
    nav_file = make_nav(tmp_path, 12)
    for target in (None, (1500.5, 33.3, 120.25)):
        want, wnav = gps.scenario(nav_file, *LOC, seconds=35, start=START, target=target)
        got, nav = gps.scenario(nav_file, *LOC, seconds=35, start=START, target=target, steer=[])
        assert got.tobytes() == want.tobytes() and nav.tobytes() == wnav.tobytes()


def test_a_motion_file_switches_interactive_mode_off(tmp_path):
    kw = dict(max_chan=12, start=START, motion_file=motion_file(tmp_path))
    nav_file = make_nav(tmp_path, 12)
    want, _ = gps.scenario(nav_file, *LOC, seconds=10, **kw)
    with gps.LiveScenario(nav_file, *LOC, 10, interactive=True, **kw) as s:
        s.advance(5)
        with pytest.raises(gps.GpsB200Error) as e:
            s.key("e")
        assert e.value.code == -1
        got = s.advance(1000)
    assert got.tobytes() == want[5:].tobytes()


def test_steering_state_follows_the_keys(tmp_path):
    with gps.LiveScenario(make_nav(tmp_path, 12), *LOC, 5, start=START, target=(10.0, 0.05, 0.0), interactive=True) as s:
        st = s.state()
        assert (st.bearing_mdeg, st.speed, st.velocity, st.vertical_speed, st.next_block) == (50.0, 0, 0, 0, 0)
        start = list(st.xyz)
        s.advance(3)
        assert list(s.state().xyz) == start                  # +0 per block without speed
        for k in "a" + "e" * 3 + "q" * 5 + "ww" + "s":
            s.key(k)
        st = s.state()
        assert (st.bearing_mdeg, st.speed, st.velocity, st.vertical_speed) == (360000.0, 0.0, 0.0, 1.0)
        s.key("d")
        assert s.state().bearing_mdeg == 0.0
        s.advance(10)
        assert s.state().next_block == 13 and s.state().xyz[:] != start
        s.key("x")
        assert s.state().end_block == 13
        with pytest.raises(gps.GpsB200Error) as e:
            s.advance(1)
        assert e.value.code == gps.ERR_END


def test_scenario_misuse_is_an_error(tmp_path):
    nav_file = make_nav(tmp_path, 12)
    with gps.LiveScenario(nav_file, *LOC, 2, start=START, interactive=True) as s:
        with pytest.raises(gps.GpsB200Error) as e:
            s.key("e")                                        # before block 1
        assert e.value.code == -1
        s.advance(1)
        for bad in ("z", "i", "\n", 0):
            with pytest.raises(gps.GpsB200Error) as e:
                s.key(bad)
            assert e.value.code == -1
        s.key("t")                                            # SDR gain: accepted, no effect
        s.key("g")
        assert s.advance(100).shape[0] == 18                  # <= n: the rest of the run
        with pytest.raises(gps.GpsB200Error) as e:
            s.advance(1)                                      # past the end
        assert e.value.code == gps.ERR_END
    with gps.LiveScenario(nav_file, *LOC, 2, start=START) as s:   # not interactive
        s.advance(1)
        with pytest.raises(gps.GpsB200Error) as e:
            s.key("e")
        assert e.value.code == -1
    with gps.LiveScenario(nav_file, *LOC, 2, start=START) as s:
        s.advance(1)
        with pytest.raises(gps.GpsB200Error):
            s.frame(5)                                        # never produced


def test_memory_of_an_opened_scenario_does_not_grow_with_the_duration(tmp_path):
    """24 h interactive, 12 channels: the batch engine would hold 864 000 x 12 x 64 B = 0.66 GB of records before
    the first sample; advancing 3000 blocks in chunks of 100 must stay far below that."""
    nav_file = make_nav(tmp_path, 12)
    code = textwrap.dedent("""
        import importlib, resource, sys
        sys.path.insert(0, %r)
        gps = importlib.import_module("multi-sdr-gps-sim_b200")
        gps.lib()
        base = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
        with gps.LiveScenario(%r, %r, %r, %r, 86400, start=%r, interactive=True) as s:
            for i in range(30):
                if i == 3:
                    s.key("e")
                assert s.advance(100).shape[0] == 100
                s.frame(int(s.advance(1)["nav_frame"][0, 0])) if i == 29 else None
        print(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss - base)
    """) % (scenario.ROOT, nav_file, LOC[0], LOC[1], LOC[2], START)
    grow_kb = int(subprocess.check_output([sys.executable, "-c", code]).decode().split()[-1])
    assert grow_kb < 50 * 1024, grow_kb
