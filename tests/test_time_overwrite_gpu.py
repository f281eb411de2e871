"""`-s now` on the GPU: the three time-overwrite fixtures (runs of the reference producer with time_overwrite set,
tests/golden/make_golden_now.py) from the RINEX file through the scenario engine and the CUDA synthesis, and through
gpsb200-sim on every path; every block's CRC equals the reference's."""
import datetime
import math
import os
import re
import subprocess
import zlib

import numpy as np
import pytest

import scenario
from scenario import gps
from test_time_overwrite import NOW, gps_time, now_case, parse_start

pytestmark = pytest.mark.gpu

CHUNK = 256


def chunked_crcs(ch, nav, chunk=CHUNK):
    """block CRCs of the stream made by one context in calls of `chunk` blocks that continue the carrier chain"""
    crcs, carr = [], None
    with gps.Context(ch.shape[1], chunk, max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        for b0 in range(0, ch.shape[0], chunk):
            part = ch[b0:b0 + chunk]
            if b0 > 0:
                part = gps.sharding.seed_slice(part, ch[b0 - 1], carr)
            out, carr = ctx.synth_blocks(part, 1)
            crcs.append(scenario.crc_blocks(out))
            if b0 == 0:
                first = out[:gps.BLOCK_ELEMS].copy()
    return np.concatenate(crcs), first


@pytest.mark.parametrize("name", NOW)
def test_stream_equals_the_reference_stream(name, tmp_path):
    g, kw = now_case(name, tmp_path)
    ch, nav = gps.scenario(**kw, time_overwrite=True)
    got, first = chunked_crcs(ch, nav)
    want = g["block_crcs"]
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, bad[:10]
    if "keep_blocks" in g:
        assert np.array_equal(first, g["keep_blocks"][list(g["keep_idx"]).index(0)])


def test_week_roll_stream_cut_into_slices_equals_the_reference_stream(tmp_path):
    """4 slices, each made by its own context from the hand-over phases alone; one cut exactly on the block whose
    receiver time is the first of the new GPS week"""
    g, kw = now_case("sky12_now_weekroll_300s_i8", tmp_path)
    ch, nav = gps.scenario(**kw, time_overwrite=True)
    week, sow = gps_time(kw["start"])
    roll = int(round((604800 - sow) * 10)) - 1            # block k runs at receiver time start + 0.1 (k + 1)
    assert roll == 1199
    edges = [0, 700, roll, 2300, ch.shape[0]]
    crcs = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        with gps.Context(ch.shape[1], hi - lo, max_nav_frames=len(nav)) as ctx:
            ctx.set_nav_frames(nav)
            part = ch[lo:hi]
            if lo > 0:
                part = gps.sharding.seed_slice(part, ch[lo - 1], gps.sharding.start_phases(ch[:lo], ctx=ctx))
            out, _ = ctx.synth_blocks(part, 1)
            crcs.append(scenario.crc_blocks(out))
    got = np.concatenate(crcs)
    bad = np.nonzero(got != g["block_crcs"])[0]
    assert bad.size == 0, bad[:10]


def _sim():
    exe = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "gpsb200-sim")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "csrc")])
    return exe


def _sim_args(kw, out):
    loc = "%r,%r,%r" % (float(kw["lat"]), float(kw["lon"]), float(kw["height"]))
    return [_sim(), "-e", kw["nav_file"], "-l", loc, "-d", "%g" % kw["seconds"], "-o", str(out)]


def _file_crcs(path):
    s = np.fromfile(path, dtype=np.int8)
    return np.array([zlib.crc32(r.tobytes()) for r in s.reshape(-1, gps.BLOCK_ELEMS)], np.uint32)


def test_cli_now_writes_the_reference_stream_on_every_path(tmp_path):
    """-s now --now DATE: the whole stream; --compat-drop: the stock program's file (blocks 0 and 7 on); --steer with
    an empty schedule: the interactive path, the same stream"""
    g, kw = now_case("sky12_now_35s_i8", tmp_path)
    want = g["block_crcs"]
    out = tmp_path / "iq.bin"
    empty = tmp_path / "empty.steer"
    empty.write_text("")
    for extra, keep in (([], range(want.size)), (["--compat-drop"], [0] + list(range(7, want.size))),
                        (["--steer", str(empty)], range(want.size))):
        r = subprocess.run(_sim_args(kw, out) + ["-s", "now", "--now", str(g["start"])] + extra, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-600:]
        assert "gpsb200-sim: start time: %s (week 2440, sow 390896)" % g["start"] in r.stderr
        got = _file_crcs(out)
        assert np.array_equal(got, want[list(keep)]), (extra, np.nonzero(got != want[list(keep)])[0][:5])
        out.unlink()


def _lon_for(start):
    """longitude that sees the sky of a two-set gen_rinex file after the overwrite at `start` (make_golden_now.py)"""
    week, sow = gps_time(start)
    gtmp = int(sow) // 7200 * 7200
    k = 0 if sow - gtmp < 3600 else 1                    # the set within +-1 h of the start
    toe = 7200.0 + 7200.0 * k
    new_toe = ((week - 2296) * 604800.0 + gtmp - 7200.0 + toe) % 604800.0
    lon = 139.766247 - math.degrees(7.2921151467e-5 * (new_toe - toe))
    return round((lon + 180.0) % 360.0 - 180.0, 6)


def test_cli_now_with_the_clock_equals_the_api_at_the_printed_start(tmp_path):
    g, kw = now_case("sky12_now_weekroll_300s_i8", tmp_path)
    t0 = datetime.datetime.now(datetime.timezone.utc).replace(tzinfo=None)
    kw.update(seconds=5.0, lon=_lon_for((t0.year, t0.month, t0.day, t0.hour, t0.minute, float(t0.second))))
    out = tmp_path / "iq.bin"
    r = subprocess.run(_sim_args(kw, out) + ["-s", "now"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-600:]
    m = re.search(r"start time: (\S+) \(week", r.stderr)
    printed = datetime.datetime.strptime(m.group(1), "%Y/%m/%d,%H:%M:%S")
    assert abs((printed - t0).total_seconds()) < 5
    ch, nav = gps.scenario(**dict(kw, start=parse_start(m.group(1))), time_overwrite=True)
    assert ch.shape[0] == 49 and (ch["prn"][0] > 0).sum() >= 1
    got = _file_crcs(out)
    want, _ = chunked_crcs(ch, nav)
    assert np.array_equal(got, want)
