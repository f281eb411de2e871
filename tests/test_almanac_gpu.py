"""Almanac on, through the whole path: RINEX + SEM file -> scenario engine -> CUDA synthesis, against the CRC-32 of
every block of the reference's own stream with its almanac enabled (tests/golden/sky*_alm_*.npz). The SEM and RINEX
files are written by oracle/gen_sem.py and oracle/gen_rinex.py."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import scenario
from scenario import gps

pytestmark = pytest.mark.gpu

LOC = (35.681298, 139.766247, 10.0)
START = (2024, 1, 7, 2, 0, 0.0)
LONG = {"sky12_alm_static_780s_i8": dict(nsat=12, loc=LOC, secs=780),
        "sky32_alm_lat60_310s_i8": dict(nsat=32, loc=(60.0, 140.0, 0.0), secs=310)}


def _files(tmp_path, nsat):
    nav, sem = tmp_path / ("sky%d.nav" % nsat), tmp_path / "almanac.sem"
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nsat),
                           "--out", str(nav)])
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_sem.py"), "--out", str(sem)])
    return str(nav), str(sem)


def _scenario(name, tmp_path):
    c = LONG[name]
    nav_file, sem = _files(tmp_path, c["nsat"])
    return gps.scenario(nav_file, *c["loc"], seconds=c["secs"], max_chan=c["nsat"], start=START, almanac_file=sem)


def _stream_crcs(ch, nav, edges):
    """Block CRCs of the stream made slice by slice: one context per slice [lo, hi), seeded only with the exact carrier
    phases chained through the blocks before it."""
    nchan = ch.shape[1]
    crcs = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        with gps.Context(nchan, hi - lo, max_nav_frames=len(nav)) as ctx:
            ctx.set_nav_frames(nav)
            part = ch[lo:hi]
            if lo > 0:
                part = gps.sharding.seed_slice(part, ch[lo - 1], gps.sharding.start_phases(ch[:lo], ctx=ctx))
            out, _ = ctx.synth_blocks(part, 1)
            crcs.append(scenario.crc_blocks(out))
    return np.concatenate(crcs)


@pytest.mark.parametrize("name", list(LONG))
def test_almanac_stream_equals_reference_stream(name, tmp_path):
    """Every block of the 780 s (a full 25-page rotation) and of the 310 s reallocation run, synthesized by one context
    in calls of 1000 blocks that continue the carrier chain, as gpsb200-sim does."""
    g = scenario.load_golden(name)
    ch, nav = _scenario(name, tmp_path)
    nblk = ch.shape[0]
    assert nblk == g["crcs"].size
    got = []
    carr = None
    with gps.Context(ch.shape[1], 1000, max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        for b0 in range(0, nblk, 1000):
            part = ch[b0:b0 + 1000]
            if b0 > 0:
                part = gps.sharding.seed_slice(part, ch[b0 - 1], carr)
            out, carr = ctx.synth_blocks(part, 1)
            got.append(scenario.crc_blocks(out))
    got = np.concatenate(got)
    bad = np.nonzero(got != g["crcs"])[0]
    assert bad.size == 0, bad[:10]


def test_almanac_780s_cut_into_8_time_slices_equals_reference_stream(tmp_path):
    """The 780 s stream made by 8 separate contexts from the hand-over phases alone; the cuts fall inside the 25-page
    rotation (a slice starts in the middle of the almanac pages)."""
    name = "sky12_alm_static_780s_i8"
    g = scenario.load_golden(name)
    ch, nav = _scenario(name, tmp_path)
    nblk = ch.shape[0]
    edges = [gps.sharding.slice_bounds(nblk, 8, r)[0] for r in range(8)] + [nblk]
    frame_of = ch["nav_frame"][:, 0]
    # a cut in mid-rotation: the page index of the frame at the cut is neither 0 nor the one at the stream start
    assert any(0 < lo < nblk and (lo + 1) // 300 % 25 not in (0, 1) for lo in edges)
    assert len(set(frame_of[edges[1:-1]])) == 7
    got = _stream_crcs(ch, nav, edges)
    bad = np.nonzero(got != g["crcs"])[0]
    assert bad.size == 0, (edges, bad[:10])


def test_cli_almanac_writes_reference_stream_and_stock_compat_file(tmp_path):
    """gpsb200-sim --almanac FILE, 30 s: the first 299 blocks of the reference's 780 s almanac stream; with --compat-drop
    the stock program's iqdata.bin (blocks 0 and 7..298)."""
    exe = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "gpsb200-sim")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "csrc")])
    g = scenario.load_golden("sky12_alm_static_780s_i8")
    nav_file, sem = _files(tmp_path, 12)
    for extra, keep in (([], list(range(299))), (["--compat-drop"], [0] + list(range(7, 299)))):
        out = tmp_path / ("iq%d.bin" % len(extra))
        r = subprocess.run([exe, "-e", nav_file, "-l", "35.681298,139.766247,10.0", "-d", "30", "-s", "2024/01/07,02:00:00",
                            "--almanac", sem, "-o", str(out)] + extra, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-600:]
        assert "almanac date: 2024/01/07,02:16:32" in r.stderr and "no almanac pages" not in r.stderr
        s = np.fromfile(out, dtype=np.int8)
        assert s.size == len(keep) * gps.BLOCK_ELEMS, (extra, s.size)
        for row, b in zip(s.reshape(len(keep), gps.BLOCK_ELEMS), keep):
            assert zlib.crc32(row.tobytes()) == g["crcs"][b], (extra, b)
        out.unlink()
