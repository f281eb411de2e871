#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: (re)generate the `-s now` fixtures tests/golden/sky12_now_*.npz from the reference itself.

Runs only where the reference sources exist; builds oracle/_ref/ref_dump_now12 with oracle/Makefile.now. That binary is
the reference producer behind ref_dump's recording FIFO with simulator_t.time_overwrite set, so the reference's own
ephemeris and UTC time overwrite (gps.c:2531-2561) runs, with the explicit -s date standing in for the clock reading.

The synthetic skies of gen_rinex.py are built around the receiver at the file's toe. The overwrite moves every toe to
another second of week, which turns the constellation in longitude by OMEGA_E * (new toe.sec - old toe.sec) (the node
longitude of satpos, gps.c:585). Each case therefore moves the receiver west by that angle, so that it sees the sky
the file was made for; the generator asserts how many channels each run allocates.

Stored, in the layout of the other fixtures: block CRC-32s of every block, every NAV frame and the frame of every
block, the slot occupancy of every block, the per-block parameters (all of them, or those around the events), and
verbatim blocks where listed. The "no current set" case (one-set file, start in the second hour of its 2-hour epoch)
is checked here -- the reference enqueues no block -- and stores nothing.
Usage: python tests/golden/make_golden_now.py [names...]
"""
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import gen_rinex  # noqa: E402
import refdump  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
LAT, HEIGHT = 35.681298, 10.0


def date_to_gps(y, m, d, hh, mm, sec):
    """date2gps (gps.c:315-339)"""
    doy = [0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334]
    ye = y - 1980
    lpdays = ye // 4 + 1
    if ye % 4 == 0 and m <= 2:
        lpdays -= 1
    de = ye * 365 + doy[m - 1] + d + lpdays - 6
    return de // 7, (de % 7) * 86400.0 + hh * 3600.0 + mm * 60.0 + sec


def parse_start(s):
    d, t = s.split(",")
    y, m, dd = (int(v) for v in d.split("/"))
    hh, mi, sec = t.split(":")
    return y, m, dd, int(hh), int(mi), float(sec)


def compensated_lon(start, set_index):
    """Receiver longitude [deg] that sees set `set_index` of a gen_rinex file as the file's own receiver does, after
    the overwrite at `start`: west of it by OMEGA_E * (shifted toe.sec - toe.sec), rounded to 1e-6 deg."""
    week, sow = date_to_gps(*start)
    gtmp = (week, (int(sow) // 7200) * 7200.0)
    dsec = (gtmp[0] - gen_rinex.WEEK) * 604800.0 + gtmp[1] - gen_rinex.TOE_SOW
    toe = gen_rinex.TOE_SOW + 7200.0 * set_index
    new_toe = (toe + dsec) % 604800.0
    lon = gen_rinex.RX_LON - math.degrees(gen_rinex.OMEGA_E * (new_toe - toe))
    return round((lon + 180.0) % 360.0 - 180.0, 6)


# name: (ephemeris sets, start, set the start selects, seconds, channels allocated in block 0,
#        blocks whose parameters are kept (None: all), verbatim blocks)
CASES = {
    # one set, start 2096 s into the first hour of its 2-hour epoch (12:00:00), on another day and second of week;
    # the NAV frames roll at 12:35:00 and 12:35:30
    "sky12_now_35s_i8": (1, "2026/10/15,12:34:56", 0, 35, 12, None, [0]),
    # two sets, start Saturday 23:58:00: the second hour of the 22:00 epoch, so set 1 is selected, its toc moved into
    # the next GPS week (week + 1, 0 s); the receiver crosses the week boundary at 120 s (block 1199)
    "sky12_now_weekroll_300s_i8": (2, "2026/10/17,23:58:00", 1, 300, 11,
                                   list(range(0, 3)) + list(range(1195, 1206)) + [2998], []),
    # two sets, start 3300 s after the 12:00:00 epoch: the run rolls to set 1 at the first 30 s event past 13:00:00
    # (block 3299) and transmits frame 17 -- subframe 4 page 18, the overwritten WNt / tot -- at 510 s
    "sky12_now_ephroll_560s_i8": (2, "2026/10/15,12:55:00", 0, 560, 12,
                                  list(range(0, 3)) + list(range(3290, 3312)) + list(range(5097, 5103)) + [5598], []),
}
# one set, start in the second hour of its 2-hour epoch: no set is within +-1 h of the start
NO_CURRENT_SET = (1, "2026/10/15,13:34:56", 0, 2)


def ref_run(td, sets, start, set_index, secs, crc=True, iq=False, params=True):
    nav = os.path.join(td, "sky%d.nav" % sets)
    if not os.path.exists(nav):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", "12", "--out", nav] +
                              (["--sets", str(sets)] if sets > 1 else []))
    loc = "%r,%r,%r" % (LAT, compensated_lon(parse_start(start), set_index), HEIGHT)
    files = {k: os.path.join(td, k + ".bin") for k in ("crc", "iq", "params")}
    args = [os.path.join(REF, "ref_dump_now12"), "-e", nav, "-l", loc, "-d", str(secs), "-s", start, "--time-overwrite"]
    for k, on in (("crc", crc), ("iq", iq), ("params", params)):
        if on:
            args += ["--" + k, files[k]]
    r = subprocess.run(args, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    return r, loc, files


def run(name):
    sets, start, set_index, secs, nchan, keep, verbatim = CASES[name]
    with tempfile.TemporaryDirectory() as td:
        r, loc, files = ref_run(td, sets, start, set_index, secs, iq=bool(verbatim))
        assert r.returncode == 0, r.stdout
        p = refdump.read_params(files["params"])
        ch = p["chans"]
        nblk = ch.shape[0]
        crcs = np.fromfile(files["crc"], dtype="<u4")
        assert nblk == int(secs * 10 + 0.5) - 1 and crcs.size == nblk, (nblk, crcs.size)
        assert int((ch["prn"][0] > 0).sum()) == nchan, (ch["prn"][0], nchan)
        nw = refdump.nav_table(p)
        frames, idx = [], np.zeros(nblk, np.int32)
        for b in range(nblk):
            if not frames or not np.array_equal(frames[-1], nw[b]):
                frames.append(nw[b])
            idx[b] = len(frames) - 1
        out = dict(max_chan=np.int32(p["max_chan"]), sample_size=np.int32(p["sample_size"]), seconds=np.float64(secs),
                   location=np.array([float(v) for v in loc.split(",")]), start=np.array(start), sets=np.int32(sets),
                   block_crcs=crcs, nav_frames=np.stack(frames), nav_frame_of_block=idx,
                   prn_of_block=ch["prn"].astype(np.int8))
        if keep is None:
            out["chans"] = ch
        else:
            out["chans_idx"] = np.array(keep, np.int32)
            out["chans"] = ch[out["chans_idx"]]
        if verbatim:
            blocks = np.fromfile(files["iq"], dtype=np.int8).reshape(nblk, 600000)
            out["keep_idx"] = np.array(verbatim, np.int32)
            out["keep_blocks"] = np.stack([blocks[i] for i in verbatim])
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name, "blocks", nblk, "frames", len(frames), "channels", nchan, "location", loc)


def check_no_current_set():
    sets, start, set_index, secs = NO_CURRENT_SET
    with tempfile.TemporaryDirectory() as td:
        r, _, _ = ref_run(td, sets, start, set_index, secs, crc=False, params=False)
        assert r.returncode != 0 and b'"blocks": 0' in r.stdout, r.stdout
    print("no current set at", start, ": the reference enqueues 0 blocks")


if __name__ == "__main__":
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.now"])
    for n in sys.argv[1:] or list(CASES):
        run(n)
    if not sys.argv[1:]:
        check_no_current_set()
