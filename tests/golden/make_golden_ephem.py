#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: (re)generate the broadcast-ephemeris fixtures tests/golden/sky*_ephvar_*.npz from the reference
itself.

Runs only where the reference sources exist; builds oracle/_ref/ref_dump{12,32} with oracle/Makefile. Every other fixture
is made from gen_rinex.py's default sky, whose records all have the same shape: argument of perigee 0, toc = toe, af2 = 0,
one sign for each clock, group-delay, harmonic and rate term, IODC < 256, URA index and health 0, and a run that starts at
toc. These runs use gen_rinex.py --varied --sets 2 (toc 02:00 and 04:00; PRNs 1-12 carry every signed field at both of its
limits) and start about an hour from a toc, where the rate terms have grown:
  * sky12_ephvar_p59m_35s_i8: start 02:58:54, set 0 at t - toc = +3534 s; 35 s, so that a tracked channel decodes
    subframes 1-3 of the frame sent from 02:59:00 (6 s to 24 s into the stream) from the stream itself;
  * sky32_ephvar_m59m_10s_i16: start 03:01:00, set 1 at t - toc = -3540 s, all 32 PRNs, int16;
  * sky12_ephvar_rinex3_3s_i8: the --v3 file of the same sky read by readRinex3 (-3), start 03:01:00.
No run crosses 03:00:00, where the reference rolls from one set to the other.

Stored, in the layout of the ionosphere fixtures: the CRC-32 of every block (no verbatim blocks), every NAV frame and the
frame of every block, the slot occupancy of every block, every block's parameters, and how the run was made (the
gen_rinex.py arguments, receiver, start).
Usage: python tests/golden/make_golden_ephem.py [names...]
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import refdump  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
LOC = (35.681298, 139.766247, 10.0)
ROLL_SOW = 10800.0                      # 03:00:00: one hour before the second set's toc

# name: (satellites = channels, start (hh, mm, ss) on 2024/01/07, seconds, int16, RINEX 3)
CASES = {
    "sky12_ephvar_p59m_35s_i8": (12, (2, 58, 54), 35, False, False),
    "sky32_ephvar_m59m_10s_i16": (32, (3, 1, 0), 10, True, False),
    "sky12_ephvar_rinex3_3s_i8": (12, (3, 1, 0), 3, False, True),
}


def rinex_args(nsat, v3):
    return ["--nsat", str(nsat), "--sets", "2", "--varied"] + (["--v3"] if v3 else [])


def run(name):
    nsat, (hh, mm, ss), secs, i16, v3 = CASES[name]
    t0 = 3600.0 * hh + 60.0 * mm + ss
    assert t0 + secs <= ROLL_SOW or t0 >= ROLL_SOW, name          # the run stays on one set
    start = "2024/01/07,%02d:%02d:%02d" % (hh, mm, ss)
    args = rinex_args(nsat, v3)
    with tempfile.TemporaryDirectory() as td:
        nav = os.path.join(td, "sky.nav")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--out", nav] + args)
        loc = "%r,%r,%r" % LOC
        crc, par = os.path.join(td, "crc.bin"), os.path.join(td, "p.bin")
        cmd = [os.path.join(REF, "ref_dump%d" % nsat), "-e", nav, "-l", loc, "-d", str(secs), "-s", start,
               "--crc", crc, "--params", par] + (["--iq16"] if i16 else []) + (["-3"] if v3 else [])
        subprocess.check_call(cmd, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        p = refdump.read_params(par)
        ch = p["chans"]
        nblk = ch.shape[0]
        crcs = np.fromfile(crc, dtype="<u4")
        assert nblk == secs * 10 - 1 and crcs.size == nblk, (nblk, crcs.size)
        assert ((ch["prn"] > 0).sum(1) == nsat).all(), (ch["prn"] > 0).sum(1)      # the whole sky, in every block
        nw = refdump.nav_table(p)
        frames, idx = [], np.zeros(nblk, np.int32)
        for b in range(nblk):
            if not frames or not np.array_equal(frames[-1], nw[b]):
                frames.append(nw[b])
            idx[b] = len(frames) - 1
        out = dict(max_chan=np.int32(p["max_chan"]), sample_size=np.int32(p["sample_size"]), seconds=np.float64(secs),
                   location=np.array(LOC, np.float64), start=np.array(start), nsat=np.int32(nsat),
                   rinex_args=np.array(args), rinex3=np.bool_(v3), block_crcs=crcs, nav_frames=np.stack(frames),
                   nav_frame_of_block=idx, prn_of_block=ch["prn"].astype(np.int8), chans=ch)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name, "blocks", nblk, "frames", len(frames), "start", start)


if __name__ == "__main__":
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    for n in sys.argv[1:] or list(CASES):
        run(n)
