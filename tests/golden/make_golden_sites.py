#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: (re)generate the ionosphere fixtures tests/golden/site_*.npz and sky12_iono_*.npz from the
reference itself.

Runs only where the reference sources exist; builds oracle/_ref/ref_dump{12,32} with oracle/Makefile. Every other fixture
is made under one sky, Tokyo at 02:00 UTC (local solar time near 11:20), so the Klobuchar term of the reference's
ionosphericDelay (gps.c:1893-1964) is only ever evaluated in its daytime, mid-latitude, northern branch. These runs
reach the rest of it:
  * three receivers, each with gen_rinex.py's constellation centred on it (--rx), at 02:00 UTC:
      66 N 100 W (local evening: the night branch, phi_i clamped at +0.416, AMP < 0 clamped, PER clamped at 72000 s,
      local time below 0), 66 S 140 E (phi_i clamped at -0.416, phi_m < 0) and 34.6 S 58.4 W (all night);
  * Tokyo with -I, the reference's ionosphere switch (ionoutc.enable false: no delay at all);
  * Tokyo from a file without ION ALPHA / ION BETA (gen_rinex.py --no-iono): ionoutc.vflg false, so a constant
    F * 5 ns delay and no subframe 4 page 18 (gps.c:806). The run lasts 520 s, so that it passes frame 17, where page 18
    would be sent.

Stored, in the layout of the `-s now` fixtures: the CRC-32 of every block (no verbatim blocks), every NAV frame and the
frame of every block, the slot occupancy of every block, the per-block parameters (all of them, or those around the
frame-17 boundary), and how the run was made (sky centre, receiver, flags).
Usage: python tests/golden/make_golden_sites.py [names...]
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
TOKYO = (35.681298, 139.766247)
START = "2024/01/07,02:00:00"

# name: (satellites = channels, sky centre (lat, lon), receiver height, seconds, int16, -I, ION ALPHA / BETA in the
#        file, blocks whose parameters are kept (None: all))
CASES = {
    "site_66n_100w_10s_i8": (32, (66.0, -100.0), 10.0, 10, False, False, True, None),
    "site_66s_140e_10s_i8": (32, (-66.0, 140.0), 10.0, 10, False, False, True, None),
    "site_34s_58w_10s_i16": (12, (-34.6, -58.4), 10.0, 10, True, False, True, None),
    "sky12_iono_off_3s_i8": (12, TOKYO, 10.0, 3, False, True, True, None),
    "sky12_iono_hdr_missing_520s_i8": (12, TOKYO, 10.0, 520, False, False, False,
                                       list(range(0, 3)) + list(range(5096, 5104)) + [5198]),
}


def run(name):
    nsat, rx, height, secs, i16, off, hdr, keep = CASES[name]
    with tempfile.TemporaryDirectory() as td:
        nav = os.path.join(td, "sky.nav")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nsat),
                               "--out", nav, "--rx=%r,%r" % rx] + ([] if hdr else ["--no-iono"]))
        loc = "%r,%r,%r" % (rx[0], rx[1], height)
        crc, par = os.path.join(td, "crc.bin"), os.path.join(td, "p.bin")
        args = [os.path.join(REF, "ref_dump%d" % nsat), "-e", nav, "-l", loc, "-d", str(secs), "-s", START,
                "--crc", crc, "--params", par] + (["--iq16"] if i16 else []) + (["-I"] if off else [])
        subprocess.check_call(args, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        p = refdump.read_params(par)
        ch = p["chans"]
        nblk = ch.shape[0]
        crcs = np.fromfile(crc, dtype="<u4")
        assert nblk == secs * 10 - 1 and crcs.size == nblk, (nblk, crcs.size)
        assert int((ch["prn"][0] > 0).sum()) == nsat, ch["prn"][0]          # the whole sky is in view
        nw = refdump.nav_table(p)
        frames, idx = [], np.zeros(nblk, np.int32)
        for b in range(nblk):
            if not frames or not np.array_equal(frames[-1], nw[b]):
                frames.append(nw[b])
            idx[b] = len(frames) - 1
        out = dict(max_chan=np.int32(p["max_chan"]), sample_size=np.int32(p["sample_size"]), seconds=np.float64(secs),
                   location=np.array([float(v) for v in loc.split(",")]), start=np.array(START), nsat=np.int32(nsat),
                   sky_centre=np.array(rx, np.float64), ionosphere=np.bool_(not off), iono_header=np.bool_(hdr),
                   block_crcs=crcs, nav_frames=np.stack(frames), nav_frame_of_block=idx,
                   prn_of_block=ch["prn"].astype(np.int8))
        if keep is None:
            out["chans"] = ch
        else:
            out["chans_idx"] = np.array(keep, np.int32)
            out["chans"] = ch[out["chans_idx"]]
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name, "blocks", nblk, "frames", len(frames), "location", loc)


if __name__ == "__main__":
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    for n in sys.argv[1:] or list(CASES):
        run(n)
