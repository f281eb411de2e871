#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: (re)generate the interactive-mode fixtures tests/golden/*steer*.npz from the reference itself.

Runs only where the reference sources exist; builds what it needs with oracle/Makefile.interactive
(oracle/_ref/ref_interactive{12,32}) and oracle/Makefile (ref_dump{12,32}). Each
fixture is one run of the reference's own main (gps-sim.c, unmodified: options, key switch) with -i, its keys
handed over by a script (oracle/ref_harness/ref_interactive.c), so that the key arithmetic is the reference's and
not a restatement. Stored: the schedule, block CRC-32s, the per-block parameters (all of them, or those around the
events) and the NAV frames. Before saving, the generator checks that the schedule really steers: the run's
parameters equal those of the reference's static run (ref_dump) up to the first key block and differ from it on.
Usage: python tests/golden/make_golden_interactive.py [names...]
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
START = "2024/01/07,02:00:00"

# name: (nsat, channels, location, seconds, extra reference options, schedule, blocks whose parameters are kept (None: all))
CASES = {
    # speed up to 25 m/s, a 22.9 deg turn, a 5 m/s climb, 'q' pressed past zero, a descent; events on both sides of
    # the 30 s NAV roll after block 299
    "sky12_steer_60s_i8": (12, 12, "35.681298,139.766247,10.0", 60, [],
                           "5,e,2500\n120,d,180\n299,w,5\n300,q,2600\n301,e,700\n420,s,8\n421,ae,3\n", None),
    # -t start point, bearing 50 mdeg: 'a' wraps below 0 to 360000, 'd' above 360000 to 0, keys in consecutive blocks
    "sky12_steer_target_30s_i16": (12, 12, "35.681298,139.766247,10.0", 30, ["-t", "1500.5,0.05,120.25", "--iq16"],
                                   "1,e,1200\n2,a\n3,d\n4,a\n5,a\n6,d,2\n7,w,3\n8,dq,2\n", None),
    # 60N: a satellite rises at 240 s, another sets at 300 s; the receiver moves fast, so ranges come from the moved
    # position while the allocation keeps using the start
    "sky32_lat60_steer_310s_i8": (32, 32, "60.0,140.0,0.0", 310, [],
                                  "1,e,30000\n1000,d,700\n2350,w,50\n2397,q,40000\n2399,e,25000\n2998,a,300\n3001,s,120\n",
                                  list(range(0, 3)) + list(range(997, 1003)) + list(range(2396, 2405)) +
                                  list(range(2996, 3005)) + [3098]),
}


def parse_schedule(text):
    return [(int(f[0]), f[1], int(f[2]) if len(f) > 2 else 1) for f in (ln.split(",") for ln in text.splitlines() if ln)]


def run(name):
    nsat, chan, loc, secs, extra, sched, keep = CASES[name]
    with tempfile.TemporaryDirectory() as td:
        nav = os.path.join(td, "sky.nav")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nsat), "--out", nav])
        steer, par, crc = (os.path.join(td, n) for n in ("steer.txt", "p.bin", "crc.bin"))
        with open(steer, "w") as f:
            f.write(sched)
        env = dict(os.environ, ORACLE_STEER=steer, ORACLE_PARAMS=par, ORACLE_CRC=crc)
        subprocess.check_call([os.path.join(REF, "ref_interactive%d" % chan), "-i", "-r", "iqfile", "--disable-almanac",
                               "-e", nav, "-l", loc, "-d", str(secs), "-s", START] + extra,
                              env=env, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        p = refdump.read_params(par)
        ch = p["chans"]
        nblk = ch.shape[0]
        crcs = np.fromfile(crc, dtype="<u4")
        assert nblk == int(secs * 10 + 0.5) - 1 and crcs.size == nblk, (nblk, crcs.size)
        # sanity: identical to the static run before the first key block, different from it on
        b_first = min(b for b, _, _ in parse_schedule(sched))
        spar = os.path.join(td, "static.bin")
        subprocess.check_call([os.path.join(REF, "ref_dump%d" % chan), "-e", nav, "-l", loc, "-d", str((b_first + 20) / 10.0),
                               "-s", START, "--params", spar] + [x for x in extra if x != "--iq16"],
                              stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        st = refdump.read_params(spar)["chans"]
        assert ch[:b_first].tobytes() == st[:b_first].tobytes(), "scheduled run differs from the static one before its first key"
        assert not np.array_equal(ch["f_carr"][b_first], st["f_carr"][b_first]), "the first key did not act on its block"
        nw = refdump.nav_table(p)
        frames, idx = [], np.zeros(nblk, np.int32)
        for b in range(nblk):
            if not frames or not np.array_equal(frames[-1], nw[b]):
                frames.append(nw[b])
            idx[b] = len(frames) - 1
        out = dict(max_chan=np.int32(p["max_chan"]), sample_size=np.int32(p["sample_size"]), seconds=np.float64(secs),
                   location=np.array([float(v) for v in loc.split(",")]), schedule=np.array(sched),
                   options=np.array(" ".join(extra)), block_crcs=crcs, nav_frames=np.stack(frames), nav_frame_of_block=idx,
                   prn_of_block=ch["prn"].astype(np.int8))
        if keep is None:
            out["chans"] = ch
        else:
            out["chans_idx"] = np.array(keep, np.int32)
            out["chans"] = ch[out["chans_idx"]]
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name, "blocks", nblk, "frames", len(frames), "first key block", b_first)


if __name__ == "__main__":
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.interactive"])
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    for n in sys.argv[1:] or list(CASES):
        run(n)
