#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: (re)generate the almanac fixtures of tests/golden from the reference itself.

Runs only where /root/reference exists (the build container); builds what it needs with oracle/Makefile.almanac:
ref_dump_alm{12,32} (ref_dump with the reference's almanac_enable = true) and alm_dump (the reference's SEM parser).
The reference reads ./almanac.sem (almanac.c:78), so every run happens in a temporary directory holding the SEM file
oracle/gen_sem.py writes. Fixtures:
  sky12_alm_trunc_3s_i8     3 s, the SEM file ends inside PRN 1's record: the partial record goes into subframe 5
                            page 1 of the first frame (gps.c:835 tests svid, not valid). Same layout as make_golden.py's.
  sky12_alm_static_780s_i8  780 s = 26 NAV frames, a full 25-page rotation (750 s)
  sky32_alm_lat60_310s_i8   the reallocation scenario (60N 140E, 32 channels): pages continue across slot reuse
                            (both long ones: --crc and --params together, no I/Q -- the 780 s stream alone would be
                            4.7 GB; kept are the CRC-32 of every block, slot occupancy of every block, every NAV frame)
  sem_edges                 the SEM edge files and what the reference's parser reads from each
Usage: python tests/golden/make_golden_almanac.py [names...]
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402
from make_golden import LOC, REF, ROOT, START, refdump  # noqa: E402

LOC60 = "60.0,140.0,0.0"
ALM_LONG = {"sky12_alm_static_780s_i8": (12, "ref_dump_alm12", 780, LOC),
            "sky32_alm_lat60_310s_i8": (32, "ref_dump_alm32", 310, LOC60)}
SEM_EDGES = {"full": [], "truncated": ["--truncate", "1"], "truncated_prn9": ["--truncate", "9"], "malformed": ["--malformed"],
             "bad_ids": ["--bad-ids"], "duplicate": ["--duplicate"], "full_week": ["--full-week"]}


def write_sem(td, args):
    subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_sem.py"), "--out", os.path.join(td, "almanac.sem")]
                          + args)


def run_trunc():
    """make_golden.run() for the almanac binary, run from a directory holding the truncated SEM file."""
    name = "sky12_alm_trunc_3s_i8"
    make_golden.SCENARIOS[name] = (12, "ref_dump_alm12", 3, [], [])
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as td:
        write_sem(td, ["--truncate", "1"])
        os.chdir(td)
        try:
            make_golden.run(name)
        finally:
            os.chdir(cwd)


def run_long(name):
    nsat, binary, secs, loc = ALM_LONG[name]
    with tempfile.TemporaryDirectory() as td:
        nav = os.path.join(td, "sky.nav")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nsat), "--out", nav])
        write_sem(td, [])
        crc, par = os.path.join(td, "crc.bin"), os.path.join(td, "p.bin")
        subprocess.check_call([os.path.join(REF, binary), "-e", nav, "-l", loc, "-d", str(secs), "-s", START,
                               "--crc", crc, "--params", par], stderr=subprocess.DEVNULL, stdout=subprocess.DEVNULL, cwd=td)
        p = refdump.read_params(par)
        crcs = np.fromfile(crc, dtype="<u4")
    nblk = p["chans"].shape[0]
    assert crcs.size == nblk == int(secs * 10 + 0.5) - 1, (crcs.size, nblk)
    nw = refdump.nav_table(p)
    frames, idx = [], np.zeros(nblk, np.int32)
    for b in range(nblk):                       # one copy per distinct frame, as make_golden.run() stores them
        if not frames or not np.array_equal(frames[-1], nw[b]):
            frames.append(nw[b])
        idx[b] = len(frames) - 1
    np.savez_compressed(os.path.join(HERE, name + ".npz"), crcs=crcs, max_chan=np.int32(p["max_chan"]),
                        sample_size=np.int32(p["sample_size"]), seconds=np.int32(secs),
                        prn_of_block=p["chans"]["prn"].astype(np.int8), nav_frames=np.stack(frames), nav_frame_of_block=idx)
    print(name, "blocks", nblk, "frames", len(frames))


def run_sem_edges():
    out = {}
    for edge, args in SEM_EDGES.items():
        with tempfile.TemporaryDirectory() as td:
            write_sem(td, args)
            with open(os.path.join(td, "almanac.sem"), "rb") as f:
                out["text_" + edge] = np.frombuffer(f.read(), np.uint8)
            lines = subprocess.check_output([os.path.join(REF, "alm_dump")], cwd=td, text=True).splitlines()
        out["valid_" + edge] = np.int32(lines[0].split()[0])
        rows = [ln.split() for ln in lines[1:]]
        assert len(rows) == 32
        out["ints_" + edge] = np.array([[int(v) for v in r[:7]] for r in rows], np.int64)
        out["doubles_" + edge] = np.array([[float.fromhex(v) for v in r[7:]] for r in rows], np.float64)
    np.savez_compressed(os.path.join(HERE, "sem_edges.npz"), **out)
    print("sem_edges", ", ".join("%s valid %d" % (e, out["valid_" + e]) for e in SEM_EDGES))


if __name__ == "__main__":
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.almanac"])
    for n in (sys.argv[1:] or ["sem_edges", "sky12_alm_trunc_3s_i8"] + list(ALM_LONG)):
        if n == "sem_edges":
            run_sem_edges()
        elif n == "sky12_alm_trunc_3s_i8":
            run_trunc()
        else:
            run_long(n)
