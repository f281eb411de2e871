#!/usr/bin/env python3
"""Latency of one live step of interactive mode: advance the opened scenario by one block, apply a key, synthesize the
block and download it (gpsb200_synth_blocks, host buffer), over 600 consecutive blocks. Real time needs every step to
finish within the 100 ms a block lasts. Prints one JSON line per channel count, with the card name and power limit read
in the same run.
usage: live_latency.py [--chan 12,32] [--blocks 600] [--out FILE.jsonl]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
gps = importlib.import_module("multi-sdr-gps-sim_b200")


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                                    text=True).strip()
        name, power, sm = [v.strip() for v in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"gpu": "unknown", "power_limit": "unknown", "sm_clock": "unknown"}


def measure(nchan, nblocks, nav_file):
    ring = 4
    keys = "edwqas"
    times = []
    with gps.LiveScenario(nav_file, 35.681298, 139.766247, 10.0, nblocks / 10.0 + 1.0, max_chan=nchan,
                          start=(2024, 1, 7, 2, 0, 0.0), interactive=True) as s, \
            gps.Context(nchan, 1, max_nav_frames=ring) as ctx:
        out = np.empty(gps.BLOCK_ELEMS, np.int8)
        carr, prev, uploaded = np.zeros(nchan), np.zeros(nchan, np.int32), -1
        for b in range(nblocks):
            t0 = time.perf_counter()
            if b >= 1:
                s.key(keys[b % len(keys)] if b % 50 else "e")
            ch = s.advance(1)
            f = int(ch["nav_frame"][0, 0])
            if f > uploaded:
                for c, words in enumerate(s.frame(f)):
                    ctx.set_nav(f % ring, c, words)
                uploaded = f
            ch["nav_frame"] %= ring
            ch[0]["carr_phase"] = np.where((ch[0]["prn"] > 0) & (ch[0]["prn"] == prev), carr, ch[0]["carr_phase"])
            _, carr = ctx.synth_blocks(ch, gps.SC08, out=out)
            prev = ch[0]["prn"].copy()
            times.append(time.perf_counter() - t0)
        kernel = ctx.synth_kernel_name(nchan)
    t = np.array(times) * 1e3
    return {"channels": nchan, "kernel": kernel, "blocks": nblocks, "sample_size": "int8",
            "step_ms_median": round(float(np.median(t)), 3), "step_ms_p99": round(float(np.percentile(t, 99)), 3),
            "step_ms_max": round(float(t.max()), 3), "first_step_ms": round(float(t[0]), 3),
            "real_time_margin": round(100.0 / float(np.percentile(t, 99)), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chan", default="12,32")
    ap.add_argument("--blocks", type=int, default=600)
    ap.add_argument("--out")
    a = ap.parse_args()
    info = card()
    lines = []
    with tempfile.TemporaryDirectory() as td:
        for n in [int(v) for v in a.chan.split(",")]:
            nav = os.path.join(td, "sky%d.nav" % n)
            subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", str(n), "--out", nav])
            r = dict(measure(n, a.blocks, nav), **info)
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
