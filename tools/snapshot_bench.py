"""Time one snapshot fix, stage by stage, on one GPU, and print one JSON line.

Workload per channel count: the first block of a fixture's stream (12 channels: sky12_static_35s_i8; 32 channels:
sky32_static_10s_i8; Tokyo, GPS week 2296, 7 200 s), synthesized into device memory first, and one 10 ms snapshot
from sample 1 000 of it (K = 10, int8). The stages, each timed in place on the device stream with device events
(median over --iters after --warmup, in --rounds rounds that alternate the stages):
  cold      gpsb200_acquire_device: 32 PRNs x 41 bins (-5000 .. 5000 Hz, 250 Hz)
  warm      gpsb200_acquire_windows_device: the channels' PRNs x 5 bins around each PRN's f_carr
  measure   gpsb200_snapshot_measure_device: the channels' PRNs, 12 code passes (DESIGN §11.5)
  fix       gpsb200_pvt_snapshot: one snapshot, the a-priori 50 km east, 1 km up and 10 s late
  search    gpsb200_pvt_snapshot_search: one snapshot, the default 262 144-node grid, the a-priori time 10 s late
The fix and search calls include their small uploads and downloads. Reported beside the times: the fix's and the
search's 3D error from the fixture's receiver position. The card's name, power limit and SM clock are read in the
same run (nvidia-smi). Writes nothing; needs a GPU.

    python tools/snapshot_bench.py [--iters 20] [--warmup 3] [--rounds 3]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
gps = importlib.import_module("multi-sdr-gps-sim_b200")
import pvt_model as PM   # noqa: E402

K, S0, STEP = 10, 1000, 250.0
LOC = (35.681298, 139.766247, 10.0)
START_SOW, START_WEEK = 7200.0, 2296
FIXTURES = {12: "sky12_static_35s_i8", 32: "sky32_static_10s_i8"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2]), float(q[3])


def inputs(nchan):
    """Block 0's records, the NAV frames, and the PVT channels (each slot's PRN, ephemeris from its frame)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", FIXTURES[nchan] + ".npz"))
    ch = np.zeros((1, nchan), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:1]
    frame = g["nav_frames"][int(g["nav_frame_of_block"][0])]
    ch["nav_frame"] = 0   # the block's frame alone goes up
    chans = np.zeros(nchan, gps.PVT_CHAN_DTYPE)
    for c in range(nchan):
        chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(frame[c]))[0]
        chans[c]["prn"] = ch[0]["prn"][c]
    chans["anchor_epoch"], chans["anchor_ms"] = -1, -1
    return frame[None], ch, chans


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--search-iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_start, clk_max = card()
    x0 = PM.llh_ecef(*LOC)
    lat, lon, _ = PM.ecef_llh(x0)
    east = np.array([-np.sin(lon), np.cos(lon), 0.0])
    up = np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)])
    ap_cfg = gps.coarse_config(x0 + 50e3 * east + 1e3 * up, START_SOW + 10.0, 0, START_WEEK)
    sc = gps.search_config(START_SOW + 10.0, 0, START_WEEK)
    out = {"tool": "snapshot_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_mhz_start": clk_start,
           "sm_clock_max_mhz": clk_max, "K": K, "s0": S0, "iters": args.iters, "rounds": args.rounds}
    stream = torch.cuda.Stream()
    for nchan, fixture in FIXTURES.items():
        frames, ch, chans = inputs(nchan)
        prns = [int(p) for p in chans["prn"]]
        fc = {int(p): float(f) for p, f in zip(ch[0]["prn"], ch[0]["f_carr"])}
        flo = np.array([STEP * round(fc[p] / STEP) - 2 * STEP for p in prns])
        dev = torch.empty(gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        with gps.Context(nchan, 1) as ctx, torch.cuda.stream(stream):
            ctx.set_nav_frames(frames)
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
            base = dict(device_ptr=dev.data_ptr(), nsamples=gps.BLOCK_SAMPLES, sample_size=gps.SC08, ms=K, s0=S0,
                        stream=stream.cuda_stream)
            cold = ctx.acquire(prns=range(1, 33), **base)
            res = cold[[p - 1 for p in prns]]
            cfg = gps.pvt_config(0, 1, 1)
            state = {}

            def measure():
                state["meas"] = ctx.snapshot_measure(res, prns=prns, **base)[None, :]
                return state["meas"]
            measure()
            arms = {"cold": lambda: ctx.acquire(prns=range(1, 33), **base),
                    "warm": lambda: ctx.acquire_windows(prns=prns, f_lo_prn=flo, step=STEP, nbins=5, **base),
                    "measure": measure,
                    "fix": lambda: ctx.pvt_snapshot(chans, state["meas"], cfg, ap_cfg),
                    "search": lambda: ctx.pvt_snapshot_search(chans, state["meas"], cfg, sc)}
            times, results = {}, {}
            for _ in range(args.rounds):
                for arm, fn in arms.items():
                    n = args.search_iters if arm == "search" else args.iters
                    for _ in range(1 if arm == "search" else args.warmup):
                        results[arm] = fn()
                    t = []
                    for _ in range(n):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record(stream)
                        results[arm] = fn()
                        b.record(stream)
                        b.synchronize()
                        t.append(a.elapsed_time(b))
                    times.setdefault(arm, []).append(round(float(np.median(t)), 4))
        fix, _ = results["fix"]
        sfix, rec = results["search"]
        err = lambda f: float(np.linalg.norm(np.array([f["x"][0], f["y"][0], f["z"][0]]) - x0))
        m = results["measure"][0]
        out["ch%d" % nchan] = {
            "fixture": fixture, "ms_median_per_round": times,
            "acquired": int(np.count_nonzero(results["cold"]["ratio"] >= 2.5)),
            "measured_ok": int(np.count_nonzero(m["status"] == gps.SNAP_OK)),
            "fix_status": int(fix["status"][0]), "fix_err_m": round(err(fix), 2),
            "search_status": int(sfix["status"][0]), "search_support": int(rec["support"][0]),
            "search_err_m": round(err(sfix), 2)}
    _, _, clk_end, _ = card()
    out["sm_clock_mhz_end"] = clk_end
    print(json.dumps(out))


if __name__ == "__main__":
    main()
