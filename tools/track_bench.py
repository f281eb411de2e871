"""Time the tracking loops on one GPU and print one JSON line per channel count.

The stream: the first 99 blocks (9.9 s) of a fixture's scenario (sky12_static_35s_i8 for 12 channels,
sky32_static_10s_i8 for 32), synthesized into device memory by the GPU path. Every PRN is acquired at the start
(gpsb200_acquire_device, 10 periods, 100 Hz bins) and then tracked in place over the whole buffer in one
gpsb200_track_device call (one CTA per channel, each a sequential loop over about 9 900 periods).

k_track is latency-bound: one dependent loop update per millisecond of signal and channel. Reported: device-event time
of the call (median over --iters, after --warmup; it covers the state upload, the kernel and the downloads), periods per
channel, milliseconds of signal per millisecond of device time (the figure of merit), and the time per period (the
per-step latency of the loop). The card's name, power limit and maximum SM clock are read in the same run
(nvidia-smi). Writes nothing; needs a GPU.

    python tools/track_bench.py [--iters 5] [--warmup 1]
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
gps = importlib.import_module("multi-sdr-gps-sim_b200")

NBLK = 99
FIXTURE = {12: "sky12_static_35s_i8", 32: "sky32_static_10s_i8"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2])


def run(nchan, iters, warmup, torch):
    g = np.load(os.path.join(ROOT, "tests", "golden", FIXTURE[nchan] + ".npz"))
    ch = np.zeros((NBLK, nchan), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:NBLK]
    ch["nav_frame"] = g["nav_frame_of_block"][:NBLK, None]
    n = NBLK * gps.BLOCK_SAMPLES
    dev = torch.empty(NBLK * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    stream = torch.cuda.Stream()
    times = []
    with gps.Context(nchan, NBLK, max_nav_frames=len(g["nav_frames"])) as ctx, torch.cuda.stream(stream):
        ctx.set_nav_frames(g["nav_frames"])
        ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
        prns = [int(p) for p in ch[0]["prn"] if p > 0]
        res = ctx.acquire(device_ptr=dev.data_ptr(), nsamples=n, sample_size=gps.SC08, prns=prns, ms=10, step=100.0,
                          nbins=101, stream=stream.cuda_stream)
        st = np.array([gps.track_start(int(r["prn"]), float(r["doppler_hz"]), int(r["delay"])) for r in res])
        kw = dict(device_ptr=dev.data_ptr(), nsamples=n, sample_size=gps.SC08, stream=stream.cuda_stream)
        for _ in range(warmup):
            eps, _ = ctx.track(st, **kw)
        for _ in range(iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            eps, _ = ctx.track(st, **kw)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
    t_ms = float(np.median(times))
    periods = max(e.size for e in eps)
    signal_ms = float(periods)          # one period is one C/A code epoch: 1 ms of signal
    locked = sum(int(e["lock"][-1]) for e in eps)
    return {"channels": nchan, "stream": FIXTURE[nchan] + " blocks 0-%d, int8, device source" % (NBLK - 1),
            "call_ms_median": round(t_ms, 3), "call_ms_min": round(float(np.min(times)), 3), "iters": iters,
            "periods_per_channel": periods, "signal_ms_per_device_ms": round(signal_ms / t_ms, 2),
            "us_per_period": round(t_ms * 1e3 / periods, 3), "locked_at_end": locked}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("track_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_mhz = card()
    for nchan in (12, 32):
        r = {"tool": "track_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_max_mhz": clk_mhz}
        r.update(run(nchan, args.iters, args.warmup, torch))
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
