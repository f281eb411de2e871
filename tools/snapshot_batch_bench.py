"""Time the snapshot batch against the loop of single calls it stands for, on one GPU, and print one JSON line.

Workload per channel count: the first 100 blocks (10 s) of a fixture's stream (12 channels: sky12_static_35s_i8;
32 channels: sky32_static_10s_i8, which holds 99 blocks), synthesized into device memory first, and 10 ms windows
(K = 10, int8) every 10 ms from sample 1 000 of it: nwin of 1, 10, 100 and 990 (989 on the 99 blocks of sky32).
Per nwin two searches, each run both ways:
  cold   the standard grid: 32 PRNs x 41 bins (-5000 .. 5000 Hz, 250 Hz), all 32 measured
  warm   the channels' PRNs x 5 bins around each channel's f_carr in the window's block (snapshot_bench.py's rows)
  batch  one gpsb200_snapshot_batch_device call over the nwin windows (DESIGN §11.6)
  loop   per window gpsb200_acquire_device (or gpsb200_acquire_windows_device) and gpsb200_snapshot_measure_device
Both ways run in place on one device stream, timed with device events around the whole call or loop (Python binding
overhead included), alternating within each of --rounds rounds; medians over the iterations of a round. Reported per
window in ms and as windows per second, with whether the batch's results and records equal the loop's byte for byte
(checked in the same run). The card's name, power limit and SM clocks are read in the same run (nvidia-smi). Writes
nothing; needs a GPU.

    python tools/snapshot_batch_bench.py [--iters 20] [--rounds 2]
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

K, S0, EVERY, STEP, NBLK = 10, 1000, 30000, 250.0, 100
FIXTURES = {12: "sky12_static_35s_i8", 32: "sky32_static_10s_i8"}
NWINS = (1, 10, 100, 990)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2]), float(q[3])


def inputs(nchan):
    """The channel records of the fixture's first blocks (up to NBLK) and its NAV frames."""
    g = np.load(os.path.join(ROOT, "tests", "golden", FIXTURES[nchan] + ".npz"))
    nblk = min(NBLK, g["chans"].shape[0])
    ch = np.zeros((nblk, nchan), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:nblk]
    ch["nav_frame"] = g["nav_frame_of_block"][:nblk][:, None]
    return g["nav_frames"], ch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_batch_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_start, clk_max = card()
    out = {"tool": "snapshot_batch_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_mhz_start": clk_start,
           "sm_clock_max_mhz": clk_max, "K": K, "s0": S0, "every_samples": EVERY, "rounds": args.rounds}
    stream = torch.cuda.Stream()
    equal_all = True
    cfg = gps.snapshot_config()
    for nchan, fixture in FIXTURES.items():
        frames, ch = inputs(nchan)
        nsamples = ch.shape[0] * gps.BLOCK_SAMPLES
        dev = torch.empty(ch.shape[0] * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        prns = [int(p) for p in ch[0]["prn"]]
        row = {"fixture": fixture, "blocks": ch.shape[0]}
        with gps.Context(nchan, ch.shape[0], max_nav_frames=len(frames)) as ctx, torch.cuda.stream(stream):
            ctx.set_nav_frames(frames)
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
            src = dict(device_ptr=dev.data_ptr(), nsamples=nsamples, sample_size=gps.SC08, stream=stream.cuda_stream)
            for nwin in NWINS:
                nwin = min(nwin, (nsamples - gps.acq_window_samples(K) - S0) // EVERY + 1)
                s0 = S0 + EVERY * np.arange(nwin, dtype=np.int64)
                blk = s0 // gps.BLOCK_SAMPLES
                fc = [{int(p): float(f) for p, f in zip(ch[b]["prn"], ch[b]["f_carr"])} for b in blk]
                flo = np.array([[STEP * round(fc[w][p] / STEP) - 2 * STEP for p in prns] for w in range(nwin)])
                modes = {"cold": dict(prns=list(range(1, 33)), nbins=41, f_lo_prn=None),
                         "warm": dict(prns=prns, nbins=5, f_lo_prn=flo)}
                for mode, m in modes.items():
                    def batch():
                        return ctx.snapshot_batch(s0, ms=K, cfg=cfg, **m, **src)

                    def loop():
                        res = np.zeros((nwin, len(m["prns"])), gps.ACQ_RESULT_DTYPE)
                        meas = np.zeros((nwin, len(m["prns"])), gps.SNAPSHOT_DTYPE)
                        for w in range(nwin):
                            if m["f_lo_prn"] is None:
                                res[w] = ctx.acquire(prns=m["prns"], ms=K, s0=int(s0[w]), nbins=41, **src)
                            else:
                                res[w] = ctx.acquire_windows(prns=m["prns"], f_lo_prn=flo[w], step=STEP, nbins=5, ms=K,
                                                             s0=int(s0[w]), **src)
                            meas[w] = ctx.snapshot_measure(res[w], ms=K, s0=int(s0[w]), cfg=cfg, **src)
                        return res, meas
                    iters = max(1, min(args.iters, 100 // nwin))
                    arms, times, got = {"batch": batch, "loop": loop}, {}, {}
                    for arm, fn in arms.items():
                        got[arm] = fn()   # warm-up: every shape of the timed calls
                    for _ in range(args.rounds):
                        for arm, fn in arms.items():
                            t = []
                            for _ in range(iters):
                                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                                a.record(stream)
                                got[arm] = fn()
                                b.record(stream)
                                b.synchronize()
                                t.append(a.elapsed_time(b))
                            times.setdefault(arm, []).append(float(np.median(t)))
                    eq = all(x.tobytes() == y.tobytes() for x, y in zip(got["batch"], got["loop"]))
                    equal_all = equal_all and eq
                    per = {arm: [round(v / nwin, 4) for v in ts] for arm, ts in times.items()}
                    row["%s_%d" % (mode, nwin)] = {
                        "nwin": nwin, "iters": iters, "ms_per_window": per,
                        "windows_per_s": {arm: round(1000.0 / min(v), 1) for arm, v in per.items()},
                        "equal": eq, "measured_ok": int(np.count_nonzero(got["batch"][1]["status"] == gps.SNAP_OK))}
        out["ch%d" % nchan] = row
        del dev
    _, _, clk_end, _ = card()
    out["sm_clock_mhz_end"] = clk_end
    out["equal"] = equal_all
    print(json.dumps(out))


if __name__ == "__main__":
    main()
