"""Time the warm-start acquisition search (per-PRN Doppler windows) beside the standard search, on one GPU, and print
one JSON line.

Arms, alternating round by round in one run (device-event time per search, median over --iters after --warmup, in
place in a device-resident 32-channel int8 stream that the GPU path synthesizes first, the sky32_static_10s_i8
fixture's first blocks; K = 10):
  standard          32 PRNs x 41 bins (-5000 .. 5000 Hz, 250 Hz) x 3000 delays, gpsb200_acquire_device
  standard_parent   the same through another build of the library (--parent LIB), e.g. the parent commit's
  warm_12x5         12 PRNs x 5 bins around each PRN's f_carr on the cold grid, gpsb200_acquire_windows_device, with
                    the split of each row's delays the library chooses
  warm_12x5_splitS  the same with the split forced to S CTAs per row (S = 1: no split; 2, 3, 4, 6)
  warm_12x9, warm_12x9_splitS   the same with 9 bins
The card's name, power limit and SM clock are read in the same run (nvidia-smi). Writes nothing; needs a GPU.

    python tools/acq_windows_bench.py [--iters 20] [--warmup 3] [--rounds 3] [--parent path/to/libgpsb200.so]
"""
import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
gps = importlib.import_module("multi-sdr-gps-sim_b200")

K, STEP, NBLK = 10, 250.0, 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2]), float(q[3])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="another libgpsb200.so to time the standard search with")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("acq_windows_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_start, clk_max = card()

    g = np.load(os.path.join(ROOT, "tests", "golden", "sky32_static_10s_i8.npz"))
    ch = np.zeros((NBLK, 32), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:NBLK]
    ch["nav_frame"] = g["nav_frame_of_block"][:NBLK, None]
    dev = torch.empty(NBLK * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    stream = torch.cuda.Stream()
    n = NBLK * gps.BLOCK_SAMPLES
    # the 12 PRNs of the warm start: the first 12 slots, windows on the cold grid around f_carr
    prns12 = [int(p) for p in ch[0]["prn"][:12]]
    fc = {int(r["prn"]): float(r["f_carr"]) for r in ch[0]}

    def windows(nbins):
        h = nbins // 2
        return np.array([STEP * round(fc[p] / STEP) - h * STEP for p in prns12])

    parent = parent_h = None
    if args.parent:
        parent = C.CDLL(args.parent)
        parent.gpsb200_acquire_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(gps.AcqConfig),
                                                  C.c_void_p, C.c_void_p, C.c_void_p]
        parent_h = C.c_void_p()
        pc = gps.Config(0, 1, 1, 1, 0, 0)
        if parent.gpsb200_create(C.byref(pc), C.byref(parent_h)):
            raise SystemExit("acq_windows_bench: cannot create a context with %s" % args.parent)
    times = {}
    results = {}
    with gps.Context(32, NBLK) as ctx, torch.cuda.stream(stream):
        ctx.set_nav_frames(g["nav_frames"])
        ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
        base = dict(device_ptr=dev.data_ptr(), nsamples=n, sample_size=gps.SC08, ms=K, stream=stream.cuda_stream)
        cfg = gps.AcqConfig()
        cfg.ms, cfg.nprn, cfg.f_lo_hz, cfg.step_hz, cfg.nbins = K, 32, -5000.0, STEP, 41
        for i in range(32):
            cfg.prn[i] = i + 1
        pres = np.zeros(32, gps.ACQ_RESULT_DTYPE)

        def run_parent():
            if parent.gpsb200_acquire_device(parent_h, C.c_void_p(dev.data_ptr()), n, gps.SC08, C.byref(cfg),
                                             pres.ctypes.data, None, C.c_void_p(stream.cuda_stream)):
                raise SystemExit("acq_windows_bench: the parent build's search failed")
            return pres.copy()

        def warm(nbins, split):
            def fn():
                ctx.debug_acq_split(12, nbins, force=split)
                return ctx.acquire_windows(prns=prns12, f_lo_prn=windows(nbins), step=STEP, nbins=nbins, **base)
            return fn

        def standard():
            ctx.debug_acq_split(32, 41, force=0)
            return ctx.acquire(prns=range(1, 33), nbins=41, **base)

        arms = {"standard": standard}
        for nb in (5, 9):
            arms["warm_12x%d" % nb] = warm(nb, 0)
            for split in (1, 2, 3, 4, 6):
                arms["warm_12x%d_split%d" % (nb, split)] = warm(nb, split)
        if parent:
            arms["standard_parent"] = run_parent
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                for _ in range(args.warmup):
                    results[arm] = fn()
                t = []
                for _ in range(args.iters):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    results[arm] = fn()
                    b.record(stream)
                    b.synchronize()
                    t.append(a.elapsed_time(b))
                times.setdefault(arm, []).append(round(float(np.median(t)), 4))
        chosen = {"12x5": ctx.debug_acq_split(12, 5, force=0), "12x9": ctx.debug_acq_split(12, 9),
                  "32x41": ctx.debug_acq_split(32, 41)}
    if parent:
        parent.gpsb200_destroy(parent_h)
        assert results["standard"].tobytes() == results["standard_parent"].tobytes()
    for nb in (5, 9):        # every split gives the same bits
        for split in (1, 2, 3, 4, 6):
            assert results["warm_12x%d_split%d" % (nb, split)].tobytes() == results["warm_12x%d" % nb].tobytes()
    _, _, clk_end, _ = card()
    out = {"tool": "acq_windows_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_mhz_start": clk_start,
           "sm_clock_mhz_end": clk_end, "sm_clock_max_mhz": clk_max,
           "sms": torch.cuda.get_device_properties(0).multi_processor_count, "K": K, "iters": args.iters,
           "rounds": args.rounds, "ms_median_per_round": times,
           "rows": {"standard": 32 * 41, "warm_12x5": 12 * 5, "warm_12x9": 12 * 9}, "split_chosen": chosen,
           "acquired": {k: int(np.count_nonzero(v["ratio"] >= 2.5)) for k, v in results.items()},
           "standard_equals_parent": bool(parent) or None}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
