"""Time the standard acquisition search on one GPU and print one JSON line.

The standard search: 32 PRNs x 41 Doppler bins (-5000 .. 5000 Hz, 250 Hz) x 3000 code delays x K = 10 coherent 1 ms
periods, int8, searched in place (gpsb200_acquire_device) in a device-resident 32-channel stream that the GPU path
synthesizes first (the sky32_static_10s_i8 fixture's first blocks).

Reported: device-event time per search (median over --iters, after --warmup; the span covers the parameter uploads,
both kernels and the result download on the search's stream), the work counted from the shapes, and the share of the
formulation's ceiling (DESIGN §9): k_acq_grid is bound by shared-memory wavefronts -- one 8-byte prefix-sum pair per
(delay, replica sign change) per thread, i.e. two 128-byte wavefronts per warp and edge, at one wavefront per SM and
clock. The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi); the ceiling uses that
clock. Writes nothing; needs a GPU.

    python tools/acq_bench.py [--iters 20] [--warmup 3]
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

NPRN, NBINS, K, CODE = 32, 41, 10, 3000
TAUS = 3072          # delays computed per row (256 threads x 12; the last 72 are discarded)


def replica_edges(prn):
    """Entries of the padded sign-change list k_acq_grid walks for prn (acquire.cu: replica_edges)."""
    ca = gps.codegen(prn).astype(np.int64)
    n = int(np.count_nonzero(ca[1:] != ca[:-1]))
    n += n & 1
    return (n + 7) // 8 * 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("acq_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_mhz = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    g = np.load(os.path.join(ROOT, "tests", "golden", "sky32_static_10s_i8.npz"))
    nblk = 2
    ch = np.zeros((nblk, 32), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:nblk]
    ch["nav_frame"] = g["nav_frame_of_block"][:nblk, None]
    dev = torch.empty(nblk * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    stream = torch.cuda.Stream()
    times = []
    with gps.Context(32, nblk) as ctx, torch.cuda.stream(stream):
        ctx.set_nav_frames(g["nav_frames"])
        ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
        kw = dict(device_ptr=dev.data_ptr(), nsamples=nblk * gps.BLOCK_SAMPLES, sample_size=gps.SC08,
                  prns=range(1, NPRN + 1), ms=K, nbins=NBINS, stream=stream.cuda_stream)
        for _ in range(args.warmup):
            res = ctx.acquire(**kw)
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            res = ctx.acquire(**kw)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
    t_ms = float(np.median(times))
    edges = sum(replica_edges(p) for p in range(1, NPRN + 1))
    # per (PRN, bin, period): TAUS threads-delays x (edges + 2 end terms) 8-byte loads; 32 per warp = 2 wavefronts
    lds = NBINS * K * TAUS * (edges + 2 * NPRN)
    wavefronts = lds / 32 * 2
    ceiling_ms = wavefronts / (sms * clk_mhz * 1e6) * 1e3
    direct_macs = 2.0 * NPRN * NBINS * K * CODE * CODE      # the defining sum: C_I and C_Q, 3000 terms per delay
    acquired = int(np.count_nonzero(res["ratio"] >= 2.5))
    print(json.dumps({
        "tool": "acq_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_max_mhz": clk_mhz, "sms": sms,
        "search": "%d PRN x %d bins x %d delays x K=%d, int8, device source" % (NPRN, NBINS, CODE, K),
        "search_ms_median": round(t_ms, 4), "search_ms_min": round(float(np.min(times)), 4), "iters": args.iters,
        "replica_edges_total": edges, "lds64_per_thread_total": lds, "smem_wavefronts": wavefronts,
        "ceiling_ms_smem": round(ceiling_ms, 4), "share_of_ceiling": round(ceiling_ms / t_ms, 4),
        "direct_macs": direct_macs, "direct_equiv_tmac_per_s": round(direct_macs / (t_ms * 1e-3) / 1e12, 3),
        "acquired_of_32": acquired}))


if __name__ == "__main__":
    main()
