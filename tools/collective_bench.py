"""Time collective detection (gpsb200_collective_device; DESIGN §11.7) on one GPU and print one JSON line.

Workload per channel count: the first block of a fixture's stream (12 channels: sky12_static_35s_i8; 32 channels:
sky32_static_10s_i8), synthesized into device memory first; one 10 ms window (K = 10, int8) from sample 1 000 searched
on the standard grid (32 PRNs x 41 bins), the ephemeris of the fixture's sky (oracle/gen_rinex.py), the a-priori
position 1.5 km east and 0.75 km north of the receiver and the a-priori time 0.5 s late. Two lattices a user would
run: +-5 km at 100 m east and north with +-1 s at 0.1 s (214 221 hypotheses), and the same with +-1 s at 0.01 s
(2 050 401, ten times as many). Per lattice:
  call    the whole call (search, normalisation, scores, pick, seeds, downloads), device events around it, median of
          --iters calls after one warm-up call
  score   k_cd_score alone: its device time in a torch.profiler trace of --iters calls (median), and the grid bytes it
          reads per second, from shapes: nused x 3000 x 2 bytes per hypothesis over that time
with the record's status, nused, error of the winner from the receiver (m) and score ratio. The card's name, power
limit and SM clocks are read in the same run (nvidia-smi). Writes nothing; needs a GPU.

    python tools/collective_bench.py [--iters 5]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
gps = importlib.import_module("multi-sdr-gps-sim_b200")

K, S0, WEEK = 10, 1000, 2296
FIXTURES = {12: "sky12_static_35s_i8", 32: "sky32_static_10s_i8"}
LOC = (35.681298, 139.766247, 10.0)
LATTICES = {"214k": (5000.0, 100.0, 1.0, 0.1), "2.05M": (5000.0, 100.0, 1.0, 0.01)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2]), float(q[3])


def inputs(nchan):
    g = np.load(os.path.join(ROOT, "tests", "golden", FIXTURES[nchan] + ".npz"))
    ch = np.zeros((1, nchan), gps.CHAN_DTYPE)
    for f in ("prn", "iword", "ibit", "icode", "f_carr", "f_code", "carr_phase", "code_phase", "gain"):
        ch[f] = g["chans"][f][:1]
    ch["nav_frame"] = g["nav_frame_of_block"][:1][:, None]
    return g["nav_frames"], ch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import pvt_model as PM
    from test_coarse import enu
    from test_track import START_SOW as sow
    if not torch.cuda.is_available():
        raise SystemExit("collective_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_start, clk_max = card()
    out = {"tool": "collective_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_mhz_start": clk_start,
           "sm_clock_max_mhz": clk_max, "K": K, "s0": S0, "iters": args.iters}
    stream = torch.cuda.Stream()
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    apri = gps.coarse_config(x0 + 1500.0 * e + 750.0 * n, sow + 0.5, 0, WEEK)
    tmp = tempfile.mkdtemp()
    for nchan, fixture in FIXTURES.items():
        nav = os.path.join(tmp, "sky%d.nav" % nchan)
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", str(nchan),
                               "--out", nav])
        eph = gps.rinex_ephemeris(nav, WEEK, sow)
        frames, ch = inputs(nchan)
        dev = torch.empty(gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        row = {"fixture": fixture}
        with gps.Context(nchan, 1, max_nav_frames=len(frames)) as ctx, torch.cuda.stream(stream):
            ctx.set_nav_frames(frames)
            ctx.synth_blocks_device(ch, gps.SC08, dev.data_ptr(), stream=stream.cuda_stream)
            src = dict(device_ptr=dev.data_ptr(), nsamples=gps.BLOCK_SAMPLES, sample_size=gps.SC08,
                       stream=stream.cuda_stream, ms=K, s0=S0)
            for lname, (ext, step, ext_s, step_s) in LATTICES.items():
                cfg = gps.collective_config(ext, step, ext_s, step_s, distinct_m=1000.0)
                nhyp = int(np.prod(cfg["n"].astype(np.int64)))

                def call():
                    return ctx.collective(eph, apri, cfg, **src)
                res, seed, rec = call()
                t = []
                for _ in range(args.iters):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    call()
                    b.record(stream)
                    b.synchronize()
                    t.append(a.elapsed_time(b))
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.iters):
                        call()
                    torch.cuda.synchronize()
                ks = [ev.device_time / 1000.0 if hasattr(ev, "device_time") else ev.cuda_time / 1000.0
                      for ev in prof.events() if "k_cd_score" in ev.name]
                other = {}
                for ev in prof.events():
                    if ev.name.startswith("_ZN7gpsb2002cd") or "k_cd_" in ev.name or "k_acq_" in ev.name:
                        key = next((k for k in ("k_cd_rowsum", "k_cd_q", "k_cd_setup", "k_cd_score", "k_cd_pick",
                                                "k_cd_seed", "k_acq_grid", "k_acq_pick") if k in ev.name), ev.name[:40])
                        dt = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
                        other.setdefault(key, []).append(dt / 1000.0)
                kms = float(np.median(ks)) if ks else None
                nbytes = int(rec["nused"]) * 3000 * 2 * nhyp
                row[lname] = {
                    "nhyp": nhyp, "call_ms": round(float(np.median(t)), 3),
                    "call_ms_all": [round(v, 3) for v in t],
                    "score_kernel_ms": None if kms is None else round(kms, 3),
                    "grid_bytes": nbytes,
                    "grid_gb_per_s": None if not kms else round(nbytes / (kms * 1e-3) / 1e9, 1),
                    "kernels_ms_median": {k: round(float(np.median(v)), 4) for k, v in other.items()},
                    "status": int(rec["status"]), "nused": int(rec["nused"]),
                    "passed_alone": int((res["ratio"] >= 2.5).sum()),
                    "winner_error_m": round(float(np.linalg.norm(rec["x"] - x0)), 2),
                    "o_t": float(rec["o_t"]),
                    "score_ratio": round(float(rec["runner_score"]) / max(1, int(rec["score"])), 4)}
        out["ch%d" % nchan] = row
        del dev
    _, _, clk_end, _ = card()
    out["sm_clock_mhz_end"] = clk_end
    print(json.dumps(out))


if __name__ == "__main__":
    main()
