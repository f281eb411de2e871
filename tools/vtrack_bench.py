"""Device-event time of gpsb200_vtrack per period and per filter update at 12 and 32 channels over 10 s of signal,
at several cluster sizes (DESIGN §10.1). Prints one JSON line per case and appends it to --out when given.

    python tools/vtrack_bench.py [--out profiles/h100_vtrack_bench.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    import tempfile
    import pathlib
    import torch
    import pvt_model as PM
    from scenario import gps
    from test_scenario import LOC
    from test_track import START_SOW
    from test_vtrack import chans_of, seed_x, stream
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--blocks", type=int, default=99)   # sky32_static_10s holds 99 blocks
    a = ap.parse_args()
    name_card = card()
    tmp = pathlib.Path(tempfile.mkdtemp())
    for name, nsat in (("sky12_static_35s_i8", 12), ("sky32_static_10s_i8", 32)):
        g, ch, iq = stream(name, a.blocks)
        prns = [int(p) for p in ch[0]["prn"] if p > 0]
        chans = chans_of(tmp, nsat, prns)
        cfg = gps.vtrack_config()
        st = gps.vtrack_seed(cfg, seed_x(PM.llh_ecef(*LOC)), START_SOW, 0, prns)
        d = torch.from_numpy(iq).cuda()
        n = iq.size // 2
        with gps.Context(32, 1) as ctx:
            for K in (1, 8, 16 if len(prns) >= 16 else len(prns)):
                ctx.debug_vtrack_cluster(K)
                ctx.vtrack(chans, cfg, st, 100000, device_ptr=d.data_ptr(), nsamples=n)   # warm-up
                times = []
                for _ in range(3):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s = torch.cuda.current_stream()
                    e0.record(s)
                    f, o, _, _ = ctx.vtrack(chans, cfg, st, 100000, device_ptr=d.data_ptr(), nsamples=n,
                                            stream=s.cuda_stream)
                    e1.record(s)
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1))
                ms = float(np.median(times))
                periods = len(f) * int(cfg["periods"])
                rec = dict(tool="vtrack_bench", card=name_card, stream=name, nchan=len(prns), cluster=K,
                           signal_s=n / 3e6, updates=len(f), call_ms=ms, us_per_period=1e3 * ms / periods,
                           us_per_update=1e3 * ms / len(f), runs_ms=times)
                line = json.dumps(rec)
                print(line)
                if a.out:
                    with open(a.out, "a") as fh:
                        fh.write(line + "\n")


if __name__ == "__main__":
    main()
