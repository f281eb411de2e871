"""Time the position fix on one GPU and print one JSON line.

Workload: 32 channels, 600 s of ideal epochs (tests/pvt_truth.py: what a perfect loop would record, built from the
scenario engine's records of the 32-satellite sky at the fixtures' Tokyo location), the ephemeris from the scenario's
NAV frames, a fix every 1 ms: 600 000 fixes in one gpsb200_pvt call. The epochs (32 x 600 001 records of 56 B, 1.08 GB)
go up in that call, from pinned host memory.

Reported: device-event time of the whole call (uploads, kernel, download; median over --iters after --warmup) and of
the kernel alone (gpsb200_pvt_replay, median over --iters), fixes per second of kernel time, the fixes' status counts,
and the largest difference from the numpy model (tests/pvt_model.py) over a seeded sample of --check fix instants. The
card's name, power limit and maximum SM clock are read in the same run (nvidia-smi). Writes nothing; needs a GPU.

With --raim SIGMA the same run also times the RAIM stage (gpsb200_pvt_raim, DESIGN §11.1) in three arms, alternating
--rounds times: the kernel without RAIM, with RAIM on the fault-free epochs, and with RAIM on epochs whose channel
--fault carries a 0.1-chip code-phase bias (about 29 m), so that every fix excludes once. Each arm's kernel time is the
median of its replays over all rounds; its verdict counts come from the call that set it up. With --araim MASK_DEG
two more arms alternate with them: the ARAIM stage (gpsb200_pvt_araim, DESIGN §11.2, the header's default allocations)
on the fault-free epochs, and with channel --fault's satellite clock (af0) off by twice the smallest bias that the
channel's own hypothesis detects (from the numpy model at the fix 1 s into the run), so that every fix excludes once.

With --coarse the same run also times coarse-time fixes (gpsb200_pvt_coarse, DESIGN §11.3) on the same epochs, the
a-priori position 50 km east and 1 km up of the truth and the a-priori time 10 s late, alternating with the plain
kernel --rounds times. Reported beside the kernel times: the Gauss-Newton iterations per fix of both arms and the
satellite evaluations (Kepler, orbit and clock) per channel and fix they imply -- 1 for gpsb200_pvt; 3 for the
prediction, one per iteration and 3 for the ambiguity check for the coarse call -- and the largest difference of the
coarse fixes from the numpy model (tests/coarse_model.py) over the --check sample.

With --search the same run also times position searches (gpsb200_pvt_search, DESIGN §11.4) on the default grid, at
2 000 fix instants spread over the run, on the 12 channels with the most epochs and on all 32, the a-priori time 10 s
late; each alternates with gpsb200_pvt_coarse at the same instants (a-priori position 50 km east, 1 km up) --rounds
times. Reported: kernel time per fix instant of both arms, the mean nodes searched and OK per instant, the status
counts, and the largest difference from the numpy model (tests/search_model.py) over --search-check seeded instants.

    python tools/pvt_bench.py [--iters 5] [--warmup 1] [--check 64] [--seconds 600] [--raim SIGMA [--fault C]]
                              [--araim MASK_DEG] [--coarse] [--search [--search-check 2]]
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
import pvt_model as PM   # noqa: E402
import pvt_truth as PT   # noqa: E402

LOC = (35.681298, 139.766247, 10.0)
START = (2024, 1, 7, 2, 0, 0.0)
START_SOW, START_WEEK = 7200.0, 2296     # START is Sunday 02:00 of GPS week 2296


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(",")
    return q[0].strip(), float(q[1]), float(q[2])


def workload(seconds):
    with tempfile.TemporaryDirectory() as d:
        nav = os.path.join(d, "sky32.nav")
        subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "gen_rinex.py"), "--nsat", "32", "--out", nav])
        ch, frames = gps.scenario(nav, *LOC, seconds=seconds + 0.2, max_chan=32, start=START)
        _, alpha, beta = PT.read_rinex(nav)
    fob = ch["nav_frame"][:, 0]
    prns = sorted({int(p) for p in np.unique(ch["prn"]) if p > 0})
    chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
    eps = []
    for c, prn in enumerate(prns):
        e, ae, ams = PT.ideal_epochs(ch, prn, frames, fob)
        eps.append(e)
        b = int(np.nonzero((ch["prn"] == prn).any(1))[0][0])
        slot = int(np.nonzero(ch[b]["prn"] == prn)[0][0])
        chans[c]["eph"] = gps.nav_ephemeris(gps.nav_words_of_frame(frames[int(fob[b])][slot]))[0]
        chans[c]["prn"], chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = prn, ae, ams
    return chans, eps, PT.klobuchar_broadcast(alpha, beta)


def replay_ms(ctx, stream, iters):
    import torch
    out = []
    ctx.pvt_replay(stream.cuda_stream)
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        ctx.pvt_replay(stream.cuda_stream)
        b.record(stream)
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def araim_bias(chans, packed, n, cfg, acfg, c):
    """Twice the smallest bias on channel c that its own hypothesis detects at the fix 1 s into the run: the bias moves
    the all-in-view fix by S0_qc b and the subset without c not at all, so it is detected once |S0_qc| b > T_c,q for some
    q (tests/araim_model.py)."""
    import araim_model as AM
    eps = [packed[k, :n[k]] for k in range(len(n))]
    one = gps.pvt_config(int(cfg["s0"]) + 1000 * int(cfg["step"]), 1, 1, (cfg["alpha"], cfg["beta"]))
    kh, kv = gps.araim_kfa(float(acfg["p_fa_vert"]), float(acfg["p_fa_horz"]))
    _, _, rec, extra = AM.araim(chans, eps, one, acfg, kh, kv)
    o = extra[0][0]
    kk = int(np.nonzero(o["idx"] == c)[0][0])
    return 2.0 * float(np.min(o["T"][kk] / np.abs(o["S0"][:, kk])))


def raim_arms(ctx, stream, chans, packed, n, cfg, args):
    """Kernel time of the three arms, alternating, and the verdict counts of each."""
    bad = packed.copy()
    add = int(round(0.1 * 2.0 ** 32))
    assert int(bad[args.fault, :n[args.fault]]["code_phase"].max()) + add < 2 ** 32
    bad[args.fault, :n[args.fault]]["code_phase"] += np.uint32(add)
    rcfg = gps.raim_config(args.raim)
    arms = {"plain": lambda: ctx.pvt(chans, packed, cfg, nepochs=n),
            "raim": lambda: ctx.pvt_raim(chans, packed, cfg, rcfg, nepochs=n),
            "raim_fault": lambda: ctx.pvt_raim(chans, bad, cfg, rcfg, nepochs=n)}
    if args.araim is not None:
        acfg = gps.araim_config(mask_deg=args.araim)
        arms["araim"] = lambda: ctx.pvt_araim(chans, packed, cfg, acfg, nepochs=n)
        bias = araim_bias(chans, packed, n, cfg, acfg, args.fault)
        achans = chans.copy()
        achans[args.fault]["eph"]["af0"] += bias / PM.C
        arms["araim_fault"] = lambda: ctx.pvt_araim(achans, packed, cfg, acfg, nepochs=n)
    times = {k: [] for k in arms}
    verdicts = {}
    for _ in range(args.rounds):
        for k, call in arms.items():
            got = call()
            if k != "plain":
                v, c = np.unique(got[1]["verdict"], return_counts=True)
                verdicts[k] = {int(a): int(b) for a, b in zip(v, c)}
                if k.endswith("_fault"):
                    tested = got[1]["verdict"] != gps.RAIM_UNAVAILABLE
                    verdicts[k + "_excluded_only_channel"] = bool(np.all(got[1]["excluded"][tested] ==
                                                                               1 << args.fault))
            times[k] += replay_ms(ctx, stream, args.iters)
    out = {"sigma": args.raim, "araim_mask_deg": args.araim, "araim_fault_bias_m": round(bias, 3) if args.araim is not None else None, "fault_channel": args.fault, "rounds": args.rounds, "verdicts": verdicts}
    for k, t in times.items():
        out[k + "_kernel_ms_median"] = round(float(np.median(t)), 3)
        out[k + "_kernel_ms_min"] = round(float(np.min(t)), 3)
    return out


def coarse_arms(ctx, stream, chans, eps, packed, n, cfg, args):
    """Kernel time of the plain and coarse arms, alternating; iterations, satellite evaluations and the model check."""
    import coarse_model as CM
    x0 = PM.llh_ecef(*LOC)
    lat, lon, _ = PM.ecef_llh(x0)
    east = np.array([-np.sin(lon), np.cos(lon), 0.0])
    up = np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)])
    ap = gps.coarse_config(x0 + 50e3 * east + 1e3 * up, START_SOW + 10.0, 0, START_WEEK)
    arms = {"plain": lambda: ctx.pvt(chans, packed, cfg, nepochs=n),
            "coarse": lambda: ctx.pvt_coarse(chans, packed, cfg, ap, want_ms=True, nepochs=n)}
    times = {k: [] for k in arms}
    got = {}
    for _ in range(args.rounds):
        for k, call in arms.items():
            got[k] = call()
            times[k] += replay_ms(ctx, stream, args.iters)
    plain = got["plain"]
    fix, rec, ms = got["coarse"]
    ok = fix["status"] == gps.FIX_OK
    it_p, it_c = float(plain["iterations"].mean()), float(fix["iterations"][ok].mean())
    worst = {f: 0.0 for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz")}
    worst["delta_s"] = 0.0
    rng = np.random.default_rng(2)
    for i in rng.choice(len(fix), size=min(args.check, len(fix)), replace=False):
        one = gps.pvt_config(int(cfg["s0"]) + int(i) * int(cfg["step"]), 1, 1, (cfg["alpha"], cfg["beta"]))
        want, wrec, _, wms = CM.coarse(chans, eps, one, ap)
        assert int(want["status"][0]) == int(fix["status"][i]) and np.array_equal(wms[0], ms[i])
        if fix["status"][i] == gps.FIX_OK:
            for f in worst:
                a, b = (rec["delta"][i], wrec["delta"][0]) if f == "delta_s" else (fix[f][i], want[f][0])
                worst[f] = max(worst[f], abs(float(a) - float(b)))
    out = {"apriori": "50 km east, 1 km up, +10 s", "rounds": args.rounds,
           "status_counts": {int(k): int(v) for k, v in zip(*np.unique(fix["status"], return_counts=True))},
           "iterations_mean": {"plain": round(it_p, 3), "coarse": round(it_c, 3)},
           "satellite_evals_per_channel_fix": {"plain": 1, "coarse": round(3 + it_c + 3, 3)},
           "max_abs_diff_vs_model": {k: float("%.3g" % v) for k, v in worst.items()}}
    for k, t in times.items():
        out[k + "_kernel_ms_median"] = round(float(np.median(t)), 3)
        out[k + "_kernel_ms_min"] = round(float(np.min(t)), 3)
    return out


def search_arms(ctx, stream, chans, eps, packed, n, iono, args):
    """Per channel count: kernel time per instant of the coarse and search arms, alternating; counts; model check."""
    import search_model as SM
    x0 = PM.llh_ecef(*LOC)
    lat, lon, _ = PM.ecef_llh(x0)
    east = np.array([-np.sin(lon), np.cos(lon), 0.0])
    up = np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)])
    ap = gps.coarse_config(x0 + 50e3 * east + 1e3 * up, START_SOW + 10.0, 0, START_WEEK)
    sc = gps.search_config(START_SOW + 10.0, 0, START_WEEK, gps.SEARCH_NODES)
    nfix = 2000
    step = (args.seconds * 3000000 - 6000) // nfix
    out = {"instants": nfix, "nodes": int(sc["nodes"]), "rounds": args.rounds}
    for nch in (12, 32):
        keep = np.sort(np.argsort(-n, kind="stable")[:nch])
        ch, pk, nn = chans[keep], np.ascontiguousarray(packed[keep]), n[keep]
        ev = [eps[k] for k in keep]
        c = gps.pvt_config(3000, step, nfix, iono)
        arms = {"coarse": lambda: ctx.pvt_coarse(ch, pk, c, ap, nepochs=nn),
                "search": lambda: ctx.pvt_search(ch, pk, c, sc, want_residuals=True, want_ms=True, nepochs=nn)}
        times = {k: [] for k in arms}
        got = {}
        for _ in range(args.rounds):
            for k, call in arms.items():
                got[k] = call()
                times[k] += replay_ms(ctx, stream, args.iters)
        fix, rec, res, ms = got["search"]
        worst = {f: 0.0 for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz", "rms")}
        worst["delta_s"] = 0.0
        differ = set()
        rng = np.random.default_rng(3)
        for i in rng.choice(nfix, size=min(args.search_check, nfix), replace=False):
            one = gps.pvt_config(int(c["s0"]) + int(i) * step, 1, 1, iono)
            want, wrec, _, wms = SM.search(ch, ev, one, sc)
            if int(want["status"][0]) != int(fix["status"][i]):
                differ.add("status")
            if not np.array_equal(wms[0], ms[i]):
                differ.add("ms")
            for f in ("winner", "searched", "ok", "support"):
                if int(wrec[f][0]) != int(rec[f][i]):
                    differ.add("%s %d/%d" % (f, int(rec[f][i]), int(wrec[f][0])))
            if rec["winner"][i] >= 0:
                for f in worst:
                    a, b = (rec["delta"][i], wrec["delta"][0]) if f == "delta_s" else (fix[f][i], want[f][0])
                    worst[f] = max(worst[f], abs(float(a) - float(b)))
        err = np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - x0, axis=1)
        t_c, t_s = float(np.median(times["coarse"])), float(np.median(times["search"]))
        out["ch%d" % nch] = {
            "coarse_kernel_ms_median": round(t_c, 3), "search_kernel_ms_median": round(t_s, 3),
            "search_kernel_ms_min": round(float(np.min(times["search"])), 3),
            "coarse_us_per_instant": round(1e3 * t_c / nfix, 3), "search_ms_per_instant": round(t_s / nfix, 4),
            "searched_mean": round(float(rec["searched"].mean()), 1), "ok_mean": round(float(rec["ok"].mean()), 2),
            "ok_max": int(rec["ok"].max()), "support_mean": round(float(rec["support"].mean()), 2),
            "status_counts": {int(k): int(v) for k, v in zip(*np.unique(fix["status"], return_counts=True))},
            "max_err_vs_truth_m": round(float(np.nanmax(err)), 4),
            "checked": min(args.search_check, nfix), "counts_differing_from_model": sorted(differ),
            "max_abs_diff_vs_model": {k: float("%.3g" % v) for k, v in worst.items()}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=64)
    ap.add_argument("--seconds", type=int, default=600)
    ap.add_argument("--raim", type=float, default=None)
    ap.add_argument("--fault", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--araim", type=float, default=None)
    ap.add_argument("--coarse", action="store_true")
    ap.add_argument("--search", action="store_true")
    ap.add_argument("--search-check", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pvt_bench: no CUDA device (this measurement has no CPU fallback)")
    name, power_w, clk_mhz = card()
    chans, eps, iono = workload(args.seconds)
    nfix = args.seconds * 1000
    cfg = gps.pvt_config(3000, 3000, nfix, iono)
    # the epochs packed once as the C call takes them, in pinned memory
    n = np.array([len(e) for e in eps], np.int32)
    host = torch.empty(len(eps) * int(n.max()) * gps.TRACK_EPOCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True)
    packed = host.numpy().view(gps.TRACK_EPOCH_DTYPE).reshape(len(eps), int(n.max()))
    for c, e in enumerate(eps):
        packed[c, :len(e)] = e
    stream = torch.cuda.Stream()
    call, kern = [], []
    with gps.Context(1, 1) as ctx:
        for _ in range(args.warmup):
            fix = ctx.pvt(chans, packed, cfg, nepochs=n)
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fix = ctx.pvt(chans, packed, cfg, nepochs=n)
            b.record(stream)
            b.synchronize()
            call.append(a.elapsed_time(b))
        ctx.pvt_replay(stream.cuda_stream)
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            ctx.pvt_replay(stream.cuda_stream)
            b.record(stream)
            b.synchronize()
            kern.append(a.elapsed_time(b))
        raim = raim_arms(ctx, stream, chans, packed, n, cfg, args) if args.raim is not None else None
        coarse = coarse_arms(ctx, stream, chans, eps, packed, n, cfg, args) if args.coarse else None
        search = search_arms(ctx, stream, chans, eps, packed, n, iono, args) if args.search else None
    rng = np.random.default_rng(1)
    worst = {f: 0.0 for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz")}
    for i in rng.choice(nfix, size=min(args.check, nfix), replace=False):
        one = gps.pvt_config(int(cfg["s0"]) + int(i) * int(cfg["step"]), 1, 1, iono)
        want, _, _ = PM.pvt(chans, eps, one)
        assert int(want["status"][0]) == int(fix["status"][i]) and int(want["mask"][0]) == int(fix["mask"][i])
        for f in worst:
            if fix["status"][i] == gps.FIX_OK:
                worst[f] = max(worst[f], abs(float(fix[f][i]) - float(want[f][0])))
    t_call, t_kern = float(np.median(call)), float(np.median(kern))
    st = {int(k): int(v) for k, v in zip(*np.unique(fix["status"], return_counts=True))}
    print(json.dumps({"tool": "pvt_bench", "gpu": name, "power_limit_w": power_w, "sm_clock_max_mhz": clk_mhz,
                      "channels": len(eps), "seconds": args.seconds, "fixes": nfix, "epochs_per_channel": max(map(len, eps)),
                      "call_ms_median": round(t_call, 3), "call_ms_min": round(float(np.min(call)), 3),
                      "kernel_ms_median": round(t_kern, 3), "kernel_ms_min": round(float(np.min(kern)), 3),
                      "iters": args.iters, "fixes_per_s_kernel": round(nfix / (t_kern * 1e-3)),
                      "status_counts": st, "checked": min(args.check, nfix),
                      "max_abs_diff_vs_model": {k: float("%.3g" % v) for k, v in worst.items()},
                      **({"raim": raim} if raim is not None else {}),
                      **({"coarse": coarse} if coarse is not None else {}),
                      **({"search": search} if search is not None else {})}), flush=True)


if __name__ == "__main__":
    main()
