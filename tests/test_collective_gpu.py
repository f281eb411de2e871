"""gpsb200_collective on the GPU: the search's results against gpsb200_acquire, the device's table of predicted cells
against tests/collective_model.py, its scores, record and seeds against the model scoring that table over the
device's own grid (byte for byte, but for the winner's position, latitude, longitude and height, within ulps), host
and device sources, the clean and weakened snapshot chains it seeds, the CLI on the weakened stream, the argument
checks, and compute-sanitizer."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import collective_model as CM
import pvt_model as PM
import scenario
from scenario import gps
from test_coarse import WEEK, enu, static_rows
from test_collective import PRNS, WEAK_POS, bound, check_seeds, ephemeris, pvt_chans, weak_block
from test_pvt import check_truth
from test_scenario import LOC
from test_snapshot import BOUNDS, S0, K, block_stream
from test_track import START_SOW

pytestmark = pytest.mark.gpu

BOUNDARY = 1e-6
LLH = dict(x=1e-6, lat_deg=1e-12, lon_deg=1e-12, height=1e-6)


@pytest.fixture(scope="module")
def ctx():
    with gps.Context(12, 1) as c:
        yield c


@pytest.fixture(scope="module")
def sky(tmp_path_factory):
    eph, iono = ephemeris(tmp_path_factory.mktemp("nav"), 12, START_SOW)
    eph32, _ = ephemeris(tmp_path_factory.mktemp("nav32"), 32, START_SOW)
    return eph, eph32, iono


def check_against_model(ctx, iq, ss, prns, eph, ap, cfg, f_lo_prn=None, nbins=41, step=250.0, f_lo=-5000.0, ms=K):
    """One call with scores and table, checked against acquire and the model; -> (res, seed, rec)."""
    kw = dict(iq=iq, sample_size=ss, prns=prns, ms=ms, s0=S0, nbins=nbins, step=step)
    if f_lo_prn is None:
        res0, P = ctx.acquire(f_lo=f_lo, want_grid=True, **kw)
        flo = np.full(len(prns), f_lo)
    else:
        res0, P = ctx.acquire_windows(f_lo_prn=f_lo_prn, want_grid=True, **kw)
        flo = np.asarray(f_lo_prn, np.float64)
    res, seed, rec, sc, tb = ctx.collective(eph, ap, cfg, f_lo=f_lo, f_lo_prn=f_lo_prn, want_scores=True,
                                            want_table=True, **kw)
    assert res.tobytes() == res0.tobytes()
    mu, _ = CM.normalise(P)
    use = CM.used(eph, prns, ap, S0, cfg["mask_deg"], mu)
    assert rec["nused"] == use.sum() and rec["used"] == int((use.astype(np.int64) << np.arange(use.size)).sum())
    mrec, mseed, S, b, _ = CM.collective(P, res0, eph, prns, ap, S0, cfg, flo, step,
                                         cells=tb.view(np.int32).reshape(tb.shape[0], len(prns), 2))
    if use.sum() >= CM.MIN_USED:
        cells, dc, jc = CM.table(eph, prns, use, ap, S0, cfg, flo, step, nbins)
        got = tb.view(np.int32).reshape(cells.shape)
        diff = (got != cells).any(-1)
        near = (np.abs(dc - np.floor(dc) - 0.5) < BOUNDARY) | (np.abs(jc - np.floor(jc) - 0.5) < BOUNDARY)
        assert not (diff & ~near).any(), np.argwhere(diff & ~near)[:5]
    assert np.array_equal(sc["score"], S) and np.array_equal(sc["shift"], b)
    mrec = np.array(mrec, dtype=gps.COLLECTIVE_DTYPE)
    # x_h* = x_a + o_e E + o_n N + o_u U takes E, N, U from the WGS-84 conversion at x_a, whose transcendentals differ
    # from numpy's by ulps: the position and its latitude, longitude and height agree within 1 um (and 1e-12 degrees)
    for f in gps.COLLECTIVE_DTYPE.names:
        if f in LLH:
            assert np.allclose(rec[f], mrec[f], rtol=0.0, atol=LLH[f], equal_nan=True), (f, rec, mrec)
        else:
            assert np.asarray(rec[f]).tobytes() == np.asarray(mrec[f]).tobytes(), (f, rec, mrec)
    assert seed.tobytes() == np.asarray(mseed, dtype=gps.ACQ_RESULT_DTYPE).tobytes()
    return res, seed, rec


def apriori(dx=np.zeros(3), dt=0.0, sow=START_SOW):
    return gps.coarse_config(PM.llh_ecef(*LOC) + dx, sow + dt, 0, WEEK)


@pytest.mark.parametrize("kind", ["int8", "int16"])
@pytest.mark.parametrize("nprn", [1, 12, 32])
@pytest.mark.parametrize("windows", [False, True])
def test_equals_the_model_on_random_input(ctx, sky, kind, nprn, windows):
    rng = np.random.default_rng(nprn * 7 + (kind == "int16") + 2 * windows)
    n = S0 + gps.acq_window_samples(K) + 10
    if kind == "int8":
        iq, ss = rng.integers(-128, 128, 2 * n, dtype=np.int8), gps.SC08
    else:
        iq, ss = rng.integers(-32768, 32768, 2 * n, dtype=np.int16), gps.SC16   # saturates the >> 4 reduction
    prns = [int(p) for p in rng.permutation(32)[:nprn] + 1]
    eph = sky[1]
    f_lo_prn = rng.uniform(-6000.0, 4000.0, nprn) if windows else None
    nb = 5 if windows else 41
    cfg = gps.collective_config(600.0, 200.0, 0.5, 0.5, mask_deg=-90.0, distinct_m=300.0)
    _, _, rec = check_against_model(ctx, iq, ss, prns, eph, apriori(), cfg, f_lo_prn, nbins=nb)
    assert rec["status"] == (gps.CD_FEW if rec["nused"] < gps.CD_MIN_USED else rec["status"])


def test_host_and_device_sources_give_the_same_bytes(ctx, sky):
    import torch
    _, ch, iq = block_stream("sky12_static_35s_i8", 0)
    cfg = gps.collective_config(1000.0, 250.0, 0.5, 0.5)
    host = ctx.collective(sky[0], apriori(), cfg, iq=iq, want_scores=True, want_table=True)
    d = torch.from_numpy(iq.copy()).cuda()
    torch.cuda.synchronize()
    dev = ctx.collective(sky[0], apriori(), cfg, device_ptr=d.data_ptr(), nsamples=iq.size // 2, want_scores=True,
                         want_table=True)
    for a, b in zip(host, dev):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("chain", ["clean", "weak"])
def test_chain_on_sky12_static(ctx, sky, chain):
    """The device call equals the model on sky12_static_35s block 0 (clean, or weakened so that only 4 PRNs pass
    alone); its seeds, measured by gpsb200_snapshot_measure with min_ratio 0 and fixed by gpsb200_pvt_snapshot from
    the winner, give a fix within the snapshot bounds."""
    g = scenario.load_golden("sky12_static_35s_i8")
    if chain == "clean":
        _, ch, iq = block_stream("sky12_static_35s_i8", 0)
    else:
        ch, iq = weak_block(g)
    eph, _, iono = sky
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    ap = apriori(1500.0 * e + 750.0 * n, 0.5)
    cfg = gps.collective_config(3500.0, 250.0, 1.5, 0.5, distinct_m=1000.0)
    res, seed, rec = check_against_model(ctx, iq, gps.SC08, PRNS, eph, ap, cfg)
    if chain == "weak":
        assert (res["ratio"] >= 2.5).sum() <= 4
    assert rec["status"] == gps.CD_OK and np.linalg.norm(rec["x"] - x0) <= bound(cfg)
    check_seeds(seed, ch, rec)
    prns = sorted(int(p) for p in ch[0]["prn"] if p > 0)
    meas = ctx.snapshot_measure(seed, iq=iq, ms=K, s0=S0, prns=PRNS, cfg=gps.snapshot_config(0.0))
    assert (meas[:12]["status"] == gps.SNAP_OK).all()
    sel = [int(np.nonzero(meas["prn"] == p)[0][0]) for p in prns]
    fixes, _ = ctx.pvt_snapshot(pvt_chans(eph, prns), meas[sel], gps.pvt_config(0, 1, 1, iono),
                                gps.coarse_config(rec["x"], float(ap["t_a"]) + float(rec["o_t"]), 0, WEEK))
    assert fixes["status"][0] == gps.FIX_OK and fixes["nused"][0] == 12
    check_truth(fixes, static_rows(ch, LOC), START_SOW, BOUNDS["pos"] if chain == "clean" else WEAK_POS, BOUNDS["time"],
                BOUNDS["vel"])


def raw_collective(ctx, iq, eph, ap, cfg, prns=range(1, 33), ms=K, s0=S0, f_lo_prn=None, nulls=()):
    """gpsb200_collective through ctypes with every output pre-filled with 0xA5 bytes and the arguments named in
    nulls passed as NULL. -> (return code, the outputs: res, seed, record, scores, table)."""
    import ctypes as C
    prns = [int(p) for p in prns]
    acq = gps.Context._acq_config(prns, ms, s0, -5000.0, 250.0, 41)
    cf = np.array(cfg, dtype=gps.COLLECTIVE_CONFIG_DTYPE).reshape(1)
    n = max(1, min(len(prns), 32))
    fill = lambda count, dt: np.full(count * dt.itemsize, 0xA5, np.uint8).view(dt)
    nhyp = 64   # room for the valid config of the test (25 hypotheses); a refused call writes nothing anywhere
    out = [fill(n, gps.ACQ_RESULT_DTYPE), fill(n, gps.ACQ_RESULT_DTYPE), fill(1, gps.COLLECTIVE_DTYPE),
           fill(nhyp, gps.CD_SCORE_DTYPE), fill(nhyp * n, gps.CD_CELL_DTYPE)]
    e = np.ascontiguousarray(eph, dtype=gps.EPHEMERIS_DTYPE)
    a = np.array(ap, dtype=gps.COARSE_CONFIG_DTYPE).reshape(1)
    flo = None if f_lo_prn is None else np.ascontiguousarray(f_lo_prn, np.float64)
    ptr = dict(iq=iq.ctypes.data, eph=e.ctypes.data, ap=a.ctypes.data, cfg=cf.ctypes.data, res=out[0].ctypes.data,
               seed=out[1].ctypes.data, out=out[2].ctypes.data)
    for k in nulls:
        ptr[k] = None
    rc = gps.lib().gpsb200_collective(ctx._h, ptr["iq"], iq.size // 2, gps.SC08, C.byref(acq),
                                      None if flo is None else flo.ctypes.data, ptr["eph"], ptr["ap"], ptr["cfg"],
                                      ptr["res"], ptr["seed"], ptr["out"], out[3].ctypes.data, out[4].ctypes.data)
    return rc, out


def test_refusals_write_nothing_and_leave_the_context_working(ctx, sky):
    """Every check of the contract, and each NULL pointer, refuses the call with GPSB200_ERR_ARG; no output byte
    changes (every one was 0xA5 before), and the next call gives the bytes it gave before."""
    _, _, iq = block_stream("sky12_static_35s_i8", 0)
    good = gps.collective_config(500.0, 250.0)
    want = ctx.collective(sky[0], apriori(), good, iq=iq, ms=K, s0=S0, want_scores=True, want_table=True)
    rc, out = raw_collective(ctx, iq, sky[0], apriori(), good)
    assert rc == 0 and out[2].tobytes() == np.asarray(want[2]).tobytes() and out[1].tobytes() == want[1].tobytes()
    bad = []
    for f, v in (("n", [0, 1, 1, 1]), ("n", [4096, 4097, 1, 1]), ("step", [np.nan, 250.0, 1.0, 1.0]),
                 ("step", [250.0, 0.0, 1.0, 1.0]), ("mask_deg", np.inf), ("distinct_m", np.nan), ("reserved", 1)):
        c = good.copy()
        c[f] = v
        if f == "step":
            c["n"] = [3, 3, 1, 1]
        bad.append(dict(cfg=c))
    bad.append(dict(ap=gps.coarse_config([np.nan, 0.0, 0.0], START_SOW)))
    bad.append(dict(ap=gps.coarse_config(PM.llh_ecef(*LOC), 604800.0)))
    bad.append(dict(ms=0))
    bad.append(dict(prns=[33]))
    bad.append(dict(f_lo_prn=np.full(32, 2e6)))
    bad.append(dict(s0=iq.size))
    for k in ("iq", "eph", "ap", "cfg", "res", "seed", "out"):
        bad.append(dict(nulls=(k,)))
    for kw in bad:
        args = dict(eph=sky[0], ap=apriori(), cfg=good)
        args.update(kw)
        rc, out = raw_collective(ctx, iq, **args)
        assert rc == gps.api.ERR_ARG, kw
        for o in out:
            assert (o.view(np.uint8) == 0xA5).all(), kw
    again = ctx.collective(sky[0], apriori(), good, iq=iq, ms=K, s0=S0, want_scores=True, want_table=True)
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(want, again))


def sanitizer_run():
    """One host and one device call of a small lattice; -> a hex digest of their outputs."""
    import hashlib
    import torch
    _, _, iq = block_stream("sky12_static_35s_i8", 0)
    import tempfile
    import pathlib
    eph, _ = ephemeris(pathlib.Path(tempfile.mkdtemp()), 12, START_SOW)
    cfg = gps.collective_config(500.0, 250.0, 0.5, 0.5)
    h = hashlib.sha256()
    with gps.Context(12, 1) as c:
        for out in (c.collective(eph, apriori(), cfg, iq=iq, prns=range(1, 13), want_scores=True, want_table=True),):
            for a in out:
                h.update(np.asarray(a).tobytes())
        d = torch.from_numpy(iq.copy()).cuda()
        torch.cuda.synchronize()
        for a in c.collective(eph, apriori(), cfg, device_ptr=d.data_ptr(), nsamples=iq.size // 2, prns=range(1, 13),
                              want_scores=True, want_table=True):
            h.update(np.asarray(a).tobytes())
    return h.hexdigest()


def test_clean_under_compute_sanitizer():
    """compute-sanitizer memcheck over one host and one device call: no error, and the same bytes as a plain run."""
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_collective_gpu as T; "
            "print('ok', T.sanitizer_run())" % (scenario.ROOT, os.path.join(scenario.ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0, plain.stderr[-2000:]
    r = subprocess.run([cs, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, "-c", code],
                       capture_output=True, text=True, timeout=1200)
    from test_coarse_gpu import _device_not_supported
    if _device_not_supported(r):   # the fallback of test_sanitizers: no CUDA error and the same bytes again
        import torch
        assert sanitizer_run() == plain.stdout.split()[-1]
        torch.cuda.synchronize()
        return
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert r.stdout.split()[-1] == plain.stdout.split()[-1]


def test_cli_collective_fixes_where_plain_fixes_are_few(tmp_path):
    """The weakened stream written to a file (one block, int8), the a-priori 1.5 km east, 0.75 km north and 0.5 s
    late: `gpsb200-acq --fix` prints FEW (at most 4 PRNs pass alone), `--fix --collective 3500,250,1.5,0.5` prints an
    OK fix from at least 10 channels within WEAK_POS of the receiver, with every PRN of the sky used and at most 4 of them passing alone."""
    from test_scenario import make_nav
    exe_dir = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200")
    if not os.path.exists(os.path.join(exe_dir, "gpsb200-acq")):
        subprocess.check_call(["make", "-C", os.path.join(exe_dir, "csrc")])
    ch, iq = weak_block(scenario.load_golden("sky12_static_35s_i8"))
    path = tmp_path / "weak.bin"
    iq.astype(np.int8).tofile(path)
    nav = make_nav(tmp_path, 12)
    x0 = PM.llh_ecef(*LOC)
    e, n, _ = enu(x0)
    lat, lon, h = PM.ecef_llh(x0 + 1500.0 * e + 750.0 * n)
    acq = [os.path.join(exe_dir, "gpsb200-acq"), str(path), "--fix", "--assist", nav, "--assist-pos",
           "%.9f,%.9f,%.3f" % (np.degrees(lat), np.degrees(lon), h), "--assist-time", "2024/01/07,02:00:00.5"]

    def lines(extra):
        r = subprocess.run(acq + extra, capture_output=True, text=True, check=True)
        return [ln.split() for ln in r.stdout.splitlines() if ln and not ln.startswith("#")]
    plain = lines([])
    assert len(plain) == 1 and plain[0][1] == "FEW", plain
    cd = lines(["--collective", "3500,250,1.5,0.5"])
    assert len(cd) == 1 and len(cd[0]) == 18, cd
    ln = cd[0]
    assert ln[1] == "OK" and ln[12] == "OK" and int(ln[9]) >= 10, ln   # the model: 10 OK records, 30.3 m
    xyz = PM.llh_ecef(float(ln[2]), float(ln[3]), float(ln[4]))
    assert np.linalg.norm(xyz - x0) <= WEAK_POS, ln
    assert abs(float(ln[15]) + 0.5) <= 0.5 and len(ln[16].split(",")) == 12 and int(ln[17]) <= 4, ln
    # --collective needs an a-priori position and --fix
    assert subprocess.run(acq[:2] + ["--collective", "3500,250"], capture_output=True).returncode == 2
