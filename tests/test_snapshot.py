"""The snapshot measurement's numpy model (tests/snapshot_model.py) on the CPU oracle's streams against the scenario's
truth, and the fixes from its records (gpsb200_pvt_snapshot's model: coarse_model's solve) against the truth.

The bounds below were fixed from the model, K = 10 coherent ms from sample 1000 of a block, 12 code iterations:
- Measurement (sky12_static_35s blocks 0 and 50, sky32_static_10s block 0): every present sky12 PRN converges, its
  refined code phase within 9.9 m of range of the truth (the acquisition's sample-quantised delay: up to 47.8 m) and
  its carrier within 6.9 Hz of f_carr (the bin: up to 110 Hz). On sky32, where 32 codes share the band, two of the
  weakest channels end NO_CONVERGENCE (their last steps alternate in sign); the others reach 23.0 m and 11.9 Hz. The
  mean range error falls to about a fifth of the unrefined one (5.4 m against 24.3 m on sky32).
- Fixes (sky12_static_35s, 20 snapshots at blocks 0, 17, ..., 323, every a-priori offset of test_coarse): all OK
  with 12 channels, 3D error at most 29.1 m (mean 11.1 m), receive time 11.7 ms, velocity 3.26 m/s. The a-priori
  time error comes back in delta to within the receive-time error. The search from one snapshot with no position is
  unique and gives the coarse fix of its winning node.
- The 12-channel int16 site at 34.6 S 58.4 W (blocks 0, 40, 97): every PRN converges, 17.8 m and 6.1 Hz; fixes 33.8 m,
  2.23 m/s, receive time 4.2 ms. The 60 s circle (blocks 0, 150, 300, 450, 597): 8.5 m and 4.7 Hz; fixes 11.4 m,
  1.28 m/s, 4.0 ms.
The limits leave a margin of about a third over those figures; the GPU tests share them."""
import numpy as np
import pytest

import acq_model as A
import pvt_model as PM
import pvt_truth as PT
import scenario
import snapshot_model as S
from scenario import gps
from test_acquire import golden_rows
from test_coarse import apriori, offsets, static_rows, unanchored
from test_pvt import check_truth, ideal_inputs, rinex
from test_scenario import LOC, START, motion_file
from test_track import START_SOW

S0, K = 1000, 10
RANGE_M = dict(sky12=13.2, sky32=31.0, site_34s_58w_10s_i16=24.0, sky12_circle_60s_i16=11.4)   # code phase, m of range
DOPPLER_HZ = dict(sky12=9.3, sky32=16.0, site_34s_58w_10s_i16=8.2, sky12_circle_60s_i16=6.3)    # carrier, Hz
BOUNDS = dict(pos=39.0, pos_mean=15.0, time=0.016, vel=4.4)
SCENE_BOUNDS = dict(site_34s_58w_10s_i16=dict(pos=45.0, vel=3.0), sky12_circle_60s_i16=dict(pos=15.2, vel=1.7))
CHIP_M = 299792458.0 / 1.023e6


def block_stream(name, b):
    g = scenario.load_golden(name)
    ch = golden_rows(g, [b])
    iq, _ = scenario.oracle_run(ch, g["nav_frames"], int(g["sample_size"]))
    assert scenario.crc_blocks(iq)[0] == g["crcs"][b, 0]
    return g, ch, iq


def scene(name, tmp_path):
    """A fixture's stream and truth for snapshots: records of every block (the fixture's own for the site, the scenario
    engine's for the 60 s circle, whose fixture keeps two blocks), their PVT channels, Klobuchar terms, truth rows and
    start second of week, and stream(b) -> (I/Q of block b with its CRC checked, that block's records)."""
    import test_sites as TS
    from test_time_overwrite import gps_time
    g = scenario.load_golden(name)
    ss = int(g["sample_size"])
    if name.startswith("site_"):
        _, kw = TS.site_case(name, tmp_path)
        ch, nav = gps.scenario(**kw)
        rows = np.repeat(PM.llh_ecef(kw["lat"], kw["lon"], kw["height"])[None], ch.shape[0] + 1, 0)
        sow = gps_time(kw["start"])[1]
        crc = lambda b: g["block_crcs"][b]
        iono_src = kw["nav_file"]
        blocks = (0, 40, 97)
    else:
        nav_file, _, _ = rinex(tmp_path, 12)
        ch, nav = gps.scenario(nav_file, *LOC, seconds=60, max_chan=12, motion_file=motion_file(tmp_path), start=START)
        rows, sow = g["motion_rows"][:, 1:4], START_SOW
        crc = lambda b: g["crcs"][b, 0]
        iono_src = nav_file
        blocks = (0, 150, 300, 450, 597)
    chans, _ = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    _, alpha, beta = PT.read_rinex(iono_src)
    iono = PT.klobuchar_broadcast(alpha, beta)

    def stream(b):
        row = ch[b:b + 1].copy()   # the carrier phase the run reaches at block b (the records restart it)
        if b > 0:
            carr = gps.carrier_chain(ch[:b])
            row[0]["carr_phase"] = np.where(ch[b]["prn"] == ch[b - 1]["prn"], carr, ch[b]["carr_phase"])
        iq, _ = scenario.oracle_run(row, nav, ss)
        assert scenario.crc_blocks(iq)[0] == crc(b)
        return iq, ch[b:b + 1]
    return dict(ss=ss, chans=unanchored(chans), iono=iono, rows=rows, sow=sow, stream=stream, blocks=blocks)


def errors(meas, ch):
    """Per present PRN: (range error of the code phase at s0, m; carrier error, Hz)."""
    held = {int(r["prn"]): r for r in ch[0] if r["prn"] > 0}
    out = []
    for m in meas:
        if int(m["prn"]) not in held:
            continue
        f, tau = A.truth(held[int(m["prn"])], S0)
        want = (-tau * float(held[int(m["prn"])]["f_code"]) / 3e6) % 1023.0
        e = (float(m["code_phase"]) / 2 ** 32 - want + 511.5) % 1023.0 - 511.5
        out.append((e * CHIP_M, float(m["carr_step"]) * 3e6 / 2 ** 32 - f))
    return np.array(out)


@pytest.mark.parametrize("name,block,key", [("sky12_static_35s_i8", 0, "sky12"), ("sky12_static_35s_i8", 50, "sky12"),
                                            ("sky32_static_10s_i8", 0, "sky32")])
def test_model_truth(name, block, key):
    g, ch, iq = block_stream(name, block)
    ss = int(g["sample_size"])
    res = A.search(iq, ss, S0, K, list(range(1, 33)), -5000.0, 250.0, 41)
    meas = S.measure(iq, ss, S0, K, res, iterations=12)
    raw = S.measure(iq, ss, S0, K, res, iterations=0)
    present = {int(p) for p in ch[0]["prn"] if p > 0}
    for m in meas:   # absent PRNs are WEAK and keep the seed
        assert (m["status"] == S.WEAK) == (int(m["prn"]) not in present)
    ok = meas["status"] == S.OK
    # every sky12 PRN converges; on sky32 two of its weakest channels end in a limit cycle (NO_CONVERGENCE)
    assert ok.sum() >= len(present) - (2 if key == "sky32" else 0), meas["status"]
    e, e0 = errors(meas[ok], ch), errors(raw[ok], ch)
    assert np.abs(e[:, 0]).max() <= RANGE_M[key], e[:, 0]
    assert np.abs(e[:, 1]).max() <= DOPPLER_HZ[key], e[:, 1]
    assert np.abs(e[:, 0]).mean() < np.abs(e0[:, 0]).mean()


def test_one_chunk_leaves_the_carrier_step():
    _, _, iq = block_stream("sky12_static_35s_i8", 0)
    res = A.search(iq, 1, S0, 1, [1, 2, 3], -5000.0, 250.0, 41)
    meas = S.measure(iq, 1, S0, 1, res, iterations=4)
    for m, r in zip(meas, res):
        w, u, _ = S.seed(r, S0)
        assert m["carr_step"] == w and m["code_step"] == u


def test_model_fixes_on_sky12_static(tmp_path):
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    chans, _ = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    prns = [int(p) for p in chans["prn"]]
    meas = []
    for b in (0, 170, 323):
        _, _, iq = block_stream("sky12_static_35s_i8", b)
        m = S.measure(iq, 1, S0, K, A.search(iq, 1, S0, K, prns, -5000.0, 250.0, 41), iterations=12)
        m["sample"] += b * PT.BLOCK
        meas.append(m)
    meas = np.stack(meas)
    rows = static_rows(ch, LOC)
    cfg = gps.pvt_config(0, 1, len(meas), iono)
    for off in offsets(rows[0]):
        fix, co, _, ms = S.coarse(unanchored(chans), meas, cfg, apriori(rows[0], START_SOW, off))
        assert (fix["nused"] == 12).all()
        fig = check_truth(fix, rows, START_SOW, BOUNDS["pos"], BOUNDS["time"], BOUNDS["vel"])
        assert np.abs(co["delta"] + off[1]).max() <= BOUNDS["time"], (co["delta"], fig)
    # a record of another PRN, or a WEAK one, is not used
    bad = meas.copy()
    bad[:, 0]["prn"] = 33
    bad[:, 1]["status"] = S.WEAK
    fix, _, _, ms = S.coarse(unanchored(chans), bad, cfg, apriori(rows[0], START_SOW))
    assert (fix["nused"] == 10).all() and (ms[:, :2] == -1).all()


def test_model_search_on_sky12_static(tmp_path):
    """One snapshot (block 170) with no a-priori position, the a-priori time 10 s late: the model's search is OK and
    unique, and equals the coarse fix from its winning node."""
    import search_model as SM
    from test_search import search_cfg
    g = scenario.load_golden("sky12_static_35s_i8")
    ch, frames = scenario.golden_chans(g)
    _, _, iono = rinex(tmp_path, 12)
    chans, _ = ideal_inputs(ch, frames, g["nav_frame_of_block"])
    chans = unanchored(chans)
    _, _, iq = block_stream("sky12_static_35s_i8", 170)
    m = S.measure(iq, 1, S0, K, A.search(iq, 1, S0, K, [int(p) for p in chans["prn"]], -5000.0, 250.0, 41))
    m["sample"] += 170 * PT.BLOCK
    meas = m[None, :]
    cfg = gps.pvt_config(0, 1, 1, iono)
    sc = search_cfg(START_SOW, 10.0)
    fix, rec, res, ms = S.search(chans, meas, cfg, sc)
    assert fix["status"][0] == gps.FIX_OK and rec["support"][0] >= 1 and np.isnan(rec["alt_rms"][0])
    rows = static_rows(ch, LOC)
    check_truth(fix, rows, START_SOW, BOUNDS["pos"], BOUNDS["time"], BOUNDS["vel"])
    node = SM.nodes(int(sc["nodes"]), [int(rec["winner"][0])])[0]
    cfix, co, cres, cms = S.coarse(chans, meas, cfg, gps.coarse_config(node, float(sc["t_a"]), 0, int(sc["week"])))
    for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz", "rms"):
        assert cfix[f][0] == fix[f][0], f
    assert np.array_equal(cms, ms) and co["delta"][0] == rec["delta"][0]


@pytest.mark.parametrize("name", ["site_34s_58w_10s_i16", "sky12_circle_60s_i16"])
def test_model_on_the_int16_site_and_the_circle(name, tmp_path):
    """The 12-channel int16 stream at 34.6 S 58.4 W and the 60 s circle (a moving receiver: the carrier step carries
    the velocity, and the code phase is held over a window in which the range rate changes): every present PRN
    refined within the bounds, and fixes from every a-priori offset within them."""
    sc = scene(name, tmp_path)
    meas = []
    for b in sc["blocks"]:
        iq, r = sc["stream"](b)
        res = A.search(iq, sc["ss"], S0, K, list(range(1, 33)), -5000.0, 250.0, 41)
        m = S.measure(iq, sc["ss"], S0, K, res)
        ok = m["status"] == S.OK
        assert ok.sum() == (r[0]["prn"] > 0).sum(), m["status"]
        e = errors(m[ok], r)
        assert np.abs(e[:, 0]).max() <= RANGE_M[name] and np.abs(e[:, 1]).max() <= DOPPLER_HZ[name], e
        sel = [int(np.nonzero(m["prn"] == p)[0][0]) for p in sc["chans"]["prn"]]
        mm = m[sel]
        mm["sample"] += b * PT.BLOCK
        meas.append(mm)
    meas = np.stack(meas)
    cfg = gps.pvt_config(0, 1, len(meas), sc["iono"])
    for off in offsets(sc["rows"][0]):
        fix, _, _, _ = S.coarse(sc["chans"], meas, cfg, apriori(sc["rows"][0], sc["sow"], off))
        check_truth(fix, sc["rows"], sc["sow"], SCENE_BOUNDS[name]["pos"], BOUNDS["time"], SCENE_BOUNDS[name]["vel"])
