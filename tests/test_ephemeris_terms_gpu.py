"""The broadcast-ephemeris fixtures on the GPU (tests/test_ephemeris_terms.py): every block's CRC equals the reference's,
from the dumped parameters and from the RINEX file through the scenario engine; the fix kernels (k_pvt, k_pvt_raim,
k_pvt_araim at masks 5 and 10 deg, k_pvt_coarse) equal their models at 12 and 32 channels an hour from toc, where omega,
toe != toc, af2, both signs and the field limits of every term enter each fix; and the whole receiver chain on
sky12_ephvar_p59m_35s -- synthesis, acquisition, tracking, the ephemeris decoded from the tracked stream, fix, and
coarse-time fixes assisted by the RINEX file -- stays within the tracked bounds."""
import numpy as np
import pytest

import araim_model as AM
import coarse_model as CM
import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_araim_gpu import assert_kernel_equals_model as assert_araim_equals_model
from test_coarse import TRACKED as COARSE_TRACKED, apriori, offsets, unanchored
from test_coarse_gpu import assert_coarse_equals_model
from test_ephemeris_terms import FIXTURES, M59, P59, V3, WEEK, ephem_case, fix_inputs
from test_pvt import IDEAL, TRACKED, check_truth
from test_pvt_gpu import assert_kernel_equals_model as assert_pvt_equals_model, gpu_track, used
from test_raim_gpu import assert_kernel_equals_model as assert_raim_equals_model
from test_receiver_edges_gpu import model_margins
from test_sites_gpu import stream_crcs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", FIXTURES)
def test_stream_equals_the_reference_stream(name, tmp_path):
    g, kw, _ = ephem_case(name, tmp_path)
    ss, want = int(g["sample_size"]), g["block_crcs"]
    ch, nav = gps.scenario(**kw)
    got = stream_crcs(ch, nav, ss)
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, bad[:10]
    dch, frames = scenario.golden_chans(g)
    got = stream_crcs(dch, frames, ss)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]


@pytest.mark.parametrize("name", [P59, M59, V3])
def test_fix_kernels_equal_their_models(name, tmp_path):
    """k_pvt, k_pvt_raim, k_pvt_araim (masks 5 and 10 deg) and k_pvt_coarse (a-priori on the truth, and 50 km east + 1 km
    up with +10 s) against the models on the fixture's ideal epochs (12 channels, 32 on sky32_ephvar_m59m), no decision
    of the fix within 1e-9 of its threshold; ARAIM passes and its HPL / VPL bound the truth."""
    chans, eps, cfg, (xyz, sow), _ = fix_inputs(name, tmp_path)
    assert len(eps) == (32 if name == M59 else 12)
    model_margins(chans, eps, cfg)
    with gps.Context(1, 1) as ctx:
        fix = assert_pvt_equals_model(ctx, chans, eps, cfg)
        rfix, _, _ = assert_raim_equals_model(ctx, chans, eps, cfg, gps.raim_config(1.0))
        for mask in (5.0, 10.0):
            afix, arec = assert_araim_equals_model(ctx, chans, eps, cfg, gps.araim_config(mask_deg=mask))
            assert (arec["verdict"] == AM.PASS).all(), arec["verdict"]
            E = AM.enu(xyz[0])
            err = (np.stack([afix["x"], afix["y"], afix["z"]], 1) - xyz[0]) @ E.T
            assert np.all(np.hypot(err[:, 0], err[:, 1]) < arec["hpl"]) and np.all(np.abs(err[:, 2]) < arec["vpl"])
        for off in offsets(xyz[0])[:2]:
            got, _, _ = assert_coarse_equals_model(ctx, chans, eps, cfg, apriori(xyz[0], sow, off))
            assert (got["status"] == gps.FIX_OK).all()
    assert (fix["status"] == gps.FIX_OK).all() and (fix["nused"] == len(eps)).all()
    assert fix.tobytes() == rfix.tobytes()
    # the RINEX-3 run's 12 channels reach 0.449 m and 1.34 ns, most of it the truncation of the broadcast terms
    # (test_ephemeris_terms.py::test_truncated_terms_are_the_ideal_error)
    check_truth(fix, xyz, sow, 0.6 if name == V3 else IDEAL["pos"], 2e-9 if name == V3 else IDEAL["time"], IDEAL["vel"])


def assert_clear_coarse_fixes_equal_the_model(ctx, chans, eps, cfg, ap, margin=1e-3):
    """k_pvt_coarse against the model on tracked epochs, where no fix instant can be chosen away from the decisions:
    the fixes none of whose Gauss-Newton steps lies within `margin` relative of the 1e-4 m convergence threshold (at
    least 99 %; kernel and model steps differ by about 1e-4 relative there) equal the model as in
    test_coarse_gpu.assert_coarse_equals_model. -> kernel fixes"""
    got, rec, res, ms = ctx.pvt_coarse(chans, eps, cfg, ap, want_residuals=True, want_ms=True)
    tr = {"half": [], "residual": [], "step": [], "runaway": []}
    want, wrec, wres, wms = CM.coarse(chans, eps, cfg, ap, trace=tr)
    clear = np.ones(want["sample"].size, bool)
    for j, step in enumerate(tr["step"]):                  # iteration j steps every fix still active
        idx = np.nonzero(want["iterations"] > j)[0]
        assert idx.size == step.size
        clear[idx] &= np.abs(step / PM.CONVERGED - 1.0) > margin
    assert clear.mean() >= 0.99, clear.mean()
    for f in ("sample", "status", "nused", "mask", "iterations"):
        assert np.array_equal(got[f][clear], want[f][clear].astype(got[f].dtype)), f
    for f in ("ref", "week", "changed"):
        assert np.array_equal(rec[f][clear], wrec[f][clear].astype(rec[f].dtype)), f
    assert np.array_equal(ms[clear], wms[clear])
    ok = clear & (got["status"] == gps.FIX_OK)
    for f in ("x", "y", "z", "clock_m", "vx", "vy", "vz", "drift", "height"):
        assert np.all(np.abs(got[f][ok] - want[f][ok]) < 1e-6), (f, np.abs(got[f][ok] - want[f][ok]).max())
    assert np.all(np.abs(got["t_rx"][ok] - want["t_rx"][ok]) < 1e-14 * 604800 + 1e-12)
    both = ~np.isnan(res[clear])
    assert np.all(np.abs(res[clear][both] - wres[clear][both]) < 1e-6)
    assert (got["status"] == want["status"]).all()
    return got


def test_chain_with_the_ephemeris_from_the_stream(tmp_path):
    """35 s from 02:58:54, an hour after set 0's toc: synthesized on the GPU (block CRCs the reference's), acquired,
    tracked; each channel's ephemeris decoded from its own tracked words (subframes 1-3 sent from 02:59:00) equals the
    record's broadcast values, and so does its anchor; fixes every 10 ms from 0.5 s equal the model and are within the
    tracked bounds. Then coarse-time fixes without anchors, assisted by gpsb200_rinex_ephemeris on the same file (the
    a-priori 50 km and 10 s off; PRNs 1, 2, 3, 8, 9, 10 and 11 from set 1, whose toe is nearer): the kernel equals the
    model away from the convergence threshold; the file's health keeps PRNs 3, 6 and 11 out; with the health the stream
    carries, all 12 channels, PRNs 1 and 7 (af0 at -2^21 and 2^21 - 1, 0.98 ms) among them, fix within the coarse
    tracked bounds (9 channels reach 35.7 m, beyond them)."""
    g, kw, recs = ephem_case(P59, tmp_path)
    ch, frames = scenario.golden_chans(g)
    ss = int(g["sample_size"])
    _, _, cfg0, (xyz, sow), _ = fix_inputs(P59, tmp_path)
    iono = (cfg0["alpha"], cfg0["beta"])
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(ch.shape[1], ch.shape[0], max_nav_frames=len(frames)) as ctx:
        ctx.set_nav_frames(frames)
        out, _ = ctx.synth_blocks(ch, ss)
        assert np.array_equal(scenario.crc_blocks(out), g["block_crcs"])
        eps = gpu_track(ctx, out, ss, prns)
        chans = np.zeros(len(prns), gps.PVT_CHAN_DTYPE)
        for c, (prn, e) in enumerate(zip(prns, eps)):
            _, words, sy = gps.nav_decode(e)
            eph, _ = gps.nav_ephemeris(words)
            assert eph["valid"] == 1, prn
            assert eph["iodc"] == int(recs[prn]["iodc"]) and eph["health"] == 0 and eph["ura"] == 0
            for f in PT.EPH_FIELDS:
                assert eph[f] == PT.eph2sbf_value(recs[prn], f), (prn, f)
            chans[c]["eph"], chans[c]["prn"] = eph, prn
            chans[c]["anchor_epoch"], chans[c]["anchor_ms"] = gps.nav_time_anchor(words, sy)
            assert chans[c]["anchor_epoch"] >= 0, prn
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        model_margins(chans, eps, cfg)
        fix = assert_pvt_equals_model(ctx, chans, eps, cfg)
        assert fix.size > 3000 and (fix["nused"] == 12).all()
        check_truth(fix, xyz, sow, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])

        assist = gps.rinex_ephemeris(kw["nav_file"], WEEK, sow)
        achans = unanchored(chans)
        for c, prn in enumerate(prns):
            achans[c]["eph"] = assist[prn - 1]
        unhealthy = [p for p in prns if assist[p - 1]["health"] != 0]
        assert unhealthy == [3, 6, 11]
        af0_limit = [c for c, p in enumerate(prns) if abs(assist[p - 1]["af0"]) > 0.976e-3]
        assert sorted(prns[c] for c in af0_limit) == [1, 7]
        ap = apriori(xyz[0], sow, offsets(xyz[0])[1])
        hfix = assert_clear_coarse_fixes_equal_the_model(ctx, achans, eps, cfg, ap)
        assert (hfix["status"] == gps.FIX_OK).all() and (hfix["nused"] == 9).all()
        for c, p in enumerate(prns):
            assert used(hfix, c).all() == (p not in unhealthy), p
        # the stream's own health bits are 0 (the reference sends 0 whatever the file says): with them, all 12 channels
        achans["eph"]["health"] = 0
        cfix = assert_clear_coarse_fixes_equal_the_model(ctx, achans, eps, cfg, ap)
    assert (cfix["nused"] == 12).all()
    for c in af0_limit:
        assert used(cfix, c).all(), prns[c]
    check_truth(cfix, xyz, sow, COARSE_TRACKED["pos"], COARSE_TRACKED["time"], COARSE_TRACKED["vel"],
                COARSE_TRACKED["pos_mean"])
