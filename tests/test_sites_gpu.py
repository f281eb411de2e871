"""The ionosphere fixtures on the GPU (tests/test_sites.py): every block's CRC equals the reference's, from the dumped
parameters and from the RINEX file through the scenario engine, and through gpsb200-sim -I; the fix kernels (k_pvt,
k_pvt_raim, k_pvt_araim at masks 5 and 10 deg, k_pvt_coarse) equal their models at every site, where the Klobuchar term
takes its night, clamped and southern branches; ARAIM bounds the truth there; and the whole receiver chain at
66 N 100 W -- synthesis, acquisition, tracking, decoding, fix -- stays within the tracked bounds."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import araim_model as AM
import scenario
from scenario import gps
from test_araim_gpu import assert_kernel_equals_model as assert_araim_equals_model
from test_coarse import apriori, offsets
from test_coarse_gpu import assert_coarse_equals_model
from test_pvt import IDEAL, TRACKED, check_truth, tracked_inputs
from test_pvt_gpu import assert_kernel_equals_model as assert_pvt_equals_model, gpu_track
from test_raim_gpu import assert_kernel_equals_model as assert_raim_equals_model
from test_receiver_edges_gpu import model_margins
from test_sites import FIXTURES, IONO_OFF, SITES, fix_inputs, site_case

pytestmark = pytest.mark.gpu

CHUNK = 256


def stream_crcs(ch, nav, ss, chunk=CHUNK):
    """block CRCs of the stream one context makes in calls of `chunk` blocks that continue the carrier chain"""
    crcs, carr = [], None
    with gps.Context(ch.shape[1], min(chunk, ch.shape[0]), max_nav_frames=len(nav)) as ctx:
        ctx.set_nav_frames(nav)
        for b0 in range(0, ch.shape[0], chunk):
            part = ch[b0:b0 + chunk]
            if b0 > 0:
                part = gps.sharding.seed_slice(part, ch[b0 - 1], carr)
            out, carr = ctx.synth_blocks(part, ss)
            crcs.append(scenario.crc_blocks(out))
    return np.concatenate(crcs)


@pytest.mark.parametrize("name", FIXTURES)
def test_stream_equals_the_reference_stream(name, tmp_path):
    g, kw = site_case(name, tmp_path)
    ss, want = int(g["sample_size"]), g["block_crcs"]
    ch, nav = gps.scenario(**kw)
    got = stream_crcs(ch, nav, ss)
    bad = np.nonzero(got != want)[0]
    assert got.size == want.size and bad.size == 0, bad[:10]
    if "chans_idx" not in g:                       # every block's parameters are in the fixture
        dch, frames = scenario.golden_chans(g)
        got = stream_crcs(dch, frames, ss)
        assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]


def test_cli_without_ionosphere_writes_the_reference_stream(tmp_path):
    g, kw = site_case(IONO_OFF, tmp_path)
    exe = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "gpsb200-sim")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "csrc")])
    out = tmp_path / "iq.bin"
    loc = "%r,%r,%r" % (float(kw["lat"]), float(kw["lon"]), float(kw["height"]))
    r = subprocess.run([exe, "-e", kw["nav_file"], "-l", loc, "-d", "%g" % kw["seconds"], "-I", "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-600:]
    s = np.fromfile(out, dtype=np.int8)
    got = np.array([zlib.crc32(b.tobytes()) for b in s.reshape(-1, gps.BLOCK_ELEMS)], np.uint32)
    assert np.array_equal(got, g["block_crcs"])


@pytest.mark.parametrize("name", SITES)
def test_fix_kernels_equal_their_models(name, tmp_path):
    """k_pvt, k_pvt_raim, k_pvt_araim (masks 5 and 10 deg) and k_pvt_coarse (a-priori on the truth and 50 km / 10 s
    off) against the models on the site's ideal epochs, no decision of the fix within 1e-9 of its threshold (the
    Klobuchar |X| = 1.57 included); ARAIM passes and its HPL / VPL bound the truth."""
    chans, eps, cfg, _, (xyz, sow), _ = fix_inputs(name, tmp_path)
    model_margins(chans, eps, cfg)
    with gps.Context(1, 1) as ctx:
        fix = assert_pvt_equals_model(ctx, chans, eps, cfg)
        rfix, rec, _ = assert_raim_equals_model(ctx, chans, eps, cfg, gps.raim_config(1.0))
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
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])


def test_chain_at_66n_100w(tmp_path):
    """10 s at 66 N 100 W, where most fixes see the night branch: synthesized on the GPU (block CRCs the reference's),
    acquired, tracked, the TOW anchor from the tracked words, the ephemeris from the scenario's frames; the kernel equals
    the model on these epochs and the fixes (every 10 ms from 0.5 s) are within the tracked bounds."""
    name = "site_66n_100w_10s_i8"
    g = scenario.load_golden(name)
    ch, frames = scenario.golden_chans(g)
    ss = int(g["sample_size"])
    _, _, _, iono, (xyz, sow), _ = fix_inputs(name, tmp_path)
    prns = [int(p) for p in ch[0]["prn"] if p > 0]
    with gps.Context(ch.shape[1], ch.shape[0], max_nav_frames=len(frames)) as ctx:
        ctx.set_nav_frames(frames)
        out, _ = ctx.synth_blocks(ch, ss)
        assert np.array_equal(scenario.crc_blocks(out), g["block_crcs"])
        eps = gpu_track(ctx, out, ss, prns)
        slot_of_prn = {p: k for k, p in enumerate(int(x) for x in ch[0]["prn"]) if p > 0}
        chans = tracked_inputs(eps, prns, frames, slot_of_prn)
        end = min(int(e["sample"][-2]) for e in eps)
        cfg = gps.pvt_config(1500000, 30000, (end - 1500000) // 30000, iono)
        model_margins(chans, eps, cfg)
        fix = assert_pvt_equals_model(ctx, chans, eps, cfg)
    assert (fix["nused"] == 32).all()
    check_truth(fix, xyz, sow, TRACKED["pos"], TRACKED["time"], TRACKED["vel"], TRACKED["pos_mean"])
