"""Interactive mode on the GPU: the steered fixtures (runs of the reference's own main with scripted keys) synthesized
live -- the scenario advanced chunk by chunk, cut at the key blocks, NAV frames in a ring of context slots, the carrier
chain continued across calls -- and through gpsb200-sim --steer / -i; every block's CRC equals the reference's."""
import os
import subprocess

import numpy as np
import pytest

import scenario
from scenario import gps
from test_interactive import STEER, steer_case

pytestmark = pytest.mark.gpu

KERNELS = (("1", "k_synth_lanes"), ("0", "k_synth"))
RING = 4


def synth_live(kw, sched, chunk, ss):
    """advance / key / synthesize: -> (per-block CRCs, kernel name)"""
    events = {}
    for b, keys, rep in sched:
        events[b] = events.get(b, "") + keys * rep
    crcs, uploaded, name = [], -1, None
    args = {k: v for k, v in kw.items() if k not in ("nav_file", "lat", "lon", "height", "seconds")}
    with gps.LiveScenario(kw["nav_file"], kw["lat"], kw["lon"], kw["height"], kw["seconds"], interactive=True, **args) as s, \
            gps.Context(s.channels, chunk, max_nav_frames=RING) as ctx:
        carr, prev, b = np.zeros(s.channels), np.zeros(s.channels, np.int32), 0
        while b < s.blocks:
            for k in events.get(b, ""):
                s.key(k)
            nxt = min([e for e in events if e > b] + [s.blocks])
            ch = s.advance(min(chunk, nxt - b))
            for f in np.unique(ch["nav_frame"]):
                if f > uploaded:
                    for c, words in enumerate(s.frame(int(f))):
                        ctx.set_nav(int(f) % RING, c, words)
                    uploaded = int(f)
            ch["nav_frame"] %= RING
            cont = (ch[0]["prn"] > 0) & (ch[0]["prn"] == prev)
            ch[0]["carr_phase"] = np.where(cont, carr, ch[0]["carr_phase"])
            out, carr = ctx.synth_blocks(ch, ss)
            prev = ch[-1]["prn"].copy()
            crcs.append(scenario.crc_blocks(out))
            b += ch.shape[0]
        name = ctx.synth_kernel_name(s.channels)
    return np.concatenate(crcs), name


@pytest.mark.parametrize("name", STEER)
def test_live_synthesis_of_steered_runs_matches_the_reference(name, tmp_path, monkeypatch):
    g, kw, sched = steer_case(name, tmp_path)
    want = g["block_crcs"]
    for lanes, kernel in KERNELS:
        monkeypatch.setenv("GPSB200_LANES", lanes)
        for chunk in (1, 7, 256):
            got, used = synth_live(kw, sched, chunk, int(g["sample_size"]))
            assert used == kernel
            bad = np.nonzero(got != want)[0]
            assert got.size == want.size and bad.size == 0, (kernel, chunk, bad[:5])


def _sim():
    exe = os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "gpsb200-sim")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(scenario.ROOT, "multi-sdr-gps-sim_b200", "csrc")])
    return exe


def _sim_args(g, kw, seconds=None):
    loc = "%r,%r,%r" % (float(kw["lat"]), float(kw["lon"]), float(kw["height"]))
    return [_sim(), "-e", kw["nav_file"], "-l", loc, "-d", "%g" % (seconds or kw["seconds"]),
            "-s", "2024/01/07,02:00:00", "--chan", str(kw["max_chan"])] + str(g["options"]).split()


@pytest.mark.parametrize("name", STEER)
def test_sim_steer_replays_the_reference_key_script(name, tmp_path):
    g, kw, _ = steer_case(name, tmp_path)
    steer, out = tmp_path / "steer.txt", tmp_path / "iq.bin"
    steer.write_text(str(g["schedule"]))
    subprocess.check_call(_sim_args(g, kw) + ["--steer", str(steer), "-o", str(out)])
    dt = np.int16 if int(g["sample_size"]) == 2 else np.int8
    got = scenario.crc_blocks(np.fromfile(out, dtype=dt))
    bad = np.nonzero(got != g["block_crcs"])[0]
    assert got.size == g["block_crcs"].size and bad.size == 0, bad[:5]


def test_live_session_log_replays_byte_identically_and_x_ends_with_a_prefix(tmp_path):
    g, kw, _ = steer_case("sky12_steer_60s_i8", tmp_path)
    base = _sim_args(g, kw, seconds=3)
    live, log, replay = tmp_path / "live.bin", tmp_path / "live.steer", tmp_path / "replay.bin"
    subprocess.run(base + ["-i", "--steer-log", str(log), "-o", str(live)], input=b"e" * 1500 + b"\nddd w\n", check=True)
    assert log.read_text().count("e") == 1500 and log.read_text().count("d") == 3
    subprocess.check_call(base + ["--steer", str(log), "-o", str(replay)])
    a, b = live.read_bytes(), replay.read_bytes()
    assert len(a) == 29 * gps.BLOCK_ELEMS and a == b
    # 'x' stops after the block in progress: a prefix of the same run without it
    xlog, xrun, full = tmp_path / "x.steer", tmp_path / "x.bin", tmp_path / "full.bin"
    subprocess.run(base + ["-i", "--steer-log", str(xlog), "-o", str(xrun)], input=b"e" * 800 + b"x", check=True)
    text = xlog.read_text()
    assert "x" in text
    noxs = tmp_path / "nox.steer"
    noxs.write_text("".join(ln.replace("x", "") + "\n" for ln in text.splitlines() if ln.replace("x", "")[-1] != ","))
    subprocess.check_call(base + ["--steer", str(noxs), "-o", str(full)])
    a, b = xrun.read_bytes(), full.read_bytes()
    assert 0 < len(a) < len(b) and b.startswith(a)
