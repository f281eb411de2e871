"""Race / memory checks: the FIFO under ThreadSanitizer (CPU), the kernels under compute-sanitizer (GPU; on a device the
tool cannot instrument, guard bands around the output, CUDA error state and run-to-run equality instead)."""
import os
import shutil
import subprocess
import sys

import pytest

import scenario

ROOT = scenario.ROOT


def test_fifo_is_race_free_under_tsan(tmp_path):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("no g++")
    exe = tmp_path / "fifo_tsan"
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-I", os.path.join(ROOT, "include"),
           "-I/usr/local/cuda/include", "-o", str(exe), os.path.join(ROOT, "tests", "native", "fifo_tsan.cpp"),
           os.path.join(ROOT, "multi-sdr-gps-sim_b200", "csrc", "fifo.cpp"),
           "-L/usr/local/cuda/lib64", "-lcudart", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("TSan build not available here: " + r.stderr[-200:])
    env = dict(os.environ, LD_LIBRARY_PATH="/usr/local/cuda/lib64:" + os.environ.get("LD_LIBRARY_PATH", ""))
    r = subprocess.run([str(exe)], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr


@pytest.mark.gpu
def test_kernels_clean_under_compute_sanitizer():
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import numpy as np, scenario; "
            "gps = scenario.gps; ch, nav = gps.synthetic_chans(2, 32, seed=5); ctx = gps.Context(32, 2); "
            "ctx.set_nav_frames(nav); out, cp = ctx.synth_blocks(ch, 1); "
            "ch12, nav12 = gps.synthetic_chans(1, 12, seed=6); c2 = gps.Context(12, 1); c2.set_nav_frames(nav12); "
            "o2, _ = c2.synth_blocks(ch12, 2); print('ok', int(np.abs(out).sum()), int(np.abs(o2.astype(np.int64)).sum()))"
            % (ROOT, os.path.join(ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "9", sys.executable, "-c", code],
                           capture_output=True, text=True, timeout=1500)
        if _device_not_supported(r):
            # The tool itself cannot instrument kernels on this device (e.g. where GPU debugging is disabled). Check what
            # it would have caught from outside instead: no write outside the output buffer, no sticky CUDA error,
            # output that does not change from run to run.
            _guarded_device_runs()
            return
        assert r.returncode == 0, (tool, r.stdout[-1500:], r.stderr[-500:])
        assert "ok" in r.stdout


def _device_not_supported(r):
    """Whether compute-sanitizer refused the device itself. Only that message sends a test to its fallback: a hazard or
    bounds error the tool reports ("========= Error: Race reported ...", "========= Invalid __shared__ read ...") fails
    the test through the error exit code."""
    return any(ln.startswith("========= Error: Device not supported") for ln in (r.stdout + r.stderr).splitlines())


@pytest.mark.gpu
def test_receiver_kernels_clean_under_compute_sanitizer():
    """The receiver kernels at the shapes of tests/test_receiver_edges_gpu.py: a 1024-bin search of K = 100 periods, 32
    channels tracked from 3001-sample periods on, and a RAIM call that excludes a channel."""
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_sanitizers as S; "
            "print('ok', S.receiver_runs())" % (ROOT, os.path.join(ROOT, "tests")))
    plain = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "ok" in plain.stdout, plain.stderr[-1500:]
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "9", sys.executable, "-c", code],
                           capture_output=True, text=True, timeout=1500)
        if _device_not_supported(r):
            # as above: the tool cannot instrument this device; check from outside instead. The receiver kernels only
            # read the sources, so the guard bands show no stray write into the context's own buffers; the repeats
            # equal to the host-source run are what would show one.
            _guarded_receiver_runs()
            return
        assert r.returncode == 0, (tool, r.stdout[-1500:], r.stderr[-500:])
        assert plain.stdout.split()[-1] == r.stdout.split()[-1]


def _receiver_inputs():
    """(search window int8, search config, tracking buffer int8, 32 start states, RAIM case)."""
    import numpy as np
    import test_raim as TR
    import track_model as T
    import test_receiver_edges as E
    gps = scenario.gps
    acq = E.full_scale(3000 * 100 + 2999, 13, -1.5e6 + 1023 * 2932.0, gps.SC08, delay=1500)
    acq_cfg = dict(prns=[13], ms=100, f_lo=-1.5e6, step=2932.0, nbins=1024)
    trk = np.random.default_rng(5).integers(-128, 128, 2 * 25 * 3001).astype(np.int8)
    st = E.limit_states(list(range(1, 33)), 0, 5)
    st["code_step"], st["code_phase"] = T.CODE_STEP_MIN, 0                        # 3001-sample first periods
    _, _, chans, eps = TR.sky("sky12_static_35s_i8", 6)
    TR.code_bias(eps, 2, 0.1)
    return acq, acq_cfg, trk, st, (chans, eps, gps.pvt_config(30000, 999983, 34), gps.raim_config(1.0))


def receiver_runs(inputs=None, acq_src=None, trk_src=None):
    """One run of every receiver shape -> a hex digest of all results. acq_src / trk_src: device pointers holding the
    search window / tracking buffer, in place of the host arrays."""
    import hashlib
    gps = scenario.gps
    acq, acq_cfg, trk, st, (chans, eps, cfg, rcfg) = inputs or _receiver_inputs()
    h = hashlib.sha256()
    with gps.Context(32, 1) as ctx:
        if acq_src is None:
            res, grid = ctx.acquire(acq, gps.SC08, want_grid=True, **acq_cfg)
        else:
            res, grid = ctx.acquire(device_ptr=acq_src, nsamples=acq.size // 2, sample_size=gps.SC08, want_grid=True,
                                    **acq_cfg)
        assert res[0]["bin"] == 1023 and res[0]["delay"] == 1500
        h.update(res.tobytes())
        h.update(grid.tobytes())
        if trk_src is None:
            out, s = ctx.track(st, trk, gps.SC08)
        else:
            out, s = ctx.track(st, device_ptr=trk_src, nsamples=trk.size // 2, sample_size=gps.SC08)
        assert all(e.size >= 20 and e["sample"][1] - e["sample"][0] == 3001 for e in out)
        for e in out:
            h.update(e.tobytes())
        h.update(s.tobytes())
        fix, rec = ctx.pvt_raim(chans, eps, cfg, rcfg)
        assert (rec["excluded"] == 1 << 2).all()
        h.update(fix.tobytes())
        h.update(rec.tobytes())
    return h.hexdigest()


def _guarded_receiver_runs(guard=1 << 16, pattern=0xA5, repeats=3):
    """The receiver shapes from device sources with guard bands on both sides: the guard bytes keep their pattern, CUDA
    reports no error, and every repeat gives the host-source results."""
    import numpy as np
    import torch
    inputs = _receiver_inputs()
    want = receiver_runs(inputs)
    for _ in range(repeats):
        bufs = []
        for a in (inputs[0], inputs[2]):
            buf = torch.full((guard + a.nbytes + guard,), pattern, dtype=torch.uint8, device="cuda")
            buf[guard:guard + a.nbytes] = torch.from_numpy(a.view(np.uint8)).cuda()
            bufs.append(buf)
        got = receiver_runs(inputs, bufs[0].data_ptr() + guard, bufs[1].data_ptr() + guard)
        torch.cuda.synchronize()                                  # raises on an illegal address or any sticky error
        for buf, a in zip(bufs, (inputs[0], inputs[2])):
            host = buf.cpu().numpy()
            assert np.all(host[:guard] == pattern) and np.all(host[guard + a.nbytes:] == pattern)
            assert np.array_equal(host[guard:guard + a.nbytes], a.view(np.uint8))
        assert got == want


def _guarded_device_runs(guard=1 << 16, pattern=0xA5, repeats=3):
    """Every kernel of the device path (carrier tables, probes, span chaining, checkpoints, both synthesis kernels) for
    32 and 12 channels, int8 and int16, into an output buffer with guard bands on both sides: the guard bytes must keep
    their pattern, CUDA must report no error, and every repeat must equal the host-destination path byte for byte."""
    import numpy as np
    import torch
    gps = scenario.gps
    saved = os.environ.get("GPSB200_LANES")
    for lanes in ("1", "0"):
        os.environ["GPSB200_LANES"] = lanes                      # read when a context is created
        try:
            for nchan, ss in ((32, 1), (32, 2), (12, 1), (12, 2)):
                nblk = 40                                         # > 2 blocks: the speculative chain kernels run
                ch, nav = gps.synthetic_chans(nblk, nchan, seed=900 + nchan + ss)
                with gps.Context(nchan, nblk) as ctx:
                    ctx.set_nav_frames(nav)
                    want, cp = ctx.synth_blocks(ch, ss)
                    assert ctx.synth_kernel_name(nchan) == ("k_synth_lanes" if lanes == "1" else "k_synth")
                    nbytes = want.nbytes
                    for _ in range(repeats):
                        buf = torch.full((guard + nbytes + guard,), pattern, dtype=torch.uint8, device="cuda")
                        cpd = ctx.synth_blocks_device(ch, ss, buf.data_ptr() + guard)
                        torch.cuda.synchronize()                  # raises on an illegal address or any sticky error
                        host = buf.cpu().numpy()
                        assert np.all(host[:guard] == pattern) and np.all(host[guard + nbytes:] == pattern), \
                            (lanes, nchan, ss, "write outside the output buffer")
                        assert np.array_equal(host[guard:guard + nbytes].view(want.dtype), want), (lanes, nchan, ss)
                        assert np.array_equal(cpd, cp), (lanes, nchan, ss)
        finally:
            if saved is None:
                del os.environ["GPSB200_LANES"]
            else:
                os.environ["GPSB200_LANES"] = saved
