"""Every entry point of the C ABI on one call of several pipeline segments (256 + 1024 + 220 blocks): the host- and
device-destination one-shot calls, the scatter call, the three-step slice call eager and lazy with either destination,
and two consecutive calls. They schedule the same segment steps differently; what they compute is identical. Also:
a validation failure found in a later segment, after earlier segments' work is enqueued, leaves the context usable;
and the link gpsb200_slice_prepare fills is the host-only gpsb200_slice_link_host bit for bit."""
import numpy as np
import pytest

from scenario import gps

pytestmark = pytest.mark.gpu

NBLK, NCHAN = 1500, 32


def _workload():
    ch, nav = gps.synthetic_chans(NBLK, NCHAN, seed=1500)
    ch["prn"][400:407, 3] = 0                              # slot 3 idle for a few blocks, then resumes
    ch["carr_phase"][407, 3] = 0.375
    ch["prn"][777:, 5] = ch["prn"][0, 5] % 32 + 1          # slot 5 reallocated in the middle of segment 1
    ch["carr_phase"][777, 5] = 0.6180339887
    return ch, nav


def _same_bytes(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


@pytest.fixture(scope="module")
def reference():
    """gpsb200_synth_blocks on a fresh context: output, carr_phase_out, run checkpoints."""
    ch, nav = _workload()
    with gps.Context(NCHAN, NBLK) as ctx:
        ctx.set_nav_frames(nav)
        out, cp = ctx.synth_blocks(ch, 1)
        ck = ctx.debug_run_checkpoints(NBLK, NCHAN)
    return ch, nav, out, cp, ck


def _slice_call(ctx, ch, eager, device):
    import torch
    n = ch.shape[0] * gps.BLOCK_ELEMS
    if device:
        buf = torch.empty(n, dtype=torch.int8, device="cuda")
        ctx.slice_prepare(ch, 1, buf.data_ptr())
    else:
        buf = torch.empty(n, dtype=torch.int8).pin_memory()
        ctx.slice_prepare(ch, 1, dst_host=buf.numpy())
    ctx.slice_probe(eager=eager)
    prn, ph = ctx.slice_finish()
    ctx.slice_wait()
    return buf.cpu().numpy().copy(), prn, ph


def test_every_entry_point_computes_the_same_multi_segment_call(reference):
    import torch
    ch, nav, want, cp0, ck0 = reference
    assert np.array_equal(cp0, gps.carrier_chain(ch, threads=8))
    prn_end = np.where(ch["prn"][-1] > 0, ch["prn"][-1], 0)
    with gps.Context(NCHAN, NBLK) as ctx:
        ctx.set_nav_frames(nav)

        def check(name, out, cp, ck_blocks=slice(0, NBLK)):
            assert _same_bytes(out, want[ck_blocks.start * gps.BLOCK_ELEMS:ck_blocks.stop * gps.BLOCK_ELEMS]), name
            assert np.array_equal(cp, cp0), name
            n = ck_blocks.stop - ck_blocks.start
            assert _same_bytes(ctx.debug_run_checkpoints(n, NCHAN), ck0[ck_blocks]), name

        # scatter: every block into its own buffer, in a shuffled order (blocks past the first segment included)
        order = np.random.default_rng(5).permutation(NBLK)
        pool = np.empty((NBLK, gps.BLOCK_ELEMS), np.int8)
        cp = ctx.synth_blocks_scatter(ch, 1, [pool[order[b]] for b in range(NBLK)])
        check("synth_blocks_scatter", pool[order].reshape(-1), cp)

        dev = torch.empty(NBLK * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
        cp = ctx.synth_blocks_device(ch, 1, dev.data_ptr())
        torch.cuda.synchronize()
        check("synth_blocks_device", dev.cpu().numpy(), cp)
        del dev

        for eager in (True, False):
            for device in (True, False):
                out, prn, ph = _slice_call(ctx, ch, eager, device)
                name = "slice eager=%s device=%s" % (eager, device)
                assert np.array_equal(prn, prn_end), name
                check(name, out, ph)

        # two consecutive calls on the same stream, the second seeded with the first's carr_phase_out
        k = 700
        assert np.all((ch["prn"][k - 1] > 0) & (ch["prn"][k] == ch["prn"][k - 1]))
        a, cpa = ctx.synth_blocks(ch[:k], 1)
        assert np.array_equal(cpa, gps.carrier_chain(ch[:k], threads=8))
        rest = ch[k:].copy()
        rest["carr_phase"][0] = cpa
        b, cpb = ctx.synth_blocks(rest, 1)
        check("second of two calls", b, cpb, slice(k, NBLK))
        assert _same_bytes(a, want[:k * gps.BLOCK_ELEMS])


def test_validation_failure_in_a_later_segment_leaves_the_context_usable(reference):
    import torch
    ch, nav, want, cp0, _ = reference
    bad_arg = ch.copy()
    bad_arg["code_phase"][1400, 9] = 1023.0                # segment 2
    bad_range = ch.copy()
    bad_range["gain"][1300, 2] = 130.0                     # segment 2: sum of amplitudes over the int16 range
    dev = torch.empty(NBLK * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
    pinned = torch.empty(NBLK * gps.BLOCK_ELEMS, dtype=torch.int8).pin_memory()
    pool = np.empty((NBLK, gps.BLOCK_ELEMS), np.int8)
    with gps.Context(NCHAN, NBLK) as ctx:
        ctx.set_nav_frames(nav)
        entry_points = {
            "synth_blocks": lambda c: ctx.synth_blocks(c, 1),
            "synth_blocks_scatter": lambda c: ctx.synth_blocks_scatter(c, 1, list(pool)),
            "synth_blocks_device": lambda c: ctx.synth_blocks_device(c, 1, dev.data_ptr()),
            "slice_prepare device": lambda c: ctx.slice_prepare(c, 1, dev.data_ptr()),
            "slice_prepare host": lambda c: ctx.slice_prepare(c, 1, dst_host=pinned.numpy()),
            "carrier_chain_device": lambda c: ctx.carrier_chain(c),
        }
        for bad, code, cause in ((bad_arg, -1, "invalid channel parameters in slot 9"),
                                 (bad_range, -3, "sum of channel amplitudes exceeds int16 range")):
            for name, call in entry_points.items():
                with pytest.raises(gps.GpsB200Error) as e:
                    call(bad)
                assert e.value.code == code and cause in str(e.value), (name, str(e.value))
                if name.startswith("slice_prepare"):
                    assert gps.lib().gpsb200_slice_probe(ctx._h, None, None, 0) == -1, name
                    assert gps.lib().gpsb200_slice_finish(ctx._h, None, None, None, None, None) == -1, name
                out, cp = ctx.synth_blocks(ch, 1)
                assert _same_bytes(out, want) and np.array_equal(cp, cp0), name


def _link_bytes(link):
    return bytes(memoryview(link))


def test_slice_prepare_link_equals_host_link(tmp_path):
    import torch
    from test_gpu_parity import _nav_file
    ch310, nav310 = gps.scenario(_nav_file(tmp_path, 32), 60.0, 140.0, 0.0, seconds=310, max_chan=32,
                                 start=(2024, 1, 7, 2, 0, 0.0))
    occ = ch310["prn"]
    change = [b for b in range(1, ch310.shape[0]) if np.any(occ[b] != occ[b - 1])]
    cases = []
    for ranks in (2, 8):
        edges = sorted(set([gps.sharding.slice_bounds(ch310.shape[0], ranks, r)[0] for r in range(ranks)] + change +
                           [ch310.shape[0]]))
        cases += [(ch310, nav310, lo, hi) for lo, hi in zip(edges[:-1], edges[1:])]
    ch, nav = _workload()
    cases += [(ch, nav, 0, NBLK), (ch, nav, 0, 700), (ch, nav, 700, NBLK), (ch, nav, 390, 800)]
    for chans, frames, lo, hi in cases:
        part = chans[lo:hi]
        with gps.Context(part.shape[1], hi - lo, max_nav_frames=len(frames)) as ctx:
            dev = torch.empty((hi - lo) * gps.BLOCK_ELEMS, dtype=torch.int8, device="cuda")
            link = ctx.slice_prepare(part, 1, dev.data_ptr())
            assert _link_bytes(link) == _link_bytes(gps.slice_link_host(part)), (lo, hi)
            ctx.slice_probe()
            ctx.slice_finish()
            ctx.slice_wait()
