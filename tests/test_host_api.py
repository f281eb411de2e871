"""CPU-side tests (no GPU): the C-ABI library loads and exports what include/gpsb200.h
declares, fails loudly without a device, and its host-only pieces (C/A code, exact
carrier fast-forward, FIFO) behave like the reference."""
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

import scenario
from scenario import gps

ROOT = scenario.ROOT


def header_functions():
    txt = open(os.path.join(ROOT, "include", "gpsb200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    names = re.findall(r"\b([a-z_0-9]+)\s*\([^;{]*\)\s*;", txt)
    return sorted(set(n for n in names if n.startswith(("gpsb200_", "fifo_"))))


def test_library_exports_every_declared_symbol():
    L = gps.lib()
    names = header_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), n
    assert set(names) == set(gps.api.EXPORTS)


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(gps.GpsB200Error) as e:
        gps.Context(12, 4)
    assert e.value.code == -2 and "no CPU fallback" in str(e.value)


def test_product_does_not_link_the_oracle():
    out = os.popen("ldd '%s'; nm -D '%s'" % (gps.lib_path(), gps.lib_path())).read()
    assert "oracle" not in out


def test_codegen_matches_reference_dump_and_is_gps200_kat():
    g = scenario.load_golden("sky32_static_10s_i8")
    for prn, ca in zip(g["code_prns"], g["codes"]):
        assert np.array_equal(gps.codegen(int(prn)), ca)
    assert int("".join(map(str, gps.codegen(1)[:10])), 2) == 0o1440
    with pytest.raises(gps.GpsB200Error):
        gps.codegen(33)


@pytest.mark.parametrize("name", ["sky12_static_35s_i8", "sky32_static_10s_i8", "sky12_circle_10s_i16"])
def test_exact_carrier_fast_forward_reproduces_reference_chain(name):
    # the reference's carr_phase at the start of block b+1 is what 300000 sequential FP64
    # additions left behind (gps.c:2821-2826); the O(#binade crossings) jump must land on
    # the same double, for every channel and block of the dumps
    g = scenario.load_golden(name)
    ch = g["chans"]
    n = 0
    for b in range(ch.shape[0] - 1):
        for c in range(ch.shape[1]):
            if ch["prn"][b, c] > 0 and ch["prn"][b + 1, c] == ch["prn"][b, c]:
                got = gps.carrier_advance(ch["carr_phase"][b, c], ch["f_carr"][b, c], 300000)
                assert got == ch["carr_phase"][b + 1, c], (b, c)
                n += 1
    assert n > 1000


def test_carrier_fast_forward_vs_brute_force_random():
    rng = np.random.default_rng(5)
    delt = 1.0 / 3000000.0
    for _ in range(60):
        x = rng.uniform(0, 1)
        f = rng.uniform(-6000, 6000) * rng.choice([1.0, 1e-2, 1e-4])
        n = int(rng.integers(1, 40000))
        c = f * delt
        y = x
        for _i in range(n):
            y = y + c
            if y >= 1.0:
                y -= 1.0
            elif y < 0.0:
                y += 1.0
        assert gps.carrier_advance(x, f, n) == y


def test_speculative_carrier_probe_is_exact_or_rejected():
    # parallel-in-time chain: a block walked from a GUESSED start phase plus the host fix-up must
    # either reproduce the sequential result bit for bit or say "rejected" -- never a wrong phase
    L = gps.lib()
    rng = np.random.default_rng(11)
    accepted = rejected = 0
    for t in range(3000):
        s = rng.uniform(0, 1)
        f = rng.uniform(-5500, 5500) if t % 9 else rng.uniform(-40, 40)
        err = rng.choice([0.0, 1e-15, 1e-13, 1e-12, 1e-10, 1e-8, 1e-6, 1e-3]) * rng.uniform(-1, 1)
        g = (s + err) % 1.0
        out = C.c_double()
        ok = L.gpsb200_carrier_probe_fixup(s, g, f, 300000, C.byref(out))
        if ok:
            accepted += 1
            assert out.value == gps.carrier_advance(s, f, 300000), (s, g, f)
        else:
            rejected += 1
    assert accepted > 1500 and rejected > 100


def test_speculation_accepts_nearly_all_blocks_of_reference_scenarios():
    # with the drift-model guesses the fix-up should almost never need the sequential fallback
    g = scenario.load_golden("sky12_static_35s_i8")
    ch = g["chans"]
    L = gps.lib()
    bad = tot = 0
    for c in range(ch.shape[1]):
        for b in range(1, ch.shape[0] - 1):
            s, f = float(ch["carr_phase"][b, c]), float(ch["f_carr"][b, c])
            guess = (s + 3e-12) % 1.0            # the size of the guess error seen over 35 s
            out = C.c_double()
            ok = L.gpsb200_carrier_probe_fixup(s, guess, f, 300000, C.byref(out))
            tot += 1
            if ok:
                assert out.value == float(ch["carr_phase"][b + 1, c])
            else:
                bad += 1
    assert bad <= 0.01 * tot, (bad, tot)


def _fifo_run(compat, nblocks=20, nbuf=8, size=1000):
    L = gps.lib()

    class IqBuf(C.Structure):
        pass
    IqBuf._fields_ = [("data8", C.POINTER(C.c_int8)), ("data16", C.POINTER(C.c_int16)),
                      ("totalLength", C.c_uint), ("validLength", C.c_uint), ("next", C.POINTER(IqBuf))]
    L.fifo_acquire.restype = C.POINTER(IqBuf)
    L.fifo_dequeue.restype = C.POINTER(IqBuf)
    L.fifo_enqueue.argtypes = [C.POINTER(IqBuf)]
    L.fifo_release.argtypes = [C.POINTER(IqBuf)]
    L.fifo_create.argtypes = [C.c_uint, C.c_uint, C.c_uint]
    L.fifo_create.restype = C.c_bool
    L.fifo_set_compat_drop.argtypes = [C.c_bool]
    L.fifo_set_compat_drop(compat)
    assert L.fifo_create(nbuf, size, 1)
    got = []

    def consumer():
        while True:
            b = L.fifo_dequeue()
            if not b:
                return
            got.append(int(b.contents.data8[0]))
            L.fifo_release(b)

    # like the reference (sdr_iqfile.c:73-77): the consumer starts once the FIFO is full
    def producer():
        for i in range(nblocks):
            b = L.fifo_acquire()
            if not b:
                return
            b.contents.data8[0] = i
            b.contents.validLength = size
            L.fifo_enqueue(b)

    tp = threading.Thread(target=producer)
    tp.start()
    L.fifo_wait_full()
    tc = threading.Thread(target=consumer)
    tc.start()
    tp.join()
    L.fifo_wait_next()
    L.fifo_halt()
    tc.join()
    L.fifo_destroy()
    L.fifo_set_compat_drop(False)
    return got


def test_fifo_delivers_every_buffer_in_order():
    assert _fifo_run(False) == list(range(20))


def test_fifo_compat_mode_reproduces_stock_loss_of_blocks_1_to_6():
    got = _fifo_run(True, nblocks=9)
    # stock program: block 0, then 7, 8, ... (SURVEY.md finding 3; fifo.c:163-168)
    assert got[:2] == [0, 7]


def test_fifo_push_reproduces_hackrf_buffer_cadence():
    # 600000-element blocks pushed into 262144-element buffers (HACKRF_TRANSFER_BUFFER_SIZE, sdr.h:34):
    # buffers fill across block boundaries, none is enqueued partly filled (gps.c:2847-2856)
    L = gps.lib()

    class IqBuf(C.Structure):
        pass
    IqBuf._fields_ = [("data8", C.POINTER(C.c_int8)), ("data16", C.POINTER(C.c_int16)),
                      ("totalLength", C.c_uint), ("validLength", C.c_uint), ("next", C.POINTER(IqBuf))]
    L.fifo_dequeue.restype = C.POINTER(IqBuf)
    L.fifo_release.argtypes = [C.POINTER(IqBuf)]
    L.fifo_create.argtypes = [C.c_uint, C.c_uint, C.c_uint]
    L.fifo_create.restype = C.c_bool
    L.gpsb200_fifo_push.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    assert L.fifo_create(8, 262144, 1)
    rng = np.random.default_rng(1)
    data = rng.integers(-128, 128, size=3 * 600000, dtype=np.int8)
    got = []

    def consumer():
        while True:
            b = L.fifo_dequeue()
            if not b:
                return
            n = b.contents.validLength
            got.append(np.ctypeslib.as_array(b.contents.data8, shape=(n,)).copy())
            L.fifo_release(b)

    t = threading.Thread(target=consumer)
    t.start()
    for blk in data.reshape(3, 600000):
        assert L.gpsb200_fifo_push(np.ascontiguousarray(blk).ctypes.data, blk.size, 1) == 0
    L.gpsb200_fifo_push_flush()
    L.fifo_wait_next()
    L.fifo_halt()
    t.join()
    L.fifo_destroy()
    sizes = [g.size for g in got]
    assert sizes[:-1] == [262144] * 6 and sizes[-1] == 1800000 - 6 * 262144
    assert np.array_equal(np.concatenate(got), data)


def test_span_level_chain_is_exact_or_rejected():
    """Second level of the parallel-in-time carrier chain (nco_exact.h: span_chain): K block probes chained
    speculatively from a GUESSED span start, then ONE fix-up with the true start. Whenever the speculation is
    accepted, every block start and the end phase equal the sequential exact chain bit for bit."""
    rng = np.random.default_rng(20240924)
    accepted = 0
    for case in range(160):
        K = int(rng.choice([2, 5, 32, 64]))
        f0 = rng.uniform(-6000, 6000) if rng.random() > 0.15 else rng.uniform(-400, 400)
        f = f0 + np.cumsum(rng.uniform(-0.1, 0.1, K))
        s = rng.uniform(0, 1)
        g = s + rng.choice([0.0, 1e-13, -1e-12, 3e-11, -2e-10, 1e-9, 1e-6])
        g = min(max(g, 0.0), np.nextafter(1.0, 0))
        out = gps.span_chain_host(f, s, g)
        if out is None:
            continue
        accepted += 1
        x, want = s, [s]
        for j in range(K):
            x = gps.carrier_advance(x, f[j], 300000)
            want.append(x)
        assert np.array_equal(out, np.array(want)), (case, K, f0)
    assert accepted > 100
    # a Doppler zero crossing inside the span changes the rounding grid: never accepted
    f = np.linspace(3.0, -3.0, 8) * 200.0
    assert gps.span_chain_host(f, 0.3, 0.3) is None


def _lanes_case(nchan, seed, force=0, scale=1.0, edge=False):
    ch, nav = gps.synthetic_chans(1, nchan, seed=seed)
    ch["f_carr"] *= scale
    ch["f_code"] = 1.023e6 + ch["f_carr"] / 1540.0
    rng = np.random.default_rng(seed)
    if edge:
        e = rng.integers(0, 4, size=nchan)
        ch["code_phase"][:, e == 1] = np.nextafter(1023.0, 0)
        ch["code_phase"][:, e == 2] = 0.0
        ch["icode"][:, e == 3] = 19
        ch["ibit"][:, e == 3] = 29
        ch["iword"][:, e == 3] = rng.integers(0, 59)
        ch["carr_phase"][0] = rng.choice([0.0, np.nextafter(1.0, 0), 0.5, 2.0 ** -40], size=nchan)
        ch["prn"][:, rng.random(nchan) < 0.15] = 0
    want, carr = scenario.oracle_run(ch, nav, 2)
    iq, carr_out, counters = gps.lanes_model_block(ch[0], nav[0], force=force)
    return np.array_equal(iq, want), counters


@pytest.mark.parametrize("nchan", [1, 5, 12, 16])
def test_lane_per_sample_model_is_bit_exact(nchan):
    """synth_lanes.h (fixed-point linear phases certified from exact anchors, residue-class chip words, band repair)
    against the oracle's FP64 recurrences (gps.c:2767-2857), one block."""
    for seed in (100, 101):
        ok, counters = _lanes_case(nchan, seed)
        assert ok, (nchan, seed, counters)
        assert counters[0] > 299000                               # nearly every sample takes the integer-only path


def test_lane_per_sample_model_many_seeds_and_code_rates():
    """More seeds, and code rates across the whole range the kernel accepts (1.0157 .. 1.0302 MHz): the carry-point
    estimate (integer multiply by a 32-bit reciprocal) against the oracle."""
    for seed in range(400, 412):
        ok, counters = _lanes_case(12, seed)
        assert ok, (seed, counters)
    for i, f_code in enumerate((1.01571e6, 1.0158e6, 1.019e6, 1.0229e6, 1.0231e6, 1.027e6, 1.03019e6)):
        ch, nav = gps.synthetic_chans(1, 6, seed=900 + i)
        ch["f_code"][:] = f_code + np.arange(6) * 0.37
        want, carr = scenario.oracle_run(ch, nav, 2)
        iq, carr_out, counters = gps.lanes_model_block(ch[0], nav[0])
        assert np.array_equal(iq, want), (f_code, counters)


def test_lane_per_sample_model_run_lengths():
    """Every run length the kernel accepts (multiples of 96 that divide 300000, up to 2400: the band widths are sized for
    2400 steps of accumulated rounding); longer ones are refused."""
    ch, nav = gps.synthetic_chans(1, 7, seed=77)
    want, carr = scenario.oracle_run(ch, nav, 2)
    for run in (96, 480, 2400):
        iq, carr_out, counters = gps.lanes_model_block(ch[0], nav[0], run_samples=run)
        assert np.array_equal(iq, want), run
    with pytest.raises(Exception):
        gps.lanes_model_block(ch[0], nav[0], run_samples=12000)


def test_lane_per_sample_model_extremes_and_forced_repairs():
    """Doppler x6 / x1e-5, phases on the wrap, NAV bit edges, idle channels; and every repair path forced on."""
    for seed, scale in ((300, 6.0), (301, 0.01), (302, 1e-5), (303, 2.5)):
        ok, counters = _lanes_case(12, seed, 0, scale, edge=True)
        assert ok, (seed, scale, counters)
    for force in (1, 2, 3, 5, 7, 8, 13):
        ok, counters = _lanes_case(8, 555, force, 1.0, edge=True)
        assert ok, (force, counters)


def test_lane_per_sample_model_adversarial_phases():
    """Anchors chosen so that some sample's LINEAR phase lands on a table-index boundary (carrier) or on a chip boundary
    (code) to within an ulp: exactly where floor(linear) and floor(FP64 recurrence) may differ, i.e. where the band tests
    have to send the sample to the exact walk. Against the oracle, and the repair counters must show the walks happened."""
    from fractions import Fraction
    delt = Fraction(1, 3000000)
    walks = 0
    rebuilt = 0
    for case, (f_carr, n_hit, k_hit) in enumerate([(2345.678, 1000, 17), (-1843.21, 77, 300), (4999.99, 2399, 511),
                                                   (-12.5, 150000, 256), (3.0e-3, 299999, 1), (-5999.0, 96, 0)]):
        ch, nav = gps.synthetic_chans(1, 4, seed=60 + case)
        # carrier of slot 0: x0 + n_hit * c == k_hit / 512 (mod 1) in exact arithmetic, then rounded to double
        c = Fraction(float(np.float64(f_carr) * np.float64(1.0 / 3.0e6)))
        x0 = (Fraction(k_hit, 512) - n_hit * c) % 1
        ch["f_carr"][0, 0] = f_carr
        ch["carr_phase"][0, 0] = min(float(x0), float(np.nextafter(1.0, 0)))
        # code of slot 1: y0 + n_hit * d == an integer chip (mod 1023)
        d = Fraction(float(np.float64(ch["f_code"][0, 1]) * np.float64(1.0 / 3.0e6)))
        y0 = (Fraction(500 + case) - n_hit * d) % 1023
        ch["code_phase"][0, 1] = float(y0)
        want, carr = scenario.oracle_run(ch, nav, 2)
        iq, carr_out, counters = gps.lanes_model_block(ch[0], nav[0])
        assert np.array_equal(iq, want), (case, counters)
        walks += int(counters[3])
        rebuilt += int(counters[2])
    assert walks > 0 and rebuilt > 0, (walks, rebuilt)


def test_lane_per_sample_model_engineered_repair_hits():
    """The engineered hits of tests/repair_cases.py (carrier-index and chip boundaries at chosen block, run, window, lane,
    residue and slot, from exact anchors of later runs and later blocks): each hit, alone in its block, makes the model
    walk (carrier) or rebuild the window's chip signs exactly (code), and every block of every case equals the oracle.
    The GPU test feeds the same cases to k_synth_lanes; its anchors are the exact walks the model takes here."""
    import repair_cases as rc
    for case in rc.CASES:
        ch, nav, decisive = rc.build(case)
        for h in case.hits:
            row = rc.chained_row(ch, h.block)[[h.slot]]
            _, _, counters = gps.lanes_model_block(row, nav[0][[h.slot]])
            assert counters[3 if h.kind == "carr" else 2] > 0, (case.name, h, counters)
            # the FP64 and the linear phase straddle the boundary: skipping the repair would change the sample
            # (window 0, sample 0 of run 0 has no rounding behind it: its linear phase is the input phase itself)
            assert decisive[h.slot] == (h.run + h.win + h.n + h.block > 0), (case.name, h)
        want, _ = scenario.oracle_run(ch, nav, 2)
        for b in range(case.nblk):
            iq, _, counters = gps.lanes_model_block(rc.chained_row(ch, b), nav[0])
            assert np.array_equal(iq, want[b * gps.BLOCK_ELEMS:(b + 1) * gps.BLOCK_ELEMS]), (case.name, b, counters)
