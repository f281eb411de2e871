"""The machine code of k_synth_lanes as built for sm_90a (cuobjdump -sass of libgpsb200.so), checked for what keeps the
kernel's instruction issue down: the look-up loop of the sample side stays at 172 instructions or fewer per 8 channels x
3 samples, the full 32-channel call has a look-up loop of its own with a fixed trip count, and
the window loop's local-memory traffic stays below what it was before the window state was cut down. Loops are found
from the backward branches: the look-up loops are the loops with the 24 table look-ups of 8 channels x 3 samples and no
call, the window loop is the largest loop inside the run loop that contains them."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "multi-sdr-gps-sim_b200", "libgpsb200.so")

LOOKUP_MAX = 172
# LDL + STL inside the window loop, per channel capacity (common and rare paths together). Before the window state was
# packed and the full-capacity loop given a fixed trip count: 33 (32-channel variants) and 41 (16-channel).
LOCAL_MAX = {32: 23, 16: 35}

INS = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


@pytest.fixture(scope="module")
def variants():
    exe = cuobjdump()
    if exe is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is missing")
    text = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "k_synth_lanes" in m.group(1) else None
            if cur:
                funcs[cur] = []
            continue
        m = INS.search(line)
        if m and cur:
            funcs[cur].append((int(m.group(1), 16), m.group(2)))
    assert len(funcs) == 4, sorted(funcs)          # int8 / int16 x 16 / 32 channels
    return funcs


def capacity(name):
    return int(re.search(r"k_synth_lanesILb[01]ELi(\d+)E", name).group(1))


def count(ins, lo, hi, pat):
    return sum(1 for a, t in ins if lo <= a <= hi and re.search(pat, t))


def loops(ins):
    out = set()
    for a, t in ins:
        m = re.search(r"\bBRA\b.*?(0x[0-9a-f]+)", t)
        if m and int(m.group(1), 16) <= a:
            out.add((int(m.group(1), 16), a))
    return sorted(out)


def lookup_loops(ins):
    return [(lo, hi) for lo, hi in loops(ins)
            if count(ins, lo, hi, r"^(@!?P\d )?LDS(\.U?32)? ") >= 24 and count(ins, lo, hi, r"\bCALL\b") == 0]


def window_loop(ins):
    inner = lookup_loops(ins)
    outer = [(lo, hi) for lo, hi in loops(ins)
             if (lo, hi) not in inner and all(lo <= a and b <= hi for a, b in inner)]
    outer.sort(key=lambda x: x[1] - x[0], reverse=True)
    assert len(outer) >= 2, outer                    # the run loop, then the window loop
    return outer[1]


def test_lookup_loop_length(variants):
    for name, ins in variants.items():
        found = lookup_loops(ins)
        # 32 channels: one loop for the full call and one for any other count; 16: one per window of a trip
        assert len(found) == 2, (name, found)
        for lo, hi in found:
            assert (hi - lo) // 16 + 1 <= LOOKUP_MAX, (name, hex(lo), (hi - lo) // 16 + 1)


def test_window_loop_local_memory(variants):
    for name, ins in variants.items():
        lo, hi = window_loop(ins)
        n = count(ins, lo, hi, r"^(@!?P\d )?(LDL|STL)\b")
        assert n <= LOCAL_MAX[capacity(name)], (name, n)
