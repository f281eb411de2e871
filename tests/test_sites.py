"""The ionosphere term away from the Tokyo noon sky, on the CPU. Every other fixture is made under one sky (Tokyo, 02:00
UTC, local solar time near 11:20), where the Klobuchar term only ever takes its daytime, mid-latitude, northern branch.
These fixtures (tests/golden/make_golden_sites.py) are runs of the unmodified reference at three receivers with the
constellation centred on each -- 66 N 100 W, 66 S 140 E, 34.6 S 58.4 W -- and at Tokyo with the ionosphere switched off
(-I) and from a file without ION ALPHA / ION BETA.

- The scenario engine's per-block records and NAV frames equal the reference's bit for bit at every one of them; the
  file without the Klobuchar lines sends no subframe 4 page 18 and its words decode to invalid Klobuchar terms.
- A traced restatement of the Klobuchar term shows which branches each site's fixes take: night and day, the phi_i clamp
  at +-0.416, the AMP and PER clamps, a local time below 0 before the day wrap, both signs of phi_m and the three
  sigma_iono bands of ARAIM. Each site must reach the branches it exists for.
- Ideal-epoch fixes stay within IDEAL at every site; ARAIM passes and bounds the truth there.
- With -I, fixes without the Klobuchar term stay within IDEAL while the page-18 term misses by metres; without the
  header lines, the constant F * 5 ns delay (alpha = 0) stays within IDEAL.
- The day wrap of the local time: the reference's loops, the model's np.mod and the kernel's floor form agree on doubles
  next to every multiple of a day the term can meet."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import araim_model as AM
import pvt_model as PM
import pvt_truth as PT
import scenario
from scenario import gps
from test_araim import kfa, new_trace, assert_margin
from test_interactive import assert_params_equal
from test_pvt import IDEAL, check_truth, ideal_inputs
from test_time_overwrite import gps_time, page18, parse_start

SITES = ["site_66n_100w_10s_i8", "site_66s_140e_10s_i8", "site_34s_58w_10s_i16"]
IONO_OFF = "sky12_iono_off_3s_i8"
NO_HEADER = "sky12_iono_hdr_missing_520s_i8"
FIXTURES = SITES + [IONO_OFF, NO_HEADER]
ALPHA0 = np.zeros(4)

# the branches of the Klobuchar term (gps.c:1893-1964) and of ARAIM's sigma_iono (include/gpsb200.h)
BRANCHES = ("day", "night", "phi_i_clamp_north", "phi_i_clamp_south", "amp_clamp", "per_clamp", "local_time_below_0",
            "phi_m_north", "phi_m_south", "sigma_band_20", "sigma_band_55", "sigma_band_polar")
# what each site is there for; a site that stops reaching one of them fails test_each_site_reaches_its_branches
REACHES = {
    "site_66n_100w_10s_i8": {"day", "night", "phi_i_clamp_north", "amp_clamp", "per_clamp", "local_time_below_0",
                             "phi_m_north", "sigma_band_polar"},
    "site_66s_140e_10s_i8": {"day", "phi_i_clamp_south", "per_clamp", "phi_m_south", "sigma_band_polar"},
    "site_34s_58w_10s_i16": {"night", "local_time_below_0", "phi_m_south", "sigma_band_20", "sigma_band_55"},
}
# and what it must not reach: the whole run in one branch where the site is chosen for that
AVOIDS = {
    "site_66s_140e_10s_i8": {"night", "local_time_below_0", "amp_clamp"},
    "site_34s_58w_10s_i16": {"day"},
}


def nav_file(g, d):
    """the fixture's RINEX file: gen_rinex.py's constellation centred on the fixture's sky centre"""
    nav = d / "sky.nav"
    c = g["sky_centre"]
    subprocess.check_call([sys.executable, os.path.join(scenario.ROOT, "oracle", "gen_rinex.py"), "--nsat",
                           str(int(g["nsat"])), "--out", str(nav), "--rx=%r,%r" % (float(c[0]), float(c[1]))] +
                          ([] if bool(g["iono_header"]) else ["--no-iono"]))
    return str(nav)


def site_case(name, tmp_path):
    """fixture -> (golden, scenario kwargs)"""
    g = scenario.load_golden(name)
    d = tmp_path / name
    d.mkdir()
    loc = g["location"]
    kw = dict(nav_file=nav_file(g, d), lat=loc[0], lon=loc[1], height=loc[2], seconds=float(g["seconds"]),
              max_chan=int(g["max_chan"]), start=parse_start(str(g["start"])), ionosphere=bool(g["ionosphere"]))
    return g, kw


def fix_inputs(name, tmp_path, nblk=99):
    """Ideal epochs of the first nblk blocks of a fixture's run (records from the scenario engine), a fix about every
    second from 0.01 s, the Klobuchar terms of the file's header (None without them). -> (chans, eps, cfg, iono,
    (truth rows, start second of week), records)"""
    g, kw = site_case(name, tmp_path)
    ch, nav = gps.scenario(**kw)
    ch = ch[:nblk]
    chans, eps = ideal_inputs(ch, nav, ch["nav_frame"][:, 0])
    _, alpha, beta = PT.read_rinex(kw["nav_file"])
    iono = PT.klobuchar_broadcast(alpha, beta) if bool(g["iono_header"]) else None
    cfg = gps.pvt_config(30000, 2999993, (nblk * PT.BLOCK - 30000 - PT.BLOCK) // 2999993, iono)
    xyz = np.repeat(PM.llh_ecef(kw["lat"], kw["lon"], kw["height"])[None], ch.shape[0] + 1, 0)
    return chans, eps, cfg, iono, (xyz, gps_time(kw["start"])[1]), ch


# ---- the reference's records --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FIXTURES)
def test_engine_equals_the_reference(name, tmp_path):
    g, kw = site_case(name, tmp_path)
    got, nav = gps.scenario(**kw)
    prn = g["prn_of_block"].astype(np.int32)
    assert got.shape == prn.shape and np.array_equal(got["prn"], prn)
    assert ((prn > 0).sum(1) == int(g["nsat"])).all()              # the whole constellation is in view all along
    idx = g["chans_idx"] if "chans_idx" in g else np.arange(prn.shape[0])
    assert_params_equal(got[idx], g["chans"], idx)
    assert np.array_equal(got["carr_phase"][0].view(np.uint64), g["chans"]["carr_phase"][0].view(np.uint64))
    frames, fidx = g["nav_frames"], g["nav_frame_of_block"]
    assert np.array_equal(got["nav_frame"][:, 0], fidx) and len(nav) == len(frames)
    assert np.array_equal(nav, frames)


def test_without_the_klobuchar_lines_no_page_18_is_sent(tmp_path):
    """The file without ION ALPHA / ION BETA: frame 17, where page 18 goes (test_pvt: the 780 s stream), is in the
    fixture; no frame of it carries page 18 and no slot decodes to valid Klobuchar terms. The same run from the file with
    the lines sends page 18 in frame 17."""
    g, kw = site_case(NO_HEADER, tmp_path)
    frames = g["nav_frames"]
    assert len(frames) == 18
    slots = [frames[f][c] for f in range(len(frames)) for c in range(frames.shape[1]) if frames[f][c].any()]
    assert len(slots) == 18 * 12
    assert all(page18(w) is None for w in slots)
    for w in slots:
        eph, iono = gps.nav_ephemeris(gps.nav_words_of_frame(w))
        assert eph["valid"] == 1 and iono["valid"] == 0
    full = dict(kw, nav_file=nav_file({"sky_centre": g["sky_centre"], "nsat": g["nsat"], "iono_header": True},
                                      tmp_path))
    _, nav = gps.scenario(**full)
    assert page18(nav[17][0]) is not None and page18(nav[16][0]) is None
    _, iono = gps.nav_ephemeris(gps.nav_words_of_frame(nav[17][0]))
    assert iono["valid"] == 1


# ---- branch coverage of the Klobuchar term --------------------------------------------------------------------------
def klobuchar_branches(alpha, beta, lat, lon, az, el, t):
    """The Klobuchar term restated with each branch recorded: -> (delay [m], {branch: bool array})."""
    PI, C = PM.PI, PM.C
    E, phi_u, lam_u = el / PI, lat / PI, lon / PI
    F = 1.0 + 16.0 * (0.53 - E) ** 3
    psi = 0.0137 / (E + 0.11) - 0.022
    raw = phi_u + psi * np.cos(az)
    phi_i = np.clip(raw, -0.416, 0.416)
    lam_i = lam_u + psi * np.sin(az) / np.cos(phi_i * PI)
    phi_m = phi_i + 0.064 * np.cos((lam_i - 1.617) * PI)
    amp = alpha[0] + alpha[1] * phi_m + alpha[2] * phi_m ** 2 + alpha[3] * phi_m ** 3
    per = beta[0] + beta[1] * phi_m + beta[2] * phi_m ** 2 + beta[3] * phi_m ** 3
    traw = 43200.0 * lam_i + t
    tl = np.mod(traw, 86400.0)
    X = 2.0 * PI * (tl - 50400.0) / np.maximum(per, 72000.0)
    night = np.abs(X) >= 1.57
    d = np.where(night, F * 5.0e-9 * C, F * (5.0e-9 + np.maximum(amp, 0.0) * (1.0 - X * X / 2.0 + X ** 4 / 24.0)) * C)
    pm = np.abs(phi_m) * 180.0
    b = dict(day=~night, night=night, phi_i_clamp_north=raw > 0.416, phi_i_clamp_south=raw < -0.416, amp_clamp=amp < 0.0,
             per_clamp=per < 72000.0, local_time_below_0=traw < 0.0, phi_m_north=phi_m > 0.0, phi_m_south=phi_m < 0.0,
             sigma_band_20=pm <= 20.0, sigma_band_55=(pm > 20.0) & (pm <= 55.0), sigma_band_polar=pm > 55.0)
    return d, {k: np.broadcast_to(v, d.shape).ravel() for k, v in b.items()}


def traced_branches(name, tmp_path, monkeypatch):
    """Ideal-epoch fixes and ARAIM at mask 5 deg on the site's first 10 s with every Klobuchar evaluation traced; the
    restatement gives the same delay as the model at each. -> {branch: count}, evaluations"""
    chans, eps, cfg, _, _, _ = fix_inputs(name, tmp_path)
    seen = []
    model = PM.klobuchar

    def traced(alpha, beta, lat, lon, az, el, t, trace=None):
        want = model(alpha, beta, lat, lon, az, el, t, trace)
        d, b = klobuchar_branches(alpha, beta, lat, lon, az, el, t)
        assert np.array_equal(np.broadcast_to(d, want.shape), want)
        seen.append(b)
        return want
    monkeypatch.setattr(PM, "klobuchar", traced)
    PM.pvt(chans, eps, cfg)
    AM.araim(chans, eps, cfg, gps.araim_config(mask_deg=5.0), *kfa(gps.araim_config(mask_deg=5.0)))
    assert seen
    return {k: int(sum(int(s[k].sum()) for s in seen)) for k in BRANCHES}, sum(s["day"].size for s in seen)


@pytest.mark.parametrize("name", SITES)
def test_each_site_reaches_its_branches(name, tmp_path, monkeypatch):
    count, n = traced_branches(name, tmp_path, monkeypatch)
    missing = [k for k in sorted(REACHES[name]) if count[k] == 0]
    assert not missing, (name, missing, count)
    reached = [k for k in sorted(AVOIDS.get(name, ())) if count[k] > 0]
    assert not reached, (name, reached, count)
    if name == "site_66n_100w_10s_i8":           # the evening terminator: both sides of |X| = 1.57 in one run
        assert count["night"] > n // 4 and count["day"] > n // 10, count
        assert count["per_clamp"] == count["local_time_below_0"] == n, count


def test_the_sites_reach_every_branch():
    """Every branch is some site's: removing a site leaves one unreached."""
    assert set(REACHES) == set(SITES)
    assert set().union(*REACHES.values()) == set(BRANCHES)
    for name in SITES:
        others = set().union(*(v for k, v in REACHES.items() if k != name))
        assert REACHES[name] - others, name


# ---- fixes ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SITES)
def test_ideal_fixes_and_araim_at_every_site(name, tmp_path):
    chans, eps, cfg, _, (xyz, sow), _ = fix_inputs(name, tmp_path)
    fix, _, _ = PM.pvt(chans, eps, cfg)
    assert (fix["nused"] == len(eps)).all()
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])
    for mask in (5.0, 10.0):
        acfg = gps.araim_config(mask_deg=mask)
        tr = new_trace()
        afix, _, rec, _ = AM.araim(chans, eps, cfg, acfg, *kfa(acfg), trace=tr)
        assert_margin(tr)
        assert (rec["verdict"] == AM.PASS).all(), rec["verdict"]
        E = AM.enu(xyz[0])
        err = (np.stack([afix["x"], afix["y"], afix["z"]], 1) - xyz[0]) @ E.T
        assert np.all(np.hypot(err[:, 0], err[:, 1]) < rec["hpl"]) and np.all(np.abs(err[:, 2]) < rec["vpl"])


def errors(fix, xyz):
    assert (fix["status"] == PM.FIX_OK).all()
    tx, _ = PT.truth_xyz(xyz, fix["sample"])
    return np.linalg.norm(np.stack([fix["x"], fix["y"], fix["z"]], 1) - tx, axis=1)


def test_ionosphere_off_stream_is_fixed_without_the_term(tmp_path):
    """-I: fixes without the Klobuchar term are within IDEAL; with the header's (page 18) terms they miss by metres."""
    chans, eps, cfg, iono, (xyz, sow), _ = fix_inputs(IONO_OFF, tmp_path, nblk=29)
    off = gps.pvt_config(int(cfg["s0"]), int(cfg["step"]), int(cfg["nfix"]))
    fix, _, _ = PM.pvt(chans, eps, off)
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])
    on, _, _ = PM.pvt(chans, eps, cfg)
    assert errors(on, xyz).min() > 3.0, errors(on, xyz)


def test_missing_klobuchar_lines_give_the_constant_delay(tmp_path):
    """Without ION ALPHA / ION BETA the delay is F * 5 ns: alpha = 0 gives exactly that and stays within IDEAL; without
    the term the fixes miss by metres."""
    chans, eps, cfg, iono, (xyz, sow), _ = fix_inputs(NO_HEADER, tmp_path, nblk=99)
    assert iono is None
    const = gps.pvt_config(int(cfg["s0"]), int(cfg["step"]), int(cfg["nfix"]), (ALPHA0, np.zeros(4)))
    fix, _, _ = PM.pvt(chans, eps, const)
    check_truth(fix, xyz, sow, IDEAL["pos"], IDEAL["time"], IDEAL["vel"])
    off, _, _ = PM.pvt(chans, eps, cfg)
    assert errors(off, xyz).min() > 1.0, errors(off, xyz)


# ---- the day wrap ---------------------------------------------------------------------------------------------------
def wrap_reference(t):
    """gps.c:1948-1951"""
    while t >= 86400.0:
        t -= 86400.0
    while t < 0:
        t += 86400.0
    return t


def wrap_kernel(t):
    """csrc/pvt.cu klobuchar(): t - 86400 floor(t / 86400) (the product is an integer below 2^53, so exact with or
    without a fused multiply-add)"""
    return t - 86400.0 * math.floor(t / 86400.0)


def test_day_wrap_forms_agree():
    """43200 lambda_i + t lies in (-43200 * 1.1, 604800 + 43200 * 1.1): days -1 to 8. On every double within 300 ulps
    of each multiple of a day there, and on a sweep across each day, the reference's loops and the model's np.mod give
    the same bits, and so does the kernel's floor form -- except below 0 by less than 86400 * 2^-1075, where the
    kernel's quotient underflows to -0 and the form returns its input. A local time there needs the receive time and
    43200 lambda_i both within 1e-300 of 0, which no fix meets, so the kernel keeps its form."""
    n = 0
    for k in range(-1, 9):
        c = 86400.0 * k
        lo, hi = [c], [c]
        for _ in range(300):
            lo.append(float(np.nextafter(lo[-1], -np.inf)))
            hi.append(float(np.nextafter(hi[-1], np.inf)))
        xs = lo + hi + list(c + np.linspace(0.0, 86400.0, 1001)[1:-1])
        for t in xs:
            r = wrap_reference(t)
            assert float(np.mod(t, 86400.0)) == r and 0.0 <= r <= 86400.0, t
            assert wrap_kernel(t) == (t if t < 0.0 and t / 86400.0 == 0.0 else r), t
            n += 1
    assert n > 10 * 1600
    for t in (-5e-324, -2e-319):
        assert wrap_kernel(t) == t and wrap_reference(t) == 86400.0 == float(np.mod(t, 86400.0))
    # the smallest magnitude that does not underflow: from there on the kernel wraps to 86400 as the reference does
    t = -86400.0 * np.finfo(np.float64).tiny
    assert wrap_kernel(t) == wrap_reference(t) == 86400.0
