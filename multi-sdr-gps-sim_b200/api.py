"""ctypes mirror of include/gpsb200.h. No compute happens here and there is no CPU
fallback: if libgpsb200.so is missing or no CUDA device is present the calls fail."""
import ctypes as C
import os

import numpy as np

BLOCK_SAMPLES = 300000
BLOCK_ELEMS = 600000
SC08, SC16 = 1, 2

_HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path():
    return os.path.join(_HERE, "libgpsb200.so")


class GpsB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("gpsb200 error %d: %s" % (code, msg))
        self.code = code


class Chan(C.Structure):
    """gpsb200_chan_t (64 bytes)."""
    _fields_ = [("prn", C.c_int32), ("iword", C.c_int32), ("ibit", C.c_int32), ("icode", C.c_int32),
                ("nav_frame", C.c_int32), ("reserved", C.c_int32),
                ("f_carr", C.c_double), ("f_code", C.c_double), ("carr_phase", C.c_double),
                ("code_phase", C.c_double), ("gain", C.c_double)]


CHAN_DTYPE = np.dtype([("prn", "<i4"), ("iword", "<i4"), ("ibit", "<i4"), ("icode", "<i4"),
                       ("nav_frame", "<i4"), ("reserved", "<i4"),
                       ("f_carr", "<f8"), ("f_code", "<f8"), ("carr_phase", "<f8"),
                       ("code_phase", "<f8"), ("gain", "<f8")])
assert CHAN_DTYPE.itemsize == C.sizeof(Chan) == 64

# one run checkpoint (gpsb200_debug_run_checkpoints): NCO state at the first sample of a run
RUN_CKPT_DTYPE = np.dtype([("x", "<f8"), ("y", "<f8"), ("nav", "<u4"), ("pad", "<u4")])
assert RUN_CKPT_DTYPE.itemsize == 24

# one carrier block probe (gpsb200_carrier_probe_host, gpsb200_debug_block_probes)
CARRIER_PROBE_DTYPE = np.dtype([("x_w", "<f8"), ("x_end", "<f8", 2), ("m_pos", "<f8", 2), ("m_neg", "<f8", 2),
                                ("n_w", "<i4"), ("pad", "<i4")])
assert CARRIER_PROBE_DTYPE.itemsize == 64


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_chan", C.c_int32), ("max_blocks", C.c_int32),
                ("max_nav_frames", C.c_int32), ("host_threads", C.c_int32), ("run_samples", C.c_int32)]


class ScenarioConfig(C.Structure):
    _fields_ = [("nav_file", C.c_char_p), ("motion_file", C.c_char_p),
                ("lat_deg", C.c_double), ("lon_deg", C.c_double), ("height_m", C.c_double),
                ("duration_ds", C.c_int32), ("max_chan", C.c_int32), ("ionosphere_enable", C.c_int32),
                ("pluto_gain", C.c_int32),
                ("start_year", C.c_int32), ("start_month", C.c_int32), ("start_day", C.c_int32),
                ("start_hour", C.c_int32), ("start_min", C.c_int32), ("rinex3", C.c_int32),
                ("start_sec", C.c_double), ("target_valid", C.c_int32), ("reserved", C.c_int32),
                ("target_distance_m", C.c_double), ("target_bearing_deg", C.c_double), ("target_height_m", C.c_double),
                ("almanac_file", C.c_char_p)]
    # the header's `interactive` field (int32 at offset 92); _fields_ keeps its former name `reserved`, so that code
    # written against the earlier mirror still runs
    interactive = property(lambda self: self.reserved, lambda self, v: setattr(self, "reserved", v))


class SteerState(C.Structure):
    """gpsb200_steer_state_t."""
    _fields_ = [("speed", C.c_double), ("velocity", C.c_double), ("bearing_mdeg", C.c_double),
                ("vertical_speed", C.c_double), ("xyz", C.c_double * 3), ("next_block", C.c_int32),
                ("end_block", C.c_int32)]


assert C.sizeof(SteerState) == 64

ERR_ARG = -1
ERR_END = -6
# the keys of the reference's interactive mode (gui.h:25-32, gps-sim.c:336-401)
KEYS = "adwseqtgxX"


ALMANAC_RECORD_DTYPE = np.dtype([("svid", "<i4"), ("svn", "<i4"), ("ura", "<i4"), ("health", "<i4"), ("config_code", "<i4"),
                                 ("valid", "<i4"), ("toa_week", "<i4"), ("reserved", "<i4"),
                                 ("e", "<f8"), ("delta_i", "<f8"), ("omegadot", "<f8"), ("sqrta", "<f8"), ("omega0", "<f8"),
                                 ("aop", "<f8"), ("m0", "<f8"), ("af0", "<f8"), ("af1", "<f8"), ("toa_sec", "<f8")])
assert ALMANAC_RECORD_DTYPE.itemsize == 112          # gpsb200_almanac_record_t


class SliceLink(C.Structure):
    """gpsb200_slice_link_t."""
    _fields_ = [("prn_first", C.c_int32 * 32), ("prn_last", C.c_int32 * 32), ("reset_inside", C.c_int32 * 32),
                ("first_phase", C.c_double * 32), ("value", C.c_double * 32)]


class Stats(C.Structure):
    _fields_ = [("host_chain_ms", C.c_double), ("h2d_ms", C.c_double), ("kernel_ms", C.c_double),
                ("d2h_ms", C.c_double), ("checkpoint_kernel_ms", C.c_double), ("synth_kernel_ms", C.c_double),
                ("probe_kernel_ms", C.c_double),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("launches", C.c_int32),
                ("chain_fallbacks", C.c_int32)]


class AcqConfig(C.Structure):
    """gpsb200_acq_config_t (168 bytes)."""
    _fields_ = [("s0", C.c_int64), ("ms", C.c_int32), ("nprn", C.c_int32), ("prn", C.c_int32 * 32),
                ("f_lo_hz", C.c_double), ("step_hz", C.c_double), ("nbins", C.c_int32), ("reserved", C.c_int32)]


assert C.sizeof(AcqConfig) == 168

# gpsb200_acq_result_t: one row per searched PRN
ACQ_RESULT_DTYPE = np.dtype([("prn", "<i4"), ("bin", "<i4"), ("delay", "<i4"), ("reserved", "<i4"),
                             ("doppler_hz", "<f8"), ("delay_chips", "<f8"), ("p1", "<u8"), ("p2", "<u8"), ("ratio", "<f8")])
assert ACQ_RESULT_DTYPE.itemsize == 56
ACQ_CODE_SAMPLES = 3000


def acq_window_samples(ms):
    """Samples an acquisition search over `ms` coherent 1 ms periods reads from s0 on: 3000 ms + 2999."""
    return ACQ_CODE_SAMPLES * int(ms) + ACQ_CODE_SAMPLES - 1


# gpsb200_track_state_t / gpsb200_track_epoch_t (DESIGN §10)
TRACK_STATE_DTYPE = np.dtype([("prn", "<i4"), ("epochs", "<i4"), ("sample", "<i8"), ("code_phase", "<u8"),
                              ("carr_freq", "<i8"), ("carr_phase", "<u4"), ("carr_step", "<i4"), ("code_step", "<u4"),
                              ("prev_i", "<i4"), ("prev_q", "<i4"), ("lock_i", "<i4"), ("lock_q", "<i4"), ("lock", "<i4")])
assert TRACK_STATE_DTYPE.itemsize == 64
TRACK_EPOCH_DTYPE = np.dtype([("sample", "<i8"), ("e_i", "<i4"), ("e_q", "<i4"), ("p_i", "<i4"), ("p_q", "<i4"),
                              ("l_i", "<i4"), ("l_q", "<i4"), ("carr_phase", "<u4"), ("carr_step", "<i4"),
                              ("code_phase", "<u4"), ("code_step", "<u4"), ("lock", "<i4"), ("reserved", "<i4")])
assert TRACK_EPOCH_DTYPE.itemsize == 56
NAV_BIT_DTYPE = np.dtype([("sample", "<i8"), ("sum", "<i8"), ("value", "<i4"), ("locked", "<i4")])
NAV_WORD_DTYPE = np.dtype([("sample", "<i8"), ("raw", "<u4"), ("data", "<u4"), ("parity_ok", "<i4"), ("subframe", "<i4"),
                           ("tow", "<i4"), ("index", "<i4")])
NAV_SYNC_DTYPE = np.dtype([("bit_edge", "<i4"), ("nbits", "<i4"), ("frame_bit", "<i4"), ("inverted", "<i4"),
                           ("nwords", "<i4"), ("words_ok", "<i4"), ("subframes", "<i4"), ("first_tow", "<i4")])
assert NAV_BIT_DTYPE.itemsize == 24 and NAV_WORD_DTYPE.itemsize == 32 and NAV_SYNC_DTYPE.itemsize == 32


def vtrack_config(**kw):
    """gpsb200_vtrack_config_default with the fields of kw replaced. -> VTRACK_CONFIG_DTYPE record."""
    c = np.zeros(1, VTRACK_CONFIG_DTYPE)
    lib().gpsb200_vtrack_config_default(c.ctypes.data)
    for k, v in kw.items():
        c[0][k] = v
    return c[0]


def vtrack_seed(cfg, x8, t_rx, s0, prns):
    """gpsb200_vtrack_seed: the state of a run from X = (x, y, z, vx, vy, vz, b, d) at stream sample s0 whose true
    receive time is t_rx (s of week), one channel per PRN. -> VTRACK_STATE_DTYPE record."""
    st = np.zeros(1, VTRACK_STATE_DTYPE)
    cf = np.array(cfg, dtype=VTRACK_CONFIG_DTYPE).reshape(1)
    x = np.ascontiguousarray(x8, np.float64)
    p = np.ascontiguousarray(prns, np.int32)
    rc = lib().gpsb200_vtrack_seed(cf.ctypes.data, x.ctypes.data, float(t_rx), int(s0), p.ctypes.data, p.size,
                                   st.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_vtrack_seed")
    return st[0]


def track_start(prn, doppler_hz, sample):
    """gpsb200_track_start: the tracking state of a channel from an acquisition (prn, Doppler, the sample where the
    code's chip 0 starts: s0 + delay). -> TRACK_STATE_DTYPE record."""
    st = np.zeros(1, TRACK_STATE_DTYPE)
    rc = lib().gpsb200_track_start(int(prn), float(doppler_hz), int(sample), st.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_track_start(%d, %r, %d)" % (prn, doppler_hz, sample))
    return st[0]


def nav_decode(epochs):
    """gpsb200_nav_decode: bit sync, frame sync and words from the epochs of one channel (TRACK_EPOCH_DTYPE, time order).
    -> (bits NAV_BIT_DTYPE[], words NAV_WORD_DTYPE[], sync NAV_SYNC_DTYPE record)."""
    e = np.ascontiguousarray(epochs, dtype=TRACK_EPOCH_DTYPE)
    n = e.size
    bits = np.zeros(max(1, n // 20), NAV_BIT_DTYPE)
    words = np.zeros(max(1, n // 600), NAV_WORD_DTYPE)
    sync = np.zeros(1, NAV_SYNC_DTYPE)
    rc = lib().gpsb200_nav_decode(e.ctypes.data if n else None, n, bits.ctypes.data, bits.size, words.ctypes.data,
                                  words.size, sync.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_nav_decode")
    s = sync[0]
    return bits[:max(0, int(s["nbits"]))], words[:max(0, int(s["nwords"]))], s


def nav_word_check(word, prev):
    """gpsb200_nav_word_check: (parity ok, 24 data bits with D30* undone) of a received 30-bit word after `prev`."""
    d = C.c_uint32(0)
    ok = lib().gpsb200_nav_word_check(int(word) & 0x3FFFFFFF, int(prev) & 0x3FFFFFFF, C.byref(d))
    return bool(ok), int(d.value)


def nav_parity(data24, d29, d30):
    """gpsb200_nav_parity: the 6 IS-GPS-200 parity bits of 24 data bits after D29*, D30*."""
    return int(lib().gpsb200_nav_parity(int(data24) & 0xFFFFFF, int(d29), int(d30)))


# gpsb200_ephemeris_t / gpsb200_iono_t / gpsb200_pvt_chan_t / gpsb200_pvt_config_t / gpsb200_fix_t (DESIGN §11)
EPHEMERIS_DTYPE = np.dtype([("valid", "<i4"), ("week", "<i4"), ("iodc", "<i4"), ("iode", "<i4"), ("health", "<i4"),
                            ("ura", "<i4"), ("reserved", "<i4", 2), ("toc", "<f8"), ("af0", "<f8"), ("af1", "<f8"),
                            ("af2", "<f8"), ("tgd", "<f8"), ("toe", "<f8"), ("m0", "<f8"), ("deltan", "<f8"), ("ecc", "<f8"),
                            ("sqrta", "<f8"), ("omg0", "<f8"), ("inc0", "<f8"), ("aop", "<f8"), ("omgdot", "<f8"),
                            ("idot", "<f8"), ("cuc", "<f8"), ("cus", "<f8"), ("crc", "<f8"), ("crs", "<f8"), ("cic", "<f8"),
                            ("cis", "<f8")])
IONO_DTYPE = np.dtype([("valid", "<i4"), ("reserved", "<i4"), ("alpha", "<f8", 4), ("beta", "<f8", 4)])
PVT_CHAN_DTYPE = np.dtype([("eph", EPHEMERIS_DTYPE), ("prn", "<i4"), ("anchor_epoch", "<i4"), ("anchor_ms", "<i8")])
PVT_CONFIG_DTYPE = np.dtype([("s0", "<i8"), ("step", "<i8"), ("nfix", "<i4"), ("iono", "<i4"), ("alpha", "<f8", 4),
                             ("beta", "<f8", 4)])
FIX_DTYPE = np.dtype([("sample", "<i8"), ("status", "<i4"), ("nused", "<i4"), ("mask", "<u4"), ("iterations", "<i4"),
                      ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("clock_m", "<f8"), ("t_rx", "<f8"), ("vx", "<f8"),
                      ("vy", "<f8"), ("vz", "<f8"), ("drift", "<f8"), ("lat_deg", "<f8"), ("lon_deg", "<f8"),
                      ("height", "<f8"), ("pdop", "<f8"), ("rms", "<f8")])
assert (EPHEMERIS_DTYPE.itemsize, IONO_DTYPE.itemsize, PVT_CHAN_DTYPE.itemsize, PVT_CONFIG_DTYPE.itemsize,
        FIX_DTYPE.itemsize) == (200, 72, 216, 88, 136)
FIX_OK, FIX_FEW, FIX_NO_CONVERGENCE = 0, 1, 2
VTRACK_CONFIG_DTYPE = np.dtype([("periods", "<i4"), ("reserved", "<i4"), ("sigma_code_m", "<f8"),
                                ("sigma_rate_mps", "<f8"), ("q_min", "<f8"), ("accel_psd", "<f8"), ("bias_psd", "<f8"),
                                ("drift_psd", "<f8"), ("sigma_pos", "<f8"), ("sigma_vel", "<f8"), ("sigma_bias", "<f8"),
                                ("sigma_drift", "<f8")])
VTRACK_CHAN_STATE_DTYPE = np.dtype([("nco", TRACK_STATE_DTYPE), ("start", "<i8"), ("e", "<i8"), ("l", "<i8"),
                                    ("p", "<i8"), ("s", "<i8"), ("dot", "<i8"), ("cross", "<i8"), ("k", "<i4"),
                                    ("used", "<i4")])
VTRACK_STATE_DTYPE = np.dtype([("s0", "<i8"), ("t0", "<f8"), ("nchan", "<i4"), ("seeded", "<i4"), ("updates", "<i4"),
                               ("reserved", "<i4"), ("t_f", "<i8"), ("x", "<f8", 8), ("P", "<f8", (8, 8)),
                               ("ch", VTRACK_CHAN_STATE_DTYPE, 32)])
VTRACK_CHAN_DTYPE = np.dtype([("sample", "<i8"), ("e", "<i8"), ("l", "<i8"), ("p", "<i8"), ("s", "<i8"),
                              ("dot", "<i8"), ("cross", "<i8"), ("prn", "<i4"), ("used", "<i4"), ("code_step", "<u4"),
                              ("carr_step", "<i4"), ("q", "<f8"), ("code_res_m", "<f8"), ("rate_res_mps", "<f8"),
                              ("sigma_code_m", "<f8"), ("sigma_rate_mps", "<f8")])
assert (VTRACK_CONFIG_DTYPE.itemsize, VTRACK_CHAN_STATE_DTYPE.itemsize, VTRACK_STATE_DTYPE.itemsize,
        VTRACK_CHAN_DTYPE.itemsize) == (88, 128, 4712, 112)
PVT_MAX_ITER = 12

# gpsb200_raim_config_t / gpsb200_raim_t (DESIGN §11.1)
RAIM_CONFIG_DTYPE = np.dtype([("sigma", "<f8"), ("p_fa", "<f8"), ("p_md", "<f8"), ("max_exclude", "<i4"),
                              ("reserved", "<i4")])
RAIM_DTYPE = np.dtype([("verdict", "<i4"), ("excluded", "<u4"), ("dof", "<i4"), ("reserved", "<i4"), ("stat", "<f8"),
                       ("threshold", "<f8"), ("hpl", "<f8"), ("vpl", "<f8")])
assert (RAIM_CONFIG_DTYPE.itemsize, RAIM_DTYPE.itemsize) == (32, 48)
RAIM_PASS, RAIM_EXCLUDED, RAIM_ALERT, RAIM_UNAVAILABLE = 0, 1, 2, 3
RAIM_MAX_DOF = 28
RAIM_MAX_EXCLUDE = 4


def raim_config(sigma, p_fa=1e-5, p_md=1e-3, max_exclude=1):
    """A RAIM_CONFIG_DTYPE record: pseudorange sigma (m), false-alarm and missed-detection probabilities, and how many
    channels a fix may exclude (0: detection only)."""
    c = np.zeros(1, RAIM_CONFIG_DTYPE)[0]
    c["sigma"], c["p_fa"], c["p_md"], c["max_exclude"] = float(sigma), float(p_fa), float(p_md), int(max_exclude)
    return c


# gpsb200_araim_config_t / gpsb200_araim_t (DESIGN §11.2)
ARAIM_CONFIG_DTYPE = np.dtype([("mask_deg", "<f8"), ("sigma_ura", "<f8"), ("sigma_ure", "<f8"), ("sigma_noise", "<f8"),
                               ("b_nom", "<f8"), ("p_sat", "<f8"), ("p_hmi_vert", "<f8"), ("p_hmi_horz", "<f8"),
                               ("p_fa_vert", "<f8"), ("p_fa_horz", "<f8"), ("max_exclude", "<i4"),
                               ("reserved", "<i4", (3,))])
ARAIM_DTYPE = np.dtype([("verdict", "<i4"), ("excluded", "<u4"), ("masked", "<u4"), ("n", "<i4"),
                        ("test_ratio", "<f8"), ("hpl", "<f8"), ("vpl", "<f8"), ("emt", "<f8"), ("sigma_acc_v", "<f8"),
                        ("p_nm", "<f8")])
assert (ARAIM_CONFIG_DTYPE.itemsize, ARAIM_DTYPE.itemsize) == (96, 64)


def araim_config(mask_deg=5.0, sigma_ura=1.0, sigma_ure=2.0 / 3.0, sigma_noise=0.36, b_nom=0.75, p_sat=1e-5,
                 p_hmi_vert=9.8e-8, p_hmi_horz=2e-9, p_fa_vert=3.9e-6, p_fa_horz=9e-8, max_exclude=1):
    """An ARAIM_CONFIG_DTYPE record; the defaults are the header's (LPV-200 allocations)."""
    c = np.zeros(1, ARAIM_CONFIG_DTYPE)[0]
    for k, v in (("mask_deg", mask_deg), ("sigma_ura", sigma_ura), ("sigma_ure", sigma_ure),
                 ("sigma_noise", sigma_noise), ("b_nom", b_nom), ("p_sat", p_sat), ("p_hmi_vert", p_hmi_vert),
                 ("p_hmi_horz", p_hmi_horz), ("p_fa_vert", p_fa_vert), ("p_fa_horz", p_fa_horz)):
        c[k] = float(v)
    c["max_exclude"] = int(max_exclude)
    return c


def araim_kfa(p_fa_vert, p_fa_horz):
    """gpsb200_araim_kfa: (K_fa,H[28], K_fa,V[28]) for n = 5..32 channels in the set."""
    kh, kv = np.zeros(RAIM_MAX_DOF), np.zeros(RAIM_MAX_DOF)
    rc = lib().gpsb200_araim_kfa(float(p_fa_vert), float(p_fa_horz), kh.ctypes.data, kv.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_araim_kfa")
    return kh, kv


# gpsb200_coarse_config_t / gpsb200_coarse_t (DESIGN §11.3)
COARSE_CONFIG_DTYPE = np.dtype([("x_a", "<f8", 3), ("t_a", "<f8"), ("s_a", "<i8"), ("week", "<i4"), ("reserved", "<i4")])
COARSE_DTYPE = np.dtype([("delta", "<f8"), ("pdop", "<f8"), ("ref", "<i4"), ("week", "<i4"), ("changed", "<u4"),
                         ("reserved", "<i4")])
assert (COARSE_CONFIG_DTYPE.itemsize, COARSE_DTYPE.itemsize) == (48, 32)
FIX_AMBIGUOUS = 3


def coarse_config(x_a, t_a, s_a=0, week=0):
    """A COARSE_CONFIG_DTYPE record: a-priori ECEF position x_a (m) and GPS time t_a (s of week `week`) at stream sample
    s_a."""
    c = np.zeros(1, COARSE_CONFIG_DTYPE)[0]
    c["x_a"], c["t_a"], c["s_a"], c["week"] = np.asarray(x_a, np.float64), float(t_a), int(s_a), int(week)
    return c


# gpsb200_search_config_t / gpsb200_search_t (DESIGN §11.4)
SEARCH_CONFIG_DTYPE = np.dtype([("t_a", "<f8"), ("s_a", "<i8"), ("week", "<i4"), ("nodes", "<i4"), ("reserved", "<i8")])
SEARCH_DTYPE = np.dtype([("winner", "<i4"), ("searched", "<i4"), ("ok", "<i4"), ("support", "<i4"), ("alt_rms", "<f8"),
                         ("alt_dist", "<f8"), ("delta", "<f8"), ("pdop", "<f8"), ("ref", "<i4"), ("week", "<i4"),
                         ("changed", "<u4"), ("reserved", "<i4")])
assert (SEARCH_CONFIG_DTYPE.itemsize, SEARCH_DTYPE.itemsize) == (32, 64)
SEARCH_NODES = 262144


def search_config(t_a, s_a=0, week=0, nodes=SEARCH_NODES):
    """A SEARCH_CONFIG_DTYPE record: a-priori GPS time t_a (s of week `week`) at stream sample s_a, and the grid's node
    count."""
    c = np.zeros(1, SEARCH_CONFIG_DTYPE)[0]
    c["t_a"], c["s_a"], c["week"], c["nodes"] = float(t_a), int(s_a), int(week), int(nodes)
    return c


# gpsb200_snapshot_config_t / gpsb200_snapshot_t (DESIGN §11.5)
SNAPSHOT_CONFIG_DTYPE = np.dtype([("min_ratio", "<f8"), ("iterations", "<i4"), ("reserved", "<i4")])
SNAPSHOT_DTYPE = np.dtype([("prn", "<i4"), ("status", "<i4"), ("sample", "<i8"), ("code_phase", "<u8"),
                           ("code_step", "<u4"), ("carr_step", "<i4"), ("iterations", "<i4"), ("last_step", "<i4"),
                           ("power", "<u8"), ("ratio", "<f8")])
assert (SNAPSHOT_CONFIG_DTYPE.itemsize, SNAPSHOT_DTYPE.itemsize) == (16, 56)
SNAP_OK, SNAP_WEAK, SNAP_NO_CONVERGENCE = 0, 1, 2
SNAP_ITERATIONS, SNAP_MAX_ITER = 12, 16
SNAP_BATCH_SCRATCH = 256 << 20   # GPSB200_SNAP_BATCH_SCRATCH: the device-scratch cap of a batch pass, bytes


def snapshot_batch_pass(nprn, nbins, ms, sample_size=SC08):
    """The windows of one pass of gpsb200_snapshot_batch (at least one): how many fit the scratch cap, as the header
    states it."""
    b = nprn * nbins * 24028 + nprn * 128 + 8 + acq_window_samples(ms) * 2 * int(sample_size)
    return max(1, SNAP_BATCH_SCRATCH // b)


def snapshot_config(min_ratio=2.5, iterations=SNAP_ITERATIONS):
    """A SNAPSHOT_CONFIG_DTYPE record: the acquisition ratio a PRN needs to be refined, and the code iterations."""
    c = np.zeros(1, SNAPSHOT_CONFIG_DTYPE)[0]
    c["min_ratio"], c["iterations"] = float(min_ratio), int(iterations)
    return c


# gpsb200_collective_config_t / gpsb200_collective_t / gpsb200_cd_score_t / gpsb200_cd_cell_t (DESIGN §11.7)
COLLECTIVE_CONFIG_DTYPE = np.dtype([("n", "<i4", 4), ("step", "<f8", 4), ("mask_deg", "<f8"), ("distinct_m", "<f8"),
                                    ("reserved", "<i8")])
COLLECTIVE_DTYPE = np.dtype([("status", "<i4"), ("nused", "<i4"), ("used", "<u4"), ("shift", "<i4"), ("winner", "<i4"),
                             ("runner", "<i4"), ("score", "<u4"), ("runner_score", "<u4"), ("o_t", "<f8"),
                             ("x", "<f8", 3), ("lat_deg", "<f8"), ("lon_deg", "<f8"), ("height", "<f8"),
                             ("runner_dist", "<f8")])
CD_SCORE_DTYPE = np.dtype([("score", "<u4"), ("shift", "<i4")])
CD_CELL_DTYPE = np.dtype([("bin", "<i4"), ("delay", "<i4")])
assert (COLLECTIVE_CONFIG_DTYPE.itemsize, COLLECTIVE_DTYPE.itemsize) == (72, 96)
CD_OK, CD_FEW, CD_AMBIGUOUS = 0, 1, 2
CD_MAX_HYP, CD_MIN_USED, CD_Q_SHIFT, CD_Q_CAP, CD_AMBIGUOUS_PCT = 1 << 24, 4, 8, 8192, 90


def collective_config(ext_m, step_m, ext_s=0.0, step_s=1.0, up_ext_m=0.0, up_step_m=1.0, mask_deg=5.0,
                      distinct_m=None):
    """A COLLECTIVE_CONFIG_DTYPE record for a lattice of +-ext_m east and north at step_m, +-up_ext_m up at up_step_m
    and +-ext_s in time at step_s: n = 2 floor(ext / step) + 1 points per axis (one where ext is 0). distinct_m
    defaults to two horizontal steps."""
    c = np.zeros(1, COLLECTIVE_CONFIG_DTYPE)[0]
    for a, (e, st) in enumerate(((ext_m, step_m), (ext_m, step_m), (up_ext_m, up_step_m), (ext_s, step_s))):
        c["n"][a] = 2 * int(np.floor(float(e) / float(st) + 1e-9)) + 1 if e > 0 else 1
        c["step"][a] = float(st)
    c["mask_deg"] = float(mask_deg)
    c["distinct_m"] = 2.0 * float(step_m) if distinct_m is None else float(distinct_m)
    return c


def search_nodes(n=SEARCH_NODES):
    """gpsb200_search_nodes: the ECEF positions float64[n, 3] of the n-node search grid."""
    xyz = np.zeros((max(1, int(n)), 3))
    rc = lib().gpsb200_search_nodes(int(n), xyz.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_search_nodes")
    return xyz


def rinex_ephemeris(path, week, sow, rinex3=False):
    """gpsb200_rinex_ephemeris: EPHEMERIS_DTYPE[32], entry prn - 1 the PRN's record of the RINEX navigation file whose
    toe is nearest to GPS time (week, sow), within 2 h (valid 0 where there is none)."""
    eph = np.zeros(32, EPHEMERIS_DTYPE)
    rc = lib().gpsb200_rinex_ephemeris(os.fsencode(str(path)), int(bool(rinex3)), int(week), float(sow), eph.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_rinex_ephemeris")
    return eph


def raim_thresholds(p_fa, p_md):
    """gpsb200_raim_thresholds: (T[28], lambda[28]) for dof 1..28; T[d - 1] is the chi^2(d) value with upper tail p_fa,
    lambda[d - 1] the noncentrality whose noncentral chi^2(d) CDF at T[d - 1] is p_md."""
    T, lam = np.zeros(RAIM_MAX_DOF), np.zeros(RAIM_MAX_DOF)
    rc = lib().gpsb200_raim_thresholds(float(p_fa), float(p_md), T.ctypes.data, lam.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_raim_thresholds")
    return T, lam


def nav_words_of_frame(words60):
    """The 60 NAV words of a frame slot as the scenario sends them (bits 29..0 used) -> NAV_WORD_DTYPE[60] records with
    index 0..59, the parity verdict and data of gpsb200_nav_word_check, subframe id and TOW on HOW words (index % 10 == 1):
    what gpsb200_nav_decode would return for a receiver that read the frame (sample = 0)."""
    w = np.asarray(words60, np.uint32) & 0x3FFFFFFF
    out = np.zeros(w.size, NAV_WORD_DTYPE)
    prev = 0
    for i, raw in enumerate(w):
        ok, data = nav_word_check(int(raw), prev)
        out[i]["raw"], out[i]["data"], out[i]["parity_ok"], out[i]["index"] = int(raw), data, int(ok), i
        out[i]["subframe"], out[i]["tow"] = ((data >> 2) & 7, (data >> 7) & 0x1FFFF) if i % 10 == 1 else (0, -1)
        prev = int(raw)
    return out


def nav_ephemeris(words):
    """gpsb200_nav_ephemeris: the ephemeris of the last complete, consistent subframe 1-3 set and the Klobuchar terms of
    the last subframe 4 page 18 in the word records (NAV_WORD_DTYPE, in order). -> (EPHEMERIS_DTYPE record, IONO_DTYPE
    record); check their `valid`."""
    w = np.ascontiguousarray(words, dtype=NAV_WORD_DTYPE)
    eph, iono = np.zeros(1, EPHEMERIS_DTYPE), np.zeros(1, IONO_DTYPE)
    rc = lib().gpsb200_nav_ephemeris(w.ctypes.data if w.size else None, w.size, eph.ctypes.data, iono.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_nav_ephemeris")
    return eph[0], iono[0]


def nav_almanac(words, week):
    """gpsb200_nav_almanac: the almanac of the subframe 4 / 5 pages in the word records (NAV_WORD_DTYPE, in order), WNa
    resolved to the full week within -128..127 of `week`. -> (ALMANAC_RECORD_DTYPE[32] indexed by svid - 1, WNa or -1)."""
    w = np.ascontiguousarray(words, dtype=NAV_WORD_DTYPE)
    rec = np.zeros(32, ALMANAC_RECORD_DTYPE)
    wna = C.c_int32(0)
    rc = lib().gpsb200_nav_almanac(w.ctypes.data if w.size else None, w.size, int(week), rec.ctypes.data, C.byref(wna))
    if rc:
        raise GpsB200Error(rc, "gpsb200_nav_almanac")
    return rec, int(wna.value)


# gpsb200_sky_t: one row per PRN 1..32
SKY_DTYPE = np.dtype([("prn", "<i4"), ("valid", "<i4"), ("el_deg", "<f8"), ("az_deg", "<f8"), ("range_m", "<f8"),
                      ("doppler_hz", "<f8")])
assert SKY_DTYPE.itemsize == 40


def almanac_predict(rec, week, sow, x_a):
    """gpsb200_almanac_predict: elevation, azimuth, range and the Doppler the acquisition peaks at of every almanac
    record (ALMANAC_RECORD_DTYPE[32], e.g. from nav_almanac or almanac_read) at GPS time (week, sow) for a static
    receiver at ECEF x_a (m). -> SKY_DTYPE[32]; rows with valid 0 were not predicted."""
    r = np.ascontiguousarray(rec, dtype=ALMANAC_RECORD_DTYPE)
    assert r.size == 32
    x = np.ascontiguousarray(x_a, dtype=np.float64).reshape(3)
    out = np.zeros(32, SKY_DTYPE)
    rc = lib().gpsb200_almanac_predict(r.ctypes.data, int(week), float(sow), x.ctypes.data, out.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_almanac_predict")
    return out


def nav_time_anchor(words, sync):
    """gpsb200_nav_time_anchor: (anchor_epoch, anchor_ms) of a tracked channel from the words and sync nav_decode
    returned for its epochs; anchor_epoch is -1 when no HOW passed parity."""
    w = np.ascontiguousarray(words, dtype=NAV_WORD_DTYPE)
    sy = np.array(sync, dtype=NAV_SYNC_DTYPE).reshape(1)
    ep, ms = C.c_int32(0), C.c_int64(0)
    rc = lib().gpsb200_nav_time_anchor(w.ctypes.data if w.size else None, w.size, sy.ctypes.data, C.byref(ep), C.byref(ms))
    if rc:
        raise GpsB200Error(rc, "gpsb200_nav_time_anchor")
    return int(ep.value), int(ms.value)


def pvt_config(s0, step, nfix, iono=None):
    """A PVT_CONFIG_DTYPE record: fixes at samples s0 + i step, i < nfix; iono: (alpha[4], beta[4]) to apply the
    Klobuchar delay with, or None for none."""
    c = np.zeros(1, PVT_CONFIG_DTYPE)[0]
    c["s0"], c["step"], c["nfix"] = int(s0), int(step), int(nfix)
    if iono is not None:
        c["iono"] = 1
        c["alpha"], c["beta"] = np.asarray(iono[0], np.float64), np.asarray(iono[1], np.float64)
    return c


HANDOFF_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_double))     # gpsb200_handoff_fn

_lib = None

EXPORTS = ["gpsb200_create", "gpsb200_destroy", "gpsb200_last_error", "gpsb200_version", "gpsb200_set_nav",
           "gpsb200_synth_blocks", "gpsb200_synth_blocks_scatter", "gpsb200_synth_blocks_device", "gpsb200_replay_device",
           "gpsb200_carrier_advance", "gpsb200_carrier_chain", "gpsb200_carrier_chain_device", "gpsb200_carrier_probe_fixup",
           "gpsb200_codegen", "gpsb200_acquire", "gpsb200_acquire_device", "gpsb200_acquire_windows",
           "gpsb200_acquire_windows_device", "gpsb200_debug_acq_split", "gpsb200_nav_almanac", "gpsb200_almanac_predict", "gpsb200_track_start",
           "gpsb200_track",
           "gpsb200_track_device", "gpsb200_nav_decode", "gpsb200_nav_word_check", "gpsb200_nav_parity",
           "gpsb200_nav_ephemeris", "gpsb200_nav_time_anchor", "gpsb200_pvt", "gpsb200_pvt_replay",
           "gpsb200_pvt_raim", "gpsb200_raim_thresholds", "gpsb200_pvt_araim", "gpsb200_araim_kfa", "gpsb200_pvt_coarse", "gpsb200_pvt_search", "gpsb200_search_nodes", "gpsb200_snapshot_measure", "gpsb200_snapshot_measure_device", "gpsb200_snapshot_batch", "gpsb200_snapshot_batch_device", "gpsb200_pvt_snapshot", "gpsb200_pvt_snapshot_search", "gpsb200_collective", "gpsb200_collective_device", "gpsb200_vtrack_config_default", "gpsb200_vtrack_seed", "gpsb200_vtrack", "gpsb200_vtrack_device", "gpsb200_debug_vtrack_cluster", "gpsb200_rinex_ephemeris", "gpsb200_bind_numa", "gpsb200_span_chain_host", "gpsb200_lanes_model_block",
           "gpsb200_lanes_window_band_host", "gpsb200_slice_prepare", "gpsb200_slice_probe",
           "gpsb200_slice_finish", "gpsb200_slice_finish_cb", "gpsb200_slice_wait", "gpsb200_link_apply", "gpsb200_slice_link_host", "gpsb200_debug_corrupt_chain", "gpsb200_synth_kernel_name",
           "gpsb200_debug_run_checkpoints", "gpsb200_checkpoint_segments_host",
           "gpsb200_carrier_probe_host", "gpsb200_debug_block_probes", "gpsb200_debug_synth_shape",
           "gpsb200_scenario_create", "gpsb200_scenario_destroy", "gpsb200_scenario_error",
           "gpsb200_scenario_blocks", "gpsb200_scenario_channels", "gpsb200_scenario_nav_frames",
           "gpsb200_scenario_chans", "gpsb200_scenario_nav", "gpsb200_scenario_almanac_date", "gpsb200_almanac_read",
           "gpsb200_scenario_open", "gpsb200_scenario_advance", "gpsb200_scenario_frame", "gpsb200_scenario_key",
           "gpsb200_scenario_steer_state", "gpsb200_scenario_open_now", "gpsb200_scenario_create_now",
           "gpsb200_scenario_start_date", "gpsb200_scenario_start_time",
           "fifo_create", "fifo_destroy", "fifo_wait_next", "fifo_wait_full", "fifo_halt", "fifo_acquire",
           "fifo_enqueue", "fifo_dequeue", "fifo_release", "fifo_set_compat_drop",
           "gpsb200_iqfile_start", "gpsb200_iqfile_stop", "gpsb200_fifo_push", "gpsb200_fifo_push_flush"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(lib_path()):
            raise GpsB200Error(-2, "libgpsb200.so not built (run __graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(lib_path())
        L.gpsb200_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
        L.gpsb200_destroy.argtypes = [C.c_void_p]
        L.gpsb200_last_error.argtypes = [C.c_void_p]
        L.gpsb200_last_error.restype = C.c_char_p
        L.gpsb200_version.restype = C.c_char_p
        L.gpsb200_set_nav.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.gpsb200_synth_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                           C.c_void_p, C.POINTER(Stats)]
        L.gpsb200_synth_blocks_scatter.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                   C.c_void_p, C.POINTER(Stats)]
        L.gpsb200_synth_blocks_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.POINTER(Stats)]
        L.gpsb200_replay_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.gpsb200_carrier_advance.argtypes = [C.c_double, C.c_double, C.c_int64]
        L.gpsb200_carrier_advance.restype = C.c_double
        L.gpsb200_codegen.argtypes = [C.c_int, C.c_void_p]
        L.gpsb200_scenario_create.argtypes = [C.POINTER(ScenarioConfig), C.POINTER(C.c_void_p)]
        L.gpsb200_scenario_destroy.argtypes = [C.c_void_p]
        L.gpsb200_scenario_error.argtypes = [C.c_void_p]
        L.gpsb200_scenario_error.restype = C.c_char_p
        for fn in ("blocks", "channels", "nav_frames"):
            getattr(L, "gpsb200_scenario_" + fn).argtypes = [C.c_void_p]
        L.gpsb200_scenario_chans.argtypes = [C.c_void_p]
        L.gpsb200_scenario_chans.restype = C.c_void_p
        L.gpsb200_scenario_nav.argtypes = [C.c_void_p]
        L.gpsb200_scenario_nav.restype = C.c_void_p
        L.gpsb200_scenario_almanac_date.argtypes = [C.c_void_p]
        L.gpsb200_scenario_almanac_date.restype = C.c_char_p
        L.gpsb200_almanac_read.argtypes = [C.c_char_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.gpsb200_scenario_open.argtypes = [C.POINTER(ScenarioConfig), C.POINTER(C.c_void_p)]
        L.gpsb200_scenario_open_now.argtypes = [C.POINTER(ScenarioConfig), C.POINTER(C.c_void_p)]
        L.gpsb200_scenario_create_now.argtypes = [C.POINTER(ScenarioConfig), C.POINTER(C.c_void_p)]
        L.gpsb200_scenario_start_date.argtypes = [C.c_void_p]
        L.gpsb200_scenario_start_date.restype = C.c_char_p
        L.gpsb200_scenario_start_time.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_double)]
        L.gpsb200_scenario_advance.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_int32)]
        L.gpsb200_scenario_frame.argtypes = [C.c_void_p, C.c_int]
        L.gpsb200_scenario_frame.restype = C.c_void_p
        L.gpsb200_scenario_key.argtypes = [C.c_void_p, C.c_int]
        L.gpsb200_scenario_steer_state.argtypes = [C.c_void_p, C.POINTER(SteerState)]
        L.gpsb200_carrier_probe_fixup.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int64, C.POINTER(C.c_double)]
        L.gpsb200_carrier_chain_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.gpsb200_carrier_chain.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        L.gpsb200_span_chain_host.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p]
        L.gpsb200_slice_prepare.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.POINTER(SliceLink)]
        L.gpsb200_slice_finish_cb.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Stats),
                                              HANDOFF_FN, C.c_void_p]
        L.gpsb200_slice_wait.argtypes = [C.c_void_p]
        L.gpsb200_slice_link_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(SliceLink)]
        L.gpsb200_slice_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.gpsb200_slice_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Stats)]
        L.gpsb200_link_apply.argtypes = [C.POINTER(SliceLink), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_debug_corrupt_chain.argtypes = [C.c_void_p, C.c_int]
        L.gpsb200_debug_run_checkpoints.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.gpsb200_checkpoint_segments_host.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int, C.c_void_p,
                                                       C.POINTER(C.c_int)]
        L.gpsb200_carrier_probe_host.argtypes = [C.c_double, C.c_double, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                                 C.c_void_p]
        L.gpsb200_debug_block_probes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_debug_synth_shape.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p),
                                                C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.gpsb200_synth_kernel_name.argtypes = [C.c_void_p, C.c_int]
        L.gpsb200_synth_kernel_name.restype = C.c_char_p
        L.gpsb200_acquire.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig), C.c_void_p,
                                      C.c_void_p]
        L.gpsb200_acquire_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig),
                                             C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_acquire_windows.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig),
                                              C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_acquire_windows_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig),
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_debug_acq_split.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.gpsb200_nav_almanac.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]
        L.gpsb200_almanac_predict.argtypes = [C.c_void_p, C.c_int32, C.c_double, C.c_void_p, C.c_void_p]
        L.gpsb200_track_start.argtypes = [C.c_int, C.c_double, C.c_int64, C.c_void_p]
        L.gpsb200_track.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int,
                                    C.c_void_p, C.c_void_p]
        L.gpsb200_track_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_nav_decode.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        L.gpsb200_nav_word_check.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.gpsb200_nav_parity.argtypes = [C.c_uint32, C.c_int, C.c_int]
        L.gpsb200_nav_parity.restype = C.c_uint32
        L.gpsb200_nav_ephemeris.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.gpsb200_nav_time_anchor.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int64)]
        L.gpsb200_pvt.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p]
        L.gpsb200_pvt_replay.argtypes = [C.c_void_p, C.c_void_p]
        L.gpsb200_pvt_raim.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_raim_thresholds.argtypes = [C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.gpsb200_pvt_araim.argtypes = L.gpsb200_pvt_raim.argtypes
        L.gpsb200_araim_kfa.argtypes = [C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.gpsb200_pvt_coarse.argtypes = L.gpsb200_pvt_raim.argtypes + [C.c_void_p]
        L.gpsb200_pvt_search.argtypes = L.gpsb200_pvt_coarse.argtypes + [C.c_void_p]
        L.gpsb200_search_nodes.argtypes = [C.c_int, C.c_void_p]
        L.gpsb200_snapshot_measure.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig),
                                               C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_snapshot_measure_device.argtypes = L.gpsb200_snapshot_measure.argtypes + [C.c_void_p]
        L.gpsb200_snapshot_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig), C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_snapshot_batch_device.argtypes = L.gpsb200_snapshot_batch.argtypes + [C.c_void_p]
        L.gpsb200_pvt_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gpsb200_pvt_snapshot_search.argtypes = L.gpsb200_pvt_snapshot.argtypes + [C.c_void_p]
        L.gpsb200_collective.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(AcqConfig), C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
        L.gpsb200_collective_device.argtypes = L.gpsb200_collective.argtypes + [C.c_void_p]
        L.gpsb200_vtrack_config_default.argtypes = [C.c_void_p]
        L.gpsb200_vtrack_config_default.restype = None
        L.gpsb200_vtrack_seed.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
        L.gpsb200_vtrack.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_void_p]
        L.gpsb200_vtrack_device.argtypes = L.gpsb200_vtrack.argtypes + [C.c_void_p]
        L.gpsb200_debug_vtrack_cluster.argtypes = [C.c_void_p, C.c_int]
        L.gpsb200_rinex_ephemeris.argtypes = [C.c_char_p, C.c_int, C.c_int32, C.c_double, C.c_void_p]
        _lib = L
    return _lib


def bind_numa(device=0):
    """gpsb200_bind_numa: pin the calling thread (and threads created later) to the GPU's NUMA node. -> node or -1."""
    L = lib()
    L.gpsb200_bind_numa.argtypes = [C.c_int]
    L.gpsb200_bind_numa.restype = C.c_int
    return int(L.gpsb200_bind_numa(int(device)))


def codegen(prn):
    ca = np.zeros(1023, np.uint8)
    rc = lib().gpsb200_codegen(prn, ca.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_codegen(%d)" % prn)
    return ca


def carrier_advance(phase, f_carr, nsamples):
    return lib().gpsb200_carrier_advance(float(phase), float(f_carr), int(nsamples))


def carrier_chain(chans, phase_in=None, threads=16):
    """Exact carrier phase of every slot after all blocks of chans[nblk, nchan] (host only)."""
    a = np.ascontiguousarray(chans, dtype=CHAN_DTYPE)
    nblk, nchan = a.shape
    out = np.zeros(nchan, np.float64)
    pin = None if phase_in is None else np.ascontiguousarray(phase_in, dtype=np.float64)
    rc = lib().gpsb200_carrier_chain(a.ctypes.data, nblk, nchan, None if pin is None else pin.ctypes.data,
                                     out.ctypes.data, threads)
    if rc:
        raise GpsB200Error(rc, "gpsb200_carrier_chain")
    return out


def lanes_model_block(chans_row, nav_frame, run_samples=2400, force=0, want_signs=False):
    """Host model of the lane = sample kernel for one block. chans_row: CHAN_DTYPE[nchan]; nav_frame: uint32[nchan, 60].
    -> (iq int16[600000], carr_out float64[nchan], counters int64[4]), and with want_signs the sign words of every window
    (uint32[nchan, 3125, 3]; word j, bit 11 (i % 3) + i // 3: chip XOR data bit of sample 32 j + i of the window)"""
    a = np.ascontiguousarray(chans_row, dtype=CHAN_DTYPE)
    nv = np.ascontiguousarray(nav_frame, dtype=np.uint32)
    iq = np.zeros(BLOCK_ELEMS, np.int16)
    co = np.zeros(a.size, np.float64)
    cnt = np.zeros(4, np.int64)
    signs = np.zeros((a.size, BLOCK_SAMPLES // 96, 3), np.uint32) if want_signs else None
    L = lib()
    L.gpsb200_lanes_model_block.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
    rc = L.gpsb200_lanes_model_block(a.ctypes.data, a.size, nv.ctypes.data, run_samples, force, iq.ctypes.data, co.ctypes.data,
                                     cnt.ctypes.data, None if signs is None else signs.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_lanes_model_block")
    return (iq, co, cnt, signs) if want_signs else (iq, co, cnt)


def lanes_window_band(steps, bases):
    """Window band certification of the lane = sample kernel for (step, base) pairs of uint32. -> bool array: some
    sample m < 96 of the window has a phase base + m * step whose low 23 bits are 2^23 - 128 or more."""
    st, bs = np.broadcast_arrays(np.asarray(steps, np.uint32), np.asarray(bases, np.uint32))
    st = np.ascontiguousarray(st.ravel())
    bs = np.ascontiguousarray(bs.ravel())
    out = np.zeros(st.size, np.uint8)
    L = lib()
    L.gpsb200_lanes_window_band_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    rc = L.gpsb200_lanes_window_band_host(st.ctypes.data, bs.ctypes.data, st.size, out.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_lanes_window_band_host")
    return out.astype(bool)


def span_chain_host(f_carr, start_true, start_guess):
    """Host model of the two-level chain for one span. -> float64[nblk + 1] exact block starts + end, or None if
    the span-level speculation was rejected."""
    f = np.ascontiguousarray(f_carr, dtype=np.float64)
    out = np.zeros(f.size + 1)
    rc = lib().gpsb200_span_chain_host(f.ctypes.data, f.size, float(start_true), float(start_guess), out.ctypes.data)
    if rc < 0:
        raise GpsB200Error(rc, "gpsb200_span_chain_host")
    return out if rc == 1 else None


def checkpoint_segments_host(start_true, start_guess, f_carr, run_samples=2400):
    """Host model of how the run-checkpoint kernel starts the checkpoint segments of one block.
    -> (accepted, starts float64[J]): starts[0] = start_true, derived start phases of the later segments (NaN for
    those walked from the block start; all NaN when the fix-up rejected the probe)."""
    out = np.zeros(8)
    nseg = C.c_int(0)
    rc = lib().gpsb200_checkpoint_segments_host(float(start_true), float(start_guess), float(f_carr), int(run_samples),
                                            out.ctypes.data, C.byref(nseg))
    if rc < 0:
        raise GpsB200Error(rc, "gpsb200_checkpoint_segments_host")
    return rc == 1, out[:nseg.value]


def carrier_probe_host(guess, f_carr, nsamples=BLOCK_SAMPLES, run_samples=2400, mode=1):
    """Host model of one carrier block probe (mode 0: each parity variant on its own, 1: both in lockstep).
    -> (probe CARRIER_PROBE_DTYPE scalar record, seg float64[2, 7] with NaN where no state is recorded)"""
    probe = np.zeros(1, CARRIER_PROBE_DTYPE)
    seg = np.zeros((2, 7))
    rc = lib().gpsb200_carrier_probe_host(float(guess), float(f_carr), int(nsamples), int(run_samples), int(mode),
                                          probe.ctypes.data, seg.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_carrier_probe_host")
    return probe[0], seg


def slice_link_host(chans):
    """gpsb200_slice_link_host: the closed-form link of a slice (host only). -> SliceLink"""
    a = np.ascontiguousarray(chans, dtype=CHAN_DTYPE)
    link = SliceLink()
    rc = lib().gpsb200_slice_link_host(a.ctypes.data, a.shape[0], a.shape[1], C.byref(link))
    if rc:
        raise GpsB200Error(rc, "gpsb200_slice_link_host")
    return link


def link_apply(link, nchan, prn_in=None, phase_in=None):
    """gpsb200_link_apply -> (prn_out int32[nchan], phase_out float64[nchan])."""
    pi = None if prn_in is None else np.ascontiguousarray(prn_in, dtype=np.int32)
    xi = None if phase_in is None else np.ascontiguousarray(phase_in, dtype=np.float64)
    po, xo = np.zeros(nchan, np.int32), np.zeros(nchan, np.float64)
    rc = lib().gpsb200_link_apply(C.byref(link), nchan, None if pi is None else pi.ctypes.data,
                                  None if xi is None else xi.ctypes.data, po.ctypes.data, xo.ctypes.data)
    if rc:
        raise GpsB200Error(rc, "gpsb200_link_apply")
    return po, xo


def almanac_read(path):
    """gpsb200_almanac_read: parse a SEM almanac file as the scenario engine does.
    -> (valid, records ALMANAC_RECORD_DTYPE[32] indexed by PRN - 1)"""
    rec = np.zeros(32, ALMANAC_RECORD_DTYPE)
    valid = C.c_int32(0)
    rc = lib().gpsb200_almanac_read(os.fsencode(path), rec.ctypes.data, C.byref(valid))
    if rc:
        raise GpsB200Error(rc, "cannot open almanac file %s" % path)
    return bool(valid.value), rec


def _scenario_config(nav_file, lat, lon, height, seconds, max_chan=12, motion_file=None, start=None,
                     ionosphere=True, pluto_gain=False, rinex3=False, target=None, almanac_file=None, interactive=False):
    cfg = ScenarioConfig()
    cfg.nav_file = os.fsencode(nav_file)
    cfg.motion_file = os.fsencode(motion_file) if motion_file else None
    cfg.lat_deg, cfg.lon_deg, cfg.height_m = lat, lon, height
    cfg.duration_ds = int(seconds * 10.0 + 0.5)
    cfg.max_chan = max_chan
    cfg.ionosphere_enable = 1 if ionosphere else 0
    cfg.pluto_gain = 1 if pluto_gain else 0
    cfg.rinex3 = 1 if rinex3 else 0
    cfg.almanac_file = os.fsencode(almanac_file) if almanac_file else None
    cfg.interactive = 1 if interactive else 0
    if target is not None:          # -t distance,bearing,height
        cfg.target_valid = 1
        cfg.target_distance_m, cfg.target_bearing_deg, cfg.target_height_m = [float(v) for v in target]
    if start:
        (cfg.start_year, cfg.start_month, cfg.start_day, cfg.start_hour, cfg.start_min) = [int(v) for v in start[:5]]
        cfg.start_sec = float(start[5])
    return cfg


def scenario(nav_file, lat, lon, height, seconds, max_chan=12, motion_file=None, start=None,
             ionosphere=True, pluto_gain=False, rinex3=False, target=None, almanac_file=None, info=None, steer=None,
             time_overwrite=False):
    """Run the host scenario engine. -> (chans[nblk, max_chan] CHAN_DTYPE, nav[nframes, max_chan, 60] uint32).
    start: (y, m, d, hh, mm, sec) or None for the first ephemeris epoch. almanac_file: SEM almanac to transmit in
    subframes 4 and 5 (None: no almanac, the reference's --disable-almanac). info: optional dict that receives
    "almanac_date" ("yyyy/mm/dd,hh:mm:ss", or None when no valid almanac record was read) and "start_date" (the
    resolved start, "yyyy/mm/dd,hh:mm:ss").
    steer: interactive run, [(block, keys, repeat), ...]: the string `keys`, `repeat` times, before `block` (>= 1);
    built on the incremental engine (LiveScenario). [] is an interactive run without keys.
    time_overwrite: the reference's `-s now` (gpsb200_scenario_create_now): `start` is the clock reading, and the
    ephemeris and UTC reference times of the file are moved to it."""
    kw = dict(max_chan=max_chan, motion_file=motion_file, start=start, ionosphere=ionosphere, pluto_gain=pluto_gain,
              rinex3=rinex3, target=target, almanac_file=almanac_file)
    if steer is not None:
        with LiveScenario(nav_file, lat, lon, height, seconds, interactive=True, time_overwrite=time_overwrite, **kw) as s:
            chans, nav = s.run(steer)
            if info is not None:
                info["almanac_date"] = s.almanac_date
                info["start_date"] = s.start_date
            return chans, nav
    cfg = _scenario_config(nav_file, lat, lon, height, seconds, **kw)
    h = C.c_void_p()
    L = lib()
    create = L.gpsb200_scenario_create_now if time_overwrite else L.gpsb200_scenario_create
    rc = create(C.byref(cfg), C.byref(h))
    try:
        if rc:
            raise GpsB200Error(rc, L.gpsb200_scenario_error(h).decode() if h else "gpsb200_scenario_create")
        nblk, nch, nfr = (L.gpsb200_scenario_blocks(h), L.gpsb200_scenario_channels(h),
                          L.gpsb200_scenario_nav_frames(h))
        chans = np.frombuffer(C.string_at(L.gpsb200_scenario_chans(h), nblk * nch * 64), dtype=CHAN_DTYPE)
        nav = np.frombuffer(C.string_at(L.gpsb200_scenario_nav(h), nfr * nch * 60 * 4), dtype=np.uint32)
        if info is not None:
            d = L.gpsb200_scenario_almanac_date(h)
            info["almanac_date"] = d.decode() if d else None
            info["start_date"] = L.gpsb200_scenario_start_date(h).decode()
        return chans.reshape(nblk, nch).copy(), nav.reshape(nfr, nch, 60).copy()
    finally:
        if h:
            L.gpsb200_scenario_destroy(h)


def parse_steer(text):
    """The `B,KEYS[,REPEAT]` schedule format (one event per line, as gpsb200-sim --steer reads it) -> [(B, KEYS, REPEAT)]."""
    out = []
    for line in text.splitlines():
        line = line.strip()
        if not line or line.startswith("#"):
            continue
        f = line.split(",")
        out.append((int(f[0]), f[1], int(f[2]) if len(f) > 2 else 1))
    return out


class LiveScenario:
    """An opened scenario (gpsb200_scenario_open), advanced block range by block range and steered in between:
    open -> advance(n) / key(k) / frame(f) / state() -> close. time_overwrite: the reference's `-s now`
    (gpsb200_scenario_open_now), `start` being the clock reading."""

    def __init__(self, nav_file, lat, lon, height, seconds, time_overwrite=False, **kw):
        self._h = C.c_void_p()
        cfg = _scenario_config(nav_file, lat, lon, height, seconds, **kw)
        L = lib()
        open_ = L.gpsb200_scenario_open_now if time_overwrite else L.gpsb200_scenario_open
        rc = open_(C.byref(cfg), C.byref(self._h))
        if rc:
            msg = L.gpsb200_scenario_error(self._h).decode() if self._h else "gpsb200_scenario_open"
            self.close()
            raise GpsB200Error(rc, msg)
        self.blocks = L.gpsb200_scenario_blocks(self._h)
        self.channels = L.gpsb200_scenario_channels(self._h)
        d = L.gpsb200_scenario_almanac_date(self._h)
        self.almanac_date = d.decode() if d else None
        self.start_date = L.gpsb200_scenario_start_date(self._h).decode()

    def close(self):
        if self._h:
            lib().gpsb200_scenario_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc):
        if rc:
            raise GpsB200Error(rc, lib().gpsb200_scenario_error(self._h).decode())

    def advance(self, nblk):
        """The next <= nblk blocks -> chans[got, channels] CHAN_DTYPE (nav_frame: global frame number)."""
        out = np.zeros((nblk, self.channels), CHAN_DTYPE)
        got = C.c_int32(0)
        self._check(lib().gpsb200_scenario_advance(self._h, int(nblk), out.ctypes.data, C.byref(got)))
        return out[:got.value]

    def frame(self, f):
        """NAV words uint32[channels, 60] of global frame f (one the last advance referenced)."""
        p = lib().gpsb200_scenario_frame(self._h, int(f))
        if not p:
            raise GpsB200Error(-1, "NAV frame %d is not held (only those of the last advance are)" % f)
        return np.frombuffer(C.string_at(p, self.channels * 60 * 4), dtype=np.uint32).reshape(self.channels, 60).copy()

    def key(self, k):
        """One key ('a', 'd', 'w', 's', 'e', 'q', 't', 'g', 'x'); acts on the next block advance produces."""
        self._check(lib().gpsb200_scenario_key(self._h, ord(k) if isinstance(k, str) else int(k)))

    def state(self):
        st = SteerState()
        self._check(lib().gpsb200_scenario_steer_state(self._h, C.byref(st)))
        return st

    def run(self, steer, chunk=None):
        """Advance to the end of the run, pressing the keys of `steer` [(block, keys, repeat)] before their blocks.
        chunk: largest advance (None: from key block to key block). -> (chans[nblk, C], nav[nframes, C, 60])."""
        events = {}
        for b, keys, rep in steer:
            events[int(b)] = events.get(int(b), "") + keys * int(rep)
        parts, frames = [], {}
        b = 0
        while True:
            if b in events:
                for k in events.pop(b):
                    self.key(k)
            st = self.state()
            if st.next_block >= st.end_block:
                break
            nxt = min([e for e in events if e > b] + [st.end_block])
            n = nxt - b if chunk is None else min(chunk, nxt - b)
            ch = self.advance(n)
            for f in np.unique(ch["nav_frame"]):
                if f not in frames:
                    frames[int(f)] = self.frame(int(f))
            parts.append(ch)
            b += ch.shape[0]
        chans = np.concatenate(parts) if parts else np.zeros((0, self.channels), CHAN_DTYPE)
        nav = np.stack([frames[f] for f in sorted(frames)]) if frames else np.zeros((0, self.channels, 60), np.uint32)
        return chans, nav


class Context:
    """gpsb200_ctx_t. `chans` arguments are numpy arrays of CHAN_DTYPE shaped [nblk, nchan]."""

    def __init__(self, max_chan, max_blocks, device=0, max_nav_frames=1, host_threads=0, run_samples=0):
        self._h = C.c_void_p()
        self.cfg = Config(device, max_chan, max_blocks, max_nav_frames, host_threads, run_samples)
        rc = lib().gpsb200_create(C.byref(self.cfg), C.byref(self._h))
        if rc:
            msg = lib().gpsb200_last_error(self._h).decode() if self._h else "gpsb200_create: bad configuration"
            if self._h:
                lib().gpsb200_destroy(self._h)
                self._h = C.c_void_p()
            raise GpsB200Error(rc, msg)

    def close(self):
        if self._h:
            lib().gpsb200_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc):
        if rc:
            raise GpsB200Error(rc, lib().gpsb200_last_error(self._h).decode())

    def set_nav(self, frame, chan, words):
        w = np.ascontiguousarray(words, dtype=np.uint32)
        assert w.size == 60
        self._check(lib().gpsb200_set_nav(self._h, frame, chan, w.ctypes.data))

    def set_nav_frames(self, frames):
        """frames: uint32[nframes, nchan, 60]."""
        for f in range(frames.shape[0]):
            for c in range(frames.shape[1]):
                self.set_nav(f, c, frames[f, c])

    @staticmethod
    def _chans(chans):
        a = np.ascontiguousarray(chans, dtype=CHAN_DTYPE)
        assert a.ndim == 2
        return a

    def synth_blocks(self, chans, sample_size=SC08, out=None, want_stats=False):
        """Host-destination path (H2D params + kernels + D2H result). Returns (iq, carr_phase_out[, Stats])."""
        a = self._chans(chans)
        nblk, nchan = a.shape
        dt = np.int16 if sample_size == SC16 else np.int8
        if out is None:
            out = np.empty(nblk * BLOCK_ELEMS, dt)
        assert out.dtype == dt and out.size >= nblk * BLOCK_ELEMS and out.flags.c_contiguous
        cp = np.zeros(nchan, np.float64)
        st = Stats()
        self._check(lib().gpsb200_synth_blocks(self._h, a.ctypes.data, nblk, nchan, sample_size,
                                               out.ctypes.data, cp.ctypes.data, C.byref(st)))
        return (out, cp, st) if want_stats else (out, cp)

    def synth_blocks_scatter(self, chans, sample_size, blocks, want_stats=False):
        """Host-destination path, block b into its own host buffer blocks[b] (BLOCK_ELEMS elements).
        Returns carr_phase_out[, Stats]."""
        a = self._chans(chans)
        nblk, nchan = a.shape
        dt = np.int16 if sample_size == SC16 else np.int8
        assert len(blocks) == nblk and all(b.dtype == dt and b.size >= BLOCK_ELEMS and b.flags.c_contiguous for b in blocks)
        ptrs = (C.c_void_p * nblk)(*[b.ctypes.data for b in blocks])
        cp = np.zeros(nchan, np.float64)
        st = Stats()
        self._check(lib().gpsb200_synth_blocks_scatter(self._h, a.ctypes.data, nblk, nchan, sample_size,
                                                       C.cast(ptrs, C.c_void_p), cp.ctypes.data, C.byref(st)))
        return (cp, st) if want_stats else cp

    def synth_blocks_device(self, chans, sample_size, dst_ptr, stream=0, want_stats=False):
        """Device-destination path: dst_ptr is a raw device pointer (e.g. torch tensor .data_ptr())."""
        a = self._chans(chans)
        nblk, nchan = a.shape
        cp = np.zeros(nchan, np.float64)
        st = Stats()
        self._check(lib().gpsb200_synth_blocks_device(self._h, a.ctypes.data, nblk, nchan, sample_size,
                                                      C.c_void_p(dst_ptr), C.c_void_p(stream), cp.ctypes.data,
                                                      C.byref(st) if want_stats else None))
        return (cp, st) if want_stats else cp

    def slice_prepare(self, chans, sample_size, dst_ptr=0, stream=0, dst_host=None):
        """Step 1 of the time-slice hand-over. dst_ptr: raw device pointer and/or dst_host: numpy array in pinned
        memory. -> SliceLink"""
        a = self._chans(chans)
        nblk, nchan = a.shape
        link = SliceLink()
        hp = None if dst_host is None else C.c_void_p(dst_host.ctypes.data)
        self._check(lib().gpsb200_slice_prepare(self._h, a.ctypes.data, nblk, nchan, sample_size, C.c_void_p(dst_ptr),
                                                hp, C.c_void_p(stream), C.byref(link)))
        self._slice_nchan = nchan
        return link

    def slice_probe(self, prn_in=None, phase_guess_in=None, eager=False):
        """Step 2. eager: all speculative work up front (a successor is waiting for this slice's outgoing state)."""
        pi = None if prn_in is None else np.ascontiguousarray(prn_in, dtype=np.int32)
        xi = None if phase_guess_in is None else np.ascontiguousarray(phase_guess_in, dtype=np.float64)
        self._check(lib().gpsb200_slice_probe(self._h, None if pi is None else pi.ctypes.data,
                                              None if xi is None else xi.ctypes.data, 1 if eager else 0))

    def slice_finish(self, prn_in=None, phase_in=None, want_stats=False, handoff=None):
        """Step 3. -> (prn_out, phase_out[, Stats]): the exact chain state after the slice. handoff(prn, phase), if
        given, is called with that state as soon as the host scan has it -- for an eager slice before the long kernels
        are enqueued (gpsb200_slice_finish_cb)."""
        n = self._slice_nchan
        pi = None if prn_in is None else np.ascontiguousarray(prn_in, dtype=np.int32)
        xi = None if phase_in is None else np.ascontiguousarray(phase_in, dtype=np.float64)
        po, xo = np.zeros(n, np.int32), np.zeros(n, np.float64)
        st = Stats()

        def _cb(_user, p_prn, p_ph):
            handoff(np.ctypeslib.as_array(p_prn, shape=(n,)).copy(), np.ctypeslib.as_array(p_ph, shape=(n,)).copy())

        cb = HANDOFF_FN(_cb) if handoff is not None else C.cast(None, HANDOFF_FN)
        self._check(lib().gpsb200_slice_finish_cb(self._h, None if pi is None else pi.ctypes.data,
                                                  None if xi is None else xi.ctypes.data, po.ctypes.data, xo.ctypes.data,
                                                  C.byref(st), cb, None))
        return (po, xo, st) if want_stats else (po, xo)

    def slice_wait(self):
        self._check(lib().gpsb200_slice_wait(self._h))

    def synth_kernel_name(self, nchan):
        return lib().gpsb200_synth_kernel_name(self._h, int(nchan)).decode()

    def debug_corrupt_chain(self, on):
        """on: False/0 off, True/1 corrupt the resolved chain, 2 corrupt a recorded checkpoint-segment state."""
        self._check(lib().gpsb200_debug_corrupt_chain(self._h, int(on)))

    def debug_run_checkpoints(self, nblk, nchan):
        """The previous call's run checkpoints -> structured array [nblk, runs per block, nchan] (x, y, nav, pad)."""
        nruns = BLOCK_SAMPLES // (self.cfg.run_samples or 2400)
        out = np.zeros((nblk, nruns, nchan), RUN_CKPT_DTYPE)
        self._check(lib().gpsb200_debug_run_checkpoints(self._h, nblk, nchan, out.ctypes.data))
        return out

    def debug_block_probes(self, nblk, nchan):
        """The previous call's carrier block probes -> (CARRIER_PROBE_DTYPE [nblk, nchan], seg float64[nblk, nchan, 2, 7]
        as carrier_probe_host orders them (entries a probe did not record are undefined), guess float64[nblk, nchan]:
        the start phases the probes walked from)."""
        probes = np.zeros((nblk, nchan), CARRIER_PROBE_DTYPE)
        seg = np.zeros((nblk, nchan, 2, 7))
        guess = np.zeros((nblk, nchan))
        self._check(lib().gpsb200_debug_block_probes(self._h, nblk, nchan, probes.ctypes.data, seg.ctypes.data,
                                                     guess.ctypes.data))
        return probes, seg, guess

    def debug_synth_shape(self, nblk, nchan, sample_size=SC08):
        """Shape of one synthesis launch over nblk blocks on this context's device -> (kernel name, CTAs per block,
        runs per CTA)."""
        name, per_block, per_cta = C.c_char_p(), C.c_int(0), C.c_int(0)
        self._check(lib().gpsb200_debug_synth_shape(self._h, int(nblk), int(nchan), int(sample_size), C.byref(name),
                                                    C.byref(per_block), C.byref(per_cta)))
        return name.value.decode(), per_block.value, per_cta.value

    def carrier_chain(self, chans, phase_in=None):
        """Exact carrier phases after all blocks of chans (device probe + host fix-up, no synthesis)."""
        a = self._chans(chans)
        nblk, nchan = a.shape
        out = np.zeros(nchan, np.float64)
        pin = None if phase_in is None else np.ascontiguousarray(phase_in, dtype=np.float64)
        self._check(lib().gpsb200_carrier_chain_device(self._h, a.ctypes.data, nblk, nchan,
                                                       None if pin is None else pin.ctypes.data, out.ctypes.data))
        return out

    def acquire(self, iq=None, sample_size=SC08, prns=range(1, 33), ms=10, s0=0, f_lo=-5000.0, step=250.0, nbins=41,
                want_grid=False, device_ptr=None, nsamples=None, stream=0):
        """GPS L1 C/A acquisition search (gpsb200_acquire; DESIGN §9) over code delay x Doppler bin f_lo + j * step,
        `ms` coherent 1 ms periods from sample s0, for each PRN of `prns`.
        Source: iq, a numpy array of interleaved I,Q (int8 for SC08, int16 for SC16), or device_ptr (a raw 16-byte
        aligned device pointer, e.g. the buffer synth_blocks_device filled) holding nsamples samples, searched in place
        on `stream` behind the work it holds.
        -> results ACQ_RESULT_DTYPE[nprn] (prn, bin, delay, doppler_hz, delay_chips, p1, p2, ratio), and with want_grid
        also the whole power grid uint64[nprn, nbins, 3000]."""
        return self._acquire(None, iq, sample_size, [int(p) for p in prns], ms, s0, f_lo, step, nbins, want_grid,
                             device_ptr, nsamples, stream)

    def acquire_windows(self, iq=None, sample_size=SC08, prns=(), f_lo_prn=(), step=250.0, nbins=5, ms=10, s0=0,
                        want_grid=False, device_ptr=None, nsamples=None, stream=0):
        """The acquisition search with a Doppler window per PRN (gpsb200_acquire_windows; DESIGN §9.1): bin j of
        prns[p] is f_lo_prn[p] + j * step, j < nbins; everything else as acquire, whose arguments these are. Row p
        equals acquire(prns=[prns[p]], f_lo=f_lo_prn[p], ...) bit for bit.
        -> results ACQ_RESULT_DTYPE[nprn], and with want_grid also the power grid uint64[nprn, nbins, 3000]."""
        prns = [int(p) for p in prns]
        flo = np.ascontiguousarray(f_lo_prn, dtype=np.float64).reshape(-1)
        if flo.size != len(prns):
            raise GpsB200Error(ERR_ARG, "acquire_windows: %d first bins for %d PRNs" % (flo.size, len(prns)))
        return self._acquire(flo, iq, sample_size, prns, ms, s0, 0.0, step, nbins, want_grid, device_ptr, nsamples,
                             stream)

    def _acquire(self, f_lo_prn, iq, sample_size, prns, ms, s0, f_lo, step, nbins, want_grid, device_ptr, nsamples,
                 stream):
        """acquire, or with f_lo_prn (float64[nprn], the first bins) acquire_windows."""
        cfg = self._acq_config(prns, ms, s0, f_lo, step, nbins)
        res = np.zeros(max(1, min(len(prns), 32)), ACQ_RESULT_DTYPE)
        grid = np.zeros((max(1, len(prns)), max(1, int(nbins)), ACQ_CODE_SAMPLES), np.uint64) if want_grid else None
        gp = None if grid is None else grid.ctypes.data
        src, n, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        if f_lo_prn is None:
            fn, fp = lib().gpsb200_acquire_device if dev else lib().gpsb200_acquire, ()
        else:
            fn = lib().gpsb200_acquire_windows_device if dev else lib().gpsb200_acquire_windows
            fp = (f_lo_prn.ctypes.data if f_lo_prn.size else None,)
        self._check(fn(self._h, src, n, int(sample_size), C.byref(cfg), *fp, res.ctypes.data, gp, *dev))
        return (res, grid) if want_grid else res

    @staticmethod
    def _acq_config(prns, ms, s0, f_lo, step, nbins):
        """The AcqConfig of a search of the PRNs `prns` (a list of ints) with acquire's other arguments."""
        cfg = AcqConfig()
        cfg.s0, cfg.ms, cfg.nprn = int(s0), int(ms), len(prns)
        for i, p in enumerate(prns[:32]):   # more than 32 is rejected by the library with the other argument checks
            cfg.prn[i] = p
        cfg.f_lo_hz, cfg.step_hz, cfg.nbins = float(f_lo), float(step), int(nbins)
        return cfg

    @staticmethod
    def _rx_source(iq, device_ptr, nsamples, stream):
        """The source of a receiver call: nsamples samples at device_ptr, or the numpy array iq (its first nsamples,
        default all). -> (pointer, nsamples, the arguments the _device entry point takes after its others: (stream,)
        for a device source, () for a host one)."""
        if device_ptr is not None:
            assert iq is None and nsamples is not None
            return C.c_void_p(device_ptr), int(nsamples), (C.c_void_p(stream),)
        a = np.ascontiguousarray(iq)
        n = a.size // 2 if nsamples is None else int(nsamples)
        assert n <= a.size // 2
        return a.ctypes, n, ()   # a.ctypes converts to the array's address and keeps the array alive

    def debug_acq_split(self, nprn, nbins, force=-1):
        """gpsb200_debug_acq_split: the CTAs per row a search of nprn x nbins rows uses on this context; force 0
        restores the automatic choice, 1/2/3/4/6 fixes it for every later search, -1 leaves it."""
        rc = lib().gpsb200_debug_acq_split(self._h, int(force), int(nprn), int(nbins))
        if rc < 0:
            self._check(rc)
        return rc

    def track(self, states, iq=None, sample_size=SC08, base=0, max_epochs=None, device_ptr=None, nsamples=None, stream=0):
        """Code and carrier tracking (gpsb200_track; DESIGN §10) of the channels `states` (TRACK_STATE_DTYPE[nchan], e.g.
        from track_start) over a buffer whose first sample is the stream's sample `base`.
        Source: iq, a numpy array of interleaved I,Q (int8 for SC08, int16 for SC16), or device_ptr (a raw 16-byte
        aligned device pointer) holding nsamples samples, tracked in place on `stream` behind the work it holds.
        -> (epochs: a list of TRACK_EPOCH_DTYPE arrays, one per channel, states after the call)."""
        st = np.array(states, dtype=TRACK_STATE_DTYPE).reshape(-1).copy()
        nchan = st.size
        src, n, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        me = int(max_epochs) if max_epochs is not None else n // 2999 + 1
        out = np.zeros((max(1, nchan), max(1, me)), TRACK_EPOCH_DTYPE)
        cnt = np.zeros(max(1, nchan), np.int32)
        fn = lib().gpsb200_track_device if dev else lib().gpsb200_track
        self._check(fn(self._h, src, n, int(sample_size), int(base), st.ctypes.data, nchan, me, out.ctypes.data,
                       cnt.ctypes.data, *dev))
        return [out[c, :cnt[c]].copy() for c in range(nchan)], st

    def vtrack(self, chans, cfg, state, max_updates, iq=None, sample_size=SC08, base=0, want_epochs=False,
               device_ptr=None, nsamples=None, stream=0):
        """Vector tracking (gpsb200_vtrack; DESIGN §10.1) of the channels of `state` (VTRACK_STATE_DTYPE, e.g. from
        vtrack_seed) with the ephemerides chans (PVT_CHAN_DTYPE[nchan]) and the config cfg (vtrack_config), over a
        buffer whose first sample is the stream's sample `base` (source as for track), at most max_updates filter
        updates. -> (fixes FIX_DTYPE[n], VTRACK_CHAN_DTYPE[n][nchan], epochs (a list of TRACK_EPOCH_DTYPE arrays per
        channel, or None), state after the call)."""
        st = np.array(state, dtype=VTRACK_STATE_DTYPE).reshape(()).copy()
        ch = np.ascontiguousarray(chans, dtype=PVT_CHAN_DTYPE)
        cf = np.array(cfg, dtype=VTRACK_CONFIG_DTYPE).reshape(()).copy()
        nchan = int(st["nchan"])
        src, n, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        mu = int(max_updates)
        fixes = np.zeros(max(1, mu), FIX_DTYPE)
        out = np.zeros((max(1, mu), max(1, nchan)), VTRACK_CHAN_DTYPE)
        nu = np.zeros(1, np.int32)
        me = (mu + 1) * int(cf["periods"]) if want_epochs else 0
        ep = np.zeros((max(1, nchan), max(1, me)), TRACK_EPOCH_DTYPE) if want_epochs else None
        cnt = np.zeros(max(1, nchan), np.int32)
        fn = lib().gpsb200_vtrack_device if dev else lib().gpsb200_vtrack
        self._check(fn(self._h, src, n, int(sample_size), int(base), ch.ctypes.data, cf.ctypes.data, st.ctypes.data, mu,
                       fixes.ctypes.data, out.ctypes.data, nu.ctypes.data, ep.ctypes.data if want_epochs else None, me,
                       cnt.ctypes.data, *dev))
        k = int(nu[0])
        eps = [ep[c, :cnt[c]].copy() for c in range(nchan)] if want_epochs else None
        return fixes[:k].copy(), out[:k, :nchan].copy(), eps, st

    def debug_vtrack_cluster(self, ctas):
        """gpsb200_debug_vtrack_cluster: the CTAs of the cluster of later vector-tracking calls (0: automatic)."""
        self._check(lib().gpsb200_debug_vtrack_cluster(self._h, int(ctas)))

    def pvt(self, chans, epochs, cfg, want_residuals=False, nepochs=None):
        """Position, velocity and time fixes (gpsb200_pvt; DESIGN §11). chans: PVT_CHAN_DTYPE[nchan] (ephemeris and time
        anchor of each channel); epochs: a list of TRACK_EPOCH_DTYPE arrays, one per channel, in time order (as track
        returns them, concatenated over calls), or, with nepochs (int32[nchan]), the [nchan, max_epochs] array as the C
        call takes it; cfg: PVT_CONFIG_DTYPE record (pvt_config).
        -> fixes FIX_DTYPE[nfix], and with want_residuals also the post-fit residuals float64[nfix, nchan] (NaN where a
        channel is not used)."""
        ch, nchan, ep, n, me, cf, fixes, res = self._pvt_args(chans, epochs, cfg, want_residuals, nepochs)
        self._check(lib().gpsb200_pvt(self._h, ch.ctypes.data, nchan, ep.ctypes.data, n.ctypes.data, me, cf.ctypes.data,
                                      fixes.ctypes.data, None if res is None else res.ctypes.data))
        return (fixes, res) if want_residuals else fixes

    def pvt_raim(self, chans, epochs, cfg, raim, want_residuals=False, nepochs=None):
        """Fixes with RAIM fault detection, exclusion and protection levels (gpsb200_pvt_raim; DESIGN §11.1). The
        arguments of pvt, plus raim: RAIM_CONFIG_DTYPE record (raim_config).
        -> (fixes FIX_DTYPE[nfix] of each fix's final channel set, RAIM_DTYPE[nfix]), and with want_residuals also the
        residuals float64[nfix, nchan]: the final set's post-fit residuals, an excluded channel's residual against the
        final fix, NaN elsewhere."""
        ch, nchan, ep, n, me, cf, fixes, res = self._pvt_args(chans, epochs, cfg, want_residuals, nepochs)
        rc = np.array(raim, dtype=RAIM_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, RAIM_DTYPE)
        self._check(lib().gpsb200_pvt_raim(self._h, ch.ctypes.data, nchan, ep.ctypes.data, n.ctypes.data, me,
                                           cf.ctypes.data, rc.ctypes.data, fixes.ctypes.data,
                                           None if res is None else res.ctypes.data, out.ctypes.data))
        return (fixes, out, res) if want_residuals else (fixes, out)

    def pvt_araim(self, chans, epochs, cfg, araim, want_residuals=False, nepochs=None):
        """Fixes with advanced RAIM: weighted solve, elevation mask, solution-separation test and protection levels
        (gpsb200_pvt_araim; DESIGN §11.2). The arguments of pvt, plus araim: ARAIM_CONFIG_DTYPE record (araim_config).
        -> (fixes FIX_DTYPE[nfix] of each fix's final set, ARAIM_DTYPE[nfix]), and with want_residuals also the
        residuals float64[nfix, nchan]: every measured channel's post-fit residual against the final fix."""
        ch, nchan, ep, n, me, cf, fixes, res = self._pvt_args(chans, epochs, cfg, want_residuals, nepochs)
        ac = np.array(araim, dtype=ARAIM_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, ARAIM_DTYPE)
        self._check(lib().gpsb200_pvt_araim(self._h, ch.ctypes.data, nchan, ep.ctypes.data, n.ctypes.data, me,
                                            cf.ctypes.data, ac.ctypes.data, fixes.ctypes.data,
                                            None if res is None else res.ctypes.data, out.ctypes.data))
        return (fixes, out, res) if want_residuals else (fixes, out)

    def pvt_coarse(self, chans, epochs, cfg, apriori, want_residuals=False, want_ms=False, nepochs=None):
        """Coarse-time fixes without time anchors (gpsb200_pvt_coarse; DESIGN §11.3). The arguments of pvt (anchors
        unread), plus apriori: COARSE_CONFIG_DTYPE record (coarse_config).
        -> (fixes FIX_DTYPE[nfix], COARSE_DTYPE[nfix]), then the residuals float64[nfix, nchan] with want_residuals and
        the resolved ms of week int64[nfix, nchan] (-1 where not used) with want_ms."""
        ch, nchan, ep, n, me, cf, fixes, res = self._pvt_args(chans, epochs, cfg, want_residuals, nepochs)
        ap = np.array(apriori, dtype=COARSE_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, COARSE_DTYPE)
        ms = np.zeros((fixes.size, max(1, nchan)), np.int64) if want_ms else None
        self._check(lib().gpsb200_pvt_coarse(self._h, ch.ctypes.data, nchan, ep.ctypes.data, n.ctypes.data, me,
                                             cf.ctypes.data, ap.ctypes.data, fixes.ctypes.data,
                                             None if res is None else res.ctypes.data, out.ctypes.data,
                                             None if ms is None else ms.ctypes.data))
        return (fixes, out) + ((res,) if want_residuals else ()) + ((ms,) if want_ms else ())

    def pvt_search(self, chans, epochs, cfg, search, want_residuals=False, want_ms=False, want_node_rms=False,
                   nepochs=None):
        """Position search with no a-priori position (gpsb200_pvt_search; DESIGN §11.4): coarse-time fixes from every
        node of a global grid. The arguments of pvt (anchors unread), plus search: SEARCH_CONFIG_DTYPE record
        (search_config).
        -> (fixes FIX_DTYPE[nfix], SEARCH_DTYPE[nfix]), then the residuals float64[nfix, nchan] with want_residuals, the
        resolved ms of week int64[nfix, nchan] (-1 where not used) with want_ms, and every node's rms float64[nfix,
        nodes] (NaN where pruned or not OK) with want_node_rms."""
        ch, nchan, ep, n, me, cf, fixes, res = self._pvt_args(chans, epochs, cfg, want_residuals, nepochs)
        sc = np.array(search, dtype=SEARCH_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, SEARCH_DTYPE)
        ms = np.zeros((fixes.size, max(1, nchan)), np.int64) if want_ms else None
        nr = np.zeros((fixes.size, max(1, int(sc[0]["nodes"]))), np.float64) if want_node_rms else None
        self._check(lib().gpsb200_pvt_search(self._h, ch.ctypes.data, nchan, ep.ctypes.data, n.ctypes.data, me,
                                             cf.ctypes.data, sc.ctypes.data, fixes.ctypes.data,
                                             None if res is None else res.ctypes.data, out.ctypes.data,
                                             None if ms is None else ms.ctypes.data,
                                             None if nr is None else nr.ctypes.data))
        return ((fixes, out) + ((res,) if want_residuals else ()) + ((ms,) if want_ms else ())
                + ((nr,) if want_node_rms else ()))

    def snapshot_measure(self, res, iq=None, sample_size=SC08, ms=10, s0=0, prns=None, f_lo=-5000.0, step=250.0,
                         nbins=41, cfg=None, device_ptr=None, nsamples=None, stream=0):
        """Refine acquisition results to snapshot measurements (gpsb200_snapshot_measure; DESIGN §11.5). res: the
        ACQ_RESULT_DTYPE rows a search returned; ms, s0, prns (default res["prn"]), f_lo, step and nbins: the search's
        arguments (acquire's); cfg: SNAPSHOT_CONFIG_DTYPE record (snapshot_config(), the default). Source as acquire.
        -> SNAPSHOT_DTYPE[nprn] in the order of res."""
        r = np.ascontiguousarray(res, dtype=ACQ_RESULT_DTYPE).reshape(-1)
        prns = [int(p) for p in (r["prn"] if prns is None else prns)]
        acq = self._acq_config(prns, ms, s0, f_lo, step, nbins)
        sc = np.array(snapshot_config() if cfg is None else cfg, dtype=SNAPSHOT_CONFIG_DTYPE).reshape(1)
        if r.size < len(prns):
            raise GpsB200Error(ERR_ARG, "snapshot_measure: %d results for %d PRNs" % (r.size, len(prns)))
        out = np.zeros(max(1, len(prns)), SNAPSHOT_DTYPE)
        src, n, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        fn = lib().gpsb200_snapshot_measure_device if dev else lib().gpsb200_snapshot_measure
        self._check(fn(self._h, src, n, int(sample_size), C.byref(acq), r.ctypes.data, sc.ctypes.data, out.ctypes.data,
                       *dev))
        return out[:len(prns)]

    def snapshot_batch(self, s0, iq=None, sample_size=SC08, prns=range(1, 33), ms=10, f_lo=-5000.0, step=250.0,
                       nbins=41, f_lo_prn=None, cfg=None, device_ptr=None, nsamples=None, stream=0):
        """The search and the snapshot measurement of many windows in one call (gpsb200_snapshot_batch; DESIGN §11.6):
        window w starts at sample s0[w] (windows may overlap, repeat and come in any order). Without f_lo_prn every
        window searches the standard grid f_lo + j * step, as acquire; with f_lo_prn (float64[nwin, nprn]) window w
        searches PRN prns[p] from f_lo_prn[w, p], as acquire_windows. cfg: SNAPSHOT_CONFIG_DTYPE record (snapshot_config(),
        the default). Source as acquire.
        -> (results ACQ_RESULT_DTYPE[nwin, nprn], SNAPSHOT_DTYPE[nwin, nprn]): row w equals acquire (or
        acquire_windows) with s0=s0[w] and snapshot_measure on its results, bit for bit."""
        prns = [int(p) for p in prns]
        s = np.ascontiguousarray(s0, dtype=np.int64).reshape(-1)
        nwin = s.size
        flo = None
        if f_lo_prn is not None:
            flo = np.ascontiguousarray(f_lo_prn, dtype=np.float64)
            if flo.shape != (nwin, len(prns)):
                raise GpsB200Error(ERR_ARG, "snapshot_batch: f_lo_prn of shape %s for %d windows of %d PRNs"
                                   % (flo.shape, nwin, len(prns)))
        acq = self._acq_config(prns, ms, 0, f_lo, step, nbins)
        sc = np.array(snapshot_config() if cfg is None else cfg, dtype=SNAPSHOT_CONFIG_DTYPE).reshape(1)
        shape = (max(1, nwin), max(1, min(len(prns), 32)))
        res = np.zeros(shape, ACQ_RESULT_DTYPE)
        out = np.zeros(shape, SNAPSHOT_DTYPE)
        src, n, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        fn = lib().gpsb200_snapshot_batch_device if dev else lib().gpsb200_snapshot_batch
        self._check(fn(self._h, src, n, int(sample_size), C.byref(acq), nwin, s.ctypes.data if nwin else None,
                       None if flo is None else flo.ctypes.data, sc.ctypes.data, res.ctypes.data, out.ctypes.data,
                       *dev))
        return res, out

    def collective(self, eph, apriori, cfg, iq=None, sample_size=SC08, prns=range(1, 33), ms=10, s0=0, f_lo=-5000.0,
                   step=250.0, nbins=41, f_lo_prn=None, want_scores=False, want_table=False, device_ptr=None,
                   nsamples=None, stream=0):
        """Collective detection (gpsb200_collective; DESIGN §11.7): the search of acquire (or, with f_lo_prn
        float64[nprn], of acquire_windows) over its arguments, then a lattice of receiver positions and time offsets
        around apriori (COARSE_CONFIG_DTYPE) scored against the power grids. eph: EPHEMERIS_DTYPE[32] indexed by PRN - 1
        (rinex_ephemeris); cfg: COLLECTIVE_CONFIG_DTYPE record (collective_config). Source as acquire.
        -> (results ACQ_RESULT_DTYPE[nprn], seeds ACQ_RESULT_DTYPE[nprn], COLLECTIVE_DTYPE record), then with
        want_scores CD_SCORE_DTYPE[nhyp] and with want_table CD_CELL_DTYPE[nhyp, nprn]."""
        prns = [int(p) for p in prns]
        flo = None
        if f_lo_prn is not None:
            flo = np.ascontiguousarray(f_lo_prn, dtype=np.float64).reshape(-1)
            if flo.size != len(prns):
                raise GpsB200Error(ERR_ARG, "collective: %d first bins for %d PRNs" % (flo.size, len(prns)))
        acq = self._acq_config(prns, ms, s0, f_lo, step, nbins)
        e = np.ascontiguousarray(eph, dtype=EPHEMERIS_DTYPE).reshape(-1)
        if e.size != 32:
            raise GpsB200Error(ERR_ARG, "collective: %d ephemeris records, not 32" % e.size)
        ap = np.array(apriori, dtype=COARSE_CONFIG_DTYPE).reshape(1)
        cf = np.array(cfg, dtype=COLLECTIVE_CONFIG_DTYPE).reshape(1)
        nhyp = max(1, int(np.prod(cf[0]["n"].astype(np.int64)))) if (cf[0]["n"] >= 1).all() else 1
        n = max(1, min(len(prns), 32))
        res, seed = np.zeros(n, ACQ_RESULT_DTYPE), np.zeros(n, ACQ_RESULT_DTYPE)
        rec = np.zeros(1, COLLECTIVE_DTYPE)
        sc = np.zeros(nhyp, CD_SCORE_DTYPE) if want_scores else None
        tb = np.zeros((nhyp, n), CD_CELL_DTYPE) if want_table else None
        src, ns, dev = self._rx_source(iq, device_ptr, nsamples, stream)
        fn = lib().gpsb200_collective_device if dev else lib().gpsb200_collective
        self._check(fn(self._h, src, ns, int(sample_size), C.byref(acq), None if flo is None else flo.ctypes.data,
                       e.ctypes.data, ap.ctypes.data, cf.ctypes.data, res.ctypes.data, seed.ctypes.data,
                       rec.ctypes.data, None if sc is None else sc.ctypes.data,
                       None if tb is None else tb.ctypes.data, *dev))
        return (res, seed, rec[0]) + ((sc,) if want_scores else ()) + ((tb,) if want_table else ())

    @staticmethod
    def _snapshot_args(chans, meas, cfg, want_residuals):
        ch = np.ascontiguousarray(chans, dtype=PVT_CHAN_DTYPE).reshape(-1)
        m = np.ascontiguousarray(meas, dtype=SNAPSHOT_DTYPE)
        if m.ndim == 1:
            m = m.reshape(1, -1)
        assert m.ndim == 2 and m.shape[0] >= 1 and m.shape[1] == ch.size, (m.shape, ch.size)
        cf = np.array(cfg, dtype=PVT_CONFIG_DTYPE).reshape(1).copy()
        cf[0]["nfix"] = m.shape[0]
        fixes = np.zeros(max(1, m.shape[0]), FIX_DTYPE)
        res = np.zeros((fixes.size, max(1, ch.size))) if want_residuals else None
        return ch, m, cf, fixes, res

    def pvt_snapshot(self, chans, meas, cfg, apriori, want_residuals=False, want_ms=False):
        """Coarse-time fixes from snapshot records (gpsb200_pvt_snapshot; DESIGN §11.5). meas: SNAPSHOT_DTYPE
        [nsnap, nchan], row i the records of snapshot i with column c for chans[c] (a 1-D array is one snapshot); cfg:
        PVT_CONFIG_DTYPE record whose iono terms apply (nfix is set to nsnap, s0 and step are not read); apriori:
        COARSE_CONFIG_DTYPE record. -> pvt_coarse's tuple."""
        ch, m, cf, fixes, res = self._snapshot_args(chans, meas, cfg, want_residuals)
        ap = np.array(apriori, dtype=COARSE_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, COARSE_DTYPE)
        ms = np.zeros((fixes.size, max(1, ch.size)), np.int64) if want_ms else None
        self._check(lib().gpsb200_pvt_snapshot(self._h, ch.ctypes.data, ch.size, m.ctypes.data, cf.ctypes.data,
                                               ap.ctypes.data, fixes.ctypes.data,
                                               None if res is None else res.ctypes.data, out.ctypes.data,
                                               None if ms is None else ms.ctypes.data))
        return (fixes, out) + ((res,) if want_residuals else ()) + ((ms,) if want_ms else ())

    def pvt_snapshot_search(self, chans, meas, cfg, search, want_residuals=False, want_ms=False, want_node_rms=False):
        """Position searches from snapshot records (gpsb200_pvt_snapshot_search; DESIGN §11.5): pvt_snapshot's
        arguments with search (SEARCH_CONFIG_DTYPE record) in place of apriori. -> pvt_search's tuple."""
        ch, m, cf, fixes, res = self._snapshot_args(chans, meas, cfg, want_residuals)
        sc = np.array(search, dtype=SEARCH_CONFIG_DTYPE).reshape(1)
        out = np.zeros(fixes.size, SEARCH_DTYPE)
        ms = np.zeros((fixes.size, max(1, ch.size)), np.int64) if want_ms else None
        nr = np.zeros((fixes.size, max(1, int(sc[0]["nodes"]))), np.float64) if want_node_rms else None
        self._check(lib().gpsb200_pvt_snapshot_search(self._h, ch.ctypes.data, ch.size, m.ctypes.data, cf.ctypes.data,
                                                      sc.ctypes.data, fixes.ctypes.data,
                                                      None if res is None else res.ctypes.data, out.ctypes.data,
                                                      None if ms is None else ms.ctypes.data,
                                                      None if nr is None else nr.ctypes.data))
        return ((fixes, out) + ((res,) if want_residuals else ()) + ((ms,) if want_ms else ())
                + ((nr,) if want_node_rms else ()))

    @staticmethod
    def _pvt_args(chans, epochs, cfg, want_residuals, nepochs):
        """The C call's arrays for pvt / pvt_raim: the epochs packed [nchan, max_epochs] unless they already are."""
        ch = np.ascontiguousarray(chans, dtype=PVT_CHAN_DTYPE).reshape(-1)
        nchan = ch.size
        if nepochs is not None:
            ep = np.ascontiguousarray(epochs, dtype=TRACK_EPOCH_DTYPE)
            n = np.ascontiguousarray(nepochs, dtype=np.int32)
            assert ep.ndim == 2 and ep.shape[0] == n.size == nchan
            me = ep.shape[1]
        else:
            n = np.array([len(e) for e in epochs], np.int32)
            assert n.size == nchan
            me = max(1, int(n.max()) if n.size else 1)
            ep = np.zeros((max(1, nchan), me), TRACK_EPOCH_DTYPE)
            for c, e in enumerate(epochs):
                ep[c, :len(e)] = e
        cf = np.array(cfg, dtype=PVT_CONFIG_DTYPE).reshape(1)
        nfix = max(1, int(cf[0]["nfix"]))
        fixes = np.zeros(nfix, FIX_DTYPE)
        res = np.zeros((nfix, max(1, nchan))) if want_residuals else None
        return ch, nchan, ep, n, me, cf, fixes, res

    def pvt_replay(self, stream=0):
        """Enqueue the fix kernel of the previous pvt call again on `stream`, on its device-resident inputs (timing)."""
        self._check(lib().gpsb200_pvt_replay(self._h, C.c_void_p(stream)))

    def replay_device(self, dst_ptr=0, stream=0, kernel_mask=15):
        self._check(lib().gpsb200_replay_device(self._h, C.c_void_p(dst_ptr), C.c_void_p(stream), kernel_mask))
