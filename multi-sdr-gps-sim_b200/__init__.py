"""gpsb200: H100-native GPS L1 C/A baseband synthesis (hot path of multi-sdr-gps-sim).

The product is libgpsb200.so (CUDA kernels for sm_90a behind the C ABI of
include/gpsb200.h). This package is only the host-side convenience layer used by
the tests and bench.py: ctypes bindings that mirror the C ABI one to one.
Import it with importlib (the directory name is not a Python identifier):

    gps = importlib.import_module("multi-sdr-gps-sim_b200")
"""
from .api import (  # noqa: F401
    BLOCK_ELEMS, BLOCK_SAMPLES, SC08, SC16, Chan, Config, Context, GpsB200Error, Stats,
    bind_numa, carrier_advance, span_chain_host, lanes_model_block, lanes_window_band, link_apply, slice_link_host, SliceLink, carrier_chain, codegen, scenario, lib, lib_path, CHAN_DTYPE,
    ScenarioConfig, LiveScenario, SteerState, parse_steer, KEYS, ERR_END, almanac_read, ALMANAC_RECORD_DTYPE, checkpoint_segments_host, RUN_CKPT_DTYPE,
    carrier_probe_host, CARRIER_PROBE_DTYPE, AcqConfig, ACQ_RESULT_DTYPE, ACQ_CODE_SAMPLES, acq_window_samples,
    TRACK_STATE_DTYPE, TRACK_EPOCH_DTYPE, NAV_BIT_DTYPE, NAV_WORD_DTYPE, NAV_SYNC_DTYPE, track_start, nav_decode, nav_word_check,
    nav_parity, EPHEMERIS_DTYPE, IONO_DTYPE, PVT_CHAN_DTYPE, PVT_CONFIG_DTYPE, FIX_DTYPE, FIX_OK, FIX_FEW,
    FIX_NO_CONVERGENCE, PVT_MAX_ITER, nav_words_of_frame, nav_ephemeris, nav_time_anchor, pvt_config,
    RAIM_CONFIG_DTYPE, RAIM_DTYPE, RAIM_PASS, RAIM_EXCLUDED, RAIM_ALERT, RAIM_UNAVAILABLE, RAIM_MAX_DOF,
    RAIM_MAX_EXCLUDE, raim_config, raim_thresholds, ARAIM_CONFIG_DTYPE, ARAIM_DTYPE, araim_config, araim_kfa,
    COARSE_CONFIG_DTYPE, COARSE_DTYPE, FIX_AMBIGUOUS, coarse_config, rinex_ephemeris,
    SEARCH_CONFIG_DTYPE, SEARCH_DTYPE, SEARCH_NODES, search_config, search_nodes,
    SKY_DTYPE, nav_almanac, almanac_predict,
    SNAPSHOT_CONFIG_DTYPE, SNAPSHOT_DTYPE, SNAP_OK, SNAP_WEAK, SNAP_NO_CONVERGENCE, SNAP_ITERATIONS, SNAP_MAX_ITER,
    snapshot_config, SNAP_BATCH_SCRATCH, snapshot_batch_pass,
    COLLECTIVE_CONFIG_DTYPE, COLLECTIVE_DTYPE, CD_SCORE_DTYPE, CD_CELL_DTYPE, CD_OK, CD_FEW, CD_AMBIGUOUS, CD_MAX_HYP,
    CD_MIN_USED, CD_Q_SHIFT, CD_Q_CAP, CD_AMBIGUOUS_PCT, collective_config,
    VTRACK_CONFIG_DTYPE, VTRACK_CHAN_STATE_DTYPE, VTRACK_STATE_DTYPE, VTRACK_CHAN_DTYPE, vtrack_config, vtrack_seed,
)
from .synthetic import synthetic_chans  # noqa: F401,E402
from . import sharding  # noqa: F401,E402
