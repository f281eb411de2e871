"""Numpy statement of the position search (include/gpsb200.h: gpsb200_pvt_search; DESIGN §11.4): the tests' reference.

It shares no code with the library. The per-node solve is coarse_model's coarse-time fix, run with one a-priori position
per row (every row at the same fix instant); the satellite and the WGS-84 conversion are pvt_model's. Only the grid, the
visibility prune and the choice among the nodes' fixes are stated here."""
import numpy as np

import coarse_model as CM
import pvt_model as PM

NODES_DEFAULT = 262144
NODES_MIN, NODES_MAX = 64, 1 << 22
GOLDEN = float.fromhex("0x1.8722191a02d61p-2")   # the double nearest (3 - sqrt(5)) / 2
MIN_ELEV_DEG = -5.0
SIN_MIN_ELEV = np.sin(np.radians(MIN_ELEV_DEG))
DISTINCT = 1000.0
MIN_CHANNELS = 6


def max_ok(n):
    """GPSB200_SEARCH_MAX_OK(n): the OK-list length per instant of an n-node grid."""
    return max(64, n // 256)


def grid_llh(n, idx=None):
    """Header step 1: geodetic latitude and longitude (rad) of nodes idx (default all) of the n-node grid."""
    i = np.arange(n, dtype=np.int64) if idx is None else np.asarray(idx, np.int64)
    z = 1.0 - (2.0 * i.astype(np.float64) + 1.0) / float(n)
    t = i.astype(np.float64) * GOLDEN
    return np.arcsin(z), 2.0 * np.pi * (t - np.floor(t))


def nodes(n, idx=None):
    """ECEF (m) [len, 3] of the grid's nodes at height 0 (pvt_model's conversion)."""
    lat, lon = grid_llh(n, idx)
    return PM.llh_ecef(np.degrees(lat), np.degrees(lon), 0.0).T.copy()


def visible(chans, use, tas, n):
    """Header step 3 at one fix instant: bool [n], the nodes from which every used channel's satellite (at GPS time
    tas - 0.075 s, unrotated) has sin(elevation) >= sin(-5 deg)."""
    eph = np.stack([chans[c]["eph"] for c in np.nonzero(use)[0]])[None, :]
    p, _, _, _ = PM.satellite(eph, np.full(eph.shape, tas - CM.TAU0))
    lat, lon = grid_llh(n)
    x = nodes(n)
    up = np.stack([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)], -1)
    ok = np.ones(n, bool)
    for c in range(p.shape[1]):
        l = p[0, c][None, :] - x
        ok &= (up * l).sum(-1) / np.sqrt((l * l).sum(-1)) >= SIN_MIN_ELEV
    return ok


def fix_at(chans, epochs, cfg, sc, s, xa):
    """The coarse-time fixes at instant s from a-priori positions xa [K, 3]. -> coarse_model.coarse's tuple, row k from
    xa[k]."""
    c1 = np.array(cfg).copy()
    c1["s0"], c1["step"], c1["nfix"] = s, 0, len(xa)
    ap = dict(x_a=np.asarray(xa, np.float64), t_a=float(sc["t_a"]), s_a=int(sc["s_a"]), week=int(sc["week"]))
    return CM.coarse(chans, epochs, c1, ap)


def search(chans, epochs, cfg, sc, want_node_rms=False, chunk=8192):
    """The searches of the contract. chans: PVT_CHAN records; epochs: list of TRACK_EPOCH arrays; cfg: PVT_CONFIG
    record; sc: SEARCH_CONFIG record.
    -> (fix dict [F] with FIX_DTYPE names, search dict [F] with SEARCH_DTYPE names, residuals [F, C], ms [F, C]), plus
    node_rms [F, N] with want_node_rms."""
    nf, nc, n = int(cfg["nfix"]), len(epochs), int(sc["nodes"])
    s = int(cfg["s0"]) + np.arange(nf, dtype=np.int64) * int(cfg["step"])
    u = float(sc["t_a"]) + (s - int(sc["s_a"])).astype(np.float64) / 3e6
    tas = u - 604800.0 * np.floor(u / 604800.0)
    use = CM.measure(chans, epochs, s, tas)["use"]
    nused = use.sum(1)
    fnames = ("x", "y", "z", "clock_m", "t_rx", "vx", "vy", "vz", "drift", "lat_deg", "lon_deg", "height", "pdop", "rms")
    fix = {f: np.full(nf, np.nan) for f in fnames}
    fix.update(sample=s, status=np.where(nused < MIN_CHANNELS, PM.FIX_FEW, PM.FIX_NO_CONVERGENCE), nused=nused,
               mask=(use * (1 << np.arange(nc, dtype=np.int64))).sum(1), iterations=np.zeros(nf, np.int32))
    out = dict(winner=np.full(nf, -1, np.int32), searched=np.zeros(nf, np.int32), ok=np.zeros(nf, np.int32),
               support=np.zeros(nf, np.int32), alt_rms=np.full(nf, np.nan), alt_dist=np.full(nf, np.nan),
               delta=np.full(nf, np.nan), pdop=np.full(nf, np.nan), ref=np.full(nf, -1, np.int32),
               week=np.full(nf, -1, np.int32), changed=np.zeros(nf, np.int64))
    res = np.full((nf, nc), np.nan)
    ms = np.full((nf, nc), -1, np.int64)
    node_rms = np.full((nf, n), np.nan) if want_node_rms else None
    for f in range(nf):
        if nused[f] < MIN_CHANNELS:
            continue
        idx = np.nonzero(visible(chans, use[f], tas[f], n))[0]
        out["searched"][f] = idx.size
        okn, rms, pos = [], [], []
        for k in range(0, idx.size, chunk):
            part = idx[k:k + chunk]
            fx, _, _, _ = fix_at(chans, epochs, cfg, sc, s[f], nodes(n, part))
            good = fx["status"] == PM.FIX_OK
            okn.append(part[good])
            rms.append(fx["rms"][good])
            pos.append(np.stack([fx["x"], fx["y"], fx["z"]], 1)[good])
        okn = np.concatenate(okn) if okn else np.zeros(0, np.int64)
        rms = np.concatenate(rms) if rms else np.zeros(0)
        pos = np.concatenate(pos) if pos else np.zeros((0, 3))
        out["ok"][f] = okn.size
        if want_node_rms:
            node_rms[f, okn] = rms
        if okn.size == 0:
            continue
        if okn.size > max_ok(n):
            fix["status"][f] = CM.FIX_AMBIGUOUS
            continue
        key = np.floor(rms * 1000.0)
        w = np.lexsort((okn, key))[0]
        d = np.sqrt(((pos - pos[w]) ** 2).sum(1))
        near = d <= DISTINCT
        out["support"][f] = near.sum()
        if (~near).any():
            j = np.nonzero(~near)[0]
            a = j[np.lexsort((okn[j], key[j]))[0]]
            out["alt_rms"][f], out["alt_dist"][f] = rms[a], d[a]
        out["winner"][f] = okn[w]
        fx, co, r1, m1 = fix_at(chans, epochs, cfg, sc, s[f], nodes(n, [okn[w]]))
        for k in fnames + ("status", "nused", "mask", "iterations"):
            fix[k][f] = fx[k][0]
        if (~near).any():
            fix["status"][f] = CM.FIX_AMBIGUOUS
        for k in ("delta", "pdop", "ref", "week", "changed"):
            out[k][f] = co[k][0]
        res[f], ms[f] = r1[0], m1[0]
    return (fix, out, res, ms) + ((node_rms,) if want_node_rms else ())
