"""Numpy statement of pooled collective detection (DESIGN §11.8): one lattice of collective_model scored over nwin
windows of one static receiver, with one clock shift b common to every window. Each window is searched, normalised,
tested for its used PRNs and predicted as collective_model does it at its own time t0_w; the scores add over the
windows; the pick is collective_model's; each window gets its own seeds at the winner. With one window every output is
collective_model.collective's, bit for bit."""
import numpy as np

from collective_model import CODE, MIN_USED, normalise, pick, seeds, table, used


def score_pool(qs, cells):
    """Step 5 of the pooled call: qs [nwin] of q [nprn][nbins][3000], cells [nwin, H, nprn, 2] -> (S [H] uint32,
    b [H] int32). S(h, b) = sum over windows of the single call's sum at (h, b)."""
    nwin, H, nprn, _ = cells.shape
    b = np.arange(CODE)
    S = np.zeros((H, CODE), np.uint32)
    for w in range(nwin):
        for p in range(nprn):
            j, d = cells[w, :, p, 0], cells[w, :, p, 1]
            on = j >= 0
            if not on.any():
                continue
            idx = (d[on][:, None] + b[None, :]) % CODE
            S[on] += np.take_along_axis(qs[w][p][j[on]], idx, 1).astype(np.uint32)
    best = np.argmax(S, 1)
    return S[np.arange(H), best], best.astype(np.int32)


def collective_pool(Ps, ress, eph, prns, ap, s0, cfg, f_lo_p, step_hz, cells=None):
    """The pooled call on the windows' grids Ps [nwin] and results ress [nwin]; s0 [nwin] the windows' first samples;
    f_lo_p: each PRN's first bin, [nprn] (every window) or [nwin, nprn]. cells: the table [nwin, H, nprn, 2] to score
    (default the model's own). -> (record, seeds [nwin, nprn], S [H], b [H], cells [nwin, H, nprn, 2])."""
    nwin, nbins = len(Ps), Ps[0].shape[1]
    flo = np.broadcast_to(np.asarray(f_lo_p, np.float64), (nwin, len(prns)))
    qs, uses = [], []
    for w in range(nwin):
        mu, q = normalise(Ps[w])
        qs.append(q)
        uses.append(used(eph, prns, ap, s0[w], cfg["mask_deg"], mu))
    use = np.logical_or.reduce(uses)
    nhyp = int(np.prod(cfg["n"].astype(np.int64)))
    if use.sum() < MIN_USED:
        rec = pick(None, None, cfg, ap, use)
        sd = np.stack([seeds(ress[w], Ps[w], rec, None, flo[w], step_hz) for w in range(nwin)])
        return rec, sd, np.zeros(nhyp, np.uint32), np.zeros(nhyp, np.int32), \
            np.full((nwin, nhyp, len(prns), 2), -1, np.int32)
    if cells is None:
        cells = np.stack([table(eph, prns, uses[w], ap, s0[w], cfg, flo[w], step_hz, nbins)[0] for w in range(nwin)])
    S, b = score_pool(qs, cells)
    rec = pick(S, b, cfg, ap, use)
    wn = int(rec["winner"])
    sd = np.stack([seeds(ress[w], Ps[w], rec, cells[w, wn], flo[w], step_hz) for w in range(nwin)])
    return rec, sd, S, b, cells
