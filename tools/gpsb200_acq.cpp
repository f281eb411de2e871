// gpsb200-acq: GPS L1 C/A acquisition search over a 3 Msps I/Q file (gpsb200-sim's output, the reference's iqdata.bin,
// any capture in these formats: int8 or, with --iq16, int16 I,Q interleaved). Reads only the searched window --
// 3000 K + 2999 samples from the start offset -- and runs gpsb200_acquire on it; prints one line per PRN: best Doppler
// bin, code delay (samples from the window start to the code's chip 0, and in chips), P1/P2 and whether P1/P2 reaches
// the threshold. The search and its arithmetic are those of include/gpsb200.h (DESIGN §9).
//
// Warm start (--almanac, DESIGN §9.1): with a SEM almanac, an a-priori position and the GPS time of the window's first
// sample, gpsb200_almanac_predict gives each PRN's elevation and Doppler; only the PRNs predicted at or above the mask
// are searched, each over 2h + 1 bins of the --doppler step around its prediction (h = ceil(window / step)), starting
// at step * round(f / step) - h * step so that the bins lie on the cold search's grid (gpsb200_acquire_windows). Each
// line then also shows the predicted Doppler and elevation.
//
// Snapshot fixes (--fix, DESIGN §11.5): with a RINEX navigation file (--assist), the GPS time of the first window's
// first sample (--assist-time) and an a-priori position (--assist-pos LAT,LON,H) or none (--assist-pos search), every
// --every ms from the start offset (--count windows) the search runs on its window, gpsb200_snapshot_measure refines
// the PRNs at or above the threshold, and gpsb200_pvt_snapshot (gpsb200_pvt_snapshot_search over the default global
// grid with search) fixes from them, with the ephemeris valid at the assist time. One line per snapshot: sample,
// status, position, clock, velocity, channels used, PDOP and delta (the solved a-priori time error), plus support with
// search. No tracking, no navigation message: each fix comes from its K ms window alone. The windows are read, searched
// and measured up to 100 at a time (gpsb200_snapshot_batch, DESIGN §11.6); the fixes stay one call per window. With
// --almanac and an a-priori position the windows are warm started: each window's sky is predicted at its own time (the
// assist time plus its offset from the first window), every window of a chunk searches the PRNs predicted at or above
// the mask in any of them, each over the warm start's bins around that window's own prediction.
// Collective detection (--fix --collective, DESIGN §11.7): with an a-priori position, per window one
// gpsb200_collective call scores a lattice of positions and time offsets around the a-priori against the powers of all
// searched PRNs, so that satellites below the threshold still count; the seeds at the winner's cells are refined
// (gpsb200_snapshot_measure, min_ratio 0) and fixed from the winner (gpsb200_pvt_snapshot). Without --collective the
// output is unchanged.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../include/gpsb200.h"
#include "rx_cli.h"

// P1/P2 at or above which a PRN counts as acquired. Without noise, absent PRNs of the project's streams stay below 1.6
// and present ones are far above 3 (tests/test_acquire.py fixes the bounds of both from the model).
static const double kDefaultThreshold = 2.5;
// Warm start: half-width of each PRN's Doppler window and the elevation mask. The almanac predicts the Doppler of the
// project's streams to within 146 Hz (tests/test_almanac_decode.py), so +-500 Hz (5 bins at 250 Hz) holds it with room
// for an a-priori a few tens of km and seconds off.
static const double kDefaultWindow = 500.0, kDefaultMask = -5.0;
// --collective: the runner-up lies farther than this (or two lattice steps) from the winner. On the model a clean
// winner's neighbours within 1 km keep most of its score (DESIGN §11.7).
static const double kDistinct = 1000.0;

static void usage() {
    fprintf(stderr,
            "gpsb200-acq FILE [--iq16] [--block B] [--offset-ms N] [--ms K] [--doppler LO,HI,STEP] [--prn LIST]\n"
            "            [--threshold R] [--device D]\n"
            "            [--almanac FILE.sem --assist-pos LAT,LON,H --assist-time YYYY/MM/DD,hh:mm:ss[.s]\n"
            "             [--window HZ] [--mask DEG]]\n"
            "            [--fix --assist NAV_FILE[,3] --assist-pos LAT,LON,H|search --assist-time YYYY/MM/DD,hh:mm:ss[.s]\n"
            "             [--every MS] [--count N] [--iono a0,a1,a2,a3,b0,b1,b2,b3]\n"
            "             [--almanac FILE.sem [--window HZ] [--mask DEG]]\n"
            "             [--collective EXT_M,STEP_M[,EXT_S,STEP_S] [--mask DEG]]]\n"
            "  FILE              interleaved I,Q at 3 Msps, int8 (default) or int16 (--iq16)\n"
            "  --block B         start at 0.1 s block B (sample 300000 B); --offset-ms N adds N ms (3000 N samples)\n"
            "  --ms K            coherent 1 ms periods summed, 1..100 (default 10)\n"
            "  --doppler L,H,S   Doppler bins L, L+S, .. up to H, in Hz (default -5000,5000,250)\n"
            "  --prn LIST        e.g. 1-32 (default), 3,7,12-15\n"
            "  --threshold R     P1/P2 at or above R counts as acquired (default %.1f)\n"
            "  --almanac         warm start: search the PRNs of --prn predicted at or above the mask from the SEM file\n"
            "                    at --assist-pos / --assist-time (GPS time of the window's first sample), each over\n"
            "                    the bins of the --doppler step within --window Hz of its prediction (default %.0f)\n"
            "  --mask DEG        elevation mask of the warm start (default %.0f)\n"
            "  --fix             snapshot fixes from the window alone: the acquired PRNs refined (gpsb200_snapshot_measure),\n"
            "                    then a coarse-time fix from --assist-pos, or a search over a global grid with 'search';\n"
            "                    ephemeris from the RINEX file of --assist (,3: RINEX 3) at --assist-time, the GPS time\n"
            "                    of the first window's first sample; one window every --every ms (default 100), --count\n"
            "                    windows (default 1); --iono: the Klobuchar alpha / beta to apply; --almanac (with\n"
            "                    LAT,LON,H only): warm start every window from its own predicted sky\n"
            "  --collective      (with --fix and LAT,LON,H) collective detection per window: a lattice of +-EXT_M at\n"
            "                    STEP_M east and north and +-EXT_S at STEP_S in time (default 0: none) around the\n"
            "                    a-priori, scored over every PRN of the search (used: ephemeris valid, elevation at or\n"
            "                    above --mask); its seeds refined and fixed from the winner; the line adds the lattice\n"
            "                    status, runner-up / winner score, clock shift, time offset, used PRNs and how many of\n"
            "                    them passed --threshold alone\n",
            kDefaultThreshold, kDefaultWindow, kDefaultMask);
    exit(2);
}

// --fix: windows of a chunk go up packed and are searched and measured in one gpsb200_snapshot_batch call, at most
// kChunk at a time; each is then fixed alone. A batch call ends at a window whose Doppler result lies beyond the
// measurement's +-10 kHz before its pass is measured, where the single calls end at that window: with bins beyond
// +-10 kHz the windows go one per call, so that the lines printed before such a failure stay those of the single calls.
static const int kChunk = 100;

// The PRNs of the chunk's warm start: of the list, those predicted at or above the mask in any window of the chunk (the
// window at sample s[w] predicted at assist time sow + (s[w] - s0) / 3 MHz), each window with its own first bins f_lo
// [n][nprn] on the standard grid. false when the almanac cannot be predicted.
static bool warm_chunk(const gpsb200_almanac_record_t *alm, int32_t week, double sow, const double *x_a, long long s0,
                       const std::vector<long long> &s, double step, double window, double mask,
                       gpsb200_acq_config_t &cfg, std::vector<double> &f_lo) {
    const int n = (int) s.size(), h = (int) std::ceil(window / step - 1e-9);
    std::vector<gpsb200_sky_t> sky((size_t) n * 32);
    for (int w = 0; w < n; w++)
        if (gpsb200_almanac_predict(alm, week, sow + (double) (s[w] - s0) / 3e6, x_a, &sky[(size_t) w * 32]) != GPSB200_OK)
            return false;
    int np = 0;
    for (int i = 0; i < cfg.nprn; i++) {
        bool up = false;
        for (int w = 0; w < n; w++) {
            const gpsb200_sky_t &k = sky[(size_t) w * 32 + cfg.prn[i] - 1];
            up = up || (k.valid && k.el_deg >= mask);
        }
        if (up) cfg.prn[np++] = cfg.prn[i];
    }
    cfg.nprn = np;
    cfg.nbins = 2 * h + 1;
    f_lo.resize((size_t) n * np);
    for (int w = 0; w < n; w++)
        for (int q = 0; q < np; q++)
            f_lo[(size_t) w * np + q] = step * std::round(sky[(size_t) w * 32 + cfg.prn[q] - 1].doppler_hz / step) - h * step;
    return true;
}

// --fix: count windows every every_ms from sample s0, each searched on the standard grid (or, with an almanac, warm
// started), measured and fixed alone.
static int snapshot_fixes(const char *path, int ss, int device, long long s0, gpsb200_acq_config_t cfg, double lo,
                          double hi, double step, double threshold, const char *nav, int nav_v3, const double *x_a,
                          int32_t week, double sow, long long every_ms, long long count, gpsb200_pvt_config_t pcfg,
                          const gpsb200_almanac_record_t *alm, const char *almanac, double window, double mask) {
    cfg.f_lo_hz = lo;
    cfg.step_hz = step;
    cfg.nbins = (int) std::floor((hi - lo) / step + 1e-9) + 1;
    gpsb200_ephemeris_t eph[32];
    if (gpsb200_rinex_ephemeris(nav, nav_v3, week, sow, eph) != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: cannot read the ephemeris of %s\n", nav);
        return 1;
    }
    const size_t elem = ss == GPSB200_SC16 ? 2 : 1;
    const long long need = (long long) GPSB200_ACQ_CODE_SAMPLES * cfg.ms + GPSB200_ACQ_CODE_SAMPLES - 1;
    const long long have = file_samples(path, elem);
    FILE *f = fopen(path, "rb");
    if (have < 0 || !f) {
        fprintf(stderr, "gpsb200-acq: cannot open %s\n", path);
        return 1;
    }
    gpsb200_ctx_t *ctx = nullptr;
    if (create_rx_context(device, &ctx) != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: cannot create a context\n");
        fclose(f);
        return 1;
    }
    gpsb200_snapshot_config_t scfg;
    memset(&scfg, 0, sizeof scfg);
    scfg.min_ratio = threshold;
    scfg.iterations = GPSB200_SNAP_ITERATIONS;
    gpsb200_coarse_config_t ap;
    memset(&ap, 0, sizeof ap);
    if (x_a) memcpy(ap.x_a, x_a, sizeof ap.x_a);
    ap.t_a = sow;
    ap.s_a = s0;
    ap.week = week;
    gpsb200_search_config_t sc;
    memset(&sc, 0, sizeof sc);
    sc.t_a = sow;
    sc.s_a = s0;
    sc.week = week;
    sc.nodes = GPSB200_SEARCH_NODES;
    pcfg.nfix = 1;
    pcfg.step = 1;
    printf("# %s: snapshot fixes, %lld window(s) of %d ms every %lld ms from sample %lld, %s, Klobuchar %s\n", path,
           count, cfg.ms, every_ms, s0, x_a ? "coarse-time fix from the a-priori position" : "search over a global grid",
           pcfg.iono ? "on" : "off");
    if (alm)
        printf("# warm start from %s: the PRNs predicted at or above %.1f deg in a chunk's windows, %d bins of %.1f Hz "
               "around each window's prediction\n", almanac, mask, 2 * (int) std::ceil(window / step - 1e-9) + 1, step);
    printf("# sample  status  lat_deg  lon_deg  height_m  clock_m  vx  vy  vz (ECEF m/s)  channels  pdop  delta_s%s\n",
           x_a ? "" : "  support");
    static const char *const kStatus[] = {"OK", "FEW", "NO_CONVERGENCE", "AMBIGUOUS"};
    int rc = GPSB200_OK;
    std::vector<char> buf, one;
    bool inside = true;   // every window so far inside the file
    for (long long i = 0; i < count && inside && rc == GPSB200_OK;) {
        // the chunk: up to kChunk windows, packed, up to the first one not inside the file
        std::vector<long long> s;
        buf.clear();
        for (; i < count && (int) s.size() < kChunk; i++) {
            const long long si = s0 + i * every_ms * GPSB200_ACQ_CODE_SAMPLES;
            if (si + need > have || !read_at(f, si, need, elem, one)) {
                inside = false;
                break;
            }
            buf.insert(buf.end(), one.begin(), one.end());
            s.push_back(si);
        }
        const int n = (int) s.size();
        gpsb200_acq_config_t c = cfg;
        std::vector<double> f_lo;   // empty: the standard grid
        if (alm && !warm_chunk(alm, week, sow, x_a, s0, s, step, window, mask, c, f_lo)) {
            fprintf(stderr, "gpsb200-acq: cannot predict the almanac of %s\n", almanac);
            fclose(f);
            gpsb200_destroy(ctx);
            return 1;
        }
        std::vector<int64_t> off(n);
        for (int w = 0; w < n; w++) off[w] = (int64_t) w * need;
        bool doppler_inside = true;   // every bin within the measurement's +-10 kHz
        for (size_t r = 0; r < (f_lo.empty() ? 1 : f_lo.size()); r++) {
            const double b0 = f_lo.empty() ? c.f_lo_hz : f_lo[r], b1 = b0 + (c.nbins - 1) * c.step_hz;
            doppler_inside = doppler_inside && std::fabs(b0) <= 10000.0 && std::fabs(b1) <= 10000.0;
        }
        const int per = doppler_inside ? std::max(n, 1) : 1, np = c.nprn;
        std::vector<gpsb200_acq_result_t> res((size_t) n * np);
        std::vector<gpsb200_snapshot_t> meas((size_t) n * np);
        for (int w0 = 0; w0 < n && rc == GPSB200_OK; w0 += per) {
            const int m = std::min(per, n - w0);
            if (np > 0)
                rc = gpsb200_snapshot_batch(ctx, buf.data(), (int64_t) n * need, ss, &c, m, off.data() + w0,
                                            f_lo.empty() ? nullptr : f_lo.data() + (size_t) w0 * np, &scfg,
                                            res.data() + (size_t) w0 * np, meas.data() + (size_t) w0 * np);
            for (int w = w0; w < w0 + m && rc == GPSB200_OK; w++) {
                // the channels: the measured PRNs with an ephemeris valid at the assist time
                std::vector<gpsb200_pvt_chan_t> chans;
                std::vector<gpsb200_snapshot_t> row;
                for (int q = 0; q < np; q++) {
                    gpsb200_snapshot_t mq = meas[(size_t) w * np + q];
                    if (mq.status != GPSB200_SNAP_OK || !eph[mq.prn - 1].valid) continue;
                    gpsb200_pvt_chan_t pc;
                    memset(&pc, 0, sizeof pc);
                    pc.eph = eph[mq.prn - 1];
                    pc.prn = mq.prn;
                    chans.push_back(pc);
                    mq.sample = s[w];
                    row.push_back(mq);
                }
                gpsb200_fix_t fx;
                gpsb200_coarse_t co;
                gpsb200_search_t sr;
                if (chans.empty()) {
                    printf("%lld  FEW\n", s[w]);
                    continue;
                }
                rc = x_a ? gpsb200_pvt_snapshot(ctx, chans.data(), (int) chans.size(), row.data(), &pcfg, &ap, &fx,
                                                nullptr, &co, nullptr)
                         : gpsb200_pvt_snapshot_search(ctx, chans.data(), (int) chans.size(), row.data(), &pcfg, &sc,
                                                       &fx, nullptr, &sr, nullptr, nullptr);
                if (rc != GPSB200_OK) break;
                printf("%lld  %s  %.8f  %.8f  %.3f  %.3f  %.3f  %.3f  %.3f  %d  %.2f  %.9f", s[w], kStatus[fx.status],
                       fx.lat_deg, fx.lon_deg, fx.height, fx.clock_m, fx.vx, fx.vy, fx.vz, fx.nused, fx.pdop,
                       x_a ? co.delta : sr.delta);
                if (!x_a) printf("  %d", sr.support);
                printf("\n");
            }
        }
    }
    fclose(f);
    if (rc != GPSB200_OK) fprintf(stderr, "gpsb200-acq: %s\n", gpsb200_last_error(ctx));
    gpsb200_destroy(ctx);
    return rc == GPSB200_OK ? 0 : 1;
}

// --collective: count windows every every_ms from sample s0, each searched on the standard grid and scored against a
// lattice around the a-priori position and time (gpsb200_collective, DESIGN §11.7), one call per window; the seeds are
// measured with min_ratio 0 (gpsb200_snapshot_measure) and fixed from the winner (gpsb200_pvt_snapshot). lat: the
// lattice's sizes and steps (the a-priori time is that of the first window's first sample).
static int collective_fixes(const char *path, int ss, int device, long long s0, gpsb200_acq_config_t cfg, double lo,
                            double hi, double step, double threshold, const char *nav, int nav_v3, const double *x_a,
                            int32_t week, double sow, long long every_ms, long long count, gpsb200_pvt_config_t pcfg,
                            const gpsb200_collective_config_t &lat) {
    cfg.f_lo_hz = lo;
    cfg.step_hz = step;
    cfg.nbins = (int) std::floor((hi - lo) / step + 1e-9) + 1;
    cfg.s0 = 0;
    gpsb200_ephemeris_t eph[32];
    if (gpsb200_rinex_ephemeris(nav, nav_v3, week, sow, eph) != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: cannot read the ephemeris of %s\n", nav);
        return 1;
    }
    const size_t elem = ss == GPSB200_SC16 ? 2 : 1;
    const long long need = (long long) GPSB200_ACQ_CODE_SAMPLES * cfg.ms + GPSB200_ACQ_CODE_SAMPLES - 1;
    const long long have = file_samples(path, elem);
    FILE *f = fopen(path, "rb");
    if (have < 0 || !f) {
        fprintf(stderr, "gpsb200-acq: cannot open %s\n", path);
        return 1;
    }
    gpsb200_ctx_t *ctx = nullptr;
    if (create_rx_context(device, &ctx) != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: cannot create a context\n");
        fclose(f);
        return 1;
    }
    gpsb200_snapshot_config_t scfg;
    memset(&scfg, 0, sizeof scfg);
    scfg.iterations = GPSB200_SNAP_ITERATIONS;   // min_ratio 0: every seeded PRN, none of the others (ratio -1)
    pcfg.nfix = 1;
    pcfg.step = 1;
    printf("# %s: collective detection and snapshot fixes, %lld window(s) of %d ms every %lld ms from sample %lld, "
           "lattice %d x %d x %d x %d (east, north, up at %.1f m, time at %.3f s), mask %.1f deg, Klobuchar %s\n", path,
           count, cfg.ms, every_ms, s0, lat.n[0], lat.n[1], lat.n[2], lat.n[3], lat.step[0], lat.step[3], lat.mask_deg,
           pcfg.iono ? "on" : "off");
    printf("# sample  status  lat_deg  lon_deg  height_m  clock_m  vx  vy  vz (ECEF m/s)  channels  pdop  delta_s  "
           "collective  score_ratio  shift  o_t_s  used_prns  alone\n");
    static const char *const kStatus[] = {"OK", "FEW", "NO_CONVERGENCE", "AMBIGUOUS"};
    static const char *const kCd[] = {"OK", "FEW", "AMBIGUOUS"};
    const int np = cfg.nprn;
    std::vector<gpsb200_acq_result_t> res(np), seed(np);
    std::vector<gpsb200_snapshot_t> meas(np);
    std::vector<char> one;
    int rc = GPSB200_OK;
    for (long long i = 0; i < count && rc == GPSB200_OK; i++) {
        const long long si = s0 + i * every_ms * GPSB200_ACQ_CODE_SAMPLES;
        if (si + need > have || !read_at(f, si, need, elem, one)) break;
        // the a-priori time at this window's first sample, in the window's own sample numbers
        gpsb200_coarse_config_t ap;
        memset(&ap, 0, sizeof ap);
        memcpy(ap.x_a, x_a, sizeof ap.x_a);
        const double t = sow + (double) (si - s0) / 3e6;
        const double kw = std::floor(t / 604800.0);
        ap.t_a = t - 604800.0 * kw;
        ap.week = week + (int32_t) kw;
        gpsb200_collective_t cd;
        rc = gpsb200_collective(ctx, one.data(), need, ss, &cfg, nullptr, eph, &ap, &lat, res.data(), seed.data(), &cd,
                                nullptr, nullptr);
        if (rc != GPSB200_OK) break;
        int alone = 0;
        std::string used;
        for (int q = 0; q < np; q++) {
            alone += (cd.used >> q & 1) && res[q].ratio >= threshold;
            if (cd.used >> q & 1) used += (used.empty() ? "" : ",") + std::to_string(cfg.prn[q]);
        }
        if (used.empty()) used = "-";
        char tail[256];
        snprintf(tail, sizeof tail, "  %s  %.4f  %d  %.3f  %s  %d", kCd[cd.status],
                 cd.score ? (double) cd.runner_score / (double) cd.score : 0.0, cd.shift, cd.o_t, used.c_str(), alone);
        if (cd.winner < 0) {
            printf("%lld  FEW%s\n", si, tail);
            continue;
        }
        rc = gpsb200_snapshot_measure(ctx, one.data(), need, ss, &cfg, seed.data(), &scfg, meas.data());
        if (rc != GPSB200_OK) break;
        std::vector<gpsb200_pvt_chan_t> chans;
        std::vector<gpsb200_snapshot_t> row;
        for (int q = 0; q < np; q++) {
            gpsb200_snapshot_t mq = meas[q];
            if (mq.status != GPSB200_SNAP_OK || !eph[mq.prn - 1].valid) continue;
            gpsb200_pvt_chan_t pc;
            memset(&pc, 0, sizeof pc);
            pc.eph = eph[mq.prn - 1];
            pc.prn = mq.prn;
            chans.push_back(pc);
            mq.sample = si;
            row.push_back(mq);
        }
        if (chans.empty()) {
            printf("%lld  FEW%s\n", si, tail);
            continue;
        }
        // the winner as the a-priori of the coarse-time fix, at this window's first sample
        gpsb200_coarse_config_t wp = ap;
        memcpy(wp.x_a, cd.x, sizeof wp.x_a);
        const double tw = ap.t_a + cd.o_t, kt = std::floor(tw / 604800.0);
        wp.t_a = tw - 604800.0 * kt;
        wp.week = ap.week + (int32_t) kt;
        wp.s_a = si;
        gpsb200_fix_t fx;
        gpsb200_coarse_t co;
        rc = gpsb200_pvt_snapshot(ctx, chans.data(), (int) chans.size(), row.data(), &pcfg, &wp, &fx, nullptr, &co,
                                  nullptr);
        if (rc != GPSB200_OK) break;
        printf("%lld  %s  %.8f  %.8f  %.3f  %.3f  %.3f  %.3f  %.3f  %d  %.2f  %.9f%s\n", si, kStatus[fx.status],
               fx.lat_deg, fx.lon_deg, fx.height, fx.clock_m, fx.vx, fx.vy, fx.vz, fx.nused, fx.pdop, co.delta, tail);
    }
    fclose(f);
    if (rc != GPSB200_OK) fprintf(stderr, "gpsb200-acq: %s\n", gpsb200_last_error(ctx));
    gpsb200_destroy(ctx);
    return rc == GPSB200_OK ? 0 : 1;
}

int main(int argc, char **argv) {
    const char *path = nullptr;
    int ss = GPSB200_SC08, device = 0;
    long long block = 0, offset_ms = 0;
    double lo = -5000.0, hi = 5000.0, step = 250.0, threshold = kDefaultThreshold;
    gpsb200_acq_config_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.ms = 10;
    const char *almanac = nullptr;
    double x_a[3] = {0.0, 0.0, 0.0}, sow = 0.0, window = kDefaultWindow, mask = kDefaultMask;
    int32_t week = 0;
    bool have_pos = false, have_time = false;
    bool fix = false, pos_search = false, collective = false;
    gpsb200_collective_config_t lattice;
    memset(&lattice, 0, sizeof lattice);
    std::string assist;
    int assist_v3 = 0;
    long long every_ms = 100, count = 1;
    gpsb200_pvt_config_t pcfg;
    memset(&pcfg, 0, sizeof pcfg);
    parse_prns("1-32", &cfg);
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto val = [&]() -> const char * {
            if (i + 1 >= argc) usage();
            return argv[++i];
        };
        if (a == "--iq16") ss = GPSB200_SC16;
        else if (a == "--block") block = atoll(val());
        else if (a == "--offset-ms") offset_ms = atoll(val());
        else if (a == "--ms") cfg.ms = atoi(val());
        else if (a == "--doppler") {
            if (sscanf(val(), "%lf,%lf,%lf", &lo, &hi, &step) != 3 || !(step > 0.0) || hi < lo) usage();
        } else if (a == "--prn") {
            if (!parse_prns(val(), &cfg)) usage();
        } else if (a == "--threshold") threshold = atof(val());
        else if (a == "--device") device = atoi(val());
        else if (a == "--almanac") almanac = val();
        else if (a == "--assist-pos" && i + 1 < argc && std::string(argv[i + 1]) == "search") {
            i++;
            have_pos = pos_search = true;
        } else if (a == "--assist-pos") {
            if (!ecef_of_llh(val(), x_a)) usage();
            have_pos = true;
        } else if (a == "--assist-time") {
            if (!gps_of_date(val(), week, sow)) usage();
            have_time = true;
        } else if (a == "--window") {
            window = atof(val());
            if (!(window >= 0.0)) usage();
        } else if (a == "--mask") mask = atof(val());
        else if (a == "--fix") fix = true;
        else if (a == "--collective") {
            double ext = 0.0, st = 0.0, ext_s = 0.0, st_s = 1.0;
            const int k = sscanf(val(), "%lf,%lf,%lf,%lf", &ext, &st, &ext_s, &st_s);
            if ((k != 2 && k != 4) || !(ext >= 0.0) || !(st > 0.0) || !(ext_s >= 0.0) || !(st_s > 0.0)) usage();
            const double ext_a[4] = {ext, ext, 0.0, ext_s}, st_a[4] = {st, st, 1.0, st_s};
            for (int ax = 0; ax < 4; ax++) {
                lattice.n[ax] = 2 * (int) std::floor(ext_a[ax] / st_a[ax] + 1e-9) + 1;
                lattice.step[ax] = st_a[ax];
            }
            lattice.distinct_m = std::max(kDistinct, 2.0 * st);
            collective = true;
        }
        else if (a == "--assist") {
            assist = val();
            const size_t k = assist.rfind(',');
            if (k != std::string::npos) {
                if (assist.substr(k + 1) != "3") usage();
                assist_v3 = 1;
                assist.resize(k);
            }
        } else if (a == "--every") every_ms = atoll(val());
        else if (a == "--count") count = atoll(val());
        else if (a == "--iono") {
            double *ab = pcfg.alpha;
            double *bb = pcfg.beta;
            if (sscanf(val(), "%lf,%lf,%lf,%lf,%lf,%lf,%lf,%lf", ab, ab + 1, ab + 2, ab + 3, bb, bb + 1, bb + 2, bb + 3) != 8)
                usage();
            pcfg.iono = 1;
        }
        else if (a[0] != '-' && !path) path = argv[i];
        else usage();
    }
    if (!path || block < 0 || offset_ms < 0 || (almanac && (!have_pos || !have_time || pos_search)) ||
        (!almanac && !fix && (have_pos || have_time)) || (fix && (assist.empty() || !have_pos || !have_time)) ||
        (!fix && (!assist.empty() || pcfg.iono)) || every_ms < 1 || count < 1 ||
        (collective && (!fix || pos_search || almanac)))
        usage();
    if (collective) {
        lattice.mask_deg = mask;
        return collective_fixes(path, ss, device, block * GPSB200_BLOCK_SAMPLES + offset_ms * GPSB200_ACQ_CODE_SAMPLES,
                                cfg, lo, hi, step, threshold, assist.c_str(), assist_v3, x_a, week, sow, every_ms, count,
                                pcfg, lattice);
    }
    if (fix) {
        gpsb200_almanac_record_t rec[32];
        int32_t valid = 0;
        if (almanac && gpsb200_almanac_read(almanac, rec, &valid) != GPSB200_OK) {
            fprintf(stderr, "gpsb200-acq: cannot read the almanac of %s\n", almanac);
            return 1;
        }
        return snapshot_fixes(path, ss, device, block * GPSB200_BLOCK_SAMPLES + offset_ms * GPSB200_ACQ_CODE_SAMPLES, cfg,
                              lo, hi, step, threshold, assist.c_str(), assist_v3, pos_search ? nullptr : x_a, week, sow,
                              every_ms, count, pcfg, almanac ? rec : nullptr, almanac, window, mask);
    }
    cfg.f_lo_hz = lo;
    cfg.step_hz = step;
    cfg.nbins = (int) std::floor((hi - lo) / step + 1e-9) + 1;
    // warm start: the PRNs of the list predicted at or above the mask, each with its own first bin
    std::vector<double> f_lo_prn;
    gpsb200_sky_t sky[32];
    if (almanac) {
        gpsb200_almanac_record_t rec[32];
        int32_t valid = 0;
        if (gpsb200_almanac_read(almanac, rec, &valid) != GPSB200_OK ||
            gpsb200_almanac_predict(rec, week, sow, x_a, sky) != GPSB200_OK) {
            fprintf(stderr, "gpsb200-acq: cannot read the almanac of %s\n", almanac);
            return 1;
        }
        const int h = (int) std::ceil(window / step - 1e-9);
        int n = 0;
        for (int i = 0; i < cfg.nprn; i++) {
            const gpsb200_sky_t &k = sky[cfg.prn[i] - 1];
            if (!k.valid || !(k.el_deg >= mask)) continue;
            cfg.prn[n++] = cfg.prn[i];
            f_lo_prn.push_back(step * std::round(k.doppler_hz / step) - h * step);
        }
        cfg.nprn = n;
        cfg.nbins = 2 * h + 1;
        if (n == 0) {
            printf("# %s: no PRN of the list is predicted at or above %.1f deg\n", path, mask);
            return 0;
        }
    }

    const size_t elem = ss == GPSB200_SC16 ? 2 : 1;
    const long long s0 = block * GPSB200_BLOCK_SAMPLES + offset_ms * GPSB200_ACQ_CODE_SAMPLES;
    const long long need = (long long) GPSB200_ACQ_CODE_SAMPLES * cfg.ms + GPSB200_ACQ_CODE_SAMPLES - 1;
    const long long have = file_samples(path, elem);
    if (have < 0) {
        fprintf(stderr, "gpsb200-acq: cannot open %s\n", path);
        return 1;
    }
    if (cfg.ms < 1 || cfg.ms > GPSB200_ACQ_MAX_MS || s0 + need > have) {
        fprintf(stderr, "gpsb200-acq: the window (sample %lld, %lld samples) is not inside %s (%lld samples)\n", s0, need,
                path, have);
        return 1;
    }
    std::vector<char> buf;
    FILE *f = fopen(path, "rb");
    if (!f || !read_at(f, s0, need, elem, buf)) {
        fprintf(stderr, "gpsb200-acq: cannot read the window of %s\n", path);
        return 1;
    }
    fclose(f);

    gpsb200_ctx_t *ctx = nullptr;
    int rc = create_rx_context(device, &ctx);
    std::vector<gpsb200_acq_result_t> res(cfg.nprn);
    if (rc == GPSB200_OK)
        rc = almanac ? gpsb200_acquire_windows(ctx, buf.data(), need, ss, &cfg, f_lo_prn.data(), res.data(), nullptr)
                     : gpsb200_acquire(ctx, buf.data(), need, ss, &cfg, res.data(), nullptr);
    if (rc != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: %s\n", ctx ? gpsb200_last_error(ctx) : "cannot create a context");
        gpsb200_destroy(ctx);
        return 1;
    }
    gpsb200_destroy(ctx);
    if (almanac) {
        printf("# %s: sample %lld, %d ms, warm start from %s: %d PRN(s) at or above %.1f deg, %d bins of %.1f Hz "
               "around each prediction, threshold P1/P2 >= %.2f\n",
               path, s0, cfg.ms, almanac, cfg.nprn, mask, cfg.nbins, step, threshold);
        printf("# PRN  doppler_hz  delay_samples  delay_chips  P1/P2  acquired  predicted_hz  elevation_deg\n");
    } else {
        printf("# %s: sample %lld, %d ms, %d bins %.1f .. %.1f Hz, threshold P1/P2 >= %.2f\n", path, s0, cfg.ms,
               cfg.nbins, lo, lo + (cfg.nbins - 1) * step, threshold);
        printf("# PRN  doppler_hz  delay_samples  delay_chips  P1/P2  acquired\n");
    }
    int nacq = 0;
    for (const auto &r : res) {
        const bool acq = r.ratio >= threshold;
        nacq += acq;
        printf("%5d  %10.1f  %13d  %11.3f  %8.3f  %s", r.prn, r.doppler_hz, r.delay, r.delay_chips, r.ratio,
               acq ? "yes" : "no");
        if (almanac) printf("  %12.1f  %13.2f", sky[r.prn - 1].doppler_hz, sky[r.prn - 1].el_deg);
        printf("\n");
    }
    printf("# %d of %d acquired\n", nacq, cfg.nprn);
    return 0;
}
