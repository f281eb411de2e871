// gpsb200-track: acquire, track and decode the navigation messages of a 3 Msps I/Q file (gpsb200-sim's output, the
// reference's iqdata.bin, any capture in these formats: int8 or, with --iq16, int16 I,Q interleaved). The acquisition
// is gpsb200_acquire at the start offset (10 coherent periods, bins of 100 Hz over +-5 kHz, so that the loops start
// within their pull-in range); every PRN whose P1/P2 reaches the threshold is tracked with gpsb200_track over the file,
// read in chunks of one second, and decoded with gpsb200_nav_decode. Prints one line per tracked PRN: locked at the
// end or not, the Doppler at the end, subframes found, words with good parity and the first TOW (DESIGN §10).
// With --fix it then computes position fixes with gpsb200_pvt from what it decoded alone: each channel's ephemeris
// (gpsb200_nav_ephemeris) and time anchor (gpsb200_nav_time_anchor); channels without both are left out. The fixes
// start 0.5 s after the acquisition window (the loops have pulled in by then) and follow every --fix-every ms; one line
// per fix with status GPSB200_FIX_OK (DESIGN §11). With --raim the fixes come from gpsb200_pvt_raim and each line gains
// the RAIM verdict, the PRNs it excluded ("-" for none) and HPL/VPL in metres (DESIGN §11.1). With --araim they come
// from gpsb200_pvt_araim and each line gains the ARAIM verdict, the excluded PRN, the PRNs below the elevation mask
// ("-" for none), HPL/VPL and the EMT in metres (DESIGN §11.2).
// With --assist the fixes are coarse-time fixes (gpsb200_pvt_coarse, DESIGN §11.3): nothing needs to be decoded. The
// ephemeris comes from a RINEX navigation file (gpsb200_rinex_ephemeris, at the assist time), the a-priori position
// from --assist-pos and the a-priori time from --assist-time, the GPS time of the first sample after --block /
// --offset-ms; each line gains delta, the solved a-priori time error in seconds. With --assist-pos search there is no
// a-priori position: the fixes come from gpsb200_pvt_search over the default global grid (DESIGN §11.4) and each line
// gains delta and then support, the number of grid nodes whose solve agreed with the fix.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../include/gpsb200.h"
#include "rx_cli.h"

static const double kDefaultThreshold = 2.5;      // as gpsb200-acq
static const int kAcqMs = 10;
static const double kAcqLo = -5000.0, kAcqHi = 5000.0, kAcqStep = 100.0;
static const long long kChunk = 3000000;          // samples per tracking call: 1 s
static const int kDefaultFixEvery = 1000;         // ms between fixes
static const long long kFixLead = 1500000;        // samples from the start to the first fix: 0.5 s of pull-in

static void usage() {
    fprintf(stderr,
            "gpsb200-track FILE [--iq16] [--block B] [--offset-ms N] [--ms K] [--prn LIST] [--threshold R] [--device D]\n"
            "              [--fix [--fix-every MS] [--iono a0,a1,a2,a3,b0,b1,b2,b3] [--raim SIGMA[,P_FA,P_MD[,MAX_EXCLUDE]]]\n"
            "               [--araim MASK_DEG[,SIGMA_URA,SIGMA_URE,B_NOM,P_SAT]]\n"
            "               [--assist NAV_FILE[,3] --assist-pos LAT,LON,H|search --assist-time YYYY/MM/DD,hh:mm:ss[.s]]]\n"
            "  FILE              interleaved I,Q at 3 Msps, int8 (default) or int16 (--iq16)\n"
            "  --block B         start at 0.1 s block B (sample 300000 B); --offset-ms N adds N ms (3000 N samples)\n"
            "  --ms K            track K ms of signal from the start (default: to the end of the file)\n"
            "  --prn LIST        PRNs searched, e.g. 1-32 (default), 3,7,12-15\n"
            "  --threshold R     P1/P2 at or above R counts as acquired and is tracked (default %.1f)\n"
            "  --fix             position, velocity and time from the decoded ephemeris and TOW, every --fix-every ms\n"
            "                    (default %d) from 0.5 s after the start; --iono: the Klobuchar alpha / beta to apply\n"
            "  --raim            fault detection and exclusion with pseudorange sigma SIGMA m (P_FA 1e-5, P_MD 1e-3,\n"
            "                    MAX_EXCLUDE 1 by default): adds the verdict, the excluded PRNs and HPL/VPL to each fix\n"
            "  --araim           advanced RAIM with elevation mask MASK_DEG (the other fields: the header's defaults): adds\n"
            "                    the verdict, the excluded PRN, the masked PRNs, HPL/VPL and the EMT to each fix\n"
            "  --assist          coarse-time fixes without decoding: ephemeris from the RINEX file (,3: RINEX 3), a-priori\n"
            "                    position (deg, deg, m) and GPS time of the first sample; adds delta (s) to each fix.\n"
            "                    --assist-pos search: no a-priori position, a search over a global grid; adds delta (s)\n"
            "                    and support\n",
            kDefaultThreshold, kDefaultFixEvery);
    exit(2);
}

static const char *const kVerdict[] = {"PASS", "EXCLUDED", "ALERT", "UNAVAILABLE"};

// Fixes from `first` every `step` samples to the last epoch of the channels, one line per fix with status OK; with
// raim (not NULL) from gpsb200_pvt_raim, with its three columns; with araim (not NULL) from gpsb200_pvt_araim, with its five;
// with ap (not NULL) from gpsb200_pvt_coarse, with delta, or with search also set from gpsb200_pvt_search over the default
// grid (ap's position unused), with delta and support.
static int print_fixes(gpsb200_ctx_t *ctx, const std::vector<gpsb200_pvt_chan_t> &chans, const std::vector<int> &of,
                       const std::vector<std::vector<gpsb200_track_epoch_t>> &eps, long long first, long long step,
                       gpsb200_pvt_config_t cfg, const gpsb200_raim_config_t *raim,
                       const gpsb200_araim_config_t *araim, const gpsb200_coarse_config_t *ap, bool search) {
    const int n = (int) chans.size();
    if (ap && search)
        printf("# position-search fixes (no a-priori position, %d-node grid): %d channel(s) with an assisted ephemeris, "
               "Klobuchar %s\n", GPSB200_SEARCH_NODES, n, cfg.iono ? "on" : "off");
    else if (ap)
        printf("# coarse-time fixes: %d channel(s) with an assisted ephemeris, Klobuchar %s\n", n, cfg.iono ? "on" : "off");
    else
        printf("# fixes: %d channel(s) with an ephemeris and a time anchor decoded, Klobuchar %s\n", n,
               cfg.iono ? "on" : "off");
    if (n == 0) return GPSB200_OK;
    size_t me = 1;
    long long end = 0;
    for (int c : of) {
        me = std::max(me, eps[c].size());
        if (!eps[c].empty()) end = std::max(end, (long long) eps[c].back().sample);
    }
    if (end < first) return GPSB200_OK;
    std::vector<gpsb200_track_epoch_t> all((size_t) n * me);
    std::vector<int32_t> cnt(n);
    for (int k = 0; k < n; k++) {
        std::copy(eps[of[k]].begin(), eps[of[k]].end(), all.begin() + (size_t) k * me);
        cnt[k] = (int32_t) eps[of[k]].size();
    }
    cfg.s0 = first;
    cfg.step = step;
    cfg.nfix = (int32_t) ((end - first) / step + 1);
    std::vector<gpsb200_fix_t> fx(cfg.nfix);
    std::vector<gpsb200_raim_t> rm(raim ? cfg.nfix : 0);
    std::vector<gpsb200_araim_t> am(araim ? cfg.nfix : 0);
    std::vector<gpsb200_coarse_t> cm(ap && !search ? cfg.nfix : 0);
    std::vector<gpsb200_search_t> sm(ap && search ? cfg.nfix : 0);
    gpsb200_search_config_t sc;
    memset(&sc, 0, sizeof sc);
    if (ap) {
        sc.t_a = ap->t_a;
        sc.s_a = ap->s_a;
        sc.week = ap->week;
        sc.nodes = GPSB200_SEARCH_NODES;
    }
    const int rc = ap && search ? gpsb200_pvt_search(ctx, chans.data(), n, all.data(), cnt.data(), (int) me, &cfg, &sc,
                                                     fx.data(), nullptr, sm.data(), nullptr, nullptr)
                   : ap ? gpsb200_pvt_coarse(ctx, chans.data(), n, all.data(), cnt.data(), (int) me, &cfg, ap, fx.data(),
                                           nullptr, cm.data(), nullptr)
                   : araim ? gpsb200_pvt_araim(ctx, chans.data(), n, all.data(), cnt.data(), (int) me, &cfg, araim,
                                             fx.data(), nullptr, am.data())
                   : raim ? gpsb200_pvt_raim(ctx, chans.data(), n, all.data(), cnt.data(), (int) me, &cfg, raim, fx.data(),
                                             nullptr, rm.data())
                          : gpsb200_pvt(ctx, chans.data(), n, all.data(), cnt.data(), (int) me, &cfg, fx.data(), nullptr);
    if (rc != GPSB200_OK) return rc;
    printf("# sample  tow_s  lat_deg  lon_deg  height_m  clock_m  vx  vy  vz (ECEF m/s)  channels  pdop%s\n",
           raim ? "  raim  excluded_prns  hpl/vpl_m"
                : (araim ? "  araim  excluded_prn  masked_prns  hpl/vpl_m  emt_m"
                         : (ap ? (search ? "  delta_s  support" : "  delta_s") : "")));
    for (int i = 0; i < cfg.nfix; i++) {
        const gpsb200_fix_t &f = fx[i];
        if (f.status != GPSB200_FIX_OK) continue;
        printf("%lld  %.9f  %.8f  %.8f  %.3f  %.3f  %.3f  %.3f  %.3f  %d  %.2f", (long long) f.sample, f.t_rx, f.lat_deg,
               f.lon_deg, f.height, f.clock_m, f.vx, f.vy, f.vz, f.nused, f.pdop);
        if (raim) {
            std::string ex;
            for (int k = 0; k < n; k++)
                if (rm[i].excluded >> k & 1u) ex += (ex.empty() ? "" : ",") + std::to_string(chans[k].prn);
            printf("  %s  %s  %.2f/%.2f", kVerdict[rm[i].verdict], ex.empty() ? "-" : ex.c_str(), rm[i].hpl, rm[i].vpl);
        }
        if (araim) {
            std::string ex, mk;
            for (int k = 0; k < n; k++) {
                if (am[i].excluded >> k & 1u) ex += (ex.empty() ? "" : ",") + std::to_string(chans[k].prn);
                if (am[i].masked >> k & 1u) mk += (mk.empty() ? "" : ",") + std::to_string(chans[k].prn);
            }
            printf("  %s  %s  %s  %.2f/%.2f  %.2f", kVerdict[am[i].verdict], ex.empty() ? "-" : ex.c_str(),
                   mk.empty() ? "-" : mk.c_str(), am[i].hpl, am[i].vpl, am[i].emt);
        }
        if (ap && search) printf("  %.9f  %d", sm[i].delta, sm[i].support);
        else if (ap) printf("  %.9f", cm[i].delta);
        printf("\n");
    }
    return GPSB200_OK;
}

int main(int argc, char **argv) {
    const char *path = nullptr;
    int ss = GPSB200_SC08, device = 0;
    long long block = 0, offset_ms = 0, ms = -1;
    double threshold = kDefaultThreshold;
    bool fix = false;
    long long fix_every = kDefaultFixEvery;
    gpsb200_pvt_config_t pcfg;
    memset(&pcfg, 0, sizeof pcfg);
    bool raim = false;
    gpsb200_raim_config_t rcfg;
    memset(&rcfg, 0, sizeof rcfg);
    bool araim = false;
    gpsb200_araim_config_t acfg;
    memset(&acfg, 0, sizeof acfg);
    std::string assist;
    int assist_v3 = 0;
    bool assist_pos = false, assist_time = false, assist_search = false;
    gpsb200_coarse_config_t ap;
    memset(&ap, 0, sizeof ap);
    gpsb200_acq_config_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.ms = kAcqMs;
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
        else if (a == "--ms") ms = atoll(val());
        else if (a == "--prn") {
            if (!parse_prns(val(), &cfg)) usage();
        } else if (a == "--threshold") threshold = atof(val());
        else if (a == "--device") device = atoi(val());
        else if (a == "--fix") fix = true;
        else if (a == "--fix-every") fix_every = atoll(val());
        else if (a == "--iono") {
            double *v[8] = {&pcfg.alpha[0], &pcfg.alpha[1], &pcfg.alpha[2], &pcfg.alpha[3],
                            &pcfg.beta[0], &pcfg.beta[1], &pcfg.beta[2], &pcfg.beta[3]};
            if (sscanf(val(), "%lf,%lf,%lf,%lf,%lf,%lf,%lf,%lf", v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]) != 8) usage();
            pcfg.iono = 1;
        } else if (a == "--raim") {
            rcfg.p_fa = 1e-5;
            rcfg.p_md = 1e-3;
            rcfg.max_exclude = 1;
            const int got = sscanf(val(), "%lf,%lf,%lf,%d", &rcfg.sigma, &rcfg.p_fa, &rcfg.p_md, &rcfg.max_exclude);
            if (got != 1 && got != 3 && got != 4) usage();
            raim = true;
        } else if (a == "--araim") {
            acfg.sigma_ura = GPSB200_ARAIM_SIGMA_URA;
            acfg.sigma_ure = GPSB200_ARAIM_SIGMA_URE;
            acfg.sigma_noise = GPSB200_ARAIM_SIGMA_NOISE;
            acfg.b_nom = GPSB200_ARAIM_B_NOM;
            acfg.p_sat = GPSB200_ARAIM_P_SAT;
            acfg.p_hmi_vert = GPSB200_ARAIM_P_HMI_VERT;
            acfg.p_hmi_horz = GPSB200_ARAIM_P_HMI_HORZ;
            acfg.p_fa_vert = GPSB200_ARAIM_P_FA_VERT;
            acfg.p_fa_horz = GPSB200_ARAIM_P_FA_HORZ;
            acfg.max_exclude = 1;
            const int got = sscanf(val(), "%lf,%lf,%lf,%lf,%lf", &acfg.mask_deg, &acfg.sigma_ura, &acfg.sigma_ure,
                                   &acfg.b_nom, &acfg.p_sat);
            if (got != 1 && got != 5) usage();
            araim = true;
        } else if (a == "--assist") {
            assist = val();
            const size_t k = assist.rfind(',');
            if (k != std::string::npos) {
                if (assist.substr(k + 1) != "3") usage();
                assist_v3 = 1;
                assist.resize(k);
            }
        } else if (a == "--assist-pos" && i + 1 < argc && std::string(argv[i + 1]) == "search") {
            i++;
            assist_pos = assist_search = true;
        } else if (a == "--assist-pos") {
            if (!ecef_of_llh(val(), ap.x_a)) usage();
            assist_pos = true;
        } else if (a == "--assist-time") {
            if (!gps_of_date(val(), ap.week, ap.t_a)) usage();
            assist_time = true;
        }
        else if (a[0] != '-' && !path) path = argv[i];
        else usage();
    }
    const bool coarse = !assist.empty();
    if (!path || block < 0 || offset_ms < 0 || ms == 0 || ms < -1 || fix_every < 1 || ((raim || araim) && !fix) ||
        (raim && araim) || (coarse && (!fix || raim || araim || !assist_pos || !assist_time)) ||
        (!coarse && (assist_pos || assist_time)))
        usage();
    cfg.f_lo_hz = kAcqLo;
    cfg.step_hz = kAcqStep;
    cfg.nbins = (int) std::floor((kAcqHi - kAcqLo) / kAcqStep + 1e-9) + 1;

    const size_t elem = ss == GPSB200_SC16 ? 2 : 1;
    const long long s0 = block * GPSB200_BLOCK_SAMPLES + offset_ms * GPSB200_ACQ_CODE_SAMPLES;
    ap.s_a = s0;
    gpsb200_ephemeris_t assisted[32];
    if (coarse && gpsb200_rinex_ephemeris(assist.c_str(), assist_v3, ap.week, ap.t_a, assisted) != GPSB200_OK) {
        fprintf(stderr, "gpsb200-track: cannot read the ephemeris of %s\n", assist.c_str());
        return 1;
    }
    const long long need = (long long) GPSB200_ACQ_CODE_SAMPLES * cfg.ms + GPSB200_ACQ_CODE_SAMPLES - 1;
    const long long have = file_samples(path, elem);
    if (have < 0) {
        fprintf(stderr, "gpsb200-track: cannot open %s\n", path);
        return 1;
    }
    if (s0 + need > have) {
        fprintf(stderr, "gpsb200-track: the acquisition window (sample %lld, %lld samples) is not inside %s (%lld samples)\n",
                s0, need, path, have);
        return 1;
    }
    const long long end = ms > 0 ? std::min(have, s0 + ms * GPSB200_ACQ_CODE_SAMPLES) : have;
    FILE *f = fopen(path, "rb");
    std::vector<char> buf;
    if (!f || !read_at(f, s0, need, elem, buf)) {
        fprintf(stderr, "gpsb200-track: cannot read the acquisition window of %s\n", path);
        if (f) fclose(f);
        return 1;
    }

    gpsb200_ctx_t *ctx = nullptr;
    int rc = create_rx_context(device, &ctx);
    std::vector<gpsb200_acq_result_t> res(cfg.nprn);
    if (rc == GPSB200_OK) rc = gpsb200_acquire(ctx, buf.data(), need, ss, &cfg, res.data(), nullptr);
    std::vector<gpsb200_track_state_t> state;
    for (const auto &r : res)
        if (rc == GPSB200_OK && r.ratio >= threshold) {
            gpsb200_track_state_t t;
            if (gpsb200_track_start(r.prn, r.doppler_hz, s0 + r.delay, &t) == GPSB200_OK) state.push_back(t);
        }
    const int nch = (int) state.size();
    std::vector<std::vector<gpsb200_track_epoch_t>> eps(nch);
    const int max_ep = (int) (kChunk / 2999 + 1);
    std::vector<gpsb200_track_epoch_t> out((size_t) std::max(nch, 1) * max_ep);
    std::vector<int32_t> n(std::max(nch, 1));
    while (rc == GPSB200_OK && nch > 0) {
        long long base = state[0].sample;
        for (const auto &t : state) base = std::min(base, (long long) t.sample);
        const long long cnt = std::min(kChunk, end - base);
        if (cnt <= 0) break;
        if (!read_at(f, base, cnt, elem, buf)) {
            fprintf(stderr, "gpsb200-track: cannot read %s at sample %lld\n", path, base);
            rc = GPSB200_ERR_ARG;
            break;
        }
        rc = gpsb200_track(ctx, buf.data(), cnt, ss, base, state.data(), nch, max_ep, out.data(), n.data());
        long long got = 0;
        for (int c = 0; c < nch && rc == GPSB200_OK; c++) {
            eps[c].insert(eps[c].end(), out.begin() + (size_t) c * max_ep, out.begin() + (size_t) c * max_ep + n[c]);
            got += n[c];
        }
        if (got == 0) break;
    }
    fclose(f);
    if (rc != GPSB200_OK) {
        fprintf(stderr, "gpsb200-track: %s\n", ctx ? gpsb200_last_error(ctx) : "cannot create a context");
        gpsb200_destroy(ctx);
        return 1;
    }
    printf("# %s: sample %lld to %lld, %d of %d PRNs acquired (P1/P2 >= %.2f) and tracked\n", path, s0, end, nch, cfg.nprn,
           threshold);
    printf("# PRN  locked  doppler_hz  subframes  words_ok  words  first_tow\n");
    std::vector<gpsb200_pvt_chan_t> fix_chans;
    std::vector<int> fix_of;
    for (int c = 0; c < nch; c++) {
        const auto &e = eps[c];
        const int64_t ne = (int64_t) e.size();
        std::vector<gpsb200_nav_bit_t> bits((size_t) (ne / 20 + 1));
        std::vector<gpsb200_nav_word_t> words((size_t) (ne / 600 + 1));
        gpsb200_nav_sync_t sy;
        gpsb200_nav_decode(e.data(), ne, bits.data(), (int64_t) bits.size(), words.data(), (int64_t) words.size(), &sy);
        const bool locked = ne > 0 && e.back().lock;
        const double dopp = ne > 0 ? e.back().carr_step * 3e6 / 4294967296.0 : 0.0;
        printf("%5d  %6s  %10.1f  %9d  %8d  %5d  %9d\n", state[c].prn, locked ? "yes" : "no", dopp, sy.subframes,
               sy.words_ok, sy.nwords, sy.first_tow);
        if (fix && coarse) {
            gpsb200_pvt_chan_t pc;
            memset(&pc, 0, sizeof pc);
            pc.eph = assisted[state[c].prn - 1];
            pc.prn = state[c].prn;
            if (pc.eph.valid) {
                fix_chans.push_back(pc);
                fix_of.push_back(c);
            }
        } else if (fix) {
            gpsb200_pvt_chan_t pc;
            memset(&pc, 0, sizeof pc);
            gpsb200_nav_ephemeris(words.data(), sy.nwords, &pc.eph, nullptr);
            gpsb200_nav_time_anchor(words.data(), sy.nwords, &sy, &pc.anchor_epoch, &pc.anchor_ms);
            pc.prn = state[c].prn;
            if (pc.eph.valid && pc.anchor_epoch >= 0) {
                fix_chans.push_back(pc);
                fix_of.push_back(c);
            }
        }
    }
    if (fix) rc = print_fixes(ctx, fix_chans, fix_of, eps, s0 + kFixLead, fix_every * GPSB200_ACQ_CODE_SAMPLES, pcfg,
                              raim ? &rcfg : nullptr, araim ? &acfg : nullptr, coarse ? &ap : nullptr, assist_search);
    if (rc != GPSB200_OK) fprintf(stderr, "gpsb200-track: %s\n", gpsb200_last_error(ctx));
    gpsb200_destroy(ctx);
    return rc == GPSB200_OK ? 0 : 1;
}
