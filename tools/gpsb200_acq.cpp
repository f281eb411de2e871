// gpsb200-acq: GPS L1 C/A acquisition search over a 3 Msps I/Q file (gpsb200-sim's output, the reference's iqdata.bin,
// any capture in these formats: int8 or, with --iq16, int16 I,Q interleaved). Reads only the searched window --
// 3000 K + 2999 samples from the start offset -- and runs gpsb200_acquire on it; prints one line per PRN: best Doppler
// bin, code delay (samples from the window start to the code's chip 0, and in chips), P1/P2 and whether P1/P2 reaches
// the threshold. The search and its arithmetic are those of include/gpsb200.h (DESIGN §9).
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

static void usage() {
    fprintf(stderr,
            "gpsb200-acq FILE [--iq16] [--block B] [--offset-ms N] [--ms K] [--doppler LO,HI,STEP] [--prn LIST]\n"
            "            [--threshold R] [--device D]\n"
            "  FILE              interleaved I,Q at 3 Msps, int8 (default) or int16 (--iq16)\n"
            "  --block B         start at 0.1 s block B (sample 300000 B); --offset-ms N adds N ms (3000 N samples)\n"
            "  --ms K            coherent 1 ms periods summed, 1..100 (default 10)\n"
            "  --doppler L,H,S   Doppler bins L, L+S, .. up to H, in Hz (default -5000,5000,250)\n"
            "  --prn LIST        e.g. 1-32 (default), 3,7,12-15\n"
            "  --threshold R     P1/P2 at or above R counts as acquired (default %.1f)\n",
            kDefaultThreshold);
    exit(2);
}

int main(int argc, char **argv) {
    const char *path = nullptr;
    int ss = GPSB200_SC08, device = 0;
    long long block = 0, offset_ms = 0;
    double lo = -5000.0, hi = 5000.0, step = 250.0, threshold = kDefaultThreshold;
    gpsb200_acq_config_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.ms = 10;
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
        else if (a[0] != '-' && !path) path = argv[i];
        else usage();
    }
    if (!path || block < 0 || offset_ms < 0) usage();
    cfg.f_lo_hz = lo;
    cfg.step_hz = step;
    cfg.nbins = (int) std::floor((hi - lo) / step + 1e-9) + 1;

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
    if (rc == GPSB200_OK) rc = gpsb200_acquire(ctx, buf.data(), need, ss, &cfg, res.data(), nullptr);
    if (rc != GPSB200_OK) {
        fprintf(stderr, "gpsb200-acq: %s\n", ctx ? gpsb200_last_error(ctx) : "cannot create a context");
        gpsb200_destroy(ctx);
        return 1;
    }
    gpsb200_destroy(ctx);
    printf("# %s: sample %lld, %d ms, %d bins %.1f .. %.1f Hz, threshold P1/P2 >= %.2f\n", path, s0, cfg.ms, cfg.nbins, lo,
           lo + (cfg.nbins - 1) * step, threshold);
    printf("# PRN  doppler_hz  delay_samples  delay_chips  P1/P2  acquired\n");
    int nacq = 0;
    for (const auto &r : res) {
        const bool acq = r.ratio >= threshold;
        nacq += acq;
        printf("%5d  %10.1f  %13d  %11.3f  %8.3f  %s\n", r.prn, r.doppler_hz, r.delay, r.delay_chips, r.ratio,
               acq ? "yes" : "no");
    }
    printf("# %d of %d acquired\n", nacq, cfg.nprn);
    return 0;
}
