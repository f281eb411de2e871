// gpsb200-sim: file-sink driver with the reference's command-line vocabulary (help.h:20-53:
// -e nav file, -l location, -t target, -d duration, -m motion file, -s start, --iq16, -I no ionosphere,
// --disable-almanac; --almanac FILE names the SEM almanac the reference would read from ./almanac.sem).
// RINEX + location -> scenario engine (host) -> CUDA synthesis -> reference-compatible FIFO ->
// iqfile writer. Output is byte-identical to the reference's enqueue stream; --compat-drop
// reproduces the stock program's iqdata.bin (which lacks blocks 1..6, fifo.c:163-168).
//
// One GPU: the FIFO is created with a batch worth of page-locked buffers; every batch is synthesized with
// gpsb200_synth_blocks_scatter, i.e. the device->host copies land straight in the acquired iq->data8/16 (no staging
// copy), and the buffers are enqueued in order.
// --gpus N: the stream is cut into N contiguous time slices, one worker thread and one context per device. The
// slices' closed-form links give every worker a guessed incoming carrier-chain state at once (gpsb200_slice_link_host
// + gpsb200_link_apply), all workers probe speculatively in parallel, and the exact states travel worker to worker
// (gpsb200_slice_prepare / _probe / _finish). Each worker downloads into a page-locked slice buffer; the main thread
// feeds the slices to the FIFO in stream order as they complete.
// -i / --steer FILE: the reference's interactive mode (gps-sim.c:363-393, gps.c:2714-2729) on one GPU. The scenario is
// opened, not built up front, and advanced chunk by chunk; keys (from stdin, paced to real time, or replayed from a
// schedule) are applied between advances. Each chunk is synthesized with gpsb200_synth_blocks_scatter, the carrier
// chain continued across calls, the NAV frames kept in a ring of context slots (global frame f in slot f mod R).
// -s now: the start is the UTC clock read while the arguments are parsed (gps-sim.c:89-102), and the scenario is opened
// with the reference's ephemeris time overwrite (gpsb200_scenario_create_now / _open_now) on every path; --now DATE
// replaces the clock reading (a session replayed, a test).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <csignal>
#include <deque>
#include <map>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <termios.h>
#include <time.h>
#include <unistd.h>

#include <cuda_runtime_api.h>

#include "../include/gpsb200.h"

static void usage() {
    fprintf(stderr,
            "gpsb200-sim -e NAV[.gz] [-3] -l lat,lon,h [-t dist,bearing,height] [-d SEC] [-m motion.csv]\n"
            "            [-s y/m/d,h:m:s | -s now [--now y/m/d,h:m:s]] [--iq16] [-I] [--pluto-gain] [--chan N] [--gpus N]\n"
            "            [-o iqdata.bin] [--compat-drop] [--almanac FILE.sem | --disable-almanac] [-i | --steer FILE]\n"
            "            [--steer-log FILE]\n"
            "  -s now          start at the current time (UTC used as GPS time, as the reference does): the ephemeris and\n"
            "                  UTC reference times of the file are moved to it, so a file of any date can be used\n"
            "  --now DATE      with -s now: use DATE instead of the clock (replay a session)\n"
            "  -i              interactive: keys from stdin (a/d heading, w/s climb, e/q speed, x end), paced to real time\n"
            "  --steer FILE    replay a schedule, one line per event \"B,KEYS[,REPEAT]\": KEYS, REPEAT times, before block B\n"
            "  --steer-log F   write the schedule that was applied (replays byte-identically with --steer)\n");
    exit(2);
}

static double now_s() {
    using namespace std::chrono;
    return duration<double>(steady_clock::now().time_since_epoch()).count();
}

namespace {
std::atomic<bool> g_stop{false};
struct termios g_tty;
bool g_tty_raw = false;

void restore_tty() {
    if (g_tty_raw) tcsetattr(0, TCSANOW, &g_tty);
    g_tty_raw = false;
}
void on_sigint(int) { g_stop = true; }          // the block in progress is finished, then the file is closed

bool read_schedule(const char *path, std::map<int, std::string> &keys) {
    FILE *fp = fopen(path, "r");
    if (!fp) return false;
    char line[8192];
    bool ok = true;
    while (ok && fgets(line, sizeof line, fp)) {
        if (line[0] == '#' || line[0] == '\n') continue;
        int b = 0, rep = 1;
        char k[8192];
        const int n = sscanf(line, "%d,%8191[^,\n],%d", &b, k, &rep);
        ok = n >= 2 && b >= 1 && rep >= 0;
        for (int r = 0; ok && r < rep; r++) keys[b] += k;
    }
    fclose(fp);
    return ok;
}

// "y/m/d,h:m:s" -> the start fields; all six are required
bool parse_date(const char *s, gpsb200_scenario_config_t &sc) {
    return sscanf(s, "%d/%d/%d,%d:%d:%lf", &sc.start_year, &sc.start_month, &sc.start_day, &sc.start_hour, &sc.start_min,
                  &sc.start_sec) == 6;
}

// the -s range check (gps-sim.c:106-114)
bool date_in_range(const gpsb200_scenario_config_t &sc) {
    return !(sc.start_year <= 1980 || sc.start_month < 1 || sc.start_month > 12 || sc.start_day < 1 || sc.start_day > 31 ||
             sc.start_hour < 0 || sc.start_hour > 23 || sc.start_min < 0 || sc.start_min > 59 || !(sc.start_sec >= 0.0) ||
             sc.start_sec >= 60.0);
}

int open_scenario(const gpsb200_scenario_config_t &sc, bool now, bool build, gpsb200_scenario_t **scn) {
    if (build) return now ? gpsb200_scenario_create_now(&sc, scn) : gpsb200_scenario_create(&sc, scn);
    return now ? gpsb200_scenario_open_now(&sc, scn) : gpsb200_scenario_open(&sc, scn);
}

void print_start(const gpsb200_scenario_t *scn) {
    int32_t week = 0;
    double sow = 0;
    gpsb200_scenario_start_time(scn, &week, &sow);
    fprintf(stderr, "gpsb200-sim: start time: %s (week %d, sow %.10g)\n", gpsb200_scenario_start_date(scn), week, sow);
}

// -i / --steer: open the scenario, then advance / key / synthesize chunk by chunk on one GPU
int run_steered(gpsb200_scenario_config_t sc, bool now, int sample_size, bool live, const char *steer_file,
                const char *log_file, const std::string &out) {
    std::map<int, std::string> sched;
    if (steer_file && !read_schedule(steer_file, sched)) {
        fprintf(stderr, "gpsb200-sim: cannot read schedule %s\n", steer_file);
        return 1;
    }
    FILE *log = nullptr;
    if (log_file && !(log = fopen(log_file, "w"))) {
        fprintf(stderr, "gpsb200-sim: cannot write %s\n", log_file);
        return 1;
    }
    sc.interactive = 1;
    gpsb200_scenario_t *scn = nullptr;
    if (open_scenario(sc, now, false, &scn) != GPSB200_OK) {
        fprintf(stderr, "scenario: %s\n", gpsb200_scenario_error(scn));
        return 1;
    }
    print_start(scn);
    const int nchan = gpsb200_scenario_channels(scn);
    const bool motion = sc.motion_file && sc.motion_file[0];
    if (motion) fprintf(stderr, "gpsb200-sim: user motion file supplied, interactive mode disabled (keys are ignored)\n");
    const int batch = live ? 1 : 256, ring = 4;       // <= 2 frames per 256 blocks (one roll per 30 s)
    const size_t blk_bytes = (size_t) GPSB200_BLOCK_ELEMS * sample_size;
    gpsb200_ctx_t *ctx = nullptr;
    gpsb200_bind_numa(0);
    gpsb200_config_t cfg{};
    cfg.max_chan = nchan;
    cfg.max_blocks = batch;
    cfg.max_nav_frames = ring;
    if (gpsb200_create(&cfg, &ctx) != GPSB200_OK) {
        fprintf(stderr, "gpsb200: %s\n", gpsb200_last_error(ctx));
        return 1;
    }
    if (!fifo_create((unsigned) batch + 8, GPSB200_BLOCK_ELEMS, sample_size)) return 1;
    // keys from stdin: a reader thread queues them; each applies to the first block not yet handed to the synthesis
    std::mutex kmu;
    std::deque<char> kq;
    if (live) {
        if (isatty(0) && tcgetattr(0, &g_tty) == 0) {
            struct termios raw = g_tty;
            raw.c_lflag &= ~(ICANON | ECHO);
            raw.c_cc[VMIN] = 1;
            raw.c_cc[VTIME] = 0;
            if (tcsetattr(0, TCSANOW, &raw) == 0) g_tty_raw = true;
            atexit(restore_tty);
        }
        std::thread([&kq, &kmu] {
            char c;
            while (read(0, &c, 1) == 1) {
                std::lock_guard<std::mutex> lk(kmu);
                kq.push_back(c);
            }
        }).detach();
    }
    signal(SIGINT, on_sigint);
    bool writer = false;
    int queued = 0, b = 0, uploaded = -1, rc = 0;
    std::vector<gpsb200_chan_t> part((size_t) batch * nchan);
    std::vector<int32_t> prev_prn(nchan, 0);
    std::vector<double> carr(nchan, 0.0);
    std::vector<void *> dsts(batch);
    std::vector<struct iq_buf *> bufs(batch);
    const double t0 = now_s();
    while (!g_stop) {
        std::string keys;
        if (b >= 1) {
            auto it = sched.find(b);
            if (it != sched.end()) keys = it->second;
            std::lock_guard<std::mutex> lk(kmu);
            for (char c : kq)
                if (strchr("adwseqtgxX", c)) keys += c;     // anything else (newlines, panels of the TUI) is ignored
            kq.clear();
        }
        bool end = false;
        for (char c : motion ? std::string() : keys) {
            const int k = gpsb200_scenario_key(scn, c);
            if (k == GPSB200_ERR_END) break;
            if (k != GPSB200_OK) {
                fprintf(stderr, "scenario: %s\n", gpsb200_scenario_error(scn));
                end = true;
                rc = 1;
                break;
            }
        }
        if (log && !keys.empty()) fprintf(log, "%d,%s\n", b, keys.c_str());
        gpsb200_steer_state_t st;
        gpsb200_scenario_steer_state(scn, &st);
        if (end || st.next_block >= st.end_block) break;
        int n = std::min(batch, st.end_block - b);
        auto nx = sched.upper_bound(b);
        if (nx != sched.end()) n = std::min(n, nx->first - b);
        int32_t got = 0;
        if (gpsb200_scenario_advance(scn, n, part.data(), &got) != GPSB200_OK) {
            fprintf(stderr, "scenario: %s\n", gpsb200_scenario_error(scn));
            rc = 1;
            break;
        }
        for (int k = 0; k < got; k++)                    // NAV ring: upload a frame before the chunk that first uses it
            for (int c = 0; c < nchan; c++) {
                gpsb200_chan_t &p = part[(size_t) k * nchan + c];
                if (p.nav_frame > uploaded) {
                    const uint32_t *w = gpsb200_scenario_frame(scn, p.nav_frame);
                    for (int cc = 0; cc < nchan; cc++)
                        gpsb200_set_nav(ctx, p.nav_frame % ring, cc, w + (size_t) cc * GPSB200_NAV_WORDS);
                    uploaded = p.nav_frame;
                }
                p.nav_frame %= ring;
            }
        for (int c = 0; c < nchan; c++)                  // continue the carrier chain across calls
            if (part[c].prn > 0 && part[c].prn == prev_prn[c]) part[c].carr_phase = carr[c];
        for (int c = 0; c < nchan; c++) prev_prn[c] = part[(size_t) (got - 1) * nchan + c].prn;
        if (live) {                                      // real time, at most 8 blocks (the reference's FIFO) ahead
            const double due = t0 + (b - 8) * 0.1 - now_s();
            if (due > 0) std::this_thread::sleep_for(std::chrono::duration<double>(due));
        }
        for (int k = 0; k < got; k++) {
            bufs[k] = fifo_acquire();
            if (!bufs[k]) return 1;
            dsts[k] = sample_size == GPSB200_SC16 ? (void *) bufs[k]->data16 : (void *) bufs[k]->data8;
        }
        if (gpsb200_synth_blocks_scatter(ctx, part.data(), got, nchan, sample_size, dsts.data(), carr.data(), nullptr) !=
            GPSB200_OK) {
            fprintf(stderr, "gpsb200: %s\n", gpsb200_last_error(ctx));
            rc = 1;
            break;
        }
        for (int k = 0; k < got; k++) {
            if (!writer && queued >= 8) {
                if (gpsb200_iqfile_start(out.c_str(), sample_size) != GPSB200_OK) return 1;
                writer = true;
            }
            bufs[k]->validLength = GPSB200_BLOCK_ELEMS;
            fifo_enqueue(bufs[k]);
            queued++;
        }
        b += got;
    }
    if (!writer && gpsb200_iqfile_start(out.c_str(), sample_size) != GPSB200_OK) return 1;
    gpsb200_iqfile_stop();
    fifo_destroy();
    gpsb200_destroy(ctx);
    restore_tty();
    if (log) fclose(log);
    gpsb200_steer_state_t st;
    gpsb200_scenario_steer_state(scn, &st);
    fprintf(stderr, "gpsb200-sim: %d blocks (%d channels), steered%s -> %s; speed %.2f m/s, heading %.3f deg, climb %.0f m/s\n", b,
            nchan, live ? " live" : "", out.c_str(), st.velocity, st.bearing_mdeg / 1000, st.vertical_speed);
    gpsb200_scenario_destroy(scn);
    return rc;
}

struct Handoff {                 // exact chain state after slice r, published by worker r
    std::mutex mu;
    std::condition_variable cv;
    bool ready = false, failed = false;
    std::vector<int32_t> prn;
    std::vector<double> phase;
};
}  // namespace

int main(int argc, char **argv) {
    gpsb200_scenario_config_t sc{};
    sc.ionosphere_enable = 1;
    sc.max_chan = 12;
    double dur = 300.0;
    int sample_size = GPSB200_SC08, gpus = 1;
    bool compat = false, live = false, have_dur = false, have_start = false, now = false;
    const char *steer_file = nullptr, *log_file = nullptr, *now_arg = nullptr;
    std::string out = "iqdata.bin";
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto need = [&]() -> const char * {
            if (i + 1 >= argc) usage();
            return argv[++i];
        };
        if (a == "-e") sc.nav_file = need();
        else if (a == "-l") sscanf(need(), "%lf,%lf,%lf", &sc.lat_deg, &sc.lon_deg, &sc.height_m);
        else if (a == "-t") {
            sc.target_valid = 1;                                    // gps-sim.c:145-148
            sscanf(need(), "%lf,%lf,%lf", &sc.target_distance_m, &sc.target_bearing_deg, &sc.target_height_m);
        } else if (a == "-d") {
            dur = atof(need());
            have_dur = true;
        } else if (a == "-i") live = true;
        else if (a == "--steer") steer_file = need();
        else if (a == "--steer-log") log_file = need();
        else if (a == "-m") sc.motion_file = need();
        else if (a == "-s") {
            const char *v = need();
            have_start = true;
            if (strncmp(v, "now", 3) == 0) {                        // gps-sim.c:89-102: whole seconds of UTC
                now = true;
                const time_t t = time(nullptr);
                struct tm g;
                gmtime_r(&t, &g);
                sc.start_year = g.tm_year + 1900;
                sc.start_month = g.tm_mon + 1;
                sc.start_day = g.tm_mday;
                sc.start_hour = g.tm_hour;
                sc.start_min = g.tm_min;
                sc.start_sec = (double) g.tm_sec;
            } else if (!parse_date(v, sc)) {
                fprintf(stderr, "gpsb200-sim: -s %s: expected y/m/d,h:m:s or now\n", v);
                return 2;
            }
        } else if (a == "--now") now_arg = need();
        else if (a == "--iq16") sample_size = GPSB200_SC16;
        else if (a == "-I") sc.ionosphere_enable = 0;
        else if (a == "-3") sc.rinex3 = 1;
        else if (a == "--pluto-gain") sc.pluto_gain = 1;
        else if (a == "--chan") sc.max_chan = atoi(need());
        else if (a == "--gpus") gpus = atoi(need());
        else if (a == "-o") out = need();
        else if (a == "--compat-drop") compat = true;
        else if (a == "--almanac") sc.almanac_file = need();
        else if (a == "--disable-almanac") sc.almanac_file = nullptr;      // gps-sim.c:165-166; also the default here
        else usage();
    }
    if (!sc.nav_file || gpus < 1) usage();
    if (now_arg) {
        if (!now) {
            fprintf(stderr, "gpsb200-sim: --now replaces the clock reading of -s now and needs it\n");
            return 2;
        }
        if (!parse_date(now_arg, sc)) {
            fprintf(stderr, "gpsb200-sim: --now %s: expected y/m/d,h:m:s\n", now_arg);
            return 2;
        }
    }
    if (have_start && !date_in_range(sc)) {
        fprintf(stderr, "gpsb200-sim: invalid date and time: %d/%d/%d,%d:%d:%g\n", sc.start_year, sc.start_month,
                sc.start_day, sc.start_hour, sc.start_min, sc.start_sec);
        return 2;
    }
    if (live && !have_dur) dur = 86400.0;                         // the reference's default (gps-sim.c:190)
    sc.duration_ds = (int) (dur * 10.0 + 0.5);                  // gps-sim.c:140
    if (live || steer_file) {
        if (gpus != 1) {
            fprintf(stderr, "gpsb200-sim: -i / --steer run on one GPU (time slices would need the keys of the future)\n");
            return 2;
        }
        if (live && steer_file) usage();
        return run_steered(sc, now, sample_size, live, steer_file, log_file, out);
    }

    gpsb200_scenario_t *scn = nullptr;
    if (open_scenario(sc, now, true, &scn) != GPSB200_OK) {
        fprintf(stderr, "scenario: %s\n", gpsb200_scenario_error(scn));
        return 1;
    }
    print_start(scn);
    const int nblk = gpsb200_scenario_blocks(scn), nchan = gpsb200_scenario_channels(scn);
    const int nframes = gpsb200_scenario_nav_frames(scn);
    const char *alm_date = gpsb200_scenario_almanac_date(scn);             // gps.c:2652-2656
    fprintf(stderr, "gpsb200-sim: almanac date: %s\n", alm_date ? alm_date : "disabled or invalid");
    if (!sc.almanac_file)
        fprintf(stderr, "gpsb200-sim: note: no almanac pages are generated -- the stream equals the reference's with its almanac "
                        "disabled (the reference sends the one in ./almanac.sem by default; pass it with --almanac FILE)\n");
    const gpsb200_chan_t *chans = gpsb200_scenario_chans(scn);
    const uint32_t *nav = gpsb200_scenario_nav(scn);
    const size_t blk_bytes = (size_t) GPSB200_BLOCK_ELEMS * sample_size;
    int ndev = 0;
    cudaGetDeviceCount(&ndev);
    if (gpus > ndev) {
        fprintf(stderr, "gpsb200-sim: --gpus %d but %d CUDA device(s) visible\n", gpus, ndev);
        return 1;
    }
    gpus = std::min(gpus, std::max(1, nblk));
    const double t0 = now_s();

    auto make_ctx = [&](int dev, int max_blocks, gpsb200_ctx_t **ctx) -> bool {
        gpsb200_config_t cfg{};
        cfg.device = dev;
        cfg.max_chan = nchan;
        cfg.max_blocks = max_blocks;
        cfg.max_nav_frames = nframes;
        if (gpsb200_create(&cfg, ctx) != GPSB200_OK) {
            fprintf(stderr, "gpsb200: %s\n", gpsb200_last_error(*ctx));
            return false;
        }
        for (int f = 0; f < nframes; f++)
            for (int c = 0; c < nchan; c++)
                gpsb200_set_nav(*ctx, f, c, nav + ((size_t) f * nchan + c) * GPSB200_NAV_WORDS);
        return true;
    };

    fifo_set_compat_drop(compat);
    bool writer = false;
    int queued = 0;
    auto start_writer_if_primed = [&](bool force) -> bool {
        // like the reference (sdr_iqfile.c:73-77) the writer starts once the FIFO is primed (or the run ends)
        if (!writer && (queued >= 8 || force)) {
            if (gpsb200_iqfile_start(out.c_str(), sample_size) != GPSB200_OK) return false;
            writer = true;
        }
        return true;
    };

    if (gpus == 1) {
        const int batch = std::min(256, nblk);
        gpsb200_ctx_t *ctx = nullptr;
        gpsb200_bind_numa(0);           // threads and pinned FIFO buffers next to the GPU (cf. thread_to_core, gps.c:2377)
        if (!make_ctx(0, batch, &ctx)) return 1;
        // a batch worth of FIFO buffers (+ the 8 the reference keeps in flight, sdr.h:24): every block of a batch is
        // downloaded straight into its own acquired buffer. --compat-drop reproduces a property of the reference's
        // 8-buffer FIFO, so it keeps that geometry and goes through a staging buffer.
        void *stage = nullptr;
        if (compat && cudaHostAlloc(&stage, blk_bytes * batch, cudaHostAllocDefault) != cudaSuccess) return 1;
        if (!fifo_create(compat ? 8u : (unsigned) batch + 8, GPSB200_BLOCK_ELEMS, sample_size)) return 1;
        std::vector<double> carr(nchan, 0.0);
        std::vector<gpsb200_chan_t> part;
        std::vector<struct iq_buf *> bufs;
        std::vector<void *> dsts;
        for (int b0 = 0; b0 < nblk; b0 += batch) {
            const int nb = std::min(batch, nblk - b0);
            part.assign(chans + (size_t) b0 * nchan, chans + (size_t) (b0 + nb) * nchan);
            if (b0 > 0)                                             // continue the carrier chain across calls
                for (int c = 0; c < nchan; c++)
                    if (part[c].prn > 0 && part[c].prn == chans[(size_t) (b0 - 1) * nchan + c].prn) part[c].carr_phase = carr[c];
            if (compat) {
                if (gpsb200_synth_blocks(ctx, part.data(), nb, nchan, sample_size, stage, carr.data(), nullptr) != GPSB200_OK) {
                    fprintf(stderr, "gpsb200: %s\n", gpsb200_last_error(ctx));
                    return 1;
                }
                for (int b = 0; b < nb; b++) {
                    if (!start_writer_if_primed(false)) return 1;
                    struct iq_buf *iq = fifo_acquire();
                    if (!iq) return 1;
                    memcpy(sample_size == GPSB200_SC16 ? (void *) iq->data16 : (void *) iq->data8,
                           (char *) stage + (size_t) b * blk_bytes, blk_bytes);
                    iq->validLength = GPSB200_BLOCK_ELEMS;
                    fifo_enqueue(iq);
                    queued++;
                }
                continue;
            }
            bufs.assign(nb, nullptr);
            dsts.assign(nb, nullptr);
            for (int b = 0; b < nb; b++) {
                bufs[b] = fifo_acquire();                           // gps.c:2698 / 2864
                if (!bufs[b]) return 1;
                dsts[b] = sample_size == GPSB200_SC16 ? (void *) bufs[b]->data16 : (void *) bufs[b]->data8;
            }
            if (gpsb200_synth_blocks_scatter(ctx, part.data(), nb, nchan, sample_size, dsts.data(), carr.data(), nullptr) !=
                GPSB200_OK) {
                fprintf(stderr, "gpsb200: %s\n", gpsb200_last_error(ctx));
                return 1;
            }
            for (int b = 0; b < nb; b++) {
                if (!start_writer_if_primed(false)) return 1;
                bufs[b]->validLength = GPSB200_BLOCK_ELEMS;
                fifo_enqueue(bufs[b]);                              // gps.c:2860
                queued++;
            }
        }
        if (!start_writer_if_primed(true)) return 1;
        gpsb200_iqfile_stop();
        fifo_destroy();
        if (stage) cudaFreeHost(stage);
        gpsb200_destroy(ctx);
    } else {
        // ---- time slices over several GPUs ----------------------------------------------------------------
        std::vector<int> lo(gpus + 1, 0);
        for (int r = 0; r < gpus; r++) {
            const int base = nblk / gpus, extra = nblk % gpus;
            lo[r + 1] = lo[r] + base + (r < extra ? 1 : 0);
        }
        // guessed incoming states from the closed-form links: no GPU work, no dependence between the workers
        std::vector<std::vector<int32_t>> gprn(gpus, std::vector<int32_t>(nchan, 0));
        std::vector<std::vector<double>> gph(gpus, std::vector<double>(nchan, 0.0));
        {
            std::vector<int32_t> p(nchan, 0), pn(nchan, 0);
            std::vector<double> x(nchan, 0.0), xn(nchan, 0.0);
            bool have = false;
            for (int r = 0; r < gpus; r++) {
                gprn[r] = p;
                gph[r] = x;
                gpsb200_slice_link_t link;
                if (gpsb200_slice_link_host(chans + (size_t) lo[r] * nchan, lo[r + 1] - lo[r], nchan, &link) != GPSB200_OK) return 1;
                gpsb200_link_apply(&link, nchan, have ? p.data() : nullptr, have ? x.data() : nullptr, pn.data(), xn.data());
                p = pn;
                x = xn;
                have = true;
            }
        }
        std::vector<Handoff> hand(gpus);
        std::vector<void *> slice_host(gpus, nullptr);
        std::vector<int> done(gpus, 0);            // 0 running, 1 ok, -1 failed
        std::mutex done_mu;
        std::condition_variable done_cv;
        std::vector<std::thread> workers;
        for (int r = 0; r < gpus; r++) {
            workers.emplace_back([&, r] {
                const int nb = lo[r + 1] - lo[r];
                bool ok = false;
                gpsb200_ctx_t *ctx = nullptr;
                std::vector<int32_t> prn_out(nchan, 0);
                std::vector<double> ph_out(nchan, 0.0);
                do {
                    if (cudaSetDevice(r) != cudaSuccess) break;
                    gpsb200_bind_numa(r);
                    if (cudaHostAlloc(&slice_host[r], blk_bytes * nb, cudaHostAllocPortable) != cudaSuccess) break;
                    if (!make_ctx(r, nb, &ctx)) break;
                    gpsb200_slice_link_t link;
                    if (gpsb200_slice_prepare(ctx, chans + (size_t) lo[r] * nchan, nb, nchan, sample_size, nullptr, slice_host[r],
                                              nullptr, &link) != GPSB200_OK) break;
                    if (gpsb200_slice_probe(ctx, r ? gprn[r].data() : nullptr, r ? gph[r].data() : nullptr, 1) != GPSB200_OK) break;
                    const int32_t *pin = nullptr;
                    const double *xin = nullptr;
                    if (r > 0) {                                        // the exact state after slice r-1
                        std::unique_lock<std::mutex> lk(hand[r - 1].mu);
                        hand[r - 1].cv.wait(lk, [&] { return hand[r - 1].ready; });
                        if (hand[r - 1].failed) break;
                        pin = hand[r - 1].prn.data();
                        xin = hand[r - 1].phase.data();
                    }
                    if (gpsb200_slice_finish(ctx, pin, xin, prn_out.data(), ph_out.data(), nullptr) != GPSB200_OK) break;
                    ok = true;
                } while (false);
                {
                    std::lock_guard<std::mutex> lk(hand[r].mu);        // hand on (or release the successor on failure)
                    hand[r].prn = prn_out;
                    hand[r].phase = ph_out;
                    hand[r].failed = !ok;
                    hand[r].ready = true;
                }
                hand[r].cv.notify_all();
                if (ok && gpsb200_slice_wait(ctx) != GPSB200_OK) ok = false;
                if (!ok && ctx) fprintf(stderr, "gpsb200 (device %d): %s\n", r, gpsb200_last_error(ctx));
                if (ctx) gpsb200_destroy(ctx);
                {
                    std::lock_guard<std::mutex> lk(done_mu);
                    done[r] = ok ? 1 : -1;
                }
                done_cv.notify_all();
            });
        }
        if (!fifo_create(8, GPSB200_BLOCK_ELEMS, sample_size)) return 1;       // sdr_iqfile.c:59, sdr.h:24
        bool failed = false;
        for (int r = 0; r < gpus && !failed; r++) {                 // one sink, stream order
            {
                std::unique_lock<std::mutex> lk(done_mu);
                done_cv.wait(lk, [&] { return done[r] != 0; });
                failed = done[r] < 0;
            }
            if (failed) break;
            for (int b = 0; b < lo[r + 1] - lo[r]; b++) {
                if (!start_writer_if_primed(false)) return 1;
                struct iq_buf *iq = fifo_acquire();
                if (!iq) return 1;
                memcpy(sample_size == GPSB200_SC16 ? (void *) iq->data16 : (void *) iq->data8,
                       (char *) slice_host[r] + (size_t) b * blk_bytes, blk_bytes);
                iq->validLength = GPSB200_BLOCK_ELEMS;
                fifo_enqueue(iq);
                queued++;
            }
        }
        for (auto &t : workers) t.join();
        if (failed) return 1;
        if (!start_writer_if_primed(true)) return 1;
        gpsb200_iqfile_stop();
        fifo_destroy();
        for (void *p : slice_host) cudaFreeHost(p);
    }
    gpsb200_scenario_destroy(scn);
    const double dt = now_s() - t0;
    fprintf(stderr, "gpsb200-sim: %d blocks (%d channels) on %d GPU(s) -> %s in %.3f s (%.1f Msamples/s incl. file sink)\n", nblk,
            nchan, gpus, out.c_str(), dt, (double) nblk * GPSB200_BLOCK_SAMPLES / dt / 1e6);
    return 0;
}
