/* TEST INFRASTRUCTURE -- not product code.
 *
 * Headless driver around the UNMODIFIED reference producer thread
 * (/root/reference/gps.c, gps_thread_ep at gps.c:2282). The reference source is
 * pulled in with #include so that
 *   - MAX_CHAN (gps.h:36, not #ifndef-guarded) can be raised to 32 without
 *     touching or copying the reference file, and
 *   - the per-block channel state that lives on gps_thread_ep's stack can be
 *     observed from a hook that expands inside its scope.
 * The FIFO entry points the producer calls (fifo.h:49,55) are provided here as
 * a recording sink: every buffer handed to fifo_enqueue() is appended, in order,
 * to the --iq file. That is the "enqueue stream" of SURVEY.md (the stock
 * fifo.c:163-168 drops queued buffers; see ref_stock_main.c for that variant).
 *
 * Build variants (oracle/Makefile):
 *   -DORACLE_MAX_CHAN=32        32-channel build
 *   -DORACLE_DUMP_PARAMS        enable the per-block parameter hook
 *                               (not used for timing runs)
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <zlib.h>

/* First inclusion of the reference headers fixes their include guards. */
#include "gps.h"
#include "gps-sim.h"
#include "sdr.h"
#include "fifo.h"
#include "gui.h"

#ifdef ORACLE_MAX_CHAN
#undef MAX_CHAN
#define MAX_CHAN (ORACLE_MAX_CHAN)
#endif

/* ------------------------------------------------------------------------ */
/* Record file: sequence of {u32 tag, u32 nbytes, payload}.                  */
enum { TAG_HEADER = 1, TAG_BLOCK = 2, TAG_NAV = 3, TAG_CODE = 4, TAG_TABLES = 5, TAG_END = 6 };

typedef struct {
    int32_t prn, iword, ibit, icode, dataBit, codeCA;
    double f_carr, f_code, carr_phase, code_phase, gain;
} dump_chan_t; /* 64 bytes */

static FILE *g_params;
static FILE *g_iq;
static FILE *g_crc;   /* --crc: one CRC-32 (zlib) per enqueued buffer instead of the bytes (long runs) */
static uint32_t g_blocks;
static uint32_t g_sample_size;
static struct timespec g_t0, g_t1;
static int g_have_t0;
static uint32_t g_last_dwrd[64][N_DWRD];
static int g_last_prn[64];

static void put_rec(uint32_t tag, const void *p, uint32_t n) {
    if (!g_params) return;
    fwrite(&tag, 4, 1, g_params);
    fwrite(&n, 4, 1, g_params);
    if (n) fwrite(p, 1, n, g_params);
}

#ifdef ORACLE_DUMP_PARAMS
/* Called at isamp == 0 of every block's sample loop (gps.c:2767), i.e. after
 * the 10 Hz update (gps.c:2731-2765) and before the first sample is made. */
static int oracle_block_hook(const channel_t *chan, const double *gain) {
    struct { uint32_t block; dump_chan_t c[MAX_CHAN]; } rec;
    memset(&rec, 0, sizeof rec);
    rec.block = g_blocks;
    for (int i = 0; i < MAX_CHAN; i++) {
        dump_chan_t *d = &rec.c[i];
        d->prn = chan[i].prn;
        if (chan[i].prn <= 0) continue;
        d->iword = chan[i].iword; d->ibit = chan[i].ibit; d->icode = chan[i].icode;
        d->dataBit = chan[i].dataBit; d->codeCA = chan[i].codeCA;
        d->f_carr = chan[i].f_carr; d->f_code = chan[i].f_code;
        d->carr_phase = chan[i].carr_phase; d->code_phase = chan[i].code_phase;
        d->gain = gain[i];
        uint32_t w[N_DWRD];
        for (int k = 0; k < N_DWRD; k++) w[k] = (uint32_t) chan[i].dwrd[k];
        if (g_last_prn[i] != chan[i].prn || memcmp(w, g_last_dwrd[i], sizeof w) != 0) {
            struct { uint32_t block, ch; uint32_t w[N_DWRD]; } nav;
            nav.block = g_blocks; nav.ch = (uint32_t) i;
            memcpy(nav.w, w, sizeof w);
            put_rec(TAG_NAV, &nav, sizeof nav);
            memcpy(g_last_dwrd[i], w, sizeof w);
        }
        if (g_last_prn[i] != chan[i].prn) {
            struct { uint32_t prn; uint8_t ca[CA_SEQ_LEN + 1]; } code;
            memset(&code, 0, sizeof code);
            code.prn = (uint32_t) chan[i].prn;
            for (int k = 0; k < CA_SEQ_LEN; k++) code.ca[k] = (uint8_t) chan[i].ca[k];
            put_rec(TAG_CODE, &code, sizeof code);
            g_last_prn[i] = chan[i].prn;
        }
    }
    put_rec(TAG_BLOCK, &rec, sizeof rec);
    return 0;
}
#undef NUM_IQ_SAMPLES
#undef IQ_BUFFER_SIZE
#define NUM_IQ_SAMPLES (((isamp == 0) ? oracle_block_hook(chan, gain) : 0), (TX_SAMPLERATE / 10))
#define IQ_BUFFER_SIZE ((TX_SAMPLERATE / 10) * 2)
#endif

/* The reference producer, verbatim. */
#include "gps.c"

/* ------------------------------------------------------------------------ */
/* Recording FIFO: two buffers are enough for a synchronous sink.            */
static struct iq_buf g_buf;

struct iq_buf *fifo_acquire(void) {
    if (!g_have_t0) { clock_gettime(CLOCK_MONOTONIC, &g_t0); g_have_t0 = 1; }
    g_buf.validLength = 0;
    g_buf.next = NULL;
    return &g_buf;
}

void fifo_enqueue(struct iq_buf *buf) {
    clock_gettime(CLOCK_MONOTONIC, &g_t1);
    if (g_iq) {
        if (g_sample_size == SC16) fwrite(buf->data16, 2, buf->validLength, g_iq);
        else fwrite(buf->data8, 1, buf->validLength, g_iq);
    }
    if (g_crc) {
        const size_t nbytes = (size_t) buf->validLength * (g_sample_size == SC16 ? 2 : 1);
        const uint32_t c = (uint32_t) crc32(0L, g_sample_size == SC16 ? (const Bytef *) buf->data16 : (const Bytef *) buf->data8,
                                            (uInt) nbytes);
        fwrite(&c, 4, 1, g_crc);
    }
    g_blocks++;
}

void set_thread_name(const char *name) { (void) name; }
int thread_to_core(int core_id) { (void) core_id; return 0; }

static void usage(void) {
    fprintf(stderr,
            "ref_dump -e NAV -l lat,lon,h -d SEC [--iq16] [-m motion.csv] [-s y/m/d,h:m:s]\n"
            "         [--iq FILE] [--crc FILE] [--params FILE] [-3] [--pluto-gain] [-I]\n");
    exit(2);
}

int main(int argc, char **argv) {
    static simulator_t sim; /* zero-initialised like gps-sim.c's global */
    const char *iq_name = NULL, *par_name = NULL, *crc_name = NULL;
    double dur = 10.0;

    sim.ionosphere_enable = true;
    sim.almanac_enable = false;
    sim.sample_size = SC08;
    sim.sdr_type = SDR_IQFILE;
    sim.sdr_name = "iqfile";
    pthread_cond_init(&sim.gps_init_done, NULL);
    pthread_mutex_init(&sim.gps_lock, NULL);

    for (int i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "-e") && i + 1 < argc) sim.nav_file_name = argv[++i];
        else if (!strcmp(argv[i], "-l") && i + 1 < argc)
            sscanf(argv[++i], "%lf,%lf,%lf", &sim.location.lat, &sim.location.lon, &sim.location.height);
        else if (!strcmp(argv[i], "-d") && i + 1 < argc) dur = atof(argv[++i]);
        else if (!strcmp(argv[i], "-m") && i + 1 < argc) sim.motion_file_name = argv[++i];
        else if (!strcmp(argv[i], "-s") && i + 1 < argc)
            sscanf(argv[++i], "%d/%d/%d,%d:%d:%lf", &sim.start.y, &sim.start.m, &sim.start.d,
                   &sim.start.hh, &sim.start.mm, &sim.start.sec);
        else if (!strcmp(argv[i], "-t") && i + 1 < argc) {                 /* as gps-sim.c:145-148 */
            sim.target.valid = true;
            sscanf(argv[++i], "%lf,%lf,%lf", &sim.target.distance, &sim.target.bearing, &sim.target.height);
            sim.target.bearing *= 1000;
        }
        else if (!strcmp(argv[i], "--iq16")) sim.sample_size = SC16;
        else if (!strcmp(argv[i], "-3")) sim.use_rinex3 = true;
        else if (!strcmp(argv[i], "-I")) sim.ionosphere_enable = false;   /* as gps-sim.c's -I */
        else if (!strcmp(argv[i], "--pluto-gain")) sim.sdr_type = SDR_PLUTOSDR;
        else if (!strcmp(argv[i], "--iq") && i + 1 < argc) iq_name = argv[++i];
        else if (!strcmp(argv[i], "--params") && i + 1 < argc) par_name = argv[++i];
        else if (!strcmp(argv[i], "--crc") && i + 1 < argc) crc_name = argv[++i];
        else usage();
    }
    if (!sim.nav_file_name) usage();
    sim.duration = (int) (dur * 10.0 + 0.5); /* gps-sim.c:140 */
    g_sample_size = (uint32_t) sim.sample_size;

    g_buf.totalLength = IQ_BUFFER_SIZE;
    if (sim.sample_size == SC16) g_buf.data16 = calloc(IQ_BUFFER_SIZE, 2);
    else g_buf.data8 = calloc(IQ_BUFFER_SIZE, 1);

    if (iq_name && !(g_iq = fopen(iq_name, "wb"))) { perror(iq_name); return 1; }
    if (par_name && !(g_params = fopen(par_name, "wb"))) { perror(par_name); return 1; }
    if (crc_name && !(g_crc = fopen(crc_name, "wb"))) { perror(crc_name); return 1; }
    memset(g_last_prn, 0, sizeof g_last_prn);

    struct { uint32_t version, max_chan, sample_size, samples_per_block; } hdr =
        { 1, MAX_CHAN, (uint32_t) sim.sample_size, TX_SAMPLERATE / 10 };
    put_rec(TAG_HEADER, &hdr, sizeof hdr);
    struct { int32_t s[512], c[512]; } tabs;
    for (int k = 0; k < 512; k++) { tabs.s[k] = sinTable512[k]; tabs.c[k] = cosTable512[k]; }
    put_rec(TAG_TABLES, &tabs, sizeof tabs);

    pthread_t th;
    pthread_attr_t attr;
    pthread_attr_init(&attr);
    pthread_attr_setstacksize(&attr, 256u << 20); /* eph[13][32] + chan[32] live on the thread stack */
    pthread_create(&th, &attr, gps_thread_ep, &sim);
    pthread_join(th, NULL);

    double secs = (g_t1.tv_sec - g_t0.tv_sec) + 1e-9 * (g_t1.tv_nsec - g_t0.tv_nsec);
    struct { uint32_t blocks, pad; double producer_seconds; } end = { g_blocks, 0, secs };
    put_rec(TAG_END, &end, sizeof end);
    if (g_iq) fclose(g_iq);
    if (g_params) fclose(g_params);
    if (g_crc) fclose(g_crc);
    /* One machine-readable line for bench.py / tests. */
    printf("{\"blocks\": %u, \"samples\": %llu, \"producer_seconds\": %.6f, \"max_chan\": %d, \"sample_size\": %d}\n",
           g_blocks, (unsigned long long) g_blocks * (TX_SAMPLERATE / 10), secs, MAX_CHAN, (int) sim.sample_size);
    return g_blocks > 0 ? 0 : 1;
}
