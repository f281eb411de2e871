/* TEST INFRASTRUCTURE -- not product code.
 *
 * The reference's interactive mode (-i), driven by a key script. Linked with the UNMODIFIED reference gps-sim.c
 * (its main, its argp options, its key switch gps-sim.c:332-414) and, through #include, the UNMODIFIED producer
 * gps.c with the per-block parameter hook of ref_dump.c. This translation unit provides what gps-sim.c and gps.c
 * leave unresolved:
 *   - the recording FIFO (fifo_acquire / fifo_enqueue; the rest are stubs): every enqueued block is recorded;
 *   - sdr_init / sdr_run / sdr_close / sdr_set_gain: "-r iqfile" selects SDR_IQFILE so that every block is
 *     enqueued whole (gps.c:2860); the gain keys change nothing, as for the reference's file sink;
 *   - the GUI (gui.h:64-77) as no-ops, except gui_getch, which hands over the scripted keys with a handshake:
 *     in fifo_enqueue of block b-1 the producer hands the keys scheduled for block b to gui_getch and waits until
 *     main calls gui_getch again after the last of them -- i.e. until main's key switch has run -- so a key acts on
 *     block b exactly (gps.c:2714-2729 reads the target at the top of block b). A key at block 0 cannot be given,
 *     as in the reference, whose main reads keys only once the producer has started. Once the last block is
 *     enqueued gui_getch returns 'x', which ends main's loop.
 * set_thread_name, thread_to_core and `simulator` come from gps-sim.c.
 *
 * Environment (gps-sim.c's argp accepts only the reference's options):
 *   ORACLE_STEER   schedule, one event per line "B,KEYS[,REPEAT]": the string KEYS, REPEAT times, before block B
 *   ORACLE_PARAMS  record file of ref_dump.c's format (tests/refdump.py) -- built with -DORACLE_DUMP_PARAMS
 *   ORACLE_CRC     one CRC-32 (zlib) per enqueued block
 *   ORACLE_IQ      the enqueued I/Q stream
 * Built by oracle/Makefile.interactive; -DORACLE_MAX_CHAN=32 for 32 channels.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <zlib.h>

#include "gps.h"
#include "gps-sim.h"
#include "sdr.h"
#include "fifo.h"
#include "gui.h"

#ifdef ORACLE_MAX_CHAN
#undef MAX_CHAN
#define MAX_CHAN (ORACLE_MAX_CHAN)
#endif

enum { TAG_HEADER = 1, TAG_BLOCK = 2, TAG_NAV = 3, TAG_CODE = 4, TAG_TABLES = 5, TAG_END = 6 };

typedef struct {
    int32_t prn, iword, ibit, icode, dataBit, codeCA;
    double f_carr, f_code, carr_phase, code_phase, gain;
} dump_chan_t; /* 64 bytes */

static FILE *g_params, *g_iq, *g_crc;
static uint32_t g_blocks, g_sample_size, g_nblocks;
static uint32_t g_last_dwrd[64][N_DWRD];
static int g_last_prn[64];
static simulator_t *g_sim;

static void put_rec(uint32_t tag, const void *p, uint32_t n) {
    if (!g_params) return;
    fwrite(&tag, 4, 1, g_params);
    fwrite(&n, 4, 1, g_params);
    if (n) fwrite(p, 1, n, g_params);
}

#ifdef ORACLE_DUMP_PARAMS
/* the hook of ref_dump.c: called at isamp == 0 of every block's sample loop (gps.c:2767) */
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

/* eph[13][32] + chan[32] live on the producer's stack; gps-sim.c creates it with default attributes */
__attribute__((constructor)) static void big_default_stack(void) {
    pthread_attr_t a;
    pthread_attr_init(&a);
    pthread_attr_setstacksize(&a, 256u << 20);
    pthread_setattr_default_np(&a);
    pthread_attr_destroy(&a);
}

/* ---- key script + handshake ------------------------------------------------------------------------------------ */
static char **g_script;            /* [block] -> keys to press before that block, or NULL */
static pthread_mutex_t g_mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t g_cv = PTHREAD_COND_INITIALIZER;
static const char *g_keys;         /* keys being handed to main */
static size_t g_kpos;
static int g_done;

static void load_script(uint32_t nblocks) {
    g_script = calloc(nblocks + 1, sizeof *g_script);
    const char *path = getenv("ORACLE_STEER");
    if (!path) return;
    FILE *fp = fopen(path, "r");
    if (!fp) { perror(path); exit(2); }
    char line[4096];
    while (fgets(line, sizeof line, fp)) {
        unsigned b = 0, rep = 1;
        char keys[4096];
        if (line[0] == '#' || line[0] == '\n') continue;
        const int n = sscanf(line, "%u,%4095[^,\n],%u", &b, keys, &rep);
        if (n < 2 || b < 1) { fprintf(stderr, "bad schedule line: %s", line); exit(2); }
        if (b >= nblocks) continue;        /* never reached */
        const size_t old = g_script[b] ? strlen(g_script[b]) : 0, add = strlen(keys) * rep;
        g_script[b] = realloc(g_script[b], old + add + 1);
        for (unsigned r = 0; r < rep; r++) memcpy(g_script[b] + old + r * strlen(keys), keys, strlen(keys));
        g_script[b][old + add] = 0;
    }
    fclose(fp);
}

static void wait_a_little(void) {
    struct timespec t;
    clock_gettime(CLOCK_REALTIME, &t);
    t.tv_nsec += 50 * 1000 * 1000;
    if (t.tv_nsec >= 1000000000) { t.tv_sec++; t.tv_nsec -= 1000000000; }
    pthread_cond_timedwait(&g_cv, &g_mu, &t);
}

int gui_getch(void) {
    pthread_mutex_lock(&g_mu);
    if (g_keys && !g_keys[g_kpos]) {       /* back after the last key: main's switch has run */
        g_keys = NULL;
        pthread_cond_broadcast(&g_cv);
    }
    while (!g_keys && !g_done && !(g_sim && g_sim->gps_thread_exit)) wait_a_little();
    int c = 'x';
    if (g_keys) c = (unsigned char) g_keys[g_kpos++];
    pthread_mutex_unlock(&g_mu);
    return c;
}

/* ---- recording FIFO ------------------------------------------------------------------------------------------- */
static struct iq_buf g_buf;

struct iq_buf *fifo_acquire(void) {
    g_buf.validLength = 0;
    g_buf.next = NULL;
    return &g_buf;
}

void fifo_enqueue(struct iq_buf *buf) {
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
    pthread_mutex_lock(&g_mu);
    if (g_blocks >= g_nblocks) {
        g_done = 1;
        pthread_cond_broadcast(&g_cv);
    } else if (g_script[g_blocks]) {
        g_keys = g_script[g_blocks];
        g_kpos = 0;
        pthread_cond_broadcast(&g_cv);
        while (g_keys && !g_sim->gps_thread_exit) wait_a_little();
    }
    pthread_mutex_unlock(&g_mu);
}

bool fifo_create(unsigned buffer_count, unsigned buffer_size, unsigned sample_size) { return true; }
void fifo_destroy() {}
void fifo_wait_next() {}
void fifo_wait_full() {}
void fifo_halt() {}
struct iq_buf *fifo_dequeue(void) { return NULL; }
void fifo_release(struct iq_buf *buf) {}

/* ---- SDR ------------------------------------------------------------------------------------------------------ */
static FILE *open_env(const char *name) {
    const char *p = getenv(name);
    if (!p) return NULL;
    FILE *f = fopen(p, "wb");
    if (!f) { perror(p); exit(2); }
    return f;
}

int sdr_init(simulator_t *s) {
    if (!s->sdr_name || strcmp(s->sdr_name, "iqfile") != 0) {
        fprintf(stderr, "ref_interactive: only -r iqfile\n");
        return -1;
    }
    s->sdr_type = SDR_IQFILE;
    g_sim = s;
    g_sample_size = (uint32_t) s->sample_size;
    g_nblocks = (uint32_t) (s->duration - 1);
    g_buf.totalLength = IQ_BUFFER_SIZE;
    g_buf.data8 = calloc(IQ_BUFFER_SIZE, 1);
    g_buf.data16 = calloc(IQ_BUFFER_SIZE, 2);
    g_params = open_env("ORACLE_PARAMS");
    g_crc = open_env("ORACLE_CRC");
    g_iq = open_env("ORACLE_IQ");
    memset(g_last_prn, 0, sizeof g_last_prn);
    load_script(g_nblocks);
    struct { uint32_t version, max_chan, sample_size, samples_per_block; } hdr =
        { 1, MAX_CHAN, (uint32_t) s->sample_size, TX_SAMPLERATE / 10 };
    put_rec(TAG_HEADER, &hdr, sizeof hdr);
    struct { int32_t s[512], c[512]; } tabs;
    for (int k = 0; k < 512; k++) { tabs.s[k] = sinTable512[k]; tabs.c[k] = cosTable512[k]; }
    put_rec(TAG_TABLES, &tabs, sizeof tabs);
    return 0;
}

int sdr_run(void) { return 0; }
int sdr_set_gain(int gain) { return gain; }

/* called by cleanup_and_exit after the producer has been joined, before exit(): close the records */
void sdr_close(void) {
    struct { uint32_t blocks, pad; double producer_seconds; } end = { g_blocks, 0, 0.0 };
    put_rec(TAG_END, &end, sizeof end);
    if (g_iq) fclose(g_iq);
    if (g_params) fclose(g_params);
    if (g_crc) fclose(g_crc);
    g_iq = g_params = g_crc = NULL;
    printf("{\"blocks\": %u, \"max_chan\": %d, \"sample_size\": %d}\n", g_blocks, MAX_CHAN, (int) g_sample_size);
}

/* ---- the rest of the GUI: no-ops ------------------------------------------------------------------------------ */
void gui_init(void) {}
void gui_destroy(void) {}
void gui_mvwprintw(window_panel_t w, int y, int x, const char *fmt, ...) {}
void gui_status_wprintw(status_color_t clr, const char *fmt, ...) {}
void gui_colorpair(window_panel_t w, unsigned clr, attr_status_t onoff) {}
void gui_top_panel(window_panel_t p) {}
void gui_toggle_current_panel(void) {}
void gui_show_panel(window_panel_t p, attr_status_t onoff) {}
void gui_show_speed(float speed) {}
void gui_show_heading(float hdg) {}
void gui_show_vertical_speed(float vs) {}
void gui_show_location(void *l) {}
void gui_show_target(void *t) {}
