/* gpsb200 -- H100-native GPS L1 C/A baseband synthesis, C ABI.
 *
 * Drop-in for the sample loop of the reference's producer thread
 * (Mictronics/multi-sdr-gps-sim, gps_thread_ep): everything between the 10 Hz
 * channel update (gps.c:2731-2765) and fifo_enqueue (gps.c:2860) -- i.e.
 * gps.c:2767-2857 -- runs as sm_90a CUDA kernels behind these entry points.
 * Plain C types only; no C++/torch types cross this boundary.
 *
 * The second half of this header re-declares, unchanged, the FIFO / sink API of
 * the reference (fifo.h:19-62, sdr.h:18-39 constants) which libgpsb200.so also
 * exports (pinned host buffers, fixed tail handling) so that the reference's
 * consumers (sdr_iqfile.c:22-55, sdr_hackrf.c:236-248, sdr_pluto.c:45-94) work
 * unmodified against it.
 */
#ifndef GPSB200_H
#define GPSB200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- constants of the reference (sdr.h:21-34, gps.h:36-57) ------------------ */
#define GPSB200_SAMPLERATE        3000000           /* TX_SAMPLERATE, sdr.h:21 */
#define GPSB200_BLOCK_SAMPLES     300000            /* NUM_IQ_SAMPLES, sdr.h:26 */
#define GPSB200_BLOCK_ELEMS       600000            /* IQ_BUFFER_SIZE, sdr.h:29 (I and Q count separately) */
#define GPSB200_MAX_CHAN          32                /* reference ships MAX_CHAN 12 (gps.h:36); 32 = all PRNs */
#define GPSB200_NAV_WORDS         60                /* N_DWRD, gps.h:52 */
#define GPSB200_CA_LEN            1023              /* CA_SEQ_LEN, gps.h:57 */
#define GPSB200_SC08              1                 /* gps-sim.h:27 */
#define GPSB200_SC16              2                 /* gps-sim.h:28 */
#define GPSB200_HACKRF_BUFFER     262144            /* HACKRF_TRANSFER_BUFFER_SIZE, sdr.h:34 */

/* ---- error codes ------------------------------------------------------------ */
enum {
    GPSB200_OK = 0,
    GPSB200_ERR_ARG = -1,        /* bad argument (NULL, count, sample size, prn, NAV index) */
    GPSB200_ERR_CUDA = -2,       /* CUDA runtime error; text via gpsb200_last_error() */
    GPSB200_ERR_RANGE = -3,      /* sum of channel amplitudes would overflow the int16 I/Q the reference stores */
    GPSB200_ERR_NOMEM = -4,
    GPSB200_ERR_INTERNAL = -5,   /* device self-check failed (would mean a bug; never returns wrong samples silently) */
    GPSB200_ERR_END = -6         /* gpsb200_scenario_advance / _key: no block of the run left */
};

/* One channel for one 0.1 s block: the fields of the reference's channel_t
 * (gps.h:213-236) and gain[] (gps.c:2300) that the sample loop reads, as left by
 * computeCodePhase (gps.c:2033-2064) and the gain update (gps.c:2749-2763).
 * dataBit/codeCA are not passed: they are functions of (iword, ibit, NAV words)
 * and (code_phase, prn) respectively (gps.c:2059-2060). */
typedef struct gpsb200_chan {
    int32_t prn;          /* 1..32; <= 0: channel unused this block (gps.c:2772) */
    int32_t iword;        /* NAV word index 0..59  (gps.c:2052) */
    int32_t ibit;         /* bit in word 0..29     (gps.c:2055) */
    int32_t icode;        /* code period in bit 0..19 (gps.c:2058) */
    int32_t nav_frame;    /* which NAV frame (set of 60 words) this block uses, see gpsb200_set_nav */
    int32_t reserved;
    double f_carr;        /* Hz, Doppler (gps.c:2043); |f_carr| < 2.9 MHz */
    double f_code;        /* Hz (gps.c:2044); 0 < f_code <= 1.07 MHz */
    double carr_phase;    /* cycles in [0,1): used for the first block of a call and whenever prn differs
                             from the previous block's prn in the same slot (allocateChannel, gps.c:2203-2210);
                             otherwise the phase is carried from the previous block (gps.c:2821-2826) */
    double code_phase;    /* chips in [0,1023) (gps.c:2049) */
    double gain;          /* gps.c:2756 (x2 for Pluto, gps.c:2759-2763) */
} gpsb200_chan_t;         /* 64 bytes */

typedef struct gpsb200_config {
    int32_t device;            /* CUDA device ordinal */
    int32_t max_chan;          /* 1..32 */
    int32_t max_blocks;        /* largest nblk of one gpsb200_synth_* call */
    int32_t max_nav_frames;    /* NAV frames held at once (>= 1) */
    int32_t host_threads;      /* threads for the exact carrier-phase chain; 0 = auto */
    int32_t run_samples;       /* device work unit, divides 300000 and is a multiple of 32; 0 = default (2400) */
} gpsb200_config_t;

typedef struct gpsb200_ctx gpsb200_ctx_t;

/* Per-call statistics (filled when the pointer is not NULL). Times in milliseconds. */
typedef struct gpsb200_stats {
    double host_chain_ms;      /* host share of the carrier chain: start-phase guesses + fix-up scan */
    double h2d_ms, kernel_ms, d2h_ms;   /* kernel_ms: CUDA-event span of the call's stream (host-destination calls only);
                                           h2d_ms / d2h_ms: reserved, always 0 (transfers overlap the kernels) */
    double checkpoint_kernel_ms, synth_kernel_ms, probe_kernel_ms;
    int64_t h2d_bytes, d2h_bytes;
    int32_t launches;          /* kernels launched by this call */
    int32_t chain_fallbacks;   /* blocks the host had to walk sequentially (their block probe was unusable) */
} gpsb200_stats_t;

/* Threading: a context may be used by one thread at a time; different contexts (same or different devices)
 * may be used concurrently from different threads, every entry point selects the context's device itself.
 * The FIFO below is process-global with one producer and one consumer, as in the reference (fifo.c:21-29). */
int gpsb200_create(const gpsb200_config_t *cfg, gpsb200_ctx_t **out);
void gpsb200_destroy(gpsb200_ctx_t *ctx);
const char *gpsb200_last_error(const gpsb200_ctx_t *ctx);
const char *gpsb200_version(void);

/* Deployment helper, the counterpart of the reference's thread_to_core() (gps-sim.c:251-262, called by
 * gps_thread_ep, gps.c:2377): bind the CALLING thread (and every thread it creates afterwards: the
 * context's host workers, the iqfile writer) to the CPUs of the NUMA node the CUDA device `device`
 * hangs off, so that page-locked result buffers allocated afterwards (fifo_create, cudaHostAlloc) are
 * local to the GPU's PCIe root. Call before gpsb200_create / fifo_create. Returns the NUMA node (>= 0),
 * -1 when the platform reports none (nothing changed), or GPSB200_ERR_CUDA. */
int gpsb200_bind_numa(int device);

/* NAV words of one channel for one 30 s frame: channel_t.dwrd (gps.h:227) as
 * built by generateNavMsg (gps.c:2066-2140); only bits 29..0 are used
 * (gps.c:2812). Copied; may be updated between synth calls. */
int gpsb200_set_nav(gpsb200_ctx_t *ctx, int frame, int chan, const uint32_t dwrd[GPSB200_NAV_WORDS]);

/* Synthesize nblk consecutive 0.1 s blocks (replaces gps.c:2767-2857 nblk times).
 *   chans       [nblk][nchan], host memory; 1 <= nchan <= cfg.max_chan (slot c of a call is NAV row c of the context)
 *   sample_size GPSB200_SC08: dst is int8  I,Q interleaved, iq >> 4 with modulo-256 narrowing (gps.c:2844)
 *               GPSB200_SC16: dst is int16 I,Q interleaved (gps.c:2842)
 *   dst         host memory (pinned is faster), nblk * 600000 elements, block after block
 *   carr_phase_out  optional [nchan]: carrier phase after the last block (what the reference
 *               leaves in channel_t.carr_phase), to seed the next call
 * Blocking: returns when dst is complete. */
int gpsb200_synth_blocks(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                         int sample_size, void *dst, double *carr_phase_out, gpsb200_stats_t *stats);

/* Same, but block b goes to its own host buffer dst_blocks[b] (600000 elements each) -- e.g. buffers handed out by
 * fifo_acquire(): the device->host copies land straight in iq->data8 / iq->data16 (SURVEY 8b ownership: the producer
 * owns a buffer between acquire and enqueue), no staging copy on the host. */
int gpsb200_synth_blocks_scatter(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                                 int sample_size, void *const *dst_blocks, double *carr_phase_out,
                                 gpsb200_stats_t *stats);

/* Same, but the output stays in device memory (dst_device: 16-byte aligned device pointer with room for
 * nblk * 600000 elements; the kernels store 16-byte words, a misaligned dst_device is GPSB200_ERR_ARG, as for
 * gpsb200_slice_prepare and gpsb200_replay_device) and the synthesis is only ENQUEUED on `stream` (a cudaStream_t,
 * 0 = the context's own stream) -- the caller synchronizes before reading dst_device. The call itself returns when
 * the speculative pre-phase (block probes, span chaining), the host scan and the run checkpoints are done and the
 * device self-check of the carrier chain has been read (a failed check returns GPSB200_ERR_INTERNAL, and nothing of the
 * call is left in flight); it never waits for the synthesis, with or without a stats request (stats then carry no
 * synthesis time). Used for kernel-resident consumers and by bench.py's one-GPU value leg. */
int gpsb200_synth_blocks_device(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                                int sample_size, void *dst_device, void *stream,
                                double *carr_phase_out, gpsb200_stats_t *stats);

/* ---- time-slice hand-over (multi-GPU: rank r makes blocks [lo_r, hi_r) of ONE stream) -----------------
 * The only state a slice needs from the blocks before it is each slot's exact carrier phase (gps.c:2821-2826
 * never resets carr_phase). Its resolution is parallel in time (block probes on the GPU chained per span, then
 * one host step per span), so a rank can do almost all of it before the incoming phases exist. One device-path
 * call is therefore offered in three steps:
 *   1. gpsb200_slice_prepare  host records, parameters up, carrier tables; fills *link: how this slice maps an
 *                             incoming chain state to the (closed-form, GUESSED) outgoing one. Ranks exchange
 *                             their links and compose them with gpsb200_link_apply() to obtain good guesses of
 *                             their incoming state without any GPU work.
 *   2. gpsb200_slice_probe    incoming state as GUESSED (NULL: the slice starts the stream): speculative block
 *                             probes + span chaining are enqueued (all of them at once if `eager`).
 *   3. gpsb200_slice_finish   incoming state EXACT (prn_in/phase_in, from the previous rank's *_out; NULL: the
 *                             stream starts here): segment by segment, as soon as a segment's probes are done, the
 *                             host scan over its span summaries, its run checkpoints (with the device self-check) and
 *                             its synthesis are enqueued -- the synthesis of early segments overlaps the probes of
 *                             later ones. prn_out/phase_out (exact state after the slice) are valid on return --
 *                             BEFORE the synthesis has run -- and are what the next rank's gpsb200_slice_finish takes.
 *   4. gpsb200_slice_wait     blocks until the slice is complete and returns the verdict of the device self-check
 *                             (GPSB200_ERR_INTERNAL: the output must not be used).
 * A slot continues the incoming phase only when it still holds the same satellite (prn_in[c] == prn of its first
 * block, > 0); otherwise its first block takes carr_phase from chans, exactly as between the blocks of one call.
 * chans must stay valid until gpsb200_slice_prepare returns. gpsb200_synth_blocks_device gives the same result as the
 * three steps with NULL incoming states; the one-call path schedules its segments as DESIGN §6 describes. */
typedef struct gpsb200_slice_link {
    int32_t prn_first[GPSB200_MAX_CHAN];    /* satellite of each slot in the slice's first block (0: idle) */
    int32_t prn_last[GPSB200_MAX_CHAN];     /* ... in its last block */
    int32_t reset_inside[GPSB200_MAX_CHAN]; /* 1: the slot was (re)allocated or idle inside the slice: value is absolute */
    double first_phase[GPSB200_MAX_CHAN];   /* carr_phase of the first block (used when the slot does not continue) */
    double value[GPSB200_MAX_CHAN];         /* guessed phase after the slice (absolute), or the advance over the slice */
} gpsb200_slice_link_t;
/* dst_device (16-byte aligned) and/or dst_host: with dst_host != NULL the synthesis is launched in chunks whose downloads into dst_host
 * (pinned memory) overlap later chunks, dst_device may then be NULL (a context-owned staging buffer is used);
 * gpsb200_slice_wait blocks until synthesis and downloads of the slice are complete and reports the self-check. */
int gpsb200_slice_prepare(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size,
                          void *dst_device, void *dst_host, void *stream, gpsb200_slice_link_t *link);
int gpsb200_slice_wait(gpsb200_ctx_t *ctx);
/* eager != 0: the speculative work of the WHOLE slice is submitted at once, ahead of everything else -- for a rank
 * whose successor waits for the outgoing state. eager == 0: only the first pipeline segment's; the others follow
 * segment by segment inside gpsb200_slice_finish, each behind the previous segment's synthesis (in whose shadow the
 * latency-bound walk kernels then run) and from guesses re-anchored on the exact state just resolved -- for the last
 * rank and for single-GPU use. */
int gpsb200_slice_probe(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_guess_in, int eager);
int gpsb200_slice_finish(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_in, int32_t *prn_out,
                         double *phase_out, gpsb200_stats_t *stats);
/* Same with a hand-over callback: invoked with the exact outgoing state as soon as the host scan has it -- for an
 * eager slice BEFORE the long kernels are enqueued, so that a message to the successor (an NCCL send is a kernel too)
 * does not queue behind this slice's own synthesis. */
typedef void (*gpsb200_handoff_fn)(void *user, const int32_t *prn_out, const double *phase_out);
int gpsb200_slice_finish_cb(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_in, int32_t *prn_out,
                            double *phase_out, gpsb200_stats_t *stats, gpsb200_handoff_fn handoff, void *user);
/* Host only: the link of a slice from its parameters alone (identical to what gpsb200_slice_prepare fills). */
int gpsb200_slice_link_host(const gpsb200_chan_t *chans, int nblk, int nchan, gpsb200_slice_link_t *link);
/* Host only: (prn_in, phase_in) -> guessed (prn_out, phase_out) after the slice `link` describes. */
int gpsb200_link_apply(const gpsb200_slice_link_t *link, int nchan, const int32_t *prn_in, const double *phase_in,
                       int32_t *prn_out, double *phase_out);

/* Test hook of the device self-check: corrupt the resolved carrier chain of the next calls by one unit of the
 * rounding grid (on == 1), or the carrier state one block probe recorded at a checkpoint-segment start (on == 2: slot 0,
 * sixth block of a pipeline segment, middle segment, both parity variants); every synth call must then fail with
 * GPSB200_ERR_INTERNAL instead of returning samples. on == 0: off. */
int gpsb200_debug_corrupt_chain(gpsb200_ctx_t *ctx, int on);

/* Test hook: copy the run checkpoints of the previous synth call (nblk x 300000/run_samples x nchan records of 24 bytes:
 * carrier phase, code phase, NAV position iword | ibit << 8 | icode << 16, pad) to host memory. Waits for the context's
 * work to complete. */
int gpsb200_debug_run_checkpoints(gpsb200_ctx_t *ctx, int nblk, int nchan, void *out);

/* Test hook: copy the carrier block probes of the previous synth call of more than two blocks to host memory:
 * probes_out gets nblk x nchan records of 64 bytes (the layout gpsb200_carrier_probe_host writes), seg_out (NULL: not
 * wanted) nblk x nchan x 14 doubles, the probes' states at the checkpoint-segment starts as gpsb200_carrier_probe_host
 * orders them (entries the probe did not record hold whatever the buffer held), guess_out (NULL: not wanted) nblk x
 * nchan doubles, the guessed start phases the probes walked from. Waits for the context's work to complete. */
int gpsb200_debug_block_probes(gpsb200_ctx_t *ctx, int nblk, int nchan, void *probes_out, double *seg_out,
                               double *guess_out);

/* Test hook: the shape of ONE synthesis launch over nblk blocks of nchan channels on this context's device as it stands
 * (nblk may exceed cfg.max_blocks): *kernel = "k_synth_lanes" or "k_synth" (as gpsb200_synth_kernel_name), how many CTAs
 * share a block and how many runs each CTA takes (the last CTA of a block may take fewer). Which launches a call makes
 * depends on its path: a host-destination call launches per chunk of at most 256 blocks, a call of at most two blocks
 * and a slice call per segment, an eager device-destination call once over the whole call. Enqueues nothing. */
int gpsb200_debug_synth_shape(gpsb200_ctx_t *ctx, int nblk, int nchan, int sample_size, const char **kernel,
                              int *ctas_per_block, int *runs_per_cta);

/* Name of the synthesis kernel a call with nchan channels launches on this context as it stands: "k_synth_lanes"
 * (lane = sample: run length a multiple of 96 up to 2400, every code rate seen so far within 1.0157 .. 1.0302 MHz,
 * GPSB200_LANES != 0) or "k_synth" (lane = channel, no such conditions). Both are bit-exact; for reporting. */
const char *gpsb200_synth_kernel_name(const gpsb200_ctx_t *ctx, int nchan);

/* Re-run the device part of the previous gpsb200_synth_blocks_device call (parameters,
 * start phases and guesses already resident in HBM): used by bench.py to time the kernels
 * alone. dst_device: 16-byte aligned, or NULL for the previous call's destination. kernel_mask bits: 8 = carrier
 * tables, 4 = carrier probe, 1 = run checkpoints, 2 = synthesis. */
int gpsb200_replay_device(gpsb200_ctx_t *ctx, void *dst_device, void *stream, int kernel_mask);

/* Exact carrier phase after n samples of Doppler f_carr (the chain of gps.c:2821-2826
 * without stepping every sample); host-only helper, also used by time-slice sharding
 * to seed a rank's first block. */
double gpsb200_carrier_advance(double carr_phase, double f_carr, int64_t nsamples);

/* Exact carrier phases after nblk blocks for every channel slot (same chaining rule as
 * gpsb200_synth_blocks; phase_in == NULL: block 0 takes chans[0][c].carr_phase, else
 * phase_in[c] continues a previous call). Host only, `threads` worker threads. A rank of a
 * time-slice sharded run calls this on the blocks BEFORE its slice to seed its first block. */
int gpsb200_carrier_chain(const gpsb200_chan_t *chans, int nblk, int nchan, const double *phase_in,
                          double *phase_out, int threads);

/* Same result as gpsb200_carrier_chain, but resolved with the context's parallel-in-time machinery
 * (device probe kernel + host fix-up scan, no synthesis)
 * instead of seconds of sequential host walking. nblk may exceed cfg.max_blocks. A rank of a
 * time-slice sharded run seeds its first block with this. */
int gpsb200_carrier_chain_device(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                                 const double *phase_in, double *phase_out);

/* Host-only view of the parallel-in-time carrier chain (what the device probe kernel plus
 * the host fix-up do per block): walk `nsamples` from the GUESSED phase, then derive the exact
 * end phase of the TRUE start phase from it. Returns 1 and *end_out when the speculation is
 * accepted (then *end_out == gpsb200_carrier_advance(start, ...), bit for bit), 0 when it is
 * rejected (the pipeline then walks that block sequentially). For tests. */
int gpsb200_carrier_probe_fixup(double start, double guess, double f_carr, int64_t nsamples, double *end_out);

/* Host-only model of the two-level (span) resolution of the chain for one satellite over nblk blocks with Doppler
 * f_carr[j]: block probes from guesses derived from start_guess, speculative chaining of the span for both parity
 * variants, ONE fix-up with the true start. Returns 1 and the exact start phase of every block plus the end phase
 * (starts_out[nblk + 1]) when the span-level speculation is accepted, 0 when it is rejected (the pipeline then
 * resolves the span block by block). For tests. */
int gpsb200_span_chain_host(const double *f_carr, int nblk, double start_true, double start_guess, double *starts_out);

/* Host-only model of how the run-checkpoint kernel starts the J checkpoint segments of ONE block (J = min(8, runs per
 * block); segment j starts at run floor(j * runs / J)): the block probe from start_guess records its trajectory at the
 * segment starts, the fix-up with the true start picks its parity variant and shift, and segment j >= 1 starts from
 * the recorded state plus the shift when it starts at or after the probe's first wrap. run_samples divides 300000.
 * starts_out[8]: starts_out[0] = start_true, derived starts for j >= 1, NaN for segments that are walked from the
 * block start instead (and past J). Returns 1 when the fix-up accepts the probe (every derived start then equals
 * gpsb200_carrier_advance(start_true, f_carr, j-th segment start) bit for bit), 0 when it rejects it. For tests. */
int gpsb200_checkpoint_segments_host(double start_true, double start_guess, double f_carr, int run_samples,
                                     double *starts_out, int *nseg_out);

/* Host-only: the carrier block probe the probe kernel computes for a walk of nsamples (< 2^31) from the guessed phase
 * `guess` at Doppler f_carr. mode 0: each parity variant walked on its own (the reference formulation); mode 1: both
 * variants in lockstep (what the kernel runs). probe_out: 64 bytes, x_w, x_end[2], m_pos[2], m_neg[2] (doubles), n_w,
 * pad (int32). seg_out (used when run_samples > 0, which must divide nsamples): 2 x 7 doubles, variant v's state at the
 * start of checkpoint segment j = 1 .. J - 1 (J = min(8, nsamples / run_samples)) at seg_out[7 v + j - 1]; NaN where
 * the walk records none (segments before the first wrap or past J - 1, an unusable variant). Both modes write the same
 * bytes. For tests. */
int gpsb200_carrier_probe_host(double guess, double f_carr, int64_t nsamples, int run_samples, int mode, void *probe_out,
                               double *seg_out);

/* Host model of the lane = sample synthesis kernel (csrc/synth_lanes.h) for ONE block: the same window / band / repair
 * logic, executed on the CPU, int16 I/Q out. force bits: 1 = repair every sample's index, 2 = exact chip signs for every
 * window, 4 = every repair walks exactly from the run anchor, 8 = carry points of every window by the FP64 second
 * opinion instead of the 32-bit estimate. counters[4] = fast samples, repaired samples, exactly
 * rebuilt sign windows, exact walks. signs (NULL: not wanted) [nchan][3125][3]: the sign words of every 96-sample
 * window of the block as the synthesis reads them (word j, bit 11 (i mod 3) + i / 3: chip XOR data bit of sample
 * 32 j + i; idle channels untouched). For tests (the algorithm against the oracle without a GPU); not a product path. */
int gpsb200_lanes_model_block(const gpsb200_chan_t *chans, int nchan, const uint32_t *nav, int run_samples, int force,
                              int16_t *iq, double *carr_out, int64_t *counters, uint32_t *signs);

/* The window band certification of the lane = sample synthesis (csrc/synth_lanes.h), for n (step, base) pairs: out[i] = 1
 * when some sample m < 96 of a window with 32-bit carrier phase base bases[i] and increment steps[i] has a phase
 * bases[i] + m * steps[i] (mod 2^32) whose low 23 bits are 2^23 - 128 or more, else 0; what the kernel decides per
 * (channel, window) from the sorted residues of the step. Consecutive equal steps share one residue list. For tests. */
int gpsb200_lanes_window_band_host(const uint32_t *steps, const uint32_t *bases, int64_t n, uint8_t *out);

/* C/A code of prn (1..32) as 0/1 chips (codegen, gps.c:272-309). */
int gpsb200_codegen(int prn, uint8_t ca[GPSB200_CA_LEN]);

/* ---- acquisition search: which satellites does an I/Q stream contain? ------------------------------------------------
 * The first step of a GPS receiver, for interleaved I/Q at 3 Msps (one C/A period = 3000 samples): for each requested PRN
 * a search over code delay tau (0..2999 samples) x Doppler bin j (f_j = f_lo_hz + j * step_hz), over K coherent 1 ms
 * periods summed non-coherently. Its results seed the tracking loops below (gpsb200_track_start); no navigation
 * solution. Exact integer
 * arithmetic, deterministic (DESIGN §9; tests/acq_model.py states it in numpy):
 *   samples    int8 as is; int16 reduced to clamp(x >> 4, -128, 127) (the int8 stream's scale, saturated where the int8
 *              stream wraps)
 *   window     samples s0 .. s0 + 3000 K + 2998 (3000 K + 2999 of them) of a buffer of nsamples; m = sample - s0
 *   carrier    u_j = (uint32) llround(f_j * 2^32 / 3e6), phase (uint32)(m * u_j), index phase >> 23 into the
 *              synthesizer's 512-entry cos/sin tables (|entry| <= 250)
 *   wipe-off   I_d = I cos + Q sin, Q_d = Q cos - I sin (int32, |.| <= 64000): the stream's e^{+j phi} is removed, so the
 *              peak is at f_j ~ f_carr of the channel record
 *   replica    c_p[n] = 2 ca_p[(n * 1023) / 3000] - 1, n < 3000 (ca_p: gpsb200_codegen)
 *   correlate  C_I(k, tau) = sum_{n<3000} c_p[n] I_d[3000 k + tau + n], C_Q likewise (int32, |.| <= 1.92e8)
 *   power      P(j, tau) = sum_{k<K} C_I^2 + C_Q^2 (uint64, <= K * 7.4e16: hence K <= 100)
 *   result     (j1, tau1) = argmax P, ties to the lowest j, then the lowest tau; p1 = P(j1, tau1); p2 = the largest
 *              P(j1, tau) with circular distance |tau - tau1| (period 3000) > 3 samples, outside the +-1-chip
 *              correlation triangle; ratio = p1 / p2 (infinity when p2 is 0). */
#define GPSB200_ACQ_MAX_MS    100
#define GPSB200_ACQ_MAX_BINS  1024
#define GPSB200_ACQ_CODE_SAMPLES 3000
typedef struct gpsb200_acq_config {
    int64_t s0;            /* first sample of the window (sample = one I,Q pair) */
    int32_t ms;            /* K, coherent 1 ms periods: 1..GPSB200_ACQ_MAX_MS */
    int32_t nprn;          /* 1..32 entries of prn[] */
    int32_t prn[32];       /* 1..32 each */
    double f_lo_hz;        /* first Doppler bin */
    double step_hz;        /* bin spacing (> 0 when nbins > 1); every bin within +-1.5 MHz */
    int32_t nbins;         /* 1..GPSB200_ACQ_MAX_BINS */
    int32_t reserved;
} gpsb200_acq_config_t;    /* 168 bytes */
typedef struct gpsb200_acq_result {
    int32_t prn;
    int32_t bin;           /* j1 */
    int32_t delay;         /* tau1: samples from s0 to where the code's chip 0 starts, modulo 3000 */
    int32_t reserved;
    double doppler_hz;     /* f_j1 */
    double delay_chips;    /* tau1 * 1023 / 3000 */
    uint64_t p1, p2;
    double ratio;          /* p1 / p2: a receiver counts the PRN as acquired above a threshold (gpsb200-acq: 2.5) */
} gpsb200_acq_result_t;    /* 56 bytes */
/* Search nsamples samples of host memory (int8 or int16 I,Q interleaved, sample_size GPSB200_SC08 / GPSB200_SC16); only
 * the window is copied to the device. res: [cfg->nprn] in the order of cfg->prn. grid (NULL: not wanted): host
 * [nprn][nbins][3000] uint64, the whole P. Every argument is checked before anything is enqueued (GPSB200_ERR_ARG).
 * Blocking; scratch is allocated on the context's device as needed. */
int gpsb200_acquire(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *cfg,
                    gpsb200_acq_result_t *res, uint64_t *grid);
/* Same for a source in device memory (16-byte aligned, as gpsb200_synth_blocks_device's dst_device, else GPSB200_ERR_ARG),
 * searched in place: the search is enqueued on `stream` (0 = the context's own stream) behind whatever it holds -- e.g.
 * the synthesis of that buffer -- and the call returns when the results (and grid, in host memory) are in. */
int gpsb200_acquire_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                           const gpsb200_acq_config_t *cfg, gpsb200_acq_result_t *res, uint64_t *grid, void *stream);
/* ---- per-PRN Doppler windows: the search above with a bin grid of each PRN's own (DESIGN §9.1) ----------------------
 * A warm start (gpsb200_almanac_predict) knows each visible PRN's Doppler to a few hundred Hz and searches a few bins
 * around it instead of the whole grid. The arguments are gpsb200_acquire's plus f_lo_prn[cfg->nprn]:
 *   bins       bin j of the p-th requested PRN (cfg->prn[p]) is f_{p,j} = f_lo_prn[p] + j * cfg->step_hz, j < cfg->nbins;
 *              cfg->f_lo_hz is ignored; every f_lo_prn[p] finite and every bin within +-1.5 MHz
 *   the rest   samples, window, u_{p,j} = (uint32) llround(f_{p,j} * 2^32 / 3e6), tables, replica, K, P, the argmax with
 *              its tie rules and p2: as above, per PRN over its own bins; res[p].doppler_hz = f_{p,j1}
 * So row p of the result (and of the grid) equals gpsb200_acquire run with prn = {cfg->prn[p]} and f_lo_hz = f_lo_prn[p],
 * bit for bit. Every argument is checked before anything is enqueued (GPSB200_ERR_ARG; f_lo_prn NULL included). */
int gpsb200_acquire_windows(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                            const gpsb200_acq_config_t *cfg, const double *f_lo_prn, gpsb200_acq_result_t *res,
                            uint64_t *grid);
/* Test hook: the CTAs per (bin, PRN) row of a search of nprn x nbins rows on this context's device (1, 2, 3, 4 or 6; a
 * split search gives the same results, DESIGN §9.1). force 0 restores the automatic choice, 1, 2, 3, 4 or 6 fixes every
 * later search of the context to that split, -1 leaves the setting; GPSB200_ERR_ARG otherwise. Enqueues nothing. */
int gpsb200_debug_acq_split(gpsb200_ctx_t *ctx, int force, int nprn, int nbins);
int gpsb200_acquire_windows_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                   const gpsb200_acq_config_t *cfg, const double *f_lo_prn, gpsb200_acq_result_t *res,
                                   uint64_t *grid, void *stream);

/* ---- tracking: code and carrier loops over an I/Q stream, one coherent period per C/A code epoch ---------------------
 * A closed loop per channel, sequential in time, in exact integer arithmetic so that it is reproducible bit for bit
 * (DESIGN §10; tests/track_model.py states it in numpy). Samples are reduced as for the acquisition search (int8 as is,
 * int16 to clamp(x >> 4, -128, 127)), and the carrier tables are the synthesizer's. ">>" is an arithmetic shift (floor),
 * "/" a division truncating toward zero, M = 1023 * 2^32, H = 2^31 (half a chip).
 *   period     starts at sample s, where the local prompt code wraps; its code phase there is phi (2^-32 chip units,
 *              phi < GPSB200_TRK_CODE_STEP_MAX) and its code step u (GPSB200_TRK_CODE_STEP_MIN..MAX per sample), so it
 *              holds L = ceil((M - phi) / u) samples, 2999 <= L <= 3001 (u >= M / 3001 gives L <= 3001;
 *              phi < u_max <= M / 2999 gives L >= 2999); the next one starts at s + L with phi' = phi + L u - M < u.
 *   carrier    theta_m = theta + m * w (uint32, w the int32 carrier step in 3e6/2^32 Hz), index theta_m >> 23;
 *              I_d = I cos + Q sin, Q_d = Q cos - I sin (the stream is code * e^{+j phase}, so a locked w ~ f_carr)
 *   replicas   c(x) = 2 ca[x >> 32] - 1; prompt at phi_m = phi + m u, early at (phi_m + H) mod M, late at (phi_m - H) mod M
 *   sums       E_I = sum_{m<L} c(early) I_d, E_Q, P_I, P_Q, L_I, L_Q likewise: int32 (|.| <= 3001 * 64000 < 2^31)
 *   angle(x,y) for x >= 0: both shifted right by max(0, bitlen(max(|x|, |y|)) - 30), then 24 CORDIC vectoring steps
 *              i = 0..23: y > 0 ? (x + (y >> i), y - (x >> i), z + A_i) : (x - (y >> i), y + (x >> i), z - A_i) from
 *              z = 0; A_i = round(atan(2^-i) / 2 pi * 2^32) (listed in csrc/track.h); z in 2^-32 turns. angle(0, 0) = 0
 *              (the steps would give -0.277 turn): a period or window of zeros steers nothing. Small vectors keep
 *              the steps' error, at most 1/r turn + 90 units at magnitude r (0.056 turn at r = 2; DESIGN §10)
 *   PLL        (x, y) = (P_I, P_Q), negated when P_I < 0 (Costas: data bits do not matter); e = angle(x, y)
 *   FLL        for 1 <= epochs < GPSB200_TRK_FLL_EPOCHS: cross = I' P_Q - Q' P_I, dot = I' P_I + Q' P_Q (int64, I', Q'
 *              the previous prompt), both negated when dot < 0; d = angle(dot, cross); F += (64 d) / 3000
 *   filter     F += e >> 12, clamped to +-2^34 (F: int64, 2^-10 carrier step units); w' = (F >> 10) + (e >> 16)
 *   DLL        E = E_I^2 + E_Q^2, L = L_I^2 + L_Q^2 (int64), both shifted right by max(0, bitlen(E + L) - 40);
 *              D = ((E - L) << 14) / (E + L) (0 when E + L = 0); u' = clamp(GPSB200_TRK_CODE_STEP_NOM + w' / 1540 +
 *              (2048 D) / 3000, GPSB200_TRK_CODE_STEP_MIN, GPSB200_TRK_CODE_STEP_MAX) (carrier aiding: f_code =
 *              1.023 MHz + f_carr / 1540)
 *   lock       A_I += (|P_I| - A_I) >> 4, A_Q += (|P_Q| - A_Q) >> 4; locked when 3 A_Q < A_I (phase error below
 *              about 18 degrees, the narrow-band indicator as a ratio of integers)
 * The next period runs with theta' = theta + L w, phi', w', u'. A call runs each channel's periods while the period lies
 * inside the buffer and fewer than max_epochs were written; the state out continues the run, so any cut of a run into
 * calls gives the epochs of one call, bit for bit. */
#define GPSB200_TRK_CODE_STEP_NOM 1464583848u   /* round(1.023e6 / 3e6 * 2^32) */
#define GPSB200_TRK_CODE_STEP_MIN 1464095816u   /* ceil(M / 3001) */
#define GPSB200_TRK_CODE_STEP_MAX 1465072205u   /* floor(M / 2999) */
#define GPSB200_TRK_FLL_EPOCHS    200
#define GPSB200_TRK_MAX_CHAN      32
typedef struct gpsb200_track_state {
    int32_t prn;           /* 1..32 */
    int32_t epochs;        /* periods tracked so far, >= 0 */
    int64_t sample;        /* first sample of the next period (absolute: the stream's sample index) */
    uint64_t code_phase;   /* prompt code phase at `sample`, 2^-32 chips, < GPSB200_TRK_CODE_STEP_MAX */
    int64_t carr_freq;     /* F: loop-filter frequency in 2^-10 carrier step units, |F| <= 2^34 */
    uint32_t carr_phase;   /* theta at `sample` */
    int32_t carr_step;     /* w of the next period: 3e6 / 2^32 Hz units */
    uint32_t code_step;    /* u of the next period: 2^-32 chips per sample */
    int32_t prev_i, prev_q;/* prompt sums of the last period (FLL) */
    int32_t lock_i, lock_q;/* A_I, A_Q, >= 0 */
    int32_t lock;          /* 1 when locked after the last period */
} gpsb200_track_state_t;   /* 64 bytes */
typedef struct gpsb200_track_epoch {
    int64_t sample;        /* first sample of the period */
    int32_t e_i, e_q, p_i, p_q, l_i, l_q;
    uint32_t carr_phase;   /* theta' at the next period's first sample */
    int32_t carr_step;     /* w' */
    uint32_t code_phase;   /* phi' */
    uint32_t code_step;    /* u' */
    int32_t lock;
    int32_t reserved;
} gpsb200_track_epoch_t;   /* 56 bytes */
/* The start of a channel from an acquisition: prn, Doppler (|doppler_hz| <= 10 kHz) and the sample where the code's chip 0
 * starts (s0 + gpsb200_acq_result_t.delay): w = (int32) llround(doppler_hz * 2^32 / 3e6), F = 1024 w, u = clamp(NOM +
 * w / 1540), phi = theta = 0, everything else 0. GPSB200_ERR_ARG on a bad argument. Host only. */
int gpsb200_track_start(int prn, double doppler_hz, int64_t sample, gpsb200_track_state_t *state);
/* Track nchan (1..GPSB200_TRK_MAX_CHAN) channels over nsamples samples of host memory (int8 / int16 I,Q interleaved) whose
 * first sample is the stream's sample `base`; every state's sample must be >= base. state: [nchan], in and out.
 * epochs: [nchan][max_epochs] (max_epochs >= 1), nepochs: [nchan] written. Every argument is checked before anything is
 * enqueued (GPSB200_ERR_ARG). Blocking. */
int gpsb200_track(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base,
                  gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                  int32_t *nepochs);
/* Same for a source in device memory (16-byte aligned), tracked in place on `stream` (0 = the context's own stream)
 * behind whatever it holds; returns when the epochs and states are in host memory. */
int gpsb200_track_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size, int64_t base,
                         gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                         int32_t *nepochs, void *stream);

/* ---- navigation message from the epochs of one tracked channel (host; csrc/navdecode.cpp) ----------------------------
 *   bit sync   histogram over the 20 epoch positions (index mod 20) of prompt-I sign changes between consecutive locked
 *              epochs; the edge is the position with most changes (the lowest on ties; none: no bits)
 *   bits       bit k = the sum of the 20 prompt I's from epoch edge + 20 k on; value (sum > 0)
 *   frame sync the first bit index i >= 2 where bits i..i+7 are the preamble 10001011 or its complement (the Costas
 *              180 degree ambiguity, resolved by inverting every bit), and, so inverted, the TLM word (bits i..i+29) and
 *              the HOW (i+30..i+59) pass IS-GPS-200 parity with D29*, D30* of the bits before each, and the HOW's
 *              subframe id is 1..5
 *   words      every complete 30-bit word from i on: the bits as transmitted (what the synthesizer's NAV word holds in
 *              bits 29..0), the 24 data bits with D30* undone, the parity verdict; subframe id and TOW of HOW words */
typedef struct gpsb200_nav_bit {
    int64_t sample;        /* first sample of the bit's first epoch */
    int64_t sum;           /* the 20 prompt I's */
    int32_t value;         /* (sum > 0), inverted when the frame sync found the inverted preamble */
    int32_t locked;        /* 1 when all 20 epochs were locked */
} gpsb200_nav_bit_t;       /* 24 bytes */
typedef struct gpsb200_nav_word {
    int64_t sample;        /* first sample of the word's first bit */
    uint32_t raw;          /* the 30 bits as transmitted, first bit in bit 29 */
    uint32_t data;         /* the 24 data bits, D30* undone */
    int32_t parity_ok;
    int32_t subframe;      /* HOW (second word of a subframe): subframe id, else 0 */
    int32_t tow;           /* HOW: the 17-bit TOW count (the next subframe's start, in 6 s units), else -1 */
    int32_t index;         /* words since frame sync: 0 is the first TLM */
} gpsb200_nav_word_t;      /* 32 bytes */
typedef struct gpsb200_nav_sync {
    int32_t bit_edge;      /* epoch index of the first bit (0..19), -1: no bit sync */
    int32_t nbits;
    int32_t frame_bit;     /* bit index of the first TLM, -1: no frame sync */
    int32_t inverted;
    int32_t nwords;
    int32_t words_ok;      /* with good parity */
    int32_t subframes;     /* HOW words with good parity */
    int32_t first_tow;     /* TOW of the first good HOW, -1: none */
} gpsb200_nav_sync_t;      /* 32 bytes */
/* Decode the n epochs of one channel (in time order). bits: [max_bits >= n / 20], words: [max_words >= n / 600]; either
 * may be NULL when its count is 0. GPSB200_ERR_ARG on a bad argument. */
int gpsb200_nav_decode(const gpsb200_track_epoch_t *epochs, int64_t n, gpsb200_nav_bit_t *bits, int64_t max_bits,
                       gpsb200_nav_word_t *words, int64_t max_words, gpsb200_nav_sync_t *sync);
/* IS-GPS-200 parity of a received word: word and prev are 30-bit words as transmitted (prev supplies D29*, D30*).
 * Returns 1 when the 6 parity bits check, 0 if not; *data (may be NULL) gets the 24 data bits with D30* undone. */
int gpsb200_nav_word_check(uint32_t word, uint32_t prev, uint32_t *data);
/* The 6 parity bits of 24 data bits given D29*, D30* (computeChecksum, gps.c:1008-1072, without the D29/D30 solving). */
uint32_t gpsb200_nav_parity(uint32_t data24, int d29, int d30);

/* ---- broadcast ephemeris, ionosphere and time anchor from decoded words (host; csrc/navdecode.cpp) -------------------
 * Input: the word records of one channel in order, words[i].index == words[0].index + i (what gpsb200_nav_decode
 * returns; a NAV frame slot of the scenario, 60 words with index 0..59, turned into records with
 * gpsb200_nav_word_check, reads the same way). A subframe starts at a word whose index is a multiple of 10; its id is
 * bits 4..2 of the HOW's data. Each term is the IS-GPS-200 integer field (two's complement where signed; M0, e, sqrt A,
 * OMEGA0, i0 and omega split 8 + 24 bits over two words) times its scale, x pi for semicircles (pi = 3.1415926535898,
 * as gps.h:91): the inverse of the reference's eph2sbf (gps.c:662-684, 706-740).
 *   ephemeris  from the LAST subframe 1, 2, 3 sequence (consecutive subframes) whose 30 words all pass parity and where
 *              IODE of subframe 2 == IODE of subframe 3 == IODC & 0xFF; valid = 0 when there is none
 *   iono       the Klobuchar alpha0..3 / beta0..3 of the last subframe 4 page 18 (data id 1, SV id 56) whose 10 words
 *              pass parity; valid = 0 when there is none */
typedef struct gpsb200_ephemeris {
    int32_t valid;         /* 1: decoded from a complete, consistent set; 0: the rest is undefined */
    int32_t week;          /* WN, the transmission week modulo 1024 (10 bits) */
    int32_t iodc, iode;
    int32_t health;        /* 6 bits; 0 = all data OK */
    int32_t ura;           /* 4 bits */
    int32_t reserved[2];
    double toc;            /* s of week (x 16) */
    double af0, af1, af2;  /* s, s/s, s/s^2 (2^-31, 2^-43, 2^-55) */
    double tgd;            /* s (2^-31) */
    double toe;            /* s of week (x 16) */
    double m0, deltan;     /* rad, rad/s */
    double ecc, sqrta;     /* -, m^1/2 */
    double omg0, inc0, aop;/* rad */
    double omgdot, idot;   /* rad/s */
    double cuc, cus;       /* rad */
    double crc, crs;       /* m */
    double cic, cis;       /* rad */
} gpsb200_ephemeris_t;     /* 200 bytes */
typedef struct gpsb200_iono {
    int32_t valid;
    int32_t reserved;
    double alpha[4];       /* s, s/semicircle, s/semicircle^2, s/semicircle^3 (2^-30, 2^-27, 2^-24, 2^-24) */
    double beta[4];        /* s, ... (2^11, 2^14, 2^16, 2^16) */
} gpsb200_iono_t;          /* 72 bytes */
/* iono may be NULL. GPSB200_ERR_ARG on a bad argument (NULL eph, n < 0, words NULL with n > 0). */
int gpsb200_nav_ephemeris(const gpsb200_nav_word_t *words, int64_t n, gpsb200_ephemeris_t *eph, gpsb200_iono_t *iono);
/* The transmit-time anchor of a tracked channel from its first HOW with good parity (words and sync as
 * gpsb200_nav_decode returned them for the channel's epochs): *anchor_epoch = bit_edge + 20 (frame_bit + 30 index), the
 * epoch whose code period starts at the HOW's first bit, and *anchor_ms = ((6 TOW - 6) 1000 + 600) mod 604800000, the
 * transmit time of that code period's start in ms of week. *anchor_epoch = -1 when there is no such HOW. */
int gpsb200_nav_time_anchor(const gpsb200_nav_word_t *words, int64_t n, const gpsb200_nav_sync_t *sync,
                            int32_t *anchor_epoch, int64_t *anchor_ms);

/* ---- position, velocity and time from tracked channels (DESIGN §11; tests/pvt_model.py states it in numpy) -----------
 * Fix instants: samples s = s0 + i step, i < nfix. Per channel c (epochs[c][0 .. nepochs[c]), in time order):
 *   period     the k >= 1 with epochs[k].sample <= s < epochs[k + 1].sample (none: the channel is not used); its code
 *              phase and step are phi_k = epochs[k-1].code_phase, u_k = epochs[k-1].code_step, its carrier step
 *              w_k = epochs[k-1].carr_step
 *   integers   phi = phi_k + (s - epochs[k].sample) u_k (2^-32 chips, uint64); T = (anchor_ms + k - anchor_epoch) mod
 *              604800000 (whole ms of week); transmit time t_sv = T / 1000 + phi / (1023 2^32) / 1000 s of week
 *   used       epochs[k-1].lock and epochs[k].lock, eph.valid, eph.health == 0 and |t_sv - toe| <= 7200 s (week-wrapped)
 * Nominal receive time: the reference channel r is the lowest c with eph.valid and health 0; A = its anchor_ms,
 * s_A = epochs[r][anchor_epoch].sample; t_nom(s) = A + 75 ms + (s - s_A) / 3e6 s. Pseudorange
 * rho = c ((A + 75 + q - T) ms + (m / 3000 - phi / (1023 2^32)) ms) with s - s_A = 3000 q + m (0 <= m < 3000) and the
 * whole-ms difference wrapped into half a week, so FP64 adds nothing above ~1 um. Range rate -lambda_L1 w_k 3e6 / 2^32.
 * Per used channel (FP64, IS-GPS-200 20.3.3.3.3 / 20.3.3.4.3, the constants of gps.h:87-102): t = t_sv - dt, dt the
 * af0..af2 polynomial at t_sv (t - toc week-wrapped); Kepler's equation by Newton from E = M until |dE| <= 1e-14 (at most
 * 10 steps); satellite position and velocity (ECEF, at t); clock dt_sv = af0 + af1 d + af2 d^2 + F e sqrtA sin E - TGD
 * (d = t - toc, F = -4.442807633e-10), clock drift af1 + 2 af2 d. Then Gauss-Newton on (x, y, z, b) from (0, 0, 0, 0),
 * iteration j = 0 .. GPSB200_PVT_MAX_ITER - 1 at the estimate X_j:
 *   flight time tau = |p - x_j| / c, p the satellite position; p rotated about z by -OMEGA_E tau (exact rotation);
 *   model rho = |p_rot - x_j| + b_j - c dt_sv + I, I the Klobuchar delay (the reference's ionosphericDelay, gps.c:1893-1964,
 *   with the config's alpha / beta, at the WGS-84 latitude / longitude of x_j, the azimuth / elevation of p_rot seen from
 *   there, and the receive time t_nom - b_j / c) when cfg.iono and |x_j| >= 6e6 m, else 0;
 *   rows (-(p_rot - x_j) / |p_rot - x_j|, 1); normal equations from the used channels; X_{j+1} = X_j + solve.
 *   Status 2 as soon as |x_{j+1}| > 1e8 m (a diverging estimate: from the Earth's centre, Gauss-Newton on exactly four
 *   satellites of poor geometry can run away) or the normal matrix is not positive definite. Otherwise converged after
 *   the first j with |dx| < 1e-4 m: the fix is X_{j+1}; none after GPSB200_PVT_MAX_ITER: status 2.
 * Velocity and clock drift: least squares with the same rows (at the last X_j) on rate + c drift_sv - e . v_sat, v_sat the
 * satellite velocity rotated like p. Residuals (post-fit, m): rho - model - row . dX of the last iteration. PDOP:
 * sqrt of the trace of the position block of (H^T H)^-1. Fewer than 4 used channels: status 1. */
#define GPSB200_PVT_MAX_ITER 12
enum { GPSB200_FIX_OK = 0, GPSB200_FIX_FEW = 1, GPSB200_FIX_NO_CONVERGENCE = 2 };
typedef struct gpsb200_pvt_chan {
    gpsb200_ephemeris_t eph;
    int32_t prn;           /* for the caller's reference only */
    int32_t anchor_epoch;  /* 0 <= anchor_epoch < nepochs[c] (gpsb200_nav_time_anchor) when eph.valid */
    int64_t anchor_ms;     /* 0 <= anchor_ms < 604800000 when eph.valid */
} gpsb200_pvt_chan_t;      /* 216 bytes */
typedef struct gpsb200_pvt_config {
    int64_t s0;            /* first fix instant (stream sample) */
    int64_t step;          /* samples between fix instants, >= 1 */
    int32_t nfix;          /* >= 1 */
    int32_t iono;          /* 1: apply the Klobuchar delay with alpha / beta; 0: none */
    double alpha[4], beta[4];
} gpsb200_pvt_config_t;    /* 88 bytes */
typedef struct gpsb200_fix {
    int64_t sample;        /* the fix instant */
    int32_t status;        /* GPSB200_FIX_*; the doubles below are NaN unless GPSB200_FIX_OK */
    int32_t nused;         /* channels used */
    uint32_t mask;         /* bit c: channel c used */
    int32_t iterations;    /* Gauss-Newton iterations run */
    double x, y, z;        /* ECEF, m */
    double clock_m;        /* receiver clock bias b, m */
    double t_rx;           /* receive time t_nom - b / c, s of week */
    double vx, vy, vz;     /* ECEF, m/s */
    double drift;          /* receiver clock drift, m/s */
    double lat_deg, lon_deg, height;   /* WGS-84 */
    double pdop;
    double rms;            /* post-fit residual RMS over the used channels, m */
} gpsb200_fix_t;           /* 136 bytes */
/* Fixes at cfg->nfix instants from nchan (1..GPSB200_TRK_MAX_CHAN) channels: chans [nchan], epochs [nchan][max_epochs]
 * host memory (row c holds nepochs[c] <= max_epochs records), fixes [nfix] out, residuals (NULL: not wanted)
 * [nfix][nchan] out (NaN for channels not used). One ephemeris per channel per call. A channel with eph.valid == 0 is
 * never used and its anchor is not checked, so a channel that has no ephemeris or no anchor yet (anchor_epoch -1) can
 * keep its slot: bit c of every mask then stays channel c. Every argument is checked before
 * anything is enqueued (GPSB200_ERR_ARG). Blocking: the epochs and channels go up once, the fixes come back in one
 * download. */
int gpsb200_pvt(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg, gpsb200_fix_t *fixes,
                double *residuals);
/* Re-run the fix kernel of the previous gpsb200_pvt or gpsb200_pvt_raim call (whichever ran last) on its device-resident
 * inputs, enqueued on `stream` (0 = the context's own stream), without transfers: for timing the kernel alone.
 * GPSB200_ERR_ARG when there was no such call. */
int gpsb200_pvt_replay(gpsb200_ctx_t *ctx, void *stream);

/* ---- integrity of the fixes: RAIM fault detection, exclusion and protection levels (DESIGN §11.1; tests/raim_model.py)
 * Per fix instant, with sigma, T_d and lambda_d below (d = degrees of freedom):
 *   1. Solve exactly as gpsb200_pvt does (the set S = the channels it uses).
 *   2. If the fix is OK and n = |S| >= 5: stat = sum over S of e_j^2 / sigma^2, e_j the post-fit residual of
 *      gpsb200_pvt; dof = n - 4. A fault is detected when stat > T_dof.
 *   3. If detected, n >= 6 and fewer than max_exclude channels have been excluded: exclude the channel j of S with the
 *      largest e_j^2 / (1 - h_jj), the lowest channel on ties; h_jj = g_j . N^-1 g_j, g_j = (row of j, 1), N the normal
 *      matrix of the last Gauss-Newton iteration. Channels with 1 - h_jj <= 1e-9 are never candidates.
 *   4. Gauss-Newton again on S without j, from the fix of step 1 (or of the previous step 4), with the same rules.
 *   5. Back to step 2's test on the new set.
 * Verdicts: PASS the test passed and nothing was excluded; EXCLUDED the final set passes after exclusions; ALERT a fault
 * is detected and not removed (dof 1, where every normalized residual is equal; max_exclude reached; no candidate; or a
 * re-solve that did not converge); UNAVAILABLE fewer than 5 used channels or the first solve not OK.
 * The fix record describes the final set (mask, nused, status, position, velocity, rms); iterations counts every pass.
 * stat, dof and threshold are those of the last test run (NaN, 0, NaN when none ran). Protection levels (Brown's slope
 * method) over the final set when its fix is OK and the verdict is not UNAVAILABLE, NaN otherwise:
 *   x_j = N^-1 g_j rotated to east / north / up at the final fix's WGS-84 latitude and longitude,
 *   Hslope_j = sqrt(x_jE^2 + x_jN^2) / sqrt(1 - h_jj), Vslope_j = |x_jU| / sqrt(1 - h_jj),
 *   HPL = max_j Hslope_j sigma sqrt(lambda_dof), VPL = max_j Vslope_j sigma sqrt(lambda_dof); +inf when some channel of
 *   the set has 1 - h_jj <= 1e-9.
 * residuals (NULL: not wanted) [nfix][nchan]: the set's channels as gpsb200_pvt reports them; excluded channels their
 * residual against the final fix (rho - model - row . dX of the final set's last iteration: the fault's size); every
 * other channel NaN (all NaN when the final fix is not OK). */
enum { GPSB200_RAIM_PASS = 0, GPSB200_RAIM_EXCLUDED = 1, GPSB200_RAIM_ALERT = 2, GPSB200_RAIM_UNAVAILABLE = 3 };
#define GPSB200_RAIM_MAX_DOF 28          /* dof 1..28: 5..32 channels */
#define GPSB200_RAIM_MAX_EXCLUDE 4
typedef struct gpsb200_raim_config {
    double sigma;          /* pseudorange sigma, m: finite, > 0 */
    double p_fa;           /* false-alarm probability of the test, 1e-12..0.5 */
    double p_md;           /* missed-detection probability of the protection levels, 1e-12..0.5 */
    int32_t max_exclude;   /* 0..GPSB200_RAIM_MAX_EXCLUDE; 0 = detection only */
    int32_t reserved;      /* 0 */
} gpsb200_raim_config_t;   /* 32 bytes */
typedef struct gpsb200_raim {
    int32_t verdict;       /* GPSB200_RAIM_* */
    uint32_t excluded;     /* bit c: channel c excluded */
    int32_t dof;           /* of the last test; 0 when none ran */
    int32_t reserved;
    double stat;           /* sum e^2 / sigma^2 of the last test */
    double threshold;      /* T_dof of the last test */
    double hpl, vpl;       /* m */
} gpsb200_raim_t;          /* 48 bytes */
/* Host: for d = 1..28, T[d-1] = the chi^2(d) value whose upper tail is p_fa, lambda[d-1] = the noncentrality at which
 * the noncentral chi^2(d, lambda) has P(<= T_d) = p_md (regularized incomplete gamma, a Poisson mixture for the
 * noncentral CDF, bisection; 1e-10 relative or better). GPSB200_ERR_ARG when p_fa or p_md is outside 1e-12..0.5 or an
 * array is NULL. */
int gpsb200_raim_thresholds(double p_fa, double p_md, double T[GPSB200_RAIM_MAX_DOF], double lambda[GPSB200_RAIM_MAX_DOF]);
/* gpsb200_pvt with the RAIM stage above: the same arguments and checks, plus the RAIM config (GPSB200_ERR_ARG outside its
 * ranges) and out [nfix], one record per fix. The tables of gpsb200_raim_thresholds go up with the kernel's arguments. */
int gpsb200_pvt_raim(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                     const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
                     const gpsb200_raim_config_t *raim, gpsb200_fix_t *fixes, double *residuals, gpsb200_raim_t *out);

/* ---- advanced RAIM: weighted fix, elevation mask, solution separation and ARAIM protection levels (DESIGN §11.2;
 * tests/araim_model.py states it in numpy). GPS L1 C/A only, single-satellite faults, at most one exclusion, no
 * constellation faults and no wrong-exclusion term (where this differs from the EU-US ARAIM Airborne Algorithm
 * Description: DESIGN §11.2). Per fix instant:
 *   1. Channel set. Channel i can enter the set S when gpsb200_pvt would use it and its broadcast eph.ura < 15.
 *      sigma_URA,i = max(cfg.sigma_ura, URA_nom(eph.ura)), URA_nom = 2.0, 2.8, 4, 5.7, 8, 11.3, 16, 32, 64, 128, 256, 512,
 *      1024, 2048, 4096 m (IS-GPS-200 20.3.3.3.1.3); sigma_URE,i = sigma_URA,i sigma_ure / sigma_ura.
 *   2. Weights, at the elevation el of the channel's line of sight (the rotated satellite position, as in gpsb200_pvt)
 *      from the current estimate X_j, in every Gauss-Newton iteration; el = 90 deg while |x_j| < 6e6 m:
 *        sigma_int,i^2 = sigma_URA,i^2 + sigma_tropo^2 + sigma_air^2 + sigma_iono^2, sigma_acc,i^2 the same with
 *        sigma_URE,i; sigma_tropo = 0.12 1.001 / sqrt(0.002001 + sin^2 el); sigma_air^2 = sigma_noise^2 +
 *        (0.13 + 0.53 exp(-el / 10 deg))^2; sigma_iono = max(I / 5, F tau(|phi_m|)) when cfg.iono and |x_j| >= 6e6 m,
 *        else 0, with I, F and phi_m the Klobuchar delay, obliquity factor and geomagnetic latitude of gpsb200_pvt's
 *        Klobuchar term and tau = 9 m for |phi_m| <= 20 deg, 4.5 m for <= 55 deg, 6 m above (DO-229 J.2.3).
 *   3. Weighted Gauss-Newton: gpsb200_pvt's solve (from the Earth's centre, the same convergence, runaway and
 *      positive-definiteness rules) with each row and residual scaled by 1 / sigma_int,i.
 *   4. Elevation mask: after the first converged solve, the channels with el (of the last iteration) < mask_deg leave
 *      S (bit c of `masked`). If any left, Gauss-Newton again from that fix (status 1 when fewer than 4 remain).
 *   5. Solution separation at the final fix, n = |S| >= 5 (else UNAVAILABLE). G = the last iteration's rows (g_i, 1),
 *      W = diag(1 / sigma_int,i^2), y = its prefit residuals, positions in east / north / up at the fix's WGS-84
 *      latitude and longitude. S0 = (G^T W G)^-1 G^T W; S(k) the same without row k (column k zero), for each k in S.
 *      dx(k) = (S(k) - S0) y; sigma_q(k)^2 = (S(k) C_int S(k)^T)_qq; sigma_ss,q(k)^2 = ((S(k) - S0) C_acc
 *      (S(k) - S0)^T)_qq; b_q(k) = sum_i |S(k)_qi| b_nom, and b_q0, sigma_q0 the same for S0; C = diag(sigma^2).
 *      UNAVAILABLE when some G^T W(k) G is not positive definite.
 *   6. Test: T_k,q = K_fa,q sigma_ss,q(k), K_fa,H = Q^-1(p_fa_horz / (4 n)) for east and north, K_fa,V =
 *      Q^-1(p_fa_vert / (2 n)) for up (Q the standard normal upper tail; gpsb200_araim_kfa). Passes when
 *      |dx_q(k)| <= T_k,q for every k and q; test_ratio = max |dx_q(k)| / T_k,q.
 *   7. Exclusion, when the test fails, max_exclude is 1 and n >= 6: the k with the largest max_q |dx_q(k)| / T_k,q
 *      (the lowest channel on ties) leaves S; Gauss-Newton again from the current fix, then 5-6 on the new set:
 *      EXCLUDED when it passes, else ALERT (also when that solve fails). Otherwise a failed test is ALERT.
 *   8. Protection levels over the final set: P_NM = 1 - (1 - p_sat)^n - n p_sat (1 - p_sat)^(n-1) (UNAVAILABLE when
 *      P_NM >= p_hmi_vert + p_hmi_horz); VPL the smallest L with
 *        2 Q((L - b_U0) / sigma_U0) + sum_k p_sat Q((L - T_k,U - b_U(k)) / sigma_U(k)) <= p_hmi_vert (1 - P_NM /
 *        (p_hmi_vert + p_hmi_horz)),
 *      HPL_E and HPL_N the same in east and north with p_hmi_horz / 2 in place of p_hmi_vert, HPL = sqrt(HPL_E^2 +
 *      HPL_N^2). Each by bisection (Q^-1(p) = sqrt(2) erfcinv(2 p) on the device): lo = the largest single-term
 *      solution (b0 + sigma0 Q^-1(rhs / 2); for each k, when rhs < p_sat, T + b + sigma Q^-1(rhs / p_sat)), hi = the
 *      same with rhs / (n + 1); halve until hi - lo <= 1e-3 m; the level is hi. EMT = max_k T_k,U, sigma_acc_v =
 *      sqrt((S0 C_acc S0^T)_UU).
 * The fix record describes the final set: mask, nused, status, position and clock; iterations counts every pass;
 * velocity and drift come from the weighted rows, and pdop = sqrt of the trace of the position block of
 * (G^T W G)^-1, in metres (the weighted solution's position sigma). residuals: every measured channel's post-fit
 * residual against the final fix (masked and excluded channels included), NaN for the others. Record fields that
 * no step computed are NaN (n, excluded, masked 0). */
typedef struct gpsb200_araim_config {
    double mask_deg;       /* elevation mask, deg: 0..90 */
    double sigma_ura;      /* floor of the integrity sigma, m: 0 < sigma_ura <= 100 */
    double sigma_ure;      /* accuracy sigma at sigma_ura, m: 0 < sigma_ure <= sigma_ura */
    double sigma_noise;    /* receiver noise sigma, m: 0..100 */
    double b_nom;          /* nominal bias, m: 0..100 */
    double p_sat;          /* prior probability of a satellite fault: 1e-12..1e-2 */
    double p_hmi_vert, p_hmi_horz;   /* integrity budgets: 1e-12..0.5 each */
    double p_fa_vert, p_fa_horz;     /* false-alarm budgets: 1e-12..0.5 each */
    int32_t max_exclude;   /* 0 or 1 */
    int32_t reserved[3];   /* 0 */
} gpsb200_araim_config_t;  /* 96 bytes */
/* Documented defaults (LPV-200 allocations; araim_config() in Python): */
#define GPSB200_ARAIM_MASK_DEG 5.0
#define GPSB200_ARAIM_SIGMA_URA 1.0
#define GPSB200_ARAIM_SIGMA_URE (2.0 / 3.0)
#define GPSB200_ARAIM_SIGMA_NOISE 0.36
#define GPSB200_ARAIM_B_NOM 0.75
#define GPSB200_ARAIM_P_SAT 1e-5
#define GPSB200_ARAIM_P_HMI_VERT 9.8e-8
#define GPSB200_ARAIM_P_HMI_HORZ 2e-9
#define GPSB200_ARAIM_P_FA_VERT 3.9e-6
#define GPSB200_ARAIM_P_FA_HORZ 9e-8
typedef struct gpsb200_araim {
    int32_t verdict;       /* GPSB200_RAIM_* */
    uint32_t excluded;     /* bit c: channel c excluded (at most one) */
    uint32_t masked;       /* bit c: channel c below the elevation mask */
    int32_t n;             /* channels in the final set */
    double test_ratio;     /* max |dx| / T of the last test */
    double hpl, vpl;       /* m */
    double emt;            /* max_k T_k,U of the last test, m */
    double sigma_acc_v;    /* m */
    double p_nm;           /* the unmonitored fault probability of the final set */
} gpsb200_araim_t;         /* 64 bytes */
/* Host: K_fa,H[n - 5] and K_fa,V[n - 5] of step 6 for n = 5..32 (1e-13 relative or better). GPSB200_ERR_ARG when a
 * probability is outside 1e-12..0.5 or an array is NULL. */
int gpsb200_araim_kfa(double p_fa_vert, double p_fa_horz, double kfa_h[GPSB200_RAIM_MAX_DOF],
                      double kfa_v[GPSB200_RAIM_MAX_DOF]);
/* gpsb200_pvt with the ARAIM stage above: the same arguments and checks, plus the ARAIM config (GPSB200_ERR_ARG outside
 * its ranges) and out [nfix]. gpsb200_pvt_replay re-runs it when it ran last. */
int gpsb200_pvt_araim(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                      const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
                      const gpsb200_araim_config_t *araim, gpsb200_fix_t *fixes, double *residuals,
                      gpsb200_araim_t *out);

/* ---- coarse-time fixes: position without the time anchor (DESIGN §11.3; tests/coarse_model.py states it in numpy) --
 * Assistance: the ephemeris (as for gpsb200_pvt), an a-priori position x_a and an a-priori GPS time t_a (s of week,
 * week `week`) at stream sample s_a. The tracked code phase gives each channel's transmit time modulo 1 ms; the whole
 * ms come from a prediction at x_a, and the a-priori time error delta becomes a fifth unknown. Per fix instant s
 * (s0 + i step, as gpsb200_pvt):
 *   1. A-priori time. ds = s - s_a = 3000 q + m (0 <= m < 3000); u = t_a + ds / 3e6 (float64), kw = floor(u / 604800),
 *      t_a(s) = u - 604800 kw. W = floor(t_a), F = t_a - W (exact).
 *   2. Measurement: gpsb200_pvt's period k, phi and carrier step; frac = phi / (1023 2^32) ms. anchor_epoch / anchor_ms
 *      are neither read nor checked. Used: epochs[k-1].lock and epochs[k].lock, eph.valid, eph.health == 0 and
 *      |t_a(s) - toe| <= 7200 s (week-wrapped, as gpsb200_pvt wraps t_sv - toe).
 *   3. Prediction of a used channel's transmit time at a position x and receive time t (here x_a and t_a(s)): tau_0 =
 *      0.075 s; three fixed-point steps i = 0, 1, 2: p, dt_sv = gpsb200_pvt's satellite position and clock at GPS time
 *      t - tau_i, p rotated about z by -OMEGA_E tau_i, tau_{i+1} = |p_rot - x| / c. pred = 1000 (t - tau_3 + dt_sv) ms,
 *      dt_sv that of step i = 2 (satellite time; TGD and the relativistic term included, no ionosphere).
 *   4. Reference channel r: the used channel with the largest sin(elevation) of p_rot (step i = 2) seen from x_a
 *      (up vector at x_a's WGS-84 latitude / longitude, gpsb200_pvt's six-step conversion); the lowest channel on ties.
 *   5. Whole ms, with round(v) = floor(v + 0.5) (exact halves go up): N_r = round(pred_r - frac_r),
 *      N_c = N_r + round((pred_c - pred_r) - (frac_c - frac_r)). The resolved ms of week is N_c mod 604800000 and the
 *      transmit time t_sv,c = (N_c mod 604800000) / 1000 + frac_c / 1000 s.
 *   6. Pseudorange rho_c = c ((1000 W + q - N_c) ms + (1000 F + m / 3000 - frac_c) ms), the whole-ms difference taken mod
 *      604800000 and wrapped into half a week (as gpsb200_pvt). It equals c (t_a(s) - t_sv,c).
 *   7. Gauss-Newton on X = (x, y, z, b, delta) from (x_a, 0, 0), iteration j = 0 .. GPSB200_PVT_MAX_ITER - 1: each used
 *      channel's satellite at satellite time t_sv,c + delta_j (GPS time by gpsb200_pvt's af0..af2 correction), then
 *      gpsb200_pvt's flight time, rotation, Klobuchar term (receive time t_a(s) + delta_j - b_j / c) and model
 *      rho = |p_rot - x_j| + b_j - c dt_sv + I; rows (-(p_rot - x_j) / R, 1, e . v_rot - c drift_sv), e = (p_rot - x_j) / R
 *      and v_rot the rotated satellite velocity; 5 x 5 normal equations; the convergence (|dx| < 1e-4 m), runaway
 *      (|x| > 1e8 m) and positive-definiteness rules of gpsb200_pvt. Fewer than 5 used channels: status 1.
 *   8. Ambiguity check after convergence: steps 3 and 5 again at the fix (x_{j+1}, t_a(s) + delta - b / c) with the
 *      same reference channel. The status is GPSB200_FIX_AMBIGUOUS (only this call returns it) if any N'_c - N'_r
 *      differs from N_c - N_r (bit c of `changed`; N_r itself moves with delta by design), or if some used channel's
 *      post-fit residual (step 9) exceeds GPSB200_COARSE_MAX_RESIDUAL in magnitude. Wrong integers usually fit a wrong
 *      position well enough that re-resolving at it gives them back; they show instead as residuals of kilometres,
 *      where right integers leave centimetres (ideal epochs) to tens of metres (tracked). With exactly 5 channels the
 *      solve fits any integers exactly, so a wrong integer cannot be seen.
 *   9. Post-fit residuals: rho - model - row . dX of the last iteration. Velocity and clock drift: gpsb200_pvt's least
 *      squares on the rows' first four columns (at the last x_j).
 *      t_rx = t_a(s) + delta - b / c, brought into 0..604800 with the week carried into the record's week.
 * The integers are right when, for every used channel, the prediction error of its transmit time differs from the
 * reference channel's by less than 0.5 ms (about 150 km). That holds for any geometry when x_a is within 50 km of the
 * truth and t_a within 10 s: the line-of-sight projections of the position error differ by at most 2 x 50 km, the range
 * rates by at most about 1.9 km/s (x 10 s = 19 km), well below 150 km.
 * The fix record: status, mask, nused, iterations as gpsb200_pvt; position, clock, velocity, drift, t_rx, rms and pdop
 * (the 5-state PDOP: sqrt of the trace of the position block of the 5 x 5 (H^T H)^-1) NaN unless GPSB200_FIX_OK.
 * residuals (NULL: not wanted) [nfix][nchan]: post-fit residuals of the used channels when OK, NaN otherwise.
 * ms (NULL: not wanted) [nfix][nchan]: the resolved ms of week of each used channel, -1 for the others. */
enum { GPSB200_FIX_AMBIGUOUS = 3 };
#define GPSB200_COARSE_MAX_RESIDUAL 1000.0   /* m */
typedef struct gpsb200_coarse_config {
    double x_a[3];         /* a-priori ECEF position, m: finite */
    double t_a;            /* a-priori GPS time at sample s_a, s of week: 0 <= t_a < 604800 */
    int64_t s_a;           /* stream sample of t_a: 0..2^62 */
    int32_t week;          /* GPS week of t_a: >= 0 */
    int32_t reserved;      /* 0 */
} gpsb200_coarse_config_t; /* 48 bytes */
typedef struct gpsb200_coarse {
    double delta;          /* the solved a-priori time error, s; NaN unless GPSB200_FIX_OK */
    double pdop;           /* the 5-state PDOP (as the fix record's); NaN unless GPSB200_FIX_OK */
    int32_t ref;           /* the reference channel r; -1 when no channel is used */
    int32_t week;          /* GPS week of t_rx; -1 unless GPSB200_FIX_OK */
    uint32_t changed;      /* bit c: channel c's integer changed in the ambiguity check */
    int32_t reserved;
} gpsb200_coarse_t;        /* 32 bytes */
/* Coarse-time fixes: gpsb200_pvt's arguments (the same checks, except that anchors are neither read nor checked), the
 * a-priori config (GPSB200_ERR_ARG unless x_a is finite, 0 <= t_a < 604800, 0 <= s_a <= 2^62, week >= 0 and reserved
 * is 0), out [nfix] records, and ms [nfix][nchan] (NULL: not wanted). gpsb200_pvt_replay re-runs it when it ran last. */
int gpsb200_pvt_coarse(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                       const gpsb200_track_epoch_t *epochs, const int32_t *nepochs, int max_epochs,
                       const gpsb200_pvt_config_t *cfg, const gpsb200_coarse_config_t *apriori, gpsb200_fix_t *fixes,
                       double *residuals, gpsb200_coarse_t *out, int64_t *ms);

/* ---- position search: coarse-time fixes with no a-priori position (DESIGN §11.4; tests/search_model.py states it in
 * numpy). gpsb200_pvt_coarse's assistance without x_a: the ephemeris, an a-priori GPS time t_a (s of week, week `week`)
 * at stream sample s_a, and a grid of `nodes` = N candidate positions over the whole Earth. Per fix instant s:
 *   1. Grid. Node i (0 <= i < N) is the Fibonacci lattice point z_i = 1 - (2 i + 1) / N, geodetic latitude asin(z_i),
 *      longitude 2 pi frac(i g) (g the double nearest (3 - sqrt(5)) / 2 = 0x1.8722191a02d61p-2), height 0 on WGS-84:
 *      x = (N_e cos lat cos lon, N_e cos lat sin lon, N_e (1 - e^2) sin lat), N_e = a / sqrt(1 - e^2 sin^2 lat).
 *      gpsb200_search_nodes returns them.
 *   2. Used channels: gpsb200_pvt_coarse step 2 (period, locks, eph.valid, health, |t_a(s) - toe| <= 7200 s); they do not
 *      depend on the node. Fewer than GPSB200_SEARCH_MIN_CHANNELS: status GPSB200_FIX_FEW and nothing is searched (with 5
 *      channels the coarse solve fits any integers exactly, so every node would return its own OK fix).
 *   3. Visibility prune: each used channel's satellite position p at GPS time t_a(s) - 0.075 s (gpsb200_pvt's satellite,
 *      unrotated). Node i is searched only if every used channel has (up_i . (p - x_i)) / |p - x_i| >=
 *      sin(GPSB200_SEARCH_MIN_ELEV_DEG), up_i the unit vector at the node's latitude / longitude. A channel is tracked
 *      only while its satellite is above the receiver's horizon (re-checked every 30 s), and a node within 50 km of the
 *      receiver sees it at most about half a degree lower.
 *   4. Per searched node: gpsb200_pvt_coarse steps 1 and 3-9 with x_a = the node and the same t_a, s_a and week. The
 *      node is OK when that returns GPSB200_FIX_OK.
 *   5. Winner: the OK node with the smallest floor(1000 rms) (post-fit rms in whole mm), the lowest node on ties. Nodes
 *      that converge to one solution leave rms values that differ by rounding only (below 1 nm), so an exact comparison
 *      would choose among them by rounding noise. The fix record, residuals, ms, delta, pdop, ref, week and changed are
 *      the winner's coarse solve (its status replaced as below).
 *   6. Uniqueness: support = the OK nodes whose fix lies within GPSB200_SEARCH_DISTINCT of the winner's (the winner
 *      included). An OK node whose fix lies farther is a distinct solution; alt_rms / alt_dist are the rms and distance
 *      from the winner of the distinct solution that step 5's ordering puts first. Any distinct solution: status
 *      GPSB200_FIX_AMBIGUOUS, the records still the winner's. No OK node: GPSB200_FIX_NO_CONVERGENCE. More than
 *      GPSB200_SEARCH_MAX_OK(N) OK nodes (the device keeps a list of that many per instant): GPSB200_FIX_AMBIGUOUS with
 *      no winner, `ok` still the exact count. The nodes that converge to one fix cover a region of fixed area, so their
 *      number grows in proportion to N: on the model a unique fix had at most 147 of 262 144 (1 in 1 783, 7 channels),
 *      and the list holds 1 in 256 (at least 64), seven times that. So this outcome means many OK nodes that cannot be
 *      one fix's, as at 6 channels (about 1 200 on the default grid).
 *      Strict on purpose. On the model, 7 or more channels gave no distinct solution over the default grid, while 6
 *      channels gave about a thousand wrong-integer fixes with rms of metres: a 6-channel search is AMBIGUOUS.
 * Guarantee: the default grid's covering radius is 33.99 km on a sphere of the WGS-84 equatorial radius (the largest
 * circumradius of its convex hull's facets). For a receiver at a height of 0-50 km some node lies within
 * gpsb200_pvt_coarse's 50 km, and with t_a within 10 s that node's integers are right (2 x 34 km + 19 km is far below
 * the 150 km limit). The winner is a different node only if that node also finds an OK fix. N = 131072 gives 48.06 km,
 * too close to 50 km.
 * Records without a winner: fix status, sample, nused and mask set, iterations 0, every double NaN; residuals NaN, ms
 * -1, delta / pdop NaN, ref -1, week -1, changed 0. */
#define GPSB200_SEARCH_NODES 262144          /* the default grid */
#define GPSB200_SEARCH_MIN_NODES 64
#define GPSB200_SEARCH_MAX_NODES 4194304     /* 2^22 */
#define GPSB200_SEARCH_MIN_ELEV_DEG (-5.0)
#define GPSB200_SEARCH_MIN_CHANNELS 6
#define GPSB200_SEARCH_DISTINCT 1000.0       /* m */
#define GPSB200_SEARCH_MAX_OK(n) ((n) / 256 > 64 ? (n) / 256 : 64)   /* OK-list length per instant, N nodes */
#define GPSB200_SEARCH_HIT_BYTES_PER_OK 40
#define GPSB200_SEARCH_HIT_BYTES (256ll << 20)   /* the device's OK lists of one pass over the instants */
typedef struct gpsb200_search_config {
    double t_a;            /* a-priori GPS time at sample s_a, s of week: 0 <= t_a < 604800 */
    int64_t s_a;           /* stream sample of t_a: 0..2^62 */
    int32_t week;          /* GPS week of t_a: >= 0 */
    int32_t nodes;         /* grid nodes N: GPSB200_SEARCH_MIN_NODES..GPSB200_SEARCH_MAX_NODES */
    int64_t reserved;      /* 0 */
} gpsb200_search_config_t; /* 32 bytes */
typedef struct gpsb200_search {
    int32_t winner;        /* the winning node; -1 when there is none */
    int32_t searched;      /* nodes that passed the visibility prune */
    int32_t ok;            /* of those, nodes whose coarse solve was OK */
    int32_t support;       /* OK nodes within GPSB200_SEARCH_DISTINCT of the winner's fix */
    double alt_rms;        /* the first distinct solution's rms (step 6), m; NaN when there is none */
    double alt_dist;       /* its distance from the winner's fix, m; NaN when there is none */
    double delta, pdop;    /* the winner's (gpsb200_coarse_t) */
    int32_t ref, week;     /* the winner's (gpsb200_coarse_t) */
    uint32_t changed;      /* the winner's (gpsb200_coarse_t) */
    int32_t reserved;
} gpsb200_search_t;        /* 64 bytes */
/* Host: xyz [n][3], the ECEF positions (m) of the n-node grid of step 1. GPSB200_ERR_ARG unless
 * GPSB200_SEARCH_MIN_NODES <= n <= GPSB200_SEARCH_MAX_NODES and xyz is not NULL. */
int gpsb200_search_nodes(int n, double *xyz);
/* Searches: gpsb200_pvt_coarse's arguments with the search config in place of the a-priori one (GPSB200_ERR_ARG unless
 * 0 <= t_a < 604800, 0 <= s_a <= 2^62, week >= 0, nodes in range and reserved 0; anchors are neither read nor checked),
 * out [nfix] records, ms [nfix][nchan] and node_rms [nfix][nodes] (NULL: not wanted): the rms of each OK node, NaN where
 * a node was pruned or not OK. Device scratch: 780 bytes per instant, plus one pass's OK lists, at most
 * GPSB200_SEARCH_HIT_BYTES (the instants run in passes of as many as that holds, 40 bytes per list entry: 6 553 on
 * the default grid, 409 at 2^22 nodes), never nfix x nodes; node_rms, when wanted, takes nfix x nodes doubles. Results do not depend on the order the device runs in. gpsb200_pvt_replay
 * re-runs it when it ran last. */
int gpsb200_pvt_search(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                       const gpsb200_track_epoch_t *epochs, const int32_t *nepochs, int max_epochs,
                       const gpsb200_pvt_config_t *cfg, const gpsb200_search_config_t *search, gpsb200_fix_t *fixes,
                       double *residuals, gpsb200_search_t *out, int64_t *ms, double *node_rms);

/* ---- snapshot measurement: a fine code phase and carrier step from an acquisition, without tracking (DESIGN §11.5;
 * tests/snapshot_model.py states it in numpy). An acquisition peak is quantised to one sample (99.9 m of range) and one
 * Doppler bin; this refines each acquired PRN, over the window the search ran on, to a measurement the coarse-time fix
 * can use. Exact integer arithmetic, with the tracker's pieces (samples, tables, wipe-off, replica c(x) = 2 ca[x >> 32]
 * - 1, M = 1023 * 2^32, H = 2^31, angle(), "/" truncating, ">>" floor; the gpsb200_track header). For each PRN p of the
 * search (res[p], K = acq->ms, window samples m = 0 .. 3000 K - 1 after s0, chunk k = samples 3000 k .. 3000 k + 2999):
 *   0. Weak: unless res[p].ratio >= cfg->min_ratio the record is the seed of step 1 with status GPSB200_SNAP_WEAK,
 *      iterations 0, last_step 0 and power 0: it is never refined.
 *   1. Seed (as gpsb200_track_start): w = (int32) llround(doppler_hz * 2^32 / 3e6), u = clamp(NOM + w / 1540, MIN, MAX),
 *      phi = (M - (delay * u) mod M) mod M: the prompt phase at s0 that wraps at s0 + delay.
 *   2. Frequency pass at (phi, u, w): prompt sums P_I,k, P_Q,k (int32) with the replica at (phi + m u) mod M and the
 *      carrier index ((uint32) (m w)) >> 23, continuous over the window. power = sum_k P_I,k^2 + P_Q,k^2. With K >= 2:
 *      per pair (k, k + 1) cross = P_I,k P_Q,k+1 - P_Q,k P_I,k+1, dot = P_I,k P_I,k+1 + P_Q,k P_Q,k+1, both negated
 *      when dot < 0 (data bits drop out, as in the FLL); d = angle(sum dot, sum cross) in 2^-32 turns per 3000 samples;
 *      w += d / 3000, u = clamp(NOM + w / 1540). K = 1 leaves w and u.
 *   3. Code: `iterations` passes at the current phi and the fixed u, w, each with the early ((p + H) mod M), late
 *      ((p - H) mod M) and prompt replicas: E = sum_k E_I,k^2 + E_Q,k^2, L and power likewise (int64); E and L shifted
 *      right by max(0, bitlen(E + L) - 40); D = ((E - L) * 2^14) / (E + L) (0 when E + L = 0); phi = (phi + D *
 *      GPSB200_SNAP_GAIN) mod M. On the ideal triangle D ~ -4 delta 2^14 for a replica delta chips ahead, so the step
 *      is half a Newton step: the full step limit-cycles on the sampled correlation. last_step = the last D.
 *   4. Status GPSB200_SNAP_NO_CONVERGENCE when iterations >= 1 and |last_step| > GPSB200_SNAP_MAX_LAST_D (a step above a
 *      thousandth of a chip), else GPSB200_SNAP_OK.
 * Bounds: |I_d|, |Q_d| <= 2 * 128 * 250, so a chunk sum is at most 3000 * 64000 = 1.92e8 < 2^31 in magnitude; |(I_d,
 * Q_d)| <= 181.02 * 250.46 (the tables' largest modulus), so a chunk's squared magnitude is at most 1.85e16 and E, L,
 * power <= K * 1.85e16, E + L <= 3.7e18 < 2^63 for K <= 100; |cross|, dot <= 1.85e16 per pair, sums <= 99 * 1.85e16. */
#define GPSB200_SNAP_MAX_ITER   16
#define GPSB200_SNAP_ITERATIONS 12            /* the default */
#define GPSB200_SNAP_GAIN       32768         /* 2^15: the step in 2^-32 chips per unit of D */
#define GPSB200_SNAP_MAX_LAST_D 131           /* 131 * 2^15 < 2^32 / 1000 */
enum { GPSB200_SNAP_OK = 0, GPSB200_SNAP_WEAK = 1, GPSB200_SNAP_NO_CONVERGENCE = 2 };
typedef struct gpsb200_snapshot_config {
    double min_ratio;      /* refined when res.ratio >= min_ratio (gpsb200-acq's threshold: 2.5); finite, >= 0 */
    int32_t iterations;    /* code passes: 0..GPSB200_SNAP_MAX_ITER */
    int32_t reserved;      /* 0 */
} gpsb200_snapshot_config_t;   /* 16 bytes */
typedef struct gpsb200_snapshot {
    int32_t prn;
    int32_t status;        /* GPSB200_SNAP_* */
    int64_t sample;        /* s0: the instant the measurement holds at */
    uint64_t code_phase;   /* prompt code phase at `sample`, 2^-32 chips, < 1023 * 2^32 */
    uint32_t code_step;    /* u, 2^-32 chips per sample */
    int32_t carr_step;     /* w, 3e6 / 2^32 Hz */
    int32_t iterations;    /* code passes run */
    int32_t last_step;     /* D of the last code pass (0 with none) */
    uint64_t power;        /* prompt power of the last pass */
    double ratio;          /* res.ratio */
} gpsb200_snapshot_t;      /* 56 bytes */
/* Refine the results res [acq->nprn] of a search run with acq on nsamples samples of host memory (the search's
 * arguments: the same window must lie in the buffer) into out [acq->nprn], in the order of acq->prn. acq may be the
 * config of gpsb200_acquire or of gpsb200_acquire_windows: its bins (f_lo_hz, step_hz, nbins) are neither read nor
 * checked. Every argument is checked before anything is enqueued (GPSB200_ERR_ARG: s0, ms, nprn, prn and the window
 * as gpsb200_acquire checks them, res[p].prn == acq->prn[p], delays 0..2999, |doppler_hz| <= 10 kHz -- the seed is
 * gpsb200_track_start's, with its range, which keeps w and the refined w far inside int32 -- the config in
 * range). Blocking. */
int gpsb200_snapshot_measure(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                             const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res,
                             const gpsb200_snapshot_config_t *cfg, gpsb200_snapshot_t *out);
/* Same for a source in device memory (16-byte aligned), measured in place on `stream` (0 = the context's own stream)
 * behind whatever it holds; returns when the records are in host memory. */
int gpsb200_snapshot_measure_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                    const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res,
                                    const gpsb200_snapshot_config_t *cfg, gpsb200_snapshot_t *out, void *stream);
/* ---- snapshot batch: the search and the measurement above over many windows of one source in one call (DESIGN §11.6)
 * Window w (0 <= w < nwin) starts at sample s0[w]; windows may overlap, repeat and come in any order. acq->s0 is not
 * read; K, the PRN list, the bins and cfg are shared by every window. Row w of res [nwin][acq->nprn] and of out
 * [nwin][acq->nprn] is, bit for bit, what these single calls give:
 *   search     gpsb200_acquire with acq->s0 = s0[w] (f_lo NULL: the standard grid from acq->f_lo_hz), or
 *              gpsb200_acquire_windows with acq->s0 = s0[w] and f_lo_prn = f_lo + w * acq->nprn (f_lo [nwin][nprn]);
 *   measure    gpsb200_snapshot_measure with acq->s0 = s0[w] on those results, with cfg.
 * Every argument is checked before anything is enqueued (GPSB200_ERR_ARG): nwin >= 1, s0 and the other pointers not
 * NULL, cfg as gpsb200_snapshot_measure checks it, and every window as its single search checks it (the window inside
 * the buffer, each f_lo row finite with its bins within +-1.5 MHz). The measurement's check of the results (|doppler_hz|
 * <= 10 kHz) can only be made after the search: a window that fails it ends the call with GPSB200_ERR_ARG before its
 * pass is measured. The search grid is not offered. Blocking.
 * Passes: the windows run in consecutive passes of P = max(1, floor(GPSB200_SNAP_BATCH_SCRATCH / B)) windows (the last
 * may hold fewer), B = nprn nbins 24028 + nprn 128 + 8 + (3000 K + 2999) 2 sample_size bytes: the device scratch one window
 * may take (the split search's powers, its rows and phase steps, the per-pair tables, records and the staged window), so
 * a pass of two windows or more stays within the cap, and its (window, PRN) pairs far below the grid's y limit. The
 * search of a pass with fewer (window, PRN, bin) rows than a full wave (3 CTAs on every SM) splits them as one search of
 * that many rows would; a larger pass runs unsplit; gpsb200_debug_acq_split forces a split for batches as for single
 * searches. Neither the passes nor the split change a result. Between the search and the measurement of a pass, the
 * results come down once and the seeded records go up once. Of a host source only the windows go up, packed. */
#define GPSB200_SNAP_BATCH_SCRATCH (256LL << 20)
int gpsb200_snapshot_batch(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                           const gpsb200_acq_config_t *acq, int nwin, const int64_t *s0, const double *f_lo,
                           const gpsb200_snapshot_config_t *cfg, gpsb200_acq_result_t *res, gpsb200_snapshot_t *out);
/* Same for a source in device memory (16-byte aligned), searched and measured in place on `stream` (0 = the context's
 * own stream) behind whatever it holds; returns when the results and records are in host memory. */
int gpsb200_snapshot_batch_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                  const gpsb200_acq_config_t *acq, int nwin, const int64_t *s0, const double *f_lo,
                                  const gpsb200_snapshot_config_t *cfg, gpsb200_acq_result_t *res,
                                  gpsb200_snapshot_t *out, void *stream);
/* ---- fixes from snapshot records (DESIGN §11.5): gpsb200_pvt_coarse and gpsb200_pvt_search with meas [nsnap][nchan]
 * in place of the epochs. Snapshot i's fix instant is its records' common `sample` (all nchan records of a row must hold
 * the same sample, 0..2^62; else GPSB200_ERR_ARG); cfg->nfix is nsnap (>= 1); cfg->iono, alpha and beta apply; cfg->s0
 * and cfg->step are not read. Channel c is used at snapshot i when meas[i][c].status is GPSB200_SNAP_OK, meas[i][c].prn
 * equals chans[c].prn, eph.valid, eph.health == 0 and |t_a(s) - toe| <= 7200 s; its measurement is frac =
 * code_phase / (1023 2^32) ms and rate = -lambda carr_step 3e6 / 2^32. Everything else is gpsb200_pvt_coarse's
 * (gpsb200_pvt_search's) procedure, records and checks, unchanged; anchors are not read. gpsb200_pvt_replay re-runs the
 * call when it ran last. */
int gpsb200_pvt_snapshot(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_snapshot_t *meas,
                         const gpsb200_pvt_config_t *cfg, const gpsb200_coarse_config_t *apriori, gpsb200_fix_t *fixes,
                         double *residuals, gpsb200_coarse_t *out, int64_t *ms);
int gpsb200_pvt_snapshot_search(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                                const gpsb200_snapshot_t *meas, const gpsb200_pvt_config_t *cfg,
                                const gpsb200_search_config_t *search, gpsb200_fix_t *fixes, double *residuals,
                                gpsb200_search_t *out, int64_t *ms, double *node_rms);

/* ---- collective detection: a position from satellites too weak to acquire alone (DESIGN §11.7;
 * tests/collective_model.py states it in numpy). Axelrad et al., "Collective Detection and Direct Positioning Using
 * Multiple GNSS Satellites", NAVIGATION 58(4), 2011. Each PRN's whole power grid P_p(j, tau) of one search is scored
 * against a lattice of candidate receiver positions and time offsets around the a-priori ones: a candidate predicts
 * every satellite's code delay and Doppler bin, and the grids' powers at those cells are added up for every common
 * receiver clock shift. The best candidate seeds the PRNs; gpsb200_snapshot_measure and gpsb200_pvt_snapshot finish.
 * Arguments: the search (acq, f_lo_prn: NULL for gpsb200_acquire's standard grid, else gpsb200_acquire_windows'
 * per-PRN first bins), eph[32] indexed by PRN - 1 (as gpsb200_rinex_ephemeris returns it), the a-priori config ap
 * (gpsb200_pvt_coarse's) and the lattice config cfg. s0 = acq->s0; "/" on integers floors.
 *   1. Search: gpsb200_acquire (gpsb200_acquire_windows) on the window, unchanged; res [nprn] is its results, bit for bit.
 *   2. Used: searched PRN p (acq->prn[p]) is used when eph[prn - 1] is valid with health 0, |t0 - toe| <= 7200 s
 *      (week-wrapped) for t0 = ap->t_a + (s0 - ap->s_a) / 3e6, its sin(elevation) from gpsb200_pvt_coarse's step 3
 *      prediction at ap->x_a, t0 (up vector at x_a) is >= sin(cfg->mask_deg pi / 180), and mu_p > 0 (step 3). Fewer than
 *      GPSB200_CD_MIN_USED used PRNs: status GPSB200_CD_FEW and nothing is scored.
 *   3. Normalise: mu_p = floor(sum_{j,tau} P_p(j, tau) / (nbins 3000)), the sum exact (128 bits: it reaches 2.3e25);
 *      q_p(j, tau) = min(floor(2^GPSB200_CD_Q_SHIFT P_p(j, tau) / mu_p), GPSB200_CD_Q_CAP) (uint16). The cap keeps one
 *      strong satellite from outvoting the others.
 *   4. Lattice: hypothesis h = ((i_t n_u + i_u) n_n + i_n) n_e + i_e, i_a < n_a; offset o_a = (i_a - (n_a - 1) / 2)
 *      step_a (real halves; 0 when n_a = 1) along east, north, up (m) and time (s); position x_h = x_a + o_e E + o_n N +
 *      o_u U (E, N, U: the unit vectors at x_a's WGS-84 latitude / longitude, gpsb200_pvt's conversion), time t_h =
 *      t0 + o_t.
 *   5. Predict, per (h, used p): pred = step 3 of gpsb200_pvt_coarse at x_h, t_h (ms, satellite time); delay d =
 *      round(3000 (1 - frac(pred))) mod 3000 (round(v) = floor(v + 0.5)), the sample after s0 where chip 0 starts;
 *      Doppler f = -(e . v_rot - c drift) / lambda_L1 with e, v_rot and drift of the prediction's last step and a static
 *      receiver (the sign of a channel's f_carr, where the acquisition peaks); bin j = round((f - f_lo_p) / step_hz),
 *      j = 0 when nbins = 1. A PRN whose j lies outside 0..nbins-1 adds nothing at h.
 *   6. Score: S(h, b) = sum_p q_p(j_p(h), (d_p(h) + b) mod 3000) for every clock shift b < 3000 (uint32: at most
 *      32 GPSB200_CD_Q_CAP = 2^18); S_h = max_b S(h, b) and b_h its lowest b.
 *   7. Pick: the winner h* has the largest S_h, the lowest h on ties. The runner-up has the largest S_h among the h
 *      whose lattice distance sqrt((o_e - o_e*)^2 + (o_n - o_n*)^2 + (o_u - o_u*)^2) exceeds cfg->distinct_m, the lowest
 *      h on ties. Status GPSB200_CD_AMBIGUOUS when 100 S_runner >= GPSB200_CD_AMBIGUOUS_PCT S_h*, else GPSB200_CD_OK.
 *   8. Seeds [nprn]: for a PRN with a cell at h* (used, j in range), res[p] as if its argmax had been forced there: bin
 *      j_p(h*), delay (d_p(h*) + b*) mod 3000, doppler_hz = f_lo_p + j step_hz, delay_chips = delay 1023 / 3000,
 *      p1 = P_p(j, delay), p2 = the largest P_p(j, tau) more than 3 samples (circular) from delay, ratio = p1 / p2
 *      (infinity when p2 is 0). Every other PRN (and every PRN when FEW): res[p] with ratio -1. So the seeds go
 *      straight into gpsb200_snapshot_measure with min_ratio 0, which refines the PRNs with a cell and leaves the others
 *      WEAK; (x*, ap->t_a + o_t*) at ap->s_a is the a-priori config of gpsb200_pvt_snapshot.
 * out: the record below; records without a winner (FEW) have winner, runner and shift -1, scores 0 and NaN doubles, a
 * winner without a runner-up has runner -1, runner_score 0 and runner_dist NaN. scores (NULL: not wanted) [nhyp]: S_h,
 * b_h (every 0 when FEW). table (NULL: not wanted) [nhyp][nprn]: (j, d) of step 5, bin -1 where j lies outside the grid,
 * both -1 for unused PRNs (every -1 when FEW).
 * Checks (GPSB200_ERR_ARG, before anything is enqueued): acq and f_lo_prn as the search checks them, eph, ap, cfg, res,
 * seed and out not NULL, ap as gpsb200_pvt_coarse checks it, every n_a >= 1 with n_e n_n n_u n_t <= GPSB200_CD_MAX_HYP,
 * step_a finite and > 0 where n_a > 1, mask_deg and distinct_m finite, reserved 0.
 * Device scratch beyond the search's (which keeps its grid): nprn nbins (6072 x 2 + 16) bytes of normalised rows and row
 * sums, 8 nhyp bytes of per-hypothesis scores (128 MiB at GPSB200_CD_MAX_HYP), and 8 nhyp nprn bytes when the table
 * is wanted. Results do not depend on the order the device runs in. Blocking. */
#define GPSB200_CD_MAX_HYP    (1 << 24)
#define GPSB200_CD_MIN_USED   4
#define GPSB200_CD_Q_SHIFT    8
#define GPSB200_CD_Q_CAP      8192
#define GPSB200_CD_AMBIGUOUS_PCT 90
enum { GPSB200_CD_OK = 0, GPSB200_CD_FEW = 1, GPSB200_CD_AMBIGUOUS = 2 };
typedef struct gpsb200_collective_config {
    int32_t n[4];          /* lattice points along east, north, up, time: >= 1 each */
    double step[4];        /* their spacing: m, m, m, s; finite and > 0 where n > 1 */
    double mask_deg;       /* elevation mask of the used PRNs at x_a, degrees: finite */
    double distinct_m;     /* the runner-up lies farther than this from the winner, m: finite */
    int64_t reserved;      /* 0 */
} gpsb200_collective_config_t;   /* 72 bytes */
typedef struct gpsb200_collective {
    int32_t status;        /* GPSB200_CD_* */
    int32_t nused;         /* used PRNs (step 2) */
    uint32_t used;         /* bit p: acq->prn[p] is used */
    int32_t shift;         /* b*: the winner's clock shift, samples; -1 without a winner */
    int32_t winner, runner;    /* hypotheses h* and the runner-up's; -1 when there is none */
    uint32_t score, runner_score;  /* their S_h; 0 when there is none */
    double o_t;            /* the winner's time offset, s */
    double x[3];           /* the winner's ECEF position x_h*, m */
    double lat_deg, lon_deg, height;   /* and its WGS-84 latitude, longitude and height (gpsb200_pvt's conversion) */
    double runner_dist;    /* the runner-up's lattice distance from the winner, m */
} gpsb200_collective_t;    /* 96 bytes */
typedef struct gpsb200_cd_score {
    uint32_t score;        /* S_h */
    int32_t shift;         /* b_h */
} gpsb200_cd_score_t;      /* 8 bytes */
typedef struct gpsb200_cd_cell {
    int32_t bin;           /* j_p(h); -1 outside the grid or unused */
    int32_t delay;         /* d_p(h); -1 unused */
} gpsb200_cd_cell_t;       /* 8 bytes */
int gpsb200_collective(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                       const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                       const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                       gpsb200_acq_result_t *res, gpsb200_acq_result_t *seed, gpsb200_collective_t *out,
                       gpsb200_cd_score_t *scores, gpsb200_cd_cell_t *table);
/* Same for a source in device memory (16-byte aligned), searched and scored in place on `stream` (0 = the context's
 * own stream) behind whatever it holds; returns when the outputs are in host memory. */
int gpsb200_collective_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                              const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                              const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                              gpsb200_acq_result_t *res, gpsb200_acq_result_t *seed, gpsb200_collective_t *out,
                              gpsb200_cd_score_t *scores, gpsb200_cd_cell_t *table, void *stream);

/* ---- vector tracking: every channel's NCOs commanded by one navigation filter (DESIGN §10.1; tests/vtrack_model.py
 * states it in numpy). Spilker 1996; Lashley, Bevly & Hung, IEEE J-STSP 3(4), 2009. A channel needs no acquisition and
 * no loop of its own: the filter predicts its code phase and Doppler, and its discriminators feed back only a correction.
 * Constants: C = 299792458 m/s, FS = 3e6, lambda_chip = C / 1.023e6, lambda = C / 1575.42e6, OMEGA_E as gpsb200_pvt;
 * integer pieces (samples, tables, wipe-off, replicas, M, H, angle(), dll(), code_step(), "/" truncating) are the
 * gpsb200_track header's.
 *   seed       gpsb200_vtrack_seed: filter state X = (x, y, z, vx, vy, vz, b, d) (ECEF m, m/s, clock bias m, drift m/s)
 *              at stream sample s0 whose true receive time is t_rx; t0 = t_rx + b / C (receive time by the receiver
 *              clock); P = diag(sp^2, sp^2, sp^2, sv^2, sv^2, sv^2, sb^2, sd^2) from the config; channels unseeded.
 *   predict    channel c at stream sample s (s >= s0) from X at filter sample t_f (FP64, this order): dt = (s - t_f) / FS,
 *              r = X[0..2] + X[3..5] dt, b = X[6] + X[7] dt; q = floor((s - s0) / 3000), m = s - s0 - 3000 q,
 *              t = t0 + q / 1000 + m / FS - b / C; tau = 0.075, three times: satellite(eph, t - tau) (gpsb200_pvt's,
 *              position p, velocity v, clock dt_sv, drift ddt), p and v turned about z by OMEGA_E tau, l = p_rot - r,
 *              tau = |l| / C. Code phase phi (chips) = 1023 frac(F0 + m / 3000 + 1000 (dt_sv - tau - b / C)),
 *              F0 = frac(1000 t0), frac(x) = x - floor(x); unit vector e = l / |l|; range rate
 *              rr = e . (v_rot - X[3..5]) - C ddt + X[7]; Doppler f = -rr / lambda.
 *   command    from X at a channel's period start s with NCO code phase phi' (2^-32 chips): w = (int32) llround(f 2^32 /
 *              FS), f clamped to +-10 kHz; err = phi 2^32 - phi' wrapped into [-M/2, M/2), llround to int64; u =
 *              clamp(NOM + w / 1540 + err / (3000 N), MIN, MAX). The code correction goes only through u, so every
 *              period keeps 2999..3001 samples and the epochs run on without a jump.
 *   first      an unseeded call starts each channel at s0 from X: w as above, u = code_step(w), phi0 = llround(phi 2^32)
 *              mod M; its first period starts where the code wraps: s0 + ceil((M - phi0) / u) with phi' = phi0 + that
 *              many u - M (s0 and phi0 itself when phi0 = 0); theta = 0. The filter sample t_f = s0.
 *   periods    per channel exactly gpsb200_track's (sums E_I..L_Q, L, theta, phi, the epoch record) with u and w held
 *              for the whole interval; the record's lock is 1 when the channel was used at the last update. Also
 *              S = sum_{m<L} I^2 + Q^2 of the reduced samples (int32: <= 3001 * 32768).
 *   interval   N periods per channel. Sums over them (int64, exact): E = sum E_I^2 + E_Q^2, L likewise, P = sum P_I^2
 *              + P_Q^2, S = sum S; over the N - 1 pairs of consecutive prompts inside the interval, dot and cross as
 *              gpsb200_track's FLL forms and folds them. Bounds (N <= 100): E, L, P <= 100 * 1.85e16; S <= 9.9e9;
 *              |dot|, |cross| <= 99 * 1.85e16; all below 2^63.
 *   update     once every channel has N periods (the call stops instead when some channel's next period leaves the
 *              buffer first, or max_updates updates ran). t_f' = the largest channel end sample; time update to t_f'
 *              with F (r += v dt, b += d dt) and the constant-velocity / two-state clock process noise, per axis
 *              [[qa dt^3/3, qa dt^2/2], [qa dt^2/2, qa dt]], clock [[qb dt + qd dt^3/3, qd dt^2/2], [qd dt^2/2, qd dt]]:
 *              P = F P F^T + Q. Per channel c at its end sample s_c, with predict at that X: power ratio
 *              q = P / (GPSB200_VTRK_NOISE_SCALE S) (0 when S = 0; about 1 + C/N0 x 1 ms); used when q >= q_min;
 *              D = dll(E, L); du = u - code_step(w); code residual r = wrap_[-511.5, 511.5)(phi'/2^32 + D / 65536 -
 *              du n / 2^33 - phi) chips (n = the interval's samples; D / 65536 chips is the signal's mean lead on
 *              the replica, du n / 2 what the correction added by the end); innovation y_c = -lambda_chip r,
 *              row (-e, 0, 0, 0, 1, 0); a = angle(dot, cross), f_m = w FS / 2^32 + a 1000 / 2^32 Hz, innovation
 *              y_r = -lambda f_m - rr, row (0, 0, 0, -e, 0, 1); variances sc^2 / ((q - 1) N) and sr^2 / ((q - 1) N).
 *              Sequential scalar updates at the used channels in channel order, code before rate: y' = y - row .
 *              (X - X_prior), g = P row^T, s = row . g + var, K = g / s, X += K y', P -= K g^T (every sum in index
 *              order). Then every channel is commanded from the new X at its end sample; its sums restart.
 *   outputs    per update a gpsb200_fix_t (sample t_f'; status OK with 4 or more used channels, else FEW; iterations
 *              1; the position, velocity and clock are the filter's, also when FEW: unlike gpsb200_pvt's record, a FEW
 *              vector fix holds the state the filter coasts on, not NaN; t_rx = t0 + (t_f' - s0) / FS - b / C; PDOP from
 *              the used code rows as gpsb200_pvt's, NaN when FEW; rms of the post-fit code residuals y_c - row .
 *              (X - X_prior) of the used channels) and a gpsb200_vtrack_chan_t per channel.
 * The state carries everything, so any cut of a run into calls gives the run of one call bit for bit. */
#define GPSB200_VTRK_MAX_PERIODS 100
#define GPSB200_VTRK_NOISE_SCALE 62500.0     /* 250^2: the carrier table's nominal squared modulus */
typedef struct gpsb200_vtrack_config {
    int32_t periods;       /* N: 1..GPSB200_VTRK_MAX_PERIODS */
    int32_t reserved;      /* 0 */
    double sigma_code_m;   /* sc > 0: sigma of a code measurement at q - 1 = 1 and N = 1 */
    double sigma_rate_mps; /* sr > 0 */
    double q_min;          /* > 1 */
    double accel_psd;      /* qa >= 0, m^2/s^3 per axis */
    double bias_psd;       /* qb >= 0, m^2/s */
    double drift_psd;      /* qd >= 0, m^2/s^3 */
    double sigma_pos, sigma_vel, sigma_bias, sigma_drift;   /* sp, sv, sb, sd > 0: the seed's P */
} gpsb200_vtrack_config_t; /* 88 bytes */
typedef struct gpsb200_vtrack_chan_state {
    gpsb200_track_state_t nco;   /* prn, sample (next period), code / carrier NCO, code_step u, carr_step w, epochs */
    int64_t start;         /* first sample of the interval */
    int64_t e, l, p, s, dot, cross;   /* the interval's sums so far */
    int32_t k;             /* periods of the interval so far, 0..N */
    int32_t used;          /* used at the last update */
} gpsb200_vtrack_chan_state_t;  /* 128 bytes */
typedef struct gpsb200_vtrack_state {
    int64_t s0;            /* the seed's sample */
    double t0;             /* receive time by the receiver clock at s0, s of week */
    int32_t nchan;         /* 1..GPSB200_TRK_MAX_CHAN */
    int32_t seeded;        /* 0 until the first call starts the channels */
    int32_t updates;       /* filter updates so far */
    int32_t reserved;
    int64_t t_f;           /* the sample X holds at */
    double x[8];
    double P[64];          /* row major */
    gpsb200_vtrack_chan_state_t ch[GPSB200_TRK_MAX_CHAN];
} gpsb200_vtrack_state_t;  /* 4712 bytes */
typedef struct gpsb200_vtrack_chan {
    int64_t sample;        /* the channel's end sample s_c of the interval */
    int64_t e, l, p, s, dot, cross;   /* the interval's sums */
    int32_t prn;
    int32_t used;
    uint32_t code_step;    /* u commanded for the next interval */
    int32_t carr_step;     /* w commanded for the next interval */
    double q;              /* power ratio */
    double code_res_m;     /* innovation y_c (m) */
    double rate_res_mps;   /* innovation y_r (m/s) */
    double sigma_code_m;   /* sqrt of the variances (inf when not used) */
    double sigma_rate_mps;
} gpsb200_vtrack_chan_t;   /* 112 bytes */
/* Fill the config with the defaults (N 20, sc 50 m, sr 10 m/s, q_min 1.2, qa 1, qb 0.1, qd 0.01, sp 100 m, sv 1 m/s,
 * sb 10 m, sd 1 m/s). */
void gpsb200_vtrack_config_default(gpsb200_vtrack_config_t *cfg);
/* The seed (see above): x8 = X, t_rx at stream sample s0 (>= 0), nchan PRNs (1..32). GPSB200_ERR_ARG on a bad argument
 * (NULL pointers, nchan out of range, a non-finite X or t_rx outside [0, 604800), the config's sigmas). Host only.
 * A PRN may appear on one channel only (here and in the state gpsb200_vtrack reads): two channels on one satellite
 * would enter the filter as independent measurements and make the PDOP's normal matrix singular. */
int gpsb200_vtrack_seed(const gpsb200_vtrack_config_t *cfg, const double *x8, double t_rx, int64_t s0,
                        const int32_t *prn, int nchan, gpsb200_vtrack_state_t *state);
/* Vector-track state->nchan channels over nsamples samples of host memory (int8 / int16 I,Q interleaved; stream sample
 * `base` first; s0 and every channel's sample >= base). chans [nchan]: the ephemeris of each channel (chans[c].prn must
 * be the channel's PRN, eph.valid; anchors not read). state in and out. fixes [max_updates] and out [max_updates][nchan]
 * get the updates (*nupdates of them, max_updates >= 1). epochs (NULL: not wanted) [nchan][max_epochs] and nepochs
 * [nchan] get each channel's period records; max_epochs >= (max_updates + 1) N. Every argument is checked before
 * anything is enqueued (GPSB200_ERR_ARG). Blocking. */
int gpsb200_vtrack(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base,
                   const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg, gpsb200_vtrack_state_t *state,
                   int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *out, int32_t *nupdates,
                   gpsb200_track_epoch_t *epochs, int max_epochs, int32_t *nepochs);
/* Same for a source in device memory (16-byte aligned), tracked in place on `stream` (0 = the context's own stream)
 * behind whatever it holds; returns when the outputs are in host memory. */
int gpsb200_vtrack_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size, int64_t base,
                          const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg,
                          gpsb200_vtrack_state_t *state, int max_updates, gpsb200_fix_t *fixes,
                          gpsb200_vtrack_chan_t *out, int32_t *nupdates, gpsb200_track_epoch_t *epochs, int max_epochs,
                          int32_t *nepochs, void *stream);
/* Test hook: the cluster size (CTAs, 1..16) of later vector-tracking calls of this context; 0 restores the automatic
 * choice (min(nchan, 8)). Channel c runs on CTA c mod K; no choice changes a result. GPSB200_ERR_ARG otherwise. */
int gpsb200_debug_vtrack_cluster(gpsb200_ctx_t *ctx, int ctas);

/* ---- scenario engine: the reference's host path outside the sample loop -------------
 * RINEX-2/3 navigation file (plain or gzip-compressed, read through zlib like the reference, gps.c:1147) +
 * location/motion -> the gpsb200_chan_t records and NAV frames the
 * synthesis consumes; bit-identical to what the reference's producer computes (RINEX reader
 * gps.c:1131-1505, satpos/computeRange/ionosphericDelay gps.c:508-611,1893-2026,
 * computeCodePhase gps.c:2033-2064, eph2sbf/generateNavMsg/computeChecksum gps.c:617-884,
 * 1008-1072,2066-2140, allocateChannel gps.c:2142-2235, the 10 Hz / 30 s loop gps.c:2703-2765,
 * 2870-2932). With almanac_file set, the almanac of a SEM file goes into subframes 4 and 5 as the reference sends it
 * by default (SEM reader almanac.c:73-184, pages gps.c:772-883, time check gps.c:2637-2651); without one, the pages
 * are those of the reference run with --disable-almanac. */
typedef struct gpsb200_scenario_config {
    const char *nav_file;          /* -e: RINEX v2 (or, with rinex3, v3) navigation file */
    const char *motion_file;       /* -m: ECEF motion csv "t,x,y,z" at 10 Hz, NULL = static */
    double lat_deg, lon_deg, height_m;   /* -l */
    int32_t duration_ds;           /* -d in 0.1 s units: (int)(seconds*10+0.5) (gps-sim.c:140); blocks = this - 1 */
    int32_t max_chan;              /* 12 as shipped (gps.h:36); up to 32 */
    int32_t ionosphere_enable;     /* 1 = reference default (-I clears it) */
    int32_t pluto_gain;            /* 1 = gain x 2 (gps.c:2759-2763) */
    int32_t start_year, start_month, start_day, start_hour, start_min;   /* -s; year 0: first ephemeris epoch;
                                                                             -s now: see gpsb200_scenario_create_now */
    int32_t rinex3;                /* -3: nav_file is RINEX v3 (gps.c:1512-1891) instead of v2 */
    double start_sec;
    /* -t distance,bearing,height (gps-sim.c:145-148, gps.c:2348-2357): static runs start at a point given by distance
     * [m] and bearing [deg] from the location, height offset [m]; ignored with a motion file, as in the reference */
    int32_t target_valid;
    /* -i: the receiver is steered by gpsb200_scenario_key between advances (gps.c:2714-2729); ignored with a motion
     * file (gps-sim.c:297-301). Without keys the run equals the static one bit for bit. */
    int32_t interactive;
    double target_distance_m, target_bearing_deg, target_height_m;
    /* SEM almanac file sent in subframe 4 pages 2-5/7-10 (PRN 25-32) and subframe 5 pages 1-25 (PRN 1-24, toa/WNa);
     * NULL = no almanac (the reference's --disable-almanac). Read as the reference reads ./almanac.sem: at most 32
     * records, records parsed before the end of the file are kept (a partly read last record too), any other parse
     * error drops the whole almanac. A file that cannot be opened, or a record whose toa is more than 4 weeks from
     * the scenario start (a file with the full week number instead of week modulo 1024), is an error. */
    const char *almanac_file;
} gpsb200_scenario_config_t;
typedef struct gpsb200_scenario gpsb200_scenario_t;

int gpsb200_scenario_create(const gpsb200_scenario_config_t *cfg, gpsb200_scenario_t **out);
void gpsb200_scenario_destroy(gpsb200_scenario_t *s);
const char *gpsb200_scenario_error(const gpsb200_scenario_t *s);
int gpsb200_scenario_blocks(const gpsb200_scenario_t *s);        /* number of 0.1 s blocks */
int gpsb200_scenario_channels(const gpsb200_scenario_t *s);
int gpsb200_scenario_nav_frames(const gpsb200_scenario_t *s);
const gpsb200_chan_t *gpsb200_scenario_chans(const gpsb200_scenario_t *s);   /* [blocks][channels] */
const uint32_t *gpsb200_scenario_nav(const gpsb200_scenario_t *s);           /* [frames][channels][60] */
/* Time of applicability of the almanac in use as "yyyy/mm/dd,hh:mm:ss" (the last valid record's, gps.c:2644-2654), or
 * NULL when no valid record was read (no almanac_file, or nothing usable in it). */
const char *gpsb200_scenario_almanac_date(const gpsb200_scenario_t *s);
/* The resolved scenario start as "yyyy/mm/dd,hh:mm:ss" (seconds rounded as the reference prints them, gps.c:2580): the
 * configured start, or the first ephemeris record's epoch when start_year is 0. NULL before the scenario is opened. */
const char *gpsb200_scenario_start_date(const gpsb200_scenario_t *s);
/* The same start as GPS week and second of week (the receiver time of the allocation, gps.c:2575-2584). */
int gpsb200_scenario_start_time(const gpsb200_scenario_t *s, int32_t *week, double *sow);

/* ---- `-s now`: the ephemeris time overwrite (gps-sim.c:89-102, gps.c:2531-2561) -------------------------------
 * gpsb200_scenario_create_now / _open_now are _create / _open with the reference's time_overwrite set. cfg->start_* is
 * the clock reading (the reference takes gmtime(time()) in whole seconds and uses UTC as GPS time, without the leap
 * seconds; a caller that mirrors it passes the same). It is required and range-checked as the reference checks -s
 * (gps-sim.c:106-114: year after 1980, month 1-12, day 1-31, 0-23 h, 0-59 min, 0 <= sec < 60), else GPSB200_ERR_ARG.
 * Then, with gtmp = (start week, start second of week truncated to a multiple of 7200 s) and dsec = gtmp - toc of the
 * first record of the file:
 *   - every record's toc and toe move by dsec (week carry included), so the file may be of any date;
 *   - the UTC reference becomes WNt = gtmp.week, tot = gtmp.sec; the iono/UTC valid flag stays as read, so subframe 4
 *     page 18 carries tot / 4096 truncated and WNt mod 256;
 *   - the ephemeris span check of an explicit start is skipped.
 * Everything after that is the ordinary path on the moved times: the set within +-1 h of the start ("no current set
 * of ephemerides" when there is none -- a one-set file and a start in the second hour of its 2-hour epoch), the
 * 4-week almanac check against the start, the 30 s ephemeris roll. A moved toe second of week turns the constellation
 * in longitude by OMEGA_E * (new toe.sec - old toe.sec) (gps.c:585), as in the reference. */
int gpsb200_scenario_create_now(const gpsb200_scenario_config_t *cfg, gpsb200_scenario_t **out);
int gpsb200_scenario_open_now(const gpsb200_scenario_config_t *cfg, gpsb200_scenario_t **out);

/* ---- incremental scenario: the same engine advanced block range by block range -------------------------------
 * gpsb200_scenario_create == gpsb200_scenario_open + one advance over the whole run. An opened scenario keeps the
 * reference producer's state between advances (channels, allocation, ephemeris set, receiver time, NAV frame table,
 * previous ranges), so its memory is bounded by the largest advance and not by the duration; any cut of a run into
 * advances gives the records and frames of the batch run. On failure *out is still set (read the error, then destroy).
 *   advance  the next min(nblk, blocks left) blocks into chans_out[nblk][channels] (*got of them); nav_frame is the
 *            global frame number. GPSB200_ERR_END when no block is left (also after key 'x').
 *   frame    the [channels][60] NAV words of global frame f, valid for the frames the last advance referenced (and
 *            until the next advance); NULL otherwise.
 *   key      one key of the reference's interactive mode (gps-sim.c:363-401, gui.h:25-32), acting on the next block
 *            advance produces: 'a'/'d' bearing -/+ 127 mdeg (below 0 -> 360000, above 360000 -> 0), 'w'/'s' vertical
 *            speed +/- 1 m/s, 'e'/'q' speed +/- 0.01 m/s (clamped at 0), 't'/'g' SDR gain (no effect on the samples),
 *            'x'/'X' end the run after the blocks already produced. GPSB200_ERR_ARG for any other key, for a scenario
 *            opened without `interactive` (or with a motion file) and before block 1 (the reference reads keys only
 *            once its producer has started); GPSB200_ERR_END when no block is left. */
typedef struct gpsb200_steer_state {
    double speed;            /* target_t.speed (gps-sim.h:36-46): key units of 0.01 m/s */
    double velocity;         /* m/s = speed / 100 */
    double bearing_mdeg;     /* millidegrees; starts at the -t bearing x 1000, else 0 */
    double vertical_speed;   /* m/s */
    double xyz[3];           /* ECEF [m] of the receiver in the last block produced (before any: the start point) */
    int32_t next_block;      /* first block of the next advance */
    int32_t end_block;       /* blocks of the run (fewer after 'x') */
} gpsb200_steer_state_t;     /* 64 bytes */
int gpsb200_scenario_open(const gpsb200_scenario_config_t *cfg, gpsb200_scenario_t **out);
int gpsb200_scenario_advance(gpsb200_scenario_t *s, int nblk, gpsb200_chan_t *chans_out, int32_t *got);
const uint32_t *gpsb200_scenario_frame(const gpsb200_scenario_t *s, int frame);
int gpsb200_scenario_key(gpsb200_scenario_t *s, int key);
int gpsb200_scenario_steer_state(const gpsb200_scenario_t *s, gpsb200_steer_state_t *out);

/* One SEM almanac record as the scenario engine reads it (the reference's almanac_prn_t, almanac.h:21-38). */
typedef struct gpsb200_almanac_record {
    int32_t svid;          /* 1..32 (file id 0 reads as 1, above 32 as 32); 0 = no record */
    int32_t svn, ura, health, config_code;   /* ura <= 15, health <= 63, config_code <= 15 */
    int32_t valid;         /* 1 = all lines read; svid != 0 with valid == 0: the record the file ended in */
    int32_t toa_week;      /* file week + 2048 */
    int32_t reserved;
    double e, delta_i, omegadot, sqrta, omega0, aop, m0, af0, af1, toa_sec;
} gpsb200_almanac_record_t;
/* Parse a SEM file into rec[0..31] (indexed by svid - 1); *valid = 1 when at least one record is complete. Returns
 * GPSB200_ERR_ARG when the file cannot be opened. For tests (the parser against the reference's, field by field). */
int gpsb200_almanac_read(const char *path, gpsb200_almanac_record_t rec[32], int32_t *valid);

/* ---- almanac from decoded words (host; csrc/navdecode.cpp) ----------------------------------------------------------
 * Input: word records of one channel, as for gpsb200_nav_ephemeris; a subframe counts when its 10 words are in sequence
 * and all pass parity. Pages read (IS-GPS-200 20.3.3.5.1.2), all with data ID 1 (bits 23-22 of word 3's data):
 *   almanac    subframe 4 or 5 with SV ID (bits 21-16 of word 3) 1..32 -- subframe 5 pages 1-24, subframe 4 pages 2-5
 *              and 7-10. Fields, two's complement where signed, times exact powers of two, in the units of
 *              gpsb200_almanac_read (angles in semicircles): e (w3 bits 15-0, 2^-21), toa (w4 23-16, 2^12 s), delta_i
 *              (w4 15-0, 2^-19), OMEGADOT (w5 23-8, 2^-38), health (w5 7-0), sqrt A (w6, 2^-11), OMEGA0 (w7, 2^-23),
 *              omega (w8, 2^-23), M0 (w9, 2^-23), af0 (11 bits: w10 23-16 above w10 4-2, 2^-20), af1 (w10 15-5, 2^-38).
 *              The last such page of an SV in the words wins; rec[svid - 1] gets svid and valid = 1; svn, ura and
 *              config_code are not broadcast and stay 0. SV ID 0 (a dummy page) decodes to nothing.
 *   WNa        subframe 5 page 25 (SV ID 51): toa (bits 15-8) and WNa (bits 7-0); the last one wins. *wna_out = WNa, or
 *              -1 when no such page was read. Every decoded record's toa_week is WNa resolved to the full week within
 *              -128..127 of `week` (the meaning gpsb200_almanac_read gives it), -1 when there is no WNa.
 * Subframe 4 page 18 (ionosphere and UTC) is gpsb200_nav_ephemeris's. Records not decoded are all 0.
 * What the scenario engine sends, and so what a decode of its stream gives:
 *   - every page's health is 0 (the reference writes 000);
 *   - a SEM record cut short by the end of the file is sent in subframe 5 with the fields that were read;
 *   - the engine scales OMEGADOT, af1 (2^-38) and OMEGA0, omega, M0 (2^-23) by decimal literals that are not exactly
 *     powers of two (3.63797880709171e-12, 1.19209289550781e-07), so its integer is trunc(SEM / literal), which can
 *     differ by one LSB from trunc(SEM / 2^-k); decoded here with 2^-k, such a field is within one LSB of the SEM value.
 * GPSB200_ERR_ARG on a bad argument (NULL rec, n < 0, words NULL with n > 0). */
int gpsb200_nav_almanac(const gpsb200_nav_word_t *words, int64_t n, int32_t week, gpsb200_almanac_record_t rec[32],
                        int32_t *wna_out);

/* ---- where each satellite is in the sky, from an almanac (host; csrc/almanac.cpp; tests/almanac_model.py) -----------
 * For rec[i] (svid i + 1) with valid != 0, svid != 0 and toa_week >= 0, at GPS time (week, sow) of a receiver at ECEF
 * x_a (m), static. FP64, pi = 3.1415926535898 for semicircles, the constants of gps.h (GM, OMEGA_E, c, lambda_L1):
 *   orbit(t)   IS-GPS-200's almanac orbit: t_k = (week_t - toa_week) 604800 + sow_t - toa_sec; A = sqrt_A^2,
 *              n = sqrt(GM / A^3), M = M0 + n t_k; E by Newton from E = M until |dE| <= 1e-14 (at most 10 steps);
 *              i = 0.30 + delta_i (semicircles); no harmonic terms, no delta n, no IDOT; OMEGA = OMEGA0 +
 *              (OMEGADOT - OMEGA_E) t_k - OMEGA_E toa_sec; position and velocity as the ephemeris orbit's (DESIGN §11)
 *              with those terms zero; clock dt = af0 + af1 t_k
 *   transmit   tau1 = |orbit(t).p - x_a| / c; the satellite is orbit(t - tau1)
 *   sight      as §11's: tau = |p - x_a| / c, p and v turned about z by OMEGA_E tau; l = p' - x_a, R = |l|; azimuth and
 *              elevation of l in the frame at x_a's geodetic latitude / longitude (six fixed-point steps, as ecef_llh)
 *   out        el_deg, az_deg (0..360) in degrees; range_m = R - c dt; range rate r = l . v' / R;
 *              doppler_hz = -(r - c af1) / lambda_L1, the sign of the scenario's f_carr, where the acquisition peaks
 * out[i].prn = i + 1; out[i].valid = 0 (the rest 0) for records not predicted. GPSB200_ERR_ARG for a NULL argument, a
 * non-finite sow or x_a. */
typedef struct gpsb200_sky {
    int32_t prn;
    int32_t valid;
    double el_deg, az_deg;
    double range_m;
    double doppler_hz;
} gpsb200_sky_t;           /* 40 bytes */
int gpsb200_almanac_predict(const gpsb200_almanac_record_t rec[32], int32_t week, double sow, const double x_a[3],
                            gpsb200_sky_t out[32]);
/* Assistance data for gpsb200_pvt_coarse: the ephemeris of a RINEX-2 (rinex3 = 0) or RINEX-3 (rinex3 = 1) navigation
 * file, read by the scenario engine's readers. eph[prn - 1] is the PRN's record whose toe (week and second) is nearest
 * to GPS time (week, sow), the first such record on ties, among those within 7200 s; valid = 0 where there is none. The
 * fields are the file's values as read (not quantised as the broadcast message would carry them); week is the toe week
 * modulo 1024, health the SV health as the engine reads it, ura 0 (the readers keep no URA). GPSB200_ERR_ARG when the
 * file cannot be read, or for a NULL argument, week < 0 or sow outside 0..604800. */
int gpsb200_rinex_ephemeris(const char *path, int rinex3, int32_t week, double sow, gpsb200_ephemeris_t eph[32]);

/* ---- FIFO / sink boundary: the reference's own API (fifo.h:19-62) --------------
 * Guarded by the reference header's own include guard (fifo.h:13-14), so that a translation unit of the reference
 * that includes both headers -- in either order -- sees the declarations once (they are identical). */
#ifndef FIFO_H
#define FIFO_H
struct iq_buf {
    signed char *data8;        /* 8 bit IQ data  */
    signed short *data16;      /* 16 bit IQ data */
    unsigned int totalLength;  /* allocated size in elements */
    unsigned int validLength;  /* valid elements */
    struct iq_buf *next;
};
bool fifo_create(unsigned buffer_count, unsigned buffer_size, unsigned sample_size);
void fifo_destroy(void);
void fifo_wait_next(void);
void fifo_wait_full(void);
void fifo_halt(void);
struct iq_buf *fifo_acquire(void);
void fifo_enqueue(struct iq_buf *buf);
struct iq_buf *fifo_dequeue(void);
void fifo_release(struct iq_buf *buf);
#endif /* FIFO_H */
/* gpsb200 extension: reproduce the stock reference's loss of buffers 1..6 of a run
 * (tail bug, fifo.c:163-168) so that iqdata.bin is byte-identical to the stock program. The guarantee covers that
 * start-up loss with the reference's geometry (8 buffers, writer started when the FIFO is primed); as in the stock
 * program, further losses while the consumer lags depend on producer/consumer timing. */
void fifo_set_compat_drop(bool on);

/* Feed a contiguous run of I/Q elements into FIFO buffers of whatever size the FIFO was created
 * with, enqueueing each buffer when full and carrying the partly filled one to the next call --
 * the HackRF cadence of the reference (262144-element buffers across 600000-element blocks,
 * gps.c:2847-2856). gpsb200_fifo_push_flush enqueues a remaining partial buffer. */
int gpsb200_fifo_push(const void *elems, size_t count, int sample_size);
int gpsb200_fifo_push_flush(void);

/* iqfile sink (sdr_iqfile.h:16-18 semantics: writes ./iqdata.bin from the FIFO). */
int gpsb200_iqfile_start(const char *path, int sample_size);
void gpsb200_iqfile_stop(void);

#ifdef __cplusplus
}
#endif
#endif /* GPSB200_H */
