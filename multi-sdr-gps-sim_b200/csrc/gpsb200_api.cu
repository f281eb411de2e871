// C ABI of libgpsb200.so (include/gpsb200.h): context, pipeline, host share of the carrier chain.
//
// (k_tables writes the per-block carrier tables k_synth fetches by TMA; it depends on the parameters only.)
// Host work per block and channel is what the reference's 10 Hz path hands to its sample loop
// (gps.c:2731-2765) plus ONE thing the loop carries implicitly: the carrier phase at the start
// of the block, which in the reference is whatever 300000 sequential FP64 additions left behind
// (gps.c:2821-2826). That chain is resolved parallel in time (nco_exact.h): the host GUESSES
// every block's start phase, k_probe walks every block from its guess on the GPU, and a cheap
// sequential host scan (carrier_fixup) turns the probes into exact start phases -- falling back to
// the exact sequential walk for the rare block whose probe cannot be used. Then k_checkpoints and
// k_synth run, in chunks whose download overlaps the synthesis of later chunks.
#include <cuda_runtime.h>
#include <sched.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gpsb200.h"
#include "acquire.h"
#include "snapshot.h"
#include "collective.h"
#include "device_buffer.h"
#include "track.h"
#include "vtrack.h"
#include "pvt.h"
#include "nco_exact.h"
#include "synth_kernels.h"
#include "synth_lanes.h"
#include "synth_tables.h"

using namespace gpsb200;

namespace {

constexpr int kSynthChunk = 256;   // blocks per synthesis launch of the host-destination path (D2H overlap)
constexpr int kSegFirst = 256;     // first carrier-chain segment of the host-destination path: small, so
                                   // that the download can start early ...
constexpr int kSegBlocks = 1024;   // ... later ones larger (their probe kernels are latency bound)
constexpr int kSpanBlocks = 32;    // blocks per span of the two-level carrier chain (nco_exact.h: span_chain)
constexpr int kHostChainBlocks = 2;   // calls of at most this many blocks (the reference's own cadence is ONE block per
                                      // call, gps.c:2703-2865) skip the speculation: the host walks the few NCO chains
                                      // exactly itself instead of two latency-bound kernel round trips

struct ChainState {
    int prn = 0;
    double phase = 0.0;
};

// Small persistent worker pool: the per-segment host passes are sub-millisecond, so thread
// creation per pass would dominate them.
class WorkerPool {
public:
    explicit WorkerPool(int n) {
        for (int i = 0; i < n; i++) th_.emplace_back([this, i] { loop(i); });
    }
    ~WorkerPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto &t : th_) t.join();
    }
    int size() const { return (int) th_.size(); }
    // run job(lo, hi) over [0, n) split into at most size() contiguous ranges; blocks until done
    void run(int n, const std::function<void(int, int)> &job) {
        const int parts = std::max(1, std::min(size(), n));
        if (parts <= 1 || th_.empty()) {
            job(0, n);
            return;
        }
        std::unique_lock<std::mutex> lk(mu_);
        job_ = &job;
        n_ = n;
        parts_ = parts;
        pending_ = parts;
        ++epoch_;
        cv_.notify_all();
        done_.wait(lk, [this] { return pending_ == 0; });
        job_ = nullptr;
    }

private:
    void loop(int id) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(int, int)> *job;
            int n, parts;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || epoch_ != seen; });
                if (stop_) return;
                seen = epoch_;
                job = job_;
                n = n_;
                parts = parts_;
            }
            if (id < parts) {
                const int per = (n + parts - 1) / parts, lo = id * per, hi = std::min(n, lo + per);
                if (lo < hi) (*job)(lo, hi);
                std::lock_guard<std::mutex> lk(mu_);
                if (--pending_ == 0) done_.notify_all();
            }
        }
    }
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    const std::function<void(int, int)> *job_ = nullptr;
    int n_ = 0, parts_ = 0, pending_ = 0;
    uint64_t epoch_ = 0;
    bool stop_ = false;
};

// Pipeline segments of a call: a short first one (its chain resolution is the lead-in of everything), then long ones.
std::vector<std::pair<int, int>> segments_of(int nblk) {
    std::vector<std::pair<int, int>> v;
    int len = kSegFirst;
    for (int b0 = 0; b0 < nblk; len = kSegBlocks) {
        const int b1 = std::min(nblk, b0 + len);
        v.emplace_back(b0, b1);
        b0 = b1;
    }
    return v;
}

// One synthesis call: what its steps (call_open, seg_params, seg_probe, seg_scan, seg_commit, call_close) share.
struct Call {
    const gpsb200_chan_t *chans = nullptr;      // the caller's records; read by seg_params only
    int nblk = 0, nchan = 0, sample_size = 0;
    void *dst = nullptr;                        // device destination (NULL: the carrier chain only, no synthesis)
    void *dst_host = nullptr;                   // host destination: one contiguous buffer ...
    void *const *scatter = nullptr;             // ... or one buffer per block
    cudaStream_t stream = nullptr;              // the caller's stream: synthesis
    std::vector<std::pair<int, int>> segs;      // pipeline segments
    std::vector<ChainState> chain;              // exact chain state after the blocks scanned so far
    std::vector<std::vector<ChainState>> after; // ... after each scanned segment
    std::vector<int64_t> slow;                  // spans of each segment the host scan resolved block by block
    int rows = 0;                               // rows of h_seg_end the committed ranges filled
    int ichunk = 0;                             // next entry of ev_done
    gpsb200_stats_t st{};
    bool active = false, eager = false, probed = false, finished = false;   // slice calls

    Call() = default;
    Call(const gpsb200_chan_t *chans_, int nblk_, int nchan_, int sample_size_, void *dst_, void *dst_host_,
         void *const *scatter_, cudaStream_t stream_)
        : chans(chans_), nblk(nblk_), nchan(nchan_), sample_size(sample_size_), dst(dst_), dst_host(dst_host_),
          scatter(scatter_), stream(stream_), chain(nchan_) {
        plan(segments_of(nblk_));
    }
    void plan(std::vector<std::pair<int, int>> s) {
        segs = std::move(s);
        after.assign(segs.size(), {});
        slow.assign(segs.size(), 0);
    }
    bool host() const { return dst_host || scatter; }
};

// Events a call records for its stats (the first segment's probe and checkpoint launches, the caller's stream).
enum { kEvCallStart, kEvProbeStart, kEvProbeEnd, kEvCkptStart, kEvCkptEnd, kEvCallEnd, kCallEvents };

}  // namespace

struct gpsb200_ctx {
    gpsb200_config_t cfg{};
    int nruns = 0;
    cudaStream_t s_compute = nullptr, s_copy = nullptr, s_pre = nullptr, s_ck = nullptr;
    cudaEvent_t ev[kCallEvents]{};
    std::vector<cudaEvent_t> ev_done;      // one per synthesis chunk
    DeviceArray<BlockChanDev> d_bc;
    PinnedArray<BlockChanDev> h_bc;
    DeviceArray<RunCkpt> d_ck;
    PinnedArray<RunCkpt> h_ck;                         // run checkpoints of small calls, computed on the host
    DeviceArray<uint32_t> d_nav;
    PinnedArray<uint32_t> h_nav;
    DeviceArray<uint32_t> d_chips;
    DeviceArray<int32_t> d_atab;           // per-block carrier tables (k_tables -> k_synth)
    DeviceArray<double> d_carr_end;
    DeviceArray<int> d_chain_errors;                   // device self-check of the carrier chain
    PinnedArray<int> h_chain_errors;
    DeviceArray<double> d_guess;                       // speculative block-start phases
    PinnedArray<double> h_guess;
    std::vector<uint8_t> h_guess_abs;                  // relative-mode marker per (block, channel), see prepare_blocks
    std::vector<uint8_t> h_span_flags;                 // per (span, channel): 1 = every block idle, 2 = one satellite throughout
    DeviceArray<double> d_carr0;                       // exact block-start phases of host-resolved (irregular) spans
    PinnedArray<double> h_carr0;
    DeviceArray<CarrierProbe> d_probe;                 // block probes in HBM (k_chain reads them)
    PinnedArray<CarrierProbe> h_probe;                 // ... and in mapped host memory (host fallback)
    DeviceArray<double> d_seg;                         // [block][chan][kSegStates] probe states at checkpoint-segment starts
    PinnedArray<CarrierProbe> h_span_sum;              // span summaries, mapped host memory
    DeviceArray<SpanBlockState> d_spec;                // speculative block-start phases
    bool lanes_on = true;                              // GPSB200_LANES=0: always k_synth (lane = channel)
    bool lanes_veto = false;                           // a channel record outside k_synth_lanes' range was seen
    DeviceArray<SpanRes> d_span_res;
    PinnedArray<SpanRes> h_span_res;
    int max_spans = 0;
    PinnedArray<double> h_seg_end;         // mapped: device-walked end phases of every pipeline segment's last block
    std::vector<double> seg_expect;        // what the chain says they must be
    std::vector<cudaEvent_t> ev_seg;       // probes of segment i complete
    int fault_inject_chain = 0;            // gpsb200_debug_corrupt_chain(): 1 = resolution, 2 = segment state
    bool trace_on = false;
    double trace_t0 = 0.0;
    Call call;                             // a slice call begun with gpsb200_slice_prepare (active until finished)
    DeviceArray<uint8_t> d_out;            // synthesis staging of host destinations
    DeviceArray<uint8_t> d_rx;             // receiver staging of host sources (acquisition window, tracking buffer)
    DeviceArray<int8_t> d_rx_chips;        // chips as +-1 of tracking and snapshots (trk::chips_upload), built once
    bool rx_chips_ready = false;           // ... when d_rx_chips holds them
    bool nav_dirty = true;
    std::unique_ptr<WorkerPool> pool;      // host passes (guesses, fix-up scan)
    SynthArgs last{};                      // replay state
    bool have_last = false;
    acq::Scratch acq;                      // acquisition searches (acquire.cu), allocated by the first one
    trk::Scratch trk;                      // tracking calls (track.cu), allocated by the first one
    pvt::Scratch pvt;                      // position fixes (pvt.cu), allocated by the first one
    snap::Scratch snap;                    // snapshot measurements (snapshot.cu), allocated by the first one
    cd::Scratch cd;                        // collective detection (collective.cu), allocated by the first one
    vtk::Scratch vtk;                      // vector tracking (vtrack.cu), allocated by the first one
    int vtk_ctas = 0;                      // gpsb200_debug_vtrack_cluster (0: automatic)
    std::string err;
};

namespace {

struct OneSatellite {          // parameter accessor of span_chain() for the host model: one satellite, increments cc[j]
    const double *cc;
    __host__ __device__ void operator()(int j, double &c, int32_t &prn) const {
        c = cc[j];
        prn = 1;
    }
};

double now_ms();
// GPSB200_TRACE=1: host time stamps of the pipeline's phases on stderr (diagnostics)
void trace(gpsb200_ctx *ctx, const char *what);

int fail(gpsb200_ctx *c, int code, const std::string &msg) {
    if (c) c->err = msg;
    return code;
}

#define CU(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(ctx, GPSB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

double now_ms() {
    using namespace std::chrono;
    return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

void trace(gpsb200_ctx *ctx, const char *what) {
    if (!ctx->trace_on) return;
    const double t = now_ms();
    fprintf(stderr, "[gpsb200 dev %d +%8.3f ms] %s (%d host workers)\n", ctx->cfg.device, t - ctx->trace_t0, what,
            ctx->pool ? ctx->pool->size() : 0);
}

// The closed-form carrier-phase guess (the phase predicted for the end of a run of blocks) of prepare_blocks,
// gpsb200_slice_link_host and gpsb200_span_chain_host: phases as 64-bit fixed point (cycles * 2^64, modulo 2^64 =
// modulo one cycle: exact integer arithmetic), truncated to a double when read.
inline uint64_t phase_to_fix(double p) { return (p >= 0.0 && p < 1.0) ? (uint64_t) (p * 0x1p64) : 0; }
inline double fix_to_phase(uint64_t a) { return (double) (a >> 11) * 0x1p-53; }
inline uint64_t step_to_fix(double c) {     // c in (-1, 1): c * 2^64 modulo 2^64 (exact for |c| >= 2^-12, else truncated)
    const uint64_t m = (uint64_t) (std::fabs(c) * 0x1p64);
    return c < 0.0 ? (uint64_t) 0 - m : m;
}
// One block: 300000 steps of c, plus the expected rounding drift of those steps. (The drift of a block is up to +-8e-12
// cycles and depends on the low bits of c, i.e. it is uncorrelated from block to block: evaluating it for every 4th
// block only was tried and made 50x more probes miss.)
inline uint64_t guess_block(uint64_t acc, double c) {
    acc += (uint64_t) GPSB200_BLOCK_SAMPLES * step_to_fix(c);
    return acc + (uint64_t) (int64_t) ((double) GPSB200_BLOCK_SAMPLES * carrier_drift_per_step(c) * 0x1p64);
}

// Host pre-pass: validate, fill the device-layout records and GUESS every block's start carrier phase.

// With link != NULL (time-slice hand-over, gpsb200_slice_prepare) the incoming chain state is not known yet:
// guesses are accumulated RELATIVE to it (h_guess holds the advance since the slice start, h_guess_abs marks
// blocks after a (re)allocation inside the slice, whose guesses are absolute) and finalize_guesses() adds the
// offset later; *link describes how the slice maps an incoming state to the guessed outgoing one.
// end_guess (optional): the GUESSED chain state after block b1-1, to seed the guesses of the next segment when that
// is prepared before this one has been resolved.
int prepare_blocks(gpsb200_ctx *ctx, const gpsb200_chan_t *chans, int b0, int b1, int nchan,
                   const std::vector<ChainState> &chain, gpsb200_slice_link_t *link = nullptr,
                   std::vector<ChainState> *end_guess = nullptr) {
    const double delt = 1.0 / (double) GPSB200_SAMPLERATE;     // gps.c:2298
    std::vector<int> status(nchan, GPSB200_OK);
    std::vector<uint8_t> lanes_bad(nchan, 0);
    ctx->pool->run(nchan, [&](int c_lo, int c_hi) {
        for (int c = c_lo; c < c_hi; c++) {
            // phase accumulator in cycles * 2^64, modulo 2^64 (= modulo one cycle): exact integer arithmetic
            uint64_t acc = phase_to_fix(chain[c].phase);    // exact phase after block b0-1 (if any)
            int prev_prn = chain[c].prn;                    // 0 at the start of a call: block 0 is "fresh"
            bool absolute = link == nullptr;                // relative mode: true once a slot was (re)allocated
            if (link) {
                acc = 0;
                prev_prn = chans[(size_t) b0 * nchan + c].prn;      // block b0 continues whatever comes in (decided later)
                link->prn_first[c] = prev_prn;
                link->first_phase[c] = prev_prn > 0 ? chans[(size_t) b0 * nchan + c].carr_phase : 0.0;
            }
            int span_first_prn = 0;
            uint8_t span_idle = 1, span_uniform = 1;
            for (int b = b0; b < b1; b++) {
                const gpsb200_chan_t &in = chans[(size_t) b * nchan + c];
                const size_t i = (size_t) b * nchan + c;
                BlockChanDev &o = ctx->h_bc[i];
                memset(&o, 0, sizeof o);
                // what the host scan wants to know about the span this block belongs to (resolve_chain)
                if (b % kSpanBlocks == 0) {
                    span_first_prn = in.prn;
                    span_idle = span_uniform = 1;
                }
                span_idle &= in.prn <= 0;
                span_uniform &= in.prn == span_first_prn;
                if ((b + 1) % kSpanBlocks == 0 || b + 1 == b1)
                    ctx->h_span_flags[(size_t) (b / kSpanBlocks) * nchan + c] = (uint8_t) (span_idle | (span_uniform << 1));
                ctx->h_guess[i] = 0.0;
                ctx->h_guess_abs[i] = absolute ? 1 : 0;
                if (in.prn <= 0) {
                    prev_prn = 0;
                    absolute = true;                        // whatever follows starts from an allocation phase
                    continue;
                }
                if (in.prn > 32 || in.iword < 0 || in.iword >= GPSB200_NAV_WORDS || in.ibit < 0 || in.ibit >= 30 ||
                    in.icode < 0 || in.icode >= 20 || in.nav_frame < 0 || in.nav_frame >= ctx->cfg.max_nav_frames ||
                    !(in.code_phase >= 0.0 && in.code_phase < 1023.0) ||
                    // the per-lane chip window holds 24 chips per 64 samples: f_code <= 1.07 MHz (GPS: 1.023 MHz +- 4 Hz)
                    !(in.f_code > 0.0 && in.f_code <= 1.07e6) ||
                    // one wrap per step keeps the phase in [0,1) only for |f_carr * delt| < 1
                    !(std::isfinite(in.f_carr) && std::fabs(in.f_carr) < 2.9e6) || !std::isfinite(in.gain)) {
                    status[c] = GPSB200_ERR_ARG;
                    return;
                }
                // a slot whose satellite changed (or the first block of a call): the caller's carr_phase applies
                if (!(in.carr_phase >= 0.0 && in.carr_phase < 1.0)) {      // read whenever a slot takes a new satellite
                    status[c] = GPSB200_ERR_ARG;
                    return;
                }
                if (in.prn != prev_prn) {
                    acc = phase_to_fix(in.carr_phase);
                    absolute = true;
                }
                ctx->h_guess_abs[i] = absolute ? 1 : 0;
                prev_prn = in.prn;
                o.c_carr = in.f_carr * delt;                    // gps.c:2821
                o.c_code = in.f_code * delt;                    // gps.c:2789
                if (!lanes::code_step_ok(o.c_code) || !(std::fabs(o.c_carr) < 0.5)) lanes_bad[c] = 1;
                o.gain = in.gain;
                o.carr_in = in.carr_phase;
                o.code0 = in.code_phase;
                o.prn = in.prn;
                o.nav0 = (uint32_t) in.iword | ((uint32_t) in.ibit << 8) | ((uint32_t) in.icode << 16);
                o.frame = in.nav_frame;
                ctx->h_guess[i] = fix_to_phase(acc);
                acc = guess_block(acc, o.c_carr);
            }
            if (end_guess) {
                (*end_guess)[c].prn = prev_prn > 0 ? prev_prn : 0;
                (*end_guess)[c].phase = prev_prn > 0 ? fix_to_phase(acc) : 0.0;
            }
            if (link) {
                link->prn_last[c] = prev_prn > 0 ? prev_prn : 0;
                link->reset_inside[c] = absolute ? 1 : 0;
                link->value[c] = fix_to_phase(acc);
            }
        }
    });
    for (int c = 0; c < nchan; c++)
        if (status[c] != GPSB200_OK) return fail(ctx, status[c], "invalid channel parameters in slot " + std::to_string(c));
    // k_synth_lanes covers every code rate a GPS receiver can see (1.0157 .. 1.0302 MHz); anything else keeps this
    // context on k_synth from here on (both are exact; the choice is sticky so that no launch mixes assumptions)
    for (int c = 0; c < nchan; c++)
        if (lanes_bad[c]) ctx->lanes_veto = true;
    // The reference stores (short)i_acc (gps.c:2834); the packed I/Q accumulation is
    // exact as long as |acc| stays inside int16, which bounds the sum of amplitudes.
    for (int b = b0; b < b1; b++) {
        double amp = 0.0;
        for (int c = 0; c < nchan; c++) amp += std::fabs(ctx->h_bc[(size_t) b * nchan + c].gain) * 250.0;
        if (amp > 32767.0) return fail(ctx, GPSB200_ERR_RANGE, "sum of channel amplitudes exceeds int16 range");
    }
    return GPSB200_OK;
}

// Second pass of the relative mode: the (guessed) incoming state is known now.
void finalize_guesses(gpsb200_ctx *ctx, int b0, int b1, int nchan, const int32_t *prn_in, const double *phase_in) {
    ctx->pool->run(nchan, [&](int c_lo, int c_hi) {
        for (int c = c_lo; c < c_hi; c++) {
            const BlockChanDev &first = ctx->h_bc[(size_t) b0 * nchan + c];
            const bool cont = prn_in && phase_in && first.prn > 0 && prn_in[c] == first.prn;
            const double off = cont ? phase_in[c] : first.carr_in;
            for (int b = b0; b < b1; b++) {
                const size_t i = (size_t) b * nchan + c;
                if (ctx->h_guess_abs[i] || ctx->h_bc[i].prn <= 0) continue;
                double g = ctx->h_guess[i] + off;
                if (g >= 1.0) g -= 1.0;
                if (!(g >= 0.0 && g < 1.0)) g = 0.0;
                ctx->h_guess[i] = g;
            }
        }
    });
}

// The exact chain state after block b0-1 is known: move the guesses of blocks [b0, b1) by the error the guess of
// block b0 turned out to have (a slot's guesses are corrected up to its next (re)allocation, whose phase is exact).
void reanchor_guesses(gpsb200_ctx *ctx, int b0, int b1, int nchan, const std::vector<ChainState> &chain) {
    ctx->pool->run(nchan, [&](int c_lo, int c_hi) {
        for (int c = c_lo; c < c_hi; c++) {
            const BlockChanDev &first = ctx->h_bc[(size_t) b0 * nchan + c];
            if (first.prn <= 0 || chain[c].prn != first.prn) continue;     // starts from an allocation phase: exact already
            double delta = chain[c].phase - ctx->h_guess[(size_t) b0 * nchan + c];
            if (delta > 0.5) delta -= 1.0;
            if (delta < -0.5) delta += 1.0;
            for (int b = b0; b < b1; b++) {
                const size_t i = (size_t) b * nchan + c;
                if (ctx->h_bc[i].prn != first.prn) break;
                double g = ctx->h_guess[i] + delta;
                if (g >= 1.0) g -= 1.0;
                if (g < 0.0) g += 1.0;
                if (!(g >= 0.0 && g < 1.0)) g = 0.0;
                ctx->h_guess[i] = g;
            }
        }
    });
}

// One block of the chain, resolved on the host from its block probe (the first level of the speculation);
// the exact sequential walk when the probe cannot be used. start_out: the block's exact start phase (k_checkpoints
// walks the block from it). Returns 1 when it had to walk.
inline int resolve_block(ChainState &st, const BlockChanDev &bc, const CarrierProbe &probe, double &start_out) {
    if (bc.prn <= 0) {
        st.prn = 0;
        start_out = 0.0;
        return 0;
    }
    if (st.prn != bc.prn) st.phase = bc.carr_in;
    st.prn = bc.prn;
    start_out = st.phase;
    double xe;
    if (carrier_fixup(st.phase, bc.c_carr, probe, xe)) {
        st.phase = xe;
        return 0;
    }
    int64_t dummy = 0;
    nco_advance<NCO_CARRIER>(st.phase, bc.c_carr, GPSB200_BLOCK_SAMPLES, dummy);
    return 1;
}

// Host scan of the two-level chain for blocks [b0, b1) (b0 is a span boundary of this launch): one
// carrier_fixup per SPAN from the span summaries k_chain left in mapped host memory; a span the device
// could not chain speculatively (reallocation inside it, Doppler zero crossing, a rejected block probe)
// or whose summary does not fit the true start phase is resolved block by block from the block probes.
// Serial over spans per channel, parallel over channels. Returns the number of blocks walked sequentially; adds the
// number of spans resolved block by block to *spans_slow.
int64_t resolve_chain(gpsb200_ctx *ctx, int b0, int b1, int nchan, std::vector<ChainState> &chain, int64_t *spans_slow) {
    std::vector<int64_t> fallbacks(nchan, 0), slow(nchan, 0);
    const int K = kSpanBlocks;
    const int nspan = (b1 - b0 + K - 1) / K;
    ctx->pool->run(nchan, [&](int c_lo, int c_hi) {
        for (int c = c_lo; c < c_hi; c++) {
            ChainState st = chain[c];
            for (int sp = 0; sp < nspan; sp++) {
                const int s0 = b0 + sp * K, s1 = std::min(b1, s0 + K);
                SpanRes &res = ctx->h_span_res[(size_t) (s0 / K) * nchan + c];
                const BlockChanDev &first = ctx->h_bc[(size_t) s0 * nchan + c];
                const uint8_t flags = ctx->h_span_flags[(size_t) (s0 / K) * nchan + c];     // from prepare_blocks
                const bool idle = flags & 1, uniform = flags & 2;
                res.start = res.shift = 0.0;
                res.variant = 0;
                if (idle) {
                    res.mode = 2;
                    st.prn = 0;
                    continue;
                }
                if (uniform && first.prn > 0) {
                    const double start = st.prn == first.prn ? st.phase : first.carr_in;
                    const CarrierProbe &sum = ctx->h_span_sum[(size_t) (s0 / K) * nchan + c];
                    double xe, d;
                    int v;
                    if (carrier_fixup(start, first.c_carr, sum, xe, &v, &d, 1.0)) {
                        res.mode = 0;
                        res.start = start;
                        res.shift = d;
                        res.variant = v;
                        st.prn = first.prn;
                        st.phase = xe;
                        continue;
                    }
                }
                // block by block (first level only)
                res.mode = 1;
                ++slow[c];
                for (int b = s0; b < s1; b++) {
                    const size_t i = (size_t) b * nchan + c;
                    fallbacks[c] += resolve_block(st, ctx->h_bc[i], ctx->h_probe[i], ctx->h_carr0[i]);
                }
            }
            chain[c] = st;
        }
    });
    // test hook of the device self-check (gpsb200_debug_corrupt_chain): corrupt the resolution of slot 0's first span
    // by one unit of the rounding grid -- the span's shift, or the start phase of block b0 + 5 when the span was
    // resolved block by block; k_checkpoints must notice
    if (ctx->fault_inject_chain == 1 && b1 - b0 > 6) {
        SpanRes &r = ctx->h_span_res[(size_t) (b0 / K) * nchan];
        if (r.mode == 0) r.shift += 0x1p-51;
        else if (r.mode == 1) ctx->h_carr0[(size_t) (b0 + 5) * nchan] += 0x1p-51;
    }
    int64_t n = 0;
    for (int c = 0; c < nchan; c++) {
        n += fallbacks[c];
        if (spans_slow) *spans_slow += slow[c];
    }
    return n;
}

SynthArgs make_args(gpsb200_ctx *ctx, int blk0, int nblk, int nchan, int sample_size, void *out) {
    // blk0 is a multiple of kSpanBlocks whenever the chain kernels are launched with these arguments
    SynthArgs a{};
    const size_t off = (size_t) blk0 * nchan;
    a.bc = ctx->d_bc.get() + off;
    a.carr0 = ctx->d_carr0.get() + off;
    a.guess = ctx->d_guess.get() + off;
    a.probe = ctx->d_probe.get() + off;
    a.probe_host = ctx->h_probe.dev() + off;
    a.seg = ctx->d_seg.get() + off * kSegStates;
    a.spec = ctx->d_spec.get() + off;
    a.span_blocks = kSpanBlocks;
    a.nspan = (nblk + kSpanBlocks - 1) / kSpanBlocks;
    a.span_sum = ctx->h_span_sum.dev() + (size_t) (blk0 / kSpanBlocks) * nchan;
    a.span_res = ctx->d_span_res.get() + (size_t) (blk0 / kSpanBlocks) * nchan;
    a.ck = ctx->d_ck.get() + off * ctx->nruns;
    a.nav = ctx->d_nav.get();
    a.nav_stride = ctx->cfg.max_chan;
    a.chipbits = ctx->d_chips.get();
    a.atab = ctx->d_atab.get() + (size_t) blk0 * kAtabRows * 32;
    a.carr_end = ctx->d_carr_end.get() + off;
    a.chain_errors = ctx->d_chain_errors.get();
    a.out = out;
    a.nblk = nblk;
    a.nchan = nchan;
    a.nruns = ctx->nruns;
    a.run_samples = ctx->cfg.run_samples;
    a.iq16 = sample_size == GPSB200_SC16;
    a.lanes = ctx->lanes_on && !ctx->lanes_veto ? 1 : 0;
    // lanes per run follow the channel count; a CTA takes up to 24 warps' worth of runs
    const int grp = nchan > 16 ? 32 : (nchan > 8 ? 16 : 8);
    const int rpw = 32 / grp;
    int per_cta = 24 * rpw;
    const int ctas = (ctx->nruns + per_cta - 1) / per_cta;
    per_cta = (ctx->nruns + ctas - 1) / ctas;
    a.runs_per_cta = per_cta;
    a.ctas_per_block = ctas;
    return a;
}

// Arguments of a call's kernels over blocks [b0, b0 + nb), synthesizing into the call's device destination.
SynthArgs call_args(gpsb200_ctx *ctx, const Call &call, int b0, int nb) {
    const size_t blk_bytes = (size_t) GPSB200_BLOCK_ELEMS * call.sample_size;
    return make_args(ctx, b0, nb, call.nchan, call.sample_size, (char *) call.dst + (size_t) b0 * blk_bytes);
}

int upload_nav(gpsb200_ctx *ctx, cudaStream_t s) {
    if (!ctx->nav_dirty) return GPSB200_OK;
    const size_t bytes = (size_t) ctx->cfg.max_nav_frames * ctx->cfg.max_chan * GPSB200_NAV_WORDS * 4;
    CU(cudaMemcpyAsync(ctx->d_nav.get(), ctx->h_nav.get(), bytes, cudaMemcpyHostToDevice, s));
    ctx->nav_dirty = false;
    return GPSB200_OK;
}

// The checks of every entry point that enqueues work, after its own argument checks: the context has a device and no
// slice call is open. Then selects the context's device.
int check_entry(gpsb200_ctx *ctx) {
    if (!ctx->s_compute) return fail(ctx, GPSB200_ERR_CUDA, "context has no CUDA device");
    if (ctx->call.active) return fail(ctx, GPSB200_ERR_ARG, "a call begun with gpsb200_slice_prepare has not been finished");
    CU(cudaSetDevice(ctx->cfg.device));     // the caller may be a thread that never selected the context's device
    return GPSB200_OK;
}

int check_call(gpsb200_ctx *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size, void *dst) {
    if (!chans || !dst || nblk < 1 || nblk > ctx->cfg.max_blocks || nchan < 1 || nchan > ctx->cfg.max_chan ||
        (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16))
        return fail(ctx, GPSB200_ERR_ARG, "bad arguments (1 <= nchan <= cfg.max_chan; 1 <= nblk <= cfg.max_blocks)");
    return check_entry(ctx);
}

// A caller's device buffer must be 16-byte aligned. Both synthesis kernels store whole 2- to 16-byte words at multiples
// of their width from the destination (k_synth_lanes always 16 bytes, k_synth up to 32 bytes per lane as 16-byte
// vectors); the receiver calls' device sources are held to the same rule. Checked before anything is enqueued;
// allocations of CUDA and torch are aligned to 256 bytes.
int check_aligned(gpsb200_ctx *ctx, const void *p, const char *fn, const char *arg) {
    if ((reinterpret_cast<uintptr_t>(p) & 15u) != 0)
        return fail(ctx, GPSB200_ERR_ARG, std::string(fn) + ": " + arg + " is not 16-byte aligned");
    return GPSB200_OK;
}

// Host destinations are staged in the context's own device buffer, sized for the context's largest call.
int ensure_staging(gpsb200_ctx *ctx, int sample_size) {
    CU(ctx->d_out.grow((size_t) ctx->cfg.max_blocks * GPSB200_BLOCK_ELEMS * sample_size));
    return GPSB200_OK;
}

// The source of a receiver call (entry point fn), after the call's own contract check: a device source is checked for
// alignment and read in place; of a host source, samples first .. first + count - 1 are copied up on s into the
// context's receiver staging buffer (every receiver call waits for its results, so no two hold it at the same time).
// *dev: the device address of sample `first`.
int rx_source(gpsb200_ctx *ctx, const char *fn, const void *iq, int64_t first, int64_t count, int sample_size,
              bool device, cudaStream_t s, const void **dev) {
    int rc = device ? check_aligned(ctx, iq, fn, "iq_device") : GPSB200_OK;
    if (!rc) rc = check_entry(ctx);
    if (rc) return rc;
    const size_t elem = sample_size == GPSB200_SC16 ? 4 : 2;
    *dev = static_cast<const char *>(iq) + (size_t) first * elem;
    if (device) return GPSB200_OK;
    CU(ctx->d_rx.grow((size_t) count * elem));
    if (count) CU(cudaMemcpyAsync(ctx->d_rx.get(), *dev, (size_t) count * elem, cudaMemcpyHostToDevice, s));
    *dev = ctx->d_rx.get();
    return GPSB200_OK;
}

// The chips as +-1 of tracking and snapshots in ctx->d_rx_chips, built by the first receiver call that needs them (and
// again by the next one when a build fails part way).
cudaError_t rx_chips(gpsb200_ctx *ctx) {
    if (!ctx->rx_chips_ready) {
        CU_RET(trk::chips_upload(ctx->d_rx_chips));
        ctx->rx_chips_ready = true;
    }
    return cudaSuccess;
}

// The one error path of every entry point that enqueues work: on a non-OK return wait for everything this context
// and the caller's stream have in flight (the caller may free its buffers once it sees the error code, so no copy into
// them may still be pending) and drop the begun slice call; the context stays usable. Leaves ctx->err alone.
int settle(gpsb200_ctx *ctx, cudaStream_t caller, int rc) {
    if (rc == GPSB200_OK) return rc;
    ctx->call.active = false;
    if (!ctx->s_compute) return rc;
    if (caller) cudaStreamSynchronize(caller);
    cudaStreamSynchronize(ctx->s_compute);
    cudaStreamSynchronize(ctx->s_pre);
    cudaStreamSynchronize(ctx->s_ck);
    cudaStreamSynchronize(ctx->s_copy);
    return rc;
}

// The stream of an entry point that takes the caller's: stream_, or the context's compute stream when it is NULL.
cudaStream_t caller_stream(gpsb200_ctx *ctx, void *stream_) {
    return stream_ ? (cudaStream_t) stream_ : ctx->s_compute;
}

// ---- the steps of a call --------------------------------------------------------------------------------------------
// A call's segments go through params -> probe -> scan -> commit; the schedules below (run_pipeline, the slice
// entry points, gpsb200_carrier_chain_device) differ only in how they order and overlap these steps (DESIGN §6).

// Start of a call's device work: the pre-phase streams wait for what the caller's stream holds so far (it may still read
// the buffers rewritten now), then NAV words up and the self-check counter cleared on s_pre.
int call_open(gpsb200_ctx *ctx, const Call &call) {
    CU(cudaEventRecord(ctx->ev[kEvCallStart], call.stream));
    CU(cudaStreamWaitEvent(ctx->s_pre, ctx->ev[kEvCallStart], 0));
    CU(cudaStreamWaitEvent(ctx->s_ck, ctx->ev[kEvCallStart], 0));
    const int rc = upload_nav(ctx, ctx->s_pre);
    if (rc) return rc;
    CU(cudaMemsetAsync(ctx->d_chain_errors.get(), 0, sizeof(int), ctx->s_pre));
    return GPSB200_OK;
}

// Params of blocks [b0, b1) on sp: host records + guesses, parameters up, carrier tables (a call without a destination
// computes the chain only and needs none). The guesses continue the call's exact chain state before b0, or with
// `guessed` a GUESSED one (advanced in place to the guessed state after b1 - 1, so that the next segment can be
// prepared before this one is resolved), or with `link` none at all (relative mode, see prepare_blocks).
int seg_params(gpsb200_ctx *ctx, Call &call, int b0, int b1, cudaStream_t sp, std::vector<ChainState> *guessed,
               gpsb200_slice_link_t *link) {
    const size_t off = (size_t) b0 * call.nchan, cnt = (size_t) (b1 - b0) * call.nchan;
    const double t0 = now_ms();
    const int rc = prepare_blocks(ctx, call.chans, b0, b1, call.nchan, guessed ? *guessed : call.chain, link, guessed);
    if (rc) return rc;
    call.st.host_chain_ms += now_ms() - t0;
    CU(cudaMemcpyAsync(ctx->d_bc.get() + off, ctx->h_bc.get() + off, cnt * sizeof(BlockChanDev), cudaMemcpyHostToDevice,
                       sp));
    call.st.h2d_bytes += (int64_t) (cnt * sizeof(BlockChanDev));
    if (call.dst) {
        CU(launch_tables(call_args(ctx, call, b0, b1 - b0), sp));     // needs only the parameters: off the critical path
        call.st.launches += 1;
    }
    return GPSB200_OK;
}

// Probe of blocks [b0, b1) on sp: everything that needs no true start phase -- guesses up, block probes (+ the code-NCO
// half of the run checkpoints, which seg_commit relies on; not for a call without a destination), span chaining.
int seg_probe(gpsb200_ctx *ctx, Call &call, int b0, int b1, cudaStream_t sp) {
    const size_t off = (size_t) b0 * call.nchan, cnt = (size_t) (b1 - b0) * call.nchan;
    SynthArgs a = make_args(ctx, b0, b1 - b0, call.nchan, call.sample_size, nullptr);
    if (!call.dst) a.ck = nullptr;
    CU(cudaMemcpyAsync(ctx->d_guess.get() + off, ctx->h_guess.get() + off, cnt * sizeof(double), cudaMemcpyHostToDevice,
                       sp));
    if (b0 == 0) CU(cudaEventRecord(ctx->ev[kEvProbeStart], sp));
    CU(launch_probe(a, sp));
    CU(launch_chain(a, sp));
    if (b0 == 0) CU(cudaEventRecord(ctx->ev[kEvProbeEnd], sp));
    call.st.launches += 2;
    call.st.h2d_bytes += (int64_t) (cnt * sizeof(double));
    call.st.d2h_bytes += (int64_t) (cnt * sizeof(CarrierProbe) + (size_t) a.nspan * call.nchan * sizeof(CarrierProbe));
    return GPSB200_OK;
}

// Host scan of segment i: wait until its probes and span summaries are in (mapped) host memory -- for `probes_done`
// when given, else for the stream that ran them -- and resolve the call's chain through the segment.
int seg_scan(gpsb200_ctx *ctx, Call &call, int i, cudaEvent_t probes_done, cudaStream_t sp) {
    if (probes_done) CU(cudaEventSynchronize(probes_done));
    else CU(cudaStreamSynchronize(sp));
    const double t0 = now_ms();
    call.slow[i] = 0;
    call.st.chain_fallbacks +=
        (int32_t) resolve_chain(ctx, call.segs[i].first, call.segs[i].second, call.nchan, call.chain, &call.slow[i]);
    call.st.host_chain_ms += now_ms() - t0;
    call.after[i] = call.chain;
    return GPSB200_OK;
}

// Blocks [b0, b1) of the call's device destination to its host destination, on stream s.
int download(gpsb200_ctx *ctx, Call &call, int b0, int b1, cudaStream_t s) {
    const size_t blk_bytes = (size_t) GPSB200_BLOCK_ELEMS * call.sample_size;
    const char *src = (const char *) call.dst;
    if (call.scatter) {          // every block straight into its own (FIFO) buffer
        for (int b = b0; b < b1; b++)
            CU(cudaMemcpyAsync(call.scatter[b], src + (size_t) b * blk_bytes, blk_bytes, cudaMemcpyDeviceToHost, s));
    } else {
        CU(cudaMemcpyAsync((char *) call.dst_host + (size_t) b0 * blk_bytes, src + (size_t) b0 * blk_bytes,
                           (size_t) (b1 - b0) * blk_bytes, cudaMemcpyDeviceToHost, s));
    }
    call.st.d2h_bytes += (int64_t) (b1 - b0) * (int64_t) blk_bytes;
    return GPSB200_OK;
}

// Commit of the scanned segments [i0, i1) as one range: resolutions up, exact run checkpoints (+ device self-check,
// which stores the end phase of the range's last block into row i0 of h_seg_end) on sp, then -- behind them on the
// caller's stream -- one synthesis launch, or with a host destination chunks each downloaded on s_copy behind it.
int seg_commit(gpsb200_ctx *ctx, Call &call, int i0, int i1, cudaStream_t sp) {
    const int b0 = call.segs[i0].first, b1 = call.segs[i1 - 1].second, nchan = call.nchan;
    const size_t off = (size_t) b0 * nchan, cnt = (size_t) (b1 - b0) * nchan;
    int64_t slow = 0;
    for (int i = i0; i < i1; i++) slow += call.slow[i];
    SynthArgs a = call_args(ctx, call, b0, b1 - b0);
    const size_t soff = (size_t) (b0 / kSpanBlocks) * nchan, scnt = (size_t) a.nspan * nchan;
    if (b0 == 0) CU(cudaEventRecord(ctx->ev[kEvCkptStart], sp));
    CU(cudaMemcpyAsync(ctx->d_span_res.get() + soff, ctx->h_span_res.get() + soff, scnt * sizeof(SpanRes),
                       cudaMemcpyHostToDevice, sp));
    call.st.h2d_bytes += (int64_t) (scnt * sizeof(SpanRes));
    if (slow > 0) {                                  // rare: block start phases of the host-resolved spans
        CU(cudaMemcpyAsync(ctx->d_carr0.get() + off, ctx->h_carr0.get() + off, cnt * sizeof(double),
                           cudaMemcpyHostToDevice, sp));
        call.st.h2d_bytes += (int64_t) (cnt * sizeof(double));
    }
    // test hook of the device self-check (gpsb200_debug_corrupt_chain mode 2): move the state that block b0 + 5's probe
    // recorded for slot 0 at the start of the middle checkpoint segment by one unit of the rounding grid (the probes
    // are complete: the host scan waited for them); k_checkpoints must notice
    const int jm = ckpt_segments(ctx->nruns) / 2;
    if (ctx->fault_inject_chain == 2 && b1 - b0 > 6 && jm >= 1) {
        double *p = ctx->d_seg.get() + (size_t) (b0 + 5) * nchan * kSegStates, h[kSegStates];
        CU(cudaMemcpyAsync(h, p, sizeof h, cudaMemcpyDeviceToHost, sp));
        CU(cudaStreamSynchronize(sp));
        h[jm - 1] += 0x1p-51;
        h[kCkptSegs - 1 + jm - 1] += 0x1p-51;
        CU(cudaMemcpyAsync(p, h, sizeof h, cudaMemcpyHostToDevice, sp));
        CU(cudaStreamSynchronize(sp));
    }
    SynthArgs ack = a;
    ack.last_end_host = ctx->h_seg_end.dev() + (size_t) i0 * nchan;
    CU(launch_checkpoints(ack, sp));
    if (b0 == 0) CU(cudaEventRecord(ctx->ev[kEvCkptEnd], sp));
    call.st.launches += 1;
    // what the chain says the device's walk of the range's last block must end on (call_verdict compares the two):
    // this extends the device self-check across pipeline-segment (and call) boundaries
    for (int c = 0; c < nchan; c++) {
        const ChainState &e = call.after[i1 - 1][c];
        const bool live = e.prn > 0 && ctx->h_bc[(size_t) (b1 - 1) * nchan + c].prn == e.prn;
        ctx->seg_expect[(size_t) i0 * nchan + c] = live ? e.phase : -1.0;       // -1: nothing to compare
    }
    call.rows = i0 + 1;
    CU(cudaEventRecord(ctx->ev_done[call.ichunk], sp));           // the synthesis waits for the checkpoints
    CU(cudaStreamWaitEvent(call.stream, ctx->ev_done[call.ichunk], 0));
    call.ichunk++;
    if (!call.host()) {
        CU(launch_synth(a, call.stream));
        call.st.launches += 1;
        return GPSB200_OK;
    }
    // the very first chunks are short, so that the download (the long pole of this path) starts early
    for (int c0 = b0, nc = 0; c0 < b1; c0 += nc, call.ichunk++) {
        nc = c0 == 0 ? 32 : (c0 == 32 ? 96 : (c0 == 128 ? 128 : kSynthChunk));
        nc = std::min(nc, b1 - c0);
        CU(launch_synth(call_args(ctx, call, c0, nc), call.stream));
        call.st.launches += 1;
        CU(cudaEventRecord(ctx->ev_done[call.ichunk], call.stream));
        CU(cudaStreamWaitEvent(ctx->s_copy, ctx->ev_done[call.ichunk], 0));
        const int rc = download(ctx, call, c0, c0 + nc, ctx->s_copy);
        if (rc) return rc;
    }
    return GPSB200_OK;
}

// End of a call's enqueued work: end event on the caller's stream, the self-check counter read back behind the
// checkpoint launches on sp; the call's device state stays resident for gpsb200_replay_device.
int call_close(gpsb200_ctx *ctx, const Call &call, cudaStream_t sp) {
    CU(cudaEventRecord(ctx->ev[kEvCallEnd], call.stream));
    CU(cudaMemcpyAsync(ctx->h_chain_errors.get(), ctx->d_chain_errors.get(), sizeof(int), cudaMemcpyDeviceToHost, sp));
    ctx->last = call_args(ctx, call, 0, call.nblk);
    ctx->have_last = true;
    return GPSB200_OK;
}

// Verdict of the device self-check (the counter read by call_close must have arrived): the per-block comparisons inside
// the checkpoint launches plus the comparisons at the end of every committed range.
int call_verdict(gpsb200_ctx *ctx, const Call &call) {
    int bad = ctx->h_chain_errors[0];
    for (int i = 0; i < call.rows; i++)
        for (int c = 0; c < call.nchan; c++) {
            const double want = ctx->seg_expect[(size_t) i * call.nchan + c];
            if (want >= 0.0 && f64_bits(want) != f64_bits(ctx->h_seg_end[(size_t) i * call.nchan + c])) ++bad;
        }
    if (bad != 0)
        return fail(ctx, GPSB200_ERR_INTERNAL, "carrier chain self-check failed on " + std::to_string(bad) + " blocks");
    return GPSB200_OK;
}

void seed_chain(std::vector<ChainState> &chain, int nchan, const int32_t *prn_in, const double *phase_in) {
    for (int c = 0; c < nchan; c++) {
        chain[c].prn = (prn_in && phase_in && prn_in[c] > 0) ? prn_in[c] : 0;
        chain[c].phase = chain[c].prn ? phase_in[c] : 0.0;
    }
}

void export_chain(const std::vector<ChainState> &chain, int nchan, int32_t *prn_out, double *phase_out) {
    for (int c = 0; c < nchan; c++) {
        if (prn_out) prn_out[c] = chain[c].prn;
        if (phase_out) phase_out[c] = chain[c].prn > 0 ? chain[c].phase : 0.0;
    }
}

// A call of one or two blocks (the reference's cadence): the host walks every NCO chain exactly (nco_exact.h) and
// hands the device ready-made run checkpoints; tables + synthesis are the only kernels. Exact by construction.
int small_call(gpsb200_ctx *ctx, Call &call, double *carr_phase_out, gpsb200_stats_t *stats) {
    const int nblk = call.nblk, nchan = call.nchan;
    cudaStream_t s = call.stream;
    double t0 = now_ms();
    int rc = prepare_blocks(ctx, call.chans, 0, nblk, nchan, call.chain);
    if (rc) return rc;
    const int nruns = ctx->nruns, run = ctx->cfg.run_samples;
    ctx->pool->run(nchan, [&](int c_lo, int c_hi) {
        for (int c = c_lo; c < c_hi; c++) {
            ChainState stc = call.chain[c];
            for (int b = 0; b < nblk; b++) {
                const BlockChanDev &p = ctx->h_bc[(size_t) b * nchan + c];
                RunCkpt *ck = ctx->h_ck.get() + (size_t) b * nruns * nchan + c;
                if (p.prn <= 0) {
                    stc.prn = 0;
                    for (int r = 0; r < nruns; r++) ck[(size_t) r * nchan] = RunCkpt{0.0, 0.0, 0u, 0u};
                    continue;
                }
                if (stc.prn != p.prn) stc.phase = p.carr_in;
                stc.prn = p.prn;
                double x = stc.phase, y = p.code0;
                int iword = p.nav0 & 0xFF, ibit = (p.nav0 >> 8) & 0xFF, icode = (p.nav0 >> 16) & 0xFF;
                const WalkConst wx = walk_const(p.c_carr), wy = walk_const(p.c_code);
                for (int r = 0; r < nruns; r++) {
                    ck[(size_t) r * nchan] = RunCkpt{x, y, (uint32_t) iword | ((uint32_t) ibit << 8) | ((uint32_t) icode << 16), 0u};
                    int64_t periods = 0, dummy = 0;
                    nco_advance<NCO_CARRIER>(x, wx, run, dummy);
                    nco_advance<NCO_CODE>(y, wy, run, periods);
                    nav_advance(iword, ibit, icode, periods);
                }
                stc.phase = x;
            }
            call.chain[c] = stc;
        }
    });
    call.st.host_chain_ms = now_ms() - t0;
    rc = upload_nav(ctx, s);
    if (rc) return rc;
    const size_t cnt = (size_t) nblk * nchan;
    CU(cudaEventRecord(ctx->ev[kEvCallStart], s));
    CU(cudaMemcpyAsync(ctx->d_bc.get(), ctx->h_bc.get(), cnt * sizeof(BlockChanDev), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(ctx->d_ck.get(), ctx->h_ck.get(), cnt * nruns * sizeof(RunCkpt), cudaMemcpyHostToDevice, s));
    const SynthArgs a = call_args(ctx, call, 0, nblk);
    CU(launch_tables(a, s));
    CU(launch_synth(a, s));
    CU(cudaEventRecord(ctx->ev[kEvCallEnd], s));
    call.st.launches = 2;
    call.st.h2d_bytes = (int64_t) (cnt * (sizeof(BlockChanDev) + nruns * sizeof(RunCkpt)));
    if (call.host()) {
        rc = download(ctx, call, 0, nblk, s);
        if (rc) return rc;
        CU(cudaStreamSynchronize(s));
    }
    ctx->have_last = false;              // nothing to replay: there were no walk kernels
    export_chain(call.chain, nchan, nullptr, carr_phase_out);
    if (stats) *stats = call.st;
    return GPSB200_OK;
}

// A one-shot call, as a pipeline of segments: the carrier-chain resolution of a segment runs on the context's
// high-priority pre-phase stream and therefore CONCURRENTLY with the synthesis kernels of earlier segments on the
// caller's stream (the walk kernels are latency bound and fit beside k_synth's CTAs) and, with a host destination, with
// the downloads of finished chunks. Only the first (short) segment's resolution is a lead-in. Without a host destination
// the results stay at call.dst and the call returns once everything is enqueued and the chain self-check has been read.
int run_pipeline(gpsb200_ctx *ctx, Call &call, double *carr_phase_out, gpsb200_stats_t *stats) {
    ctx->trace_t0 = now_ms();
    trace(ctx, "call");
    if (call.nblk <= kHostChainBlocks && !ctx->fault_inject_chain) return small_call(ctx, call, carr_phase_out, stats);
    cudaStream_t sp = ctx->s_pre;                       // stream of the pre-phase
    int rc = call_open(ctx, call);
    if (rc) return rc;
    const auto &segs = call.segs;
    const int nseg = (int) segs.size();
    if (!call.host()) {
        // Device destination (EAGER): nothing has to leave early, so everything speculative goes first -- the host
        // prepares segment after segment (guesses continue from the GUESSED end of the previous segment) while the GPU
        // already probes the earlier ones -- then the host scans the span summaries, and run checkpoints and synthesis
        // are ONE launch each over the whole call.
        std::vector<ChainState> guess = call.chain;
        for (int i = 0; i < nseg; i++) {
            // the segments' walk kernels alternate between two streams: their long tails (walk lengths differ by
            // an order of magnitude between satellites) overlap instead of adding up
            cudaStream_t sw = (i & 1) ? ctx->s_ck : sp;
            rc = seg_params(ctx, call, segs[i].first, segs[i].second, sw, &guess, nullptr);
            if (rc) return rc;
            rc = seg_probe(ctx, call, segs[i].first, segs[i].second, sw);
            if (rc) return rc;
            CU(cudaEventRecord(ctx->ev_seg[i], sw));
        }
        trace(ctx, "speculative work enqueued");
        for (int i = 0; i < nseg; i++) {
            rc = seg_scan(ctx, call, i, ctx->ev_seg[i], nullptr);
            if (rc) return rc;
        }
        CU(cudaStreamSynchronize(ctx->s_ck));           // (its last segment's event has been waited for; this orders the
        trace(ctx, "host scan done");                   //  checkpoint launch on sp behind everything on s_ck)
        rc = seg_commit(ctx, call, 0, nseg, sp);
        if (rc) return rc;
        trace(ctx, "checkpoints + synthesis enqueued");
    } else {
        // Host destination (LAZY): segment by segment from the exact chain, so that the first downloads start early
        for (int i = 0; i < nseg; i++) {
            rc = seg_params(ctx, call, segs[i].first, segs[i].second, sp, nullptr, nullptr);
            if (rc) return rc;
            rc = seg_probe(ctx, call, segs[i].first, segs[i].second, sp);
            if (rc) return rc;
            rc = seg_scan(ctx, call, i, nullptr, sp);
            if (rc) return rc;
            rc = seg_commit(ctx, call, i, i + 1, sp);
            if (rc) return rc;
        }
    }
    rc = call_close(ctx, call, sp);
    if (rc) return rc;
    export_chain(call.chain, call.nchan, nullptr, carr_phase_out);
    // the device self-check of the carrier chain is never skipped: a wrong start phase must not produce samples silently
    CU(cudaStreamSynchronize(sp));
    trace(ctx, "pre-phase stream drained (self-check read)");
    rc = call_verdict(ctx, call);
    if (rc) return rc;
    if (call.host()) {
        CU(cudaStreamSynchronize(call.stream));
        CU(cudaStreamSynchronize(ctx->s_copy));
    }
    if (stats) {
        float ms = 0;
        // per-kernel times of the FIRST segment ...
        cudaEventElapsedTime(&ms, ctx->ev[kEvProbeStart], ctx->ev[kEvProbeEnd]);
        call.st.probe_kernel_ms = ms;
        cudaEventElapsedTime(&ms, ctx->ev[kEvCkptStart], ctx->ev[kEvCkptEnd]);
        call.st.checkpoint_kernel_ms = ms;
        if (call.host()) {      // ... and the whole span of the call's stream (a device-destination call is still running)
            cudaEventElapsedTime(&ms, ctx->ev[kEvCallStart], ctx->ev[kEvCallEnd]);
            call.st.kernel_ms = ms;
        }
        *stats = call.st;
    }
    return GPSB200_OK;
}

// The three slice steps (include/gpsb200.h); the begun call lives in ctx->call between them.
int slice_prepare(gpsb200_ctx *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size, void *dst_device,
                  void *dst_host, cudaStream_t s, gpsb200_slice_link_t *link) {
    int rc = check_call(ctx, chans, nblk, nchan, sample_size, dst_device ? dst_device : dst_host);
    if (rc) return rc;
    rc = check_aligned(ctx, dst_device, "gpsb200_slice_prepare", "dst_device");
    if (rc) return rc;
    if (!dst_device) {                          // host destination only: stage in the context's own device buffer
        rc = ensure_staging(ctx, sample_size);
        if (rc) return rc;
        dst_device = ctx->d_out.get();
    }
    if (!link) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_slice_prepare: link is NULL");
    Call &call = ctx->call = Call(chans, nblk, nchan, sample_size, dst_device, dst_host, nullptr, s);
    call.active = true;
    rc = call_open(ctx, call);
    if (rc) return rc;
    memset(link, 0, sizeof *link);
    rc = seg_params(ctx, call, 0, nblk, ctx->s_pre, nullptr, link);
    if (rc) return rc;
    call.chans = nullptr;                       // the caller's records may go now
    ctx->have_last = false;
    return GPSB200_OK;
}

int slice_probe(gpsb200_ctx *ctx, const int32_t *prn_in, const double *phase_guess_in, int eager) {
    Call &call = ctx->call;
    if (!call.active || call.probed) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_slice_probe: call gpsb200_slice_prepare first");
    CU(cudaSetDevice(ctx->cfg.device));
    const double t0 = now_ms();
    finalize_guesses(ctx, 0, call.nblk, call.nchan, prn_in, phase_guess_in);
    call.st.host_chain_ms += now_ms() - t0;
    // EAGER: everything speculative at once, ONE probe and ONE chaining launch over the whole slice (no per-segment
    // tails). LAZY: only the first segment's; the others follow one by one in slice_finish.
    call.eager = eager != 0;
    const int n = call.eager ? (int) call.segs.size() : 1;
    int rc = seg_probe(ctx, call, 0, call.segs[n - 1].second, ctx->s_pre);
    if (rc) return rc;
    for (int i = 0; i < n; i++) CU(cudaEventRecord(ctx->ev_seg[i], ctx->s_pre));
    call.probed = true;
    return GPSB200_OK;
}

int slice_finish(gpsb200_ctx *ctx, const int32_t *prn_in, const double *phase_in, int32_t *prn_out, double *phase_out,
                 gpsb200_stats_t *stats, gpsb200_handoff_fn handoff, void *user) {
    Call &call = ctx->call;
    if (!call.active || !call.probed)
        return fail(ctx, GPSB200_ERR_ARG, "gpsb200_slice_finish: call gpsb200_slice_prepare and gpsb200_slice_probe first");
    CU(cudaSetDevice(ctx->cfg.device));
    const int nchan = call.nchan, nseg = (int) call.segs.size();
    cudaStream_t sk = ctx->s_ck;
    seed_chain(call.chain, nchan, prn_in, phase_in);
    std::vector<int32_t> po(nchan, 0);
    std::vector<double> xo(nchan, 0.0);
    ctx->trace_t0 = now_ms();
    trace(ctx, "slice_finish");
    int rc;
    if (call.eager) {
        // A successor waits for the outgoing state: scan EVERYTHING first (all probes were submitted up front), hand
        // the exact state on, and only then enqueue the long kernels -- a message sent behind them would wait for them.
        for (int i = 0; i < nseg; i++) {
            rc = seg_scan(ctx, call, i, ctx->ev_seg[i], sk);
            if (rc) return rc;
        }
        trace(ctx, "host scan done");
        export_chain(call.chain, nchan, po.data(), xo.data());
        if (handoff) handoff(user, po.data(), xo.data());
        trace(ctx, "handed over");
    }
    for (int i = 0; i < nseg; i++) {
        if (!call.eager) {
            // lazy: host scan of this segment as soon as ITS probes are done; checkpoints on a stream of their own
            rc = seg_scan(ctx, call, i, ctx->ev_seg[i], sk);
            if (rc) return rc;
        }
        rc = seg_commit(ctx, call, i, i + 1, sk);
        if (rc) return rc;
        if (!call.eager && i + 1 < nseg) {
            // lazy: the next segment's speculative work is submitted only now, BEHIND this segment's synthesis, from
            // guesses re-anchored on the exact state just resolved
            const int b0 = call.segs[i + 1].first, b1 = call.segs[i + 1].second;
            reanchor_guesses(ctx, b0, b1, nchan, call.chain);
            rc = seg_probe(ctx, call, b0, b1, ctx->s_pre);
            if (rc) return rc;
            CU(cudaEventRecord(ctx->ev_seg[i + 1], ctx->s_pre));
        }
    }
    if (!call.eager) {
        export_chain(call.chain, nchan, po.data(), xo.data());
        if (handoff) handoff(user, po.data(), xo.data());
    }
    rc = call_close(ctx, call, sk);
    if (rc) return rc;
    trace(ctx, "checkpoints + synthesis enqueued");
    call.active = false;
    call.finished = true;
    for (int c = 0; c < nchan; c++) {
        if (prn_out) prn_out[c] = po[c];
        if (phase_out) phase_out[c] = xo[c];
    }
    if (stats) *stats = call.st;
    return GPSB200_OK;
}

// gpsb200_synth_blocks and _scatter: staged in the context's own device buffer, downloaded to the host destination.
int synth_host(gpsb200_ctx *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size, void *dst_host,
               void *const *scatter, double *carr_phase_out, gpsb200_stats_t *stats) {
    for (int b = 0; scatter && b < nblk; b++)
        if (!scatter[b]) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_synth_blocks_scatter: NULL block destination");
    int rc = check_call(ctx, chans, nblk, nchan, sample_size, scatter ? scatter[0] : dst_host);
    if (rc) return rc;
    rc = ensure_staging(ctx, sample_size);
    if (rc) return rc;
    Call call(chans, nblk, nchan, sample_size, ctx->d_out.get(), dst_host, scatter, ctx->s_compute);
    return run_pipeline(ctx, call, carr_phase_out, stats);
}

// gpsb200_carrier_chain_device: windows of at most cfg.max_blocks, each params -> probe -> scan on the context's stream;
// the call has no destination (no carrier tables, no code walk, no checkpoints).
int carrier_chain_device(gpsb200_ctx *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, const double *phase_in,
                         double *phase_out) {
    int rc = check_entry(ctx);
    if (rc) return rc;
    cudaStream_t s = ctx->s_compute;
    Call call(chans, 0, nchan, GPSB200_SC08, nullptr, nullptr, nullptr, s);
    if (phase_in && nblk > 0)
        for (int c = 0; c < nchan; c++)
            if (chans[c].prn > 0) call.chain[c] = ChainState{chans[c].prn, phase_in[c]};
    for (int w0 = 0; w0 < nblk; w0 += ctx->cfg.max_blocks) {
        const int nw = std::min(ctx->cfg.max_blocks, nblk - w0);
        call.chans = chans + (size_t) w0 * nchan;
        call.nblk = nw;
        call.plan({std::make_pair(0, nw)});
        rc = seg_params(ctx, call, 0, nw, s, nullptr, nullptr);
        if (!rc) rc = seg_probe(ctx, call, 0, nw, s);
        if (!rc) rc = seg_scan(ctx, call, 0, nullptr, s);
        if (rc) return rc;
    }
    ctx->have_last = false;
    export_chain(call.chain, nchan, nullptr, phase_out);
    return GPSB200_OK;
}


// The acquisition search of the four entry points (acquire.cu): the standard one, and with `windows` the per-PRN Doppler
// windows starting at f_lo_prn. Everything is checked before anything is enqueued; the source is rx_source's.
int acquire(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *cfg,
            bool windows, const double *f_lo_prn, gpsb200_acq_result_t *res, uint64_t *grid, bool device,
            cudaStream_t s) {
    const char *name = windows ? "gpsb200_acquire_windows" : "gpsb200_acquire";
    if (!iq || !res) return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": NULL source or result array");
    const std::string bad = acq::check(cfg, nsamples, sample_size, windows, f_lo_prn);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": " + bad);
    const void *window;
    const int rc = rx_source(ctx, windows ? "gpsb200_acquire_windows_device" : "gpsb200_acquire_device", iq, cfg->s0,
                             acq::window_samples(cfg), sample_size, device, s, &window);
    if (rc) return rc;
    CU(acq::scratch_reserve(ctx->acq, cfg, windows, grid != nullptr));
    CU(acq::launch(ctx->acq, window, sample_size, cfg, windows ? f_lo_prn : nullptr, grid != nullptr, s));
    if (grid)
        CU(cudaMemcpy(grid, ctx->acq.d_grid.get(), (size_t) cfg->nprn * cfg->nbins * acq::kCode * sizeof(uint64_t),
                      cudaMemcpyDeviceToHost));
    memcpy(res, ctx->acq.h_res.get(), (size_t) cfg->nprn * sizeof(gpsb200_acq_result_t));
    return GPSB200_OK;
}

// The tracking of both entry points (track.cu). Everything is checked before anything is enqueued.
int track(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base, gpsb200_track_state_t *state,
          int nchan, int max_epochs, gpsb200_track_epoch_t *epochs, int32_t *nepochs, bool device, cudaStream_t s) {
    if (!iq || !epochs || !nepochs) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_track: NULL source, epochs or nepochs");
    const std::string bad = trk::check(state, nchan, max_epochs, nsamples, base, sample_size);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_track: " + bad);
    const void *src;
    const int rc = rx_source(ctx, "gpsb200_track_device", iq, 0, nsamples, sample_size, device, s, &src);
    if (rc) return rc;
    CU(rx_chips(ctx));
    CU(trk::scratch_reserve(ctx->trk, nchan, max_epochs));
    CU(trk::launch(ctx->trk, ctx->d_rx_chips.get(), src, nsamples, sample_size, base, state, nchan, max_epochs, epochs,
                   nepochs, s));
    return GPSB200_OK;
}

// The vector tracking of both entry points (vtrack.cu). Everything is checked before anything is enqueued.
int vtrack(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base,
           const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg, gpsb200_vtrack_state_t *state,
           int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *out, int32_t *nupdates,
           gpsb200_track_epoch_t *epochs, int max_epochs, int32_t *nepochs, bool device, cudaStream_t s) {
    const char *name = device ? "gpsb200_vtrack_device" : "gpsb200_vtrack";
    if (!iq || !fixes || !out || !nupdates || (epochs && !nepochs))
        return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": NULL source, fixes, out, nupdates or nepochs");
    const std::string bad = vtk::check(state, chans, cfg, max_updates, epochs != nullptr, max_epochs, nsamples, base,
                                       sample_size);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": " + bad);
    const void *src;
    const int rc = rx_source(ctx, name, iq, 0, nsamples, sample_size, device, s, &src);
    if (rc) return rc;
    CU(rx_chips(ctx));
    CU(vtk::scratch_reserve(ctx->vtk, state->nchan, max_updates, epochs ? max_epochs : 0));
    CU(vtk::launch(ctx->vtk, ctx->d_rx_chips.get(), src, nsamples, sample_size, base, chans, cfg, state, max_updates,
                   fixes, out, nupdates, epochs, max_epochs, nepochs, ctx->vtk_ctas, s));
    return GPSB200_OK;
}

// The snapshot measurement of both entry points (snapshot.cu). Everything is checked before anything is enqueued.
int snapshot_measure(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *acq,
                     const gpsb200_acq_result_t *res, const gpsb200_snapshot_config_t *cfg, gpsb200_snapshot_t *out,
                     bool device, cudaStream_t s) {
    const char *name = device ? "gpsb200_snapshot_measure_device" : "gpsb200_snapshot_measure";
    if (!iq || !out) return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": NULL source or output");
    const std::string bad = snap::check(acq, nsamples, sample_size, res, cfg);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, std::string(name) + ": " + bad);
    const void *window;
    const int rc = rx_source(ctx, name, iq, acq->s0, acq::window_samples(acq), sample_size, device, s, &window);
    if (rc) return rc;
    CU(rx_chips(ctx));
    snap::seed(acq, res, cfg, out);
    CU(snap::launch(ctx->snap, window, sample_size, acq->ms, acq->nprn, ctx->d_rx_chips.get(), cfg->iterations, out,
                    s));
    return GPSB200_OK;
}

// Collective detection of both entry points (acquire.cu, collective.cu; DESIGN §11.7): the search with its grid kept on
// the device, then the lattice scored against it. Everything is checked before anything is enqueued.
int collective(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *acq,
               const double *f_lo_prn, const gpsb200_ephemeris_t *eph, const gpsb200_coarse_config_t *ap,
               const gpsb200_collective_config_t *cfg, gpsb200_acq_result_t *res, gpsb200_acq_result_t *seed,
               gpsb200_collective_t *out, gpsb200_cd_score_t *scores, gpsb200_cd_cell_t *table, bool device,
               cudaStream_t s) {
    const char *name = device ? "gpsb200_collective_device" : "gpsb200_collective";
    const std::string at = std::string(name) + ": ";
    if (!iq || !eph || !ap || !cfg || !res || !seed || !out)
        return fail(ctx, GPSB200_ERR_ARG, at + "NULL source, ephemeris, a-priori or lattice config, results, seeds or record");
    std::string bad = acq::check(acq, nsamples, sample_size, f_lo_prn != nullptr, f_lo_prn);
    if (bad.empty()) bad = pvt::check_coarse(*ap);
    if (bad.empty()) bad = cd::check(cfg);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, at + bad);
    const void *window;
    const int rc = rx_source(ctx, name, iq, acq->s0, acq::window_samples(acq), sample_size, device, s, &window);
    if (rc) return rc;
    CU(acq::scratch_reserve(ctx->acq, acq, f_lo_prn != nullptr, true));
    CU(acq::launch(ctx->acq, window, sample_size, acq, f_lo_prn, true, s));
    memcpy(res, ctx->acq.h_res.get(), (size_t) acq->nprn * sizeof(gpsb200_acq_result_t));
    CU(cd::launch(ctx->cd, ctx->acq.d_grid.get(), ctx->acq.d_res.get(), acq, f_lo_prn, eph, ap, cfg, seed, out, scores,
                  table, s));
    return GPSB200_OK;
}

// The snapshot batch of both entry points (acquire.cu, snapshot.cu; DESIGN §11.6). Every argument of every window is
// checked before anything is enqueued. The windows then run in passes of snap::batch_pass: the search of the pass, one
// download of its results, the measurement's checks and seed on the host (snap::seed), one upload and the measurement.
// A host source goes up one window after another, packed; a device source is read in place.
int snapshot_batch(gpsb200_ctx *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *acq,
                   int nwin, const int64_t *s0, const double *f_lo, const gpsb200_snapshot_config_t *cfg,
                   gpsb200_acq_result_t *res, gpsb200_snapshot_t *out, bool device, cudaStream_t s) {
    const char *name = device ? "gpsb200_snapshot_batch_device" : "gpsb200_snapshot_batch";
    const std::string at = std::string(name) + ": ";
    if (!iq || !acq || !s0 || !cfg || !res || !out)
        return fail(ctx, GPSB200_ERR_ARG, at + "NULL source, search config, s0, snapshot config, results or output");
    if (nwin < 1) return fail(ctx, GPSB200_ERR_ARG, at + "nwin must be >= 1");
    std::string bad = snap::check_config(cfg);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, at + bad);
    gpsb200_acq_config_t one = *acq;
    for (int w = 0; w < nwin; w++) {
        one.s0 = s0[w];
        bad = acq::check(&one, nsamples, sample_size, f_lo != nullptr, f_lo ? f_lo + (size_t) w * acq->nprn : nullptr);
        if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, at + "window " + std::to_string(w) + ": " + bad);
    }
    int rc = device ? check_aligned(ctx, iq, name, "iq_device") : GPSB200_OK;
    if (!rc) rc = check_entry(ctx);
    if (rc) return rc;
    CU(rx_chips(ctx));
    const int nprn = acq->nprn, per = snap::batch_pass(acq, sample_size, nwin);
    const int64_t span = acq::window_samples(acq);
    const size_t elem = sample_size == GPSB200_SC16 ? 4 : 2;
    std::vector<int64_t> off((size_t) per);
    std::vector<double> flo(f_lo ? 0 : (size_t) per * nprn, acq->f_lo_hz);   // the standard grid: f_lo_hz every row
    for (int w0 = 0; w0 < nwin; w0 += per) {
        const int n = std::min(per, nwin - w0);
        CU(acq::batch_reserve(ctx->acq, acq, n));
        const void *src = iq;
        if (device) {
            for (int i = 0; i < n; i++) off[i] = s0[w0 + i];
        } else {
            CU(ctx->d_rx.grow((size_t) n * span * elem));
            for (int i = 0; i < n; i++) {
                off[i] = (int64_t) i * span;
                CU(cudaMemcpyAsync(ctx->d_rx.get() + (size_t) off[i] * elem,
                                   static_cast<const char *>(iq) + s0[w0 + i] * elem, (size_t) span * elem,
                                   cudaMemcpyHostToDevice, s));
            }
            src = ctx->d_rx.get();
        }
        gpsb200_acq_result_t *r = res + (size_t) w0 * nprn;
        gpsb200_snapshot_t *o = out + (size_t) w0 * nprn;
        CU(acq::launch_batch(ctx->acq, src, sample_size, acq, n, off.data(),
                             f_lo ? f_lo + (size_t) w0 * nprn : flo.data(), r, s));
        for (int i = 0; i < n; i++) {
            one.s0 = s0[w0 + i];
            bad = snap::check(&one, nsamples, sample_size, r + (size_t) i * nprn, cfg);
            if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, at + "window " + std::to_string(w0 + i) + ": " + bad);
            snap::seed(&one, r + (size_t) i * nprn, cfg, o + (size_t) i * nprn);
        }
        CU(snap::launch_batch(ctx->snap, src, sample_size, acq->ms, n, nprn, ctx->acq.d_boff.get(),
                              ctx->d_rx_chips.get(), cfg->iterations, o, s));
    }
    return GPSB200_OK;
}

// Position fixes (pvt.cu), with the stage st names (none: plain fixes). Everything is checked before anything is
// enqueued.
int pvt_fix(gpsb200_ctx *ctx, const char *fn, const gpsb200_pvt_chan_t *chans, int nchan,
            const gpsb200_track_epoch_t *epochs, const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
            gpsb200_fix_t *fixes, double *residuals, const pvt::Stage &st) {
    const std::string at = std::string(fn) + ": ";
    if (!fixes) return fail(ctx, GPSB200_ERR_ARG, at + "NULL fixes");
    const std::string bad = pvt::check(chans, nchan, epochs, nepochs, max_epochs, cfg, st);
    if (!bad.empty()) return fail(ctx, GPSB200_ERR_ARG, at + bad);
    const int rc = check_entry(ctx);
    if (rc) return rc;
    CU(pvt::run(ctx->pvt, chans, nchan, epochs, nepochs, max_epochs, cfg, fixes, residuals, st, ctx->s_compute));
    return GPSB200_OK;
}

int pvt_replay(gpsb200_ctx *ctx, cudaStream_t s) {
    if (!ctx->pvt.have_last) return fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_replay: no previous gpsb200_pvt call");
    CU(cudaSetDevice(ctx->cfg.device));
    CU(pvt::replay(ctx->pvt, s));
    return GPSB200_OK;
}

}  // namespace

extern "C" {

const char *gpsb200_version(void) { return "gpsb200 0.2 (sm_90a)"; }

int gpsb200_bind_numa(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, (int) sizeof bus, device) != cudaSuccess) {
        cudaGetLastError();
        return GPSB200_ERR_CUDA;
    }
    for (char *p = bus; *p; ++p) *p = (char) tolower((unsigned char) *p);
    int node = -1;
    if (FILE *f = fopen((std::string("/sys/bus/pci/devices/") + bus + "/numa_node").c_str(), "r")) {
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
    }
    if (node < 0) return -1;
    char list[4096] = {0};
    FILE *f = fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r");
    if (!f) return -1;
    const bool got = fgets(list, sizeof list, f) != nullptr;
    fclose(f);
    if (!got) return -1;
    cpu_set_t cur, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof cur, &cur) != 0) return -1;
    int picked = 0;
    for (const char *p = list; *p && *p != '\n';) {            // "0-31,64-95"
        char *end = nullptr;
        long a = strtol(p, &end, 10), b = a;
        if (end == p) break;
        if (*end == '-') b = strtol(end + 1, &end, 10);
        for (long c = a; c <= b && c < CPU_SETSIZE; c++)
            if (CPU_ISSET((int) c, &cur)) {
                CPU_SET((int) c, &want);
                ++picked;
            }
        p = *end == ',' ? end + 1 : end;
    }
    if (picked == 0 || sched_setaffinity(0, sizeof want, &want) != 0) return -1;
    return node;
}

const char *gpsb200_last_error(const gpsb200_ctx_t *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int gpsb200_codegen(int prn, uint8_t ca[GPSB200_CA_LEN]) { return ca_code(prn, ca) == 0 ? GPSB200_OK : GPSB200_ERR_ARG; }

double gpsb200_carrier_advance(double carr_phase, double f_carr, int64_t nsamples) {
    const double c = f_carr * (1.0 / (double) GPSB200_SAMPLERATE);
    int64_t dummy = 0;
    nco_advance<NCO_CARRIER>(carr_phase, c, nsamples, dummy);
    return carr_phase;
}

int gpsb200_carrier_probe_fixup(double start, double guess, double f_carr, int64_t nsamples, double *end_out) {
    const double c = f_carr * (1.0 / (double) GPSB200_SAMPLERATE);
    CarrierProbe p;
    carrier_probe(guess, c, nsamples, p);
    double xe = 0.0;
    const bool ok = carrier_fixup(start, c, p, xe);
    if (ok && end_out) *end_out = xe;
    return ok ? 1 : 0;
}

int gpsb200_span_chain_host(const double *f_carr, int nblk, double start_true, double start_guess, double *starts_out) {
    // Host-only model of the two-level chain for ONE span of one satellite (what k_probe + k_chain + the host scan
    // do): block probes from closed-form guesses, span_chain() for both variants, one carrier_fixup on the summary.
    if (!f_carr || nblk < 1 || !starts_out) return GPSB200_ERR_ARG;
    const double delt = 1.0 / (double) GPSB200_SAMPLERATE;
    std::vector<CarrierProbe> probes(nblk);
    std::vector<double> cc(nblk);
    std::vector<SpanBlockState> spec(nblk);
    uint64_t acc = phase_to_fix(start_guess);
    const double guess0 = fix_to_phase(acc);        // the span is chained from its first block's guess, as k_chain does
    for (int j = 0; j < nblk; j++) {
        cc[j] = f_carr[j] * delt;
        carrier_probe(fix_to_phase(acc), cc[j], GPSB200_BLOCK_SAMPLES, probes[j]);
        acc = guess_block(acc, cc[j]);
    }
    CarrierProbe sum{}, part{};
    bool ok[2];
    for (int V = 0; V < 2; V++) {
        span_chain(probes.data(), OneSatellite{cc.data()}, nblk, 1, guess0, V, part, ok[V], spec.data());
        if (V == 0) {
            sum.x_w = part.x_w;
            sum.n_w = part.n_w;
        }
        sum.x_end[V] = part.x_end[V];
        sum.m_pos[V] = ok[V] ? part.m_pos[V] : 0.0;
        sum.m_neg[V] = ok[V] ? part.m_neg[V] : 0.0;
    }
    double xe, d;
    int v;
    if (!carrier_fixup(start_true, cc[0], sum, xe, &v, &d, 1.0)) return 0;
    starts_out[0] = start_true;
    for (int j = 1; j < nblk; j++) starts_out[j] = spec[j].start[v] + d;
    starts_out[nblk] = xe;
    return 1;
}

int gpsb200_checkpoint_segments_host(double start_true, double start_guess, double f_carr, int run_samples,
                                     double *starts_out, int *nseg_out) {
    // Host-only model of ONE block of k_probe (both variants, segment-start states) and of how k_checkpoints starts
    // its segments from them
    if (!starts_out || run_samples <= 0 || GPSB200_BLOCK_SAMPLES % run_samples != 0) return GPSB200_ERR_ARG;
    const double c = f_carr * (1.0 / (double) GPSB200_SAMPLERATE);
    const int nruns = GPSB200_BLOCK_SAMPLES / run_samples, nseg = ckpt_segments(nruns);
    CarrierProbe p;
    double seg[kSegStates];
    carrier_probe_walk2(start_guess, c, GPSB200_BLOCK_SAMPLES, p, seg, nruns, run_samples);
    if (nseg_out) *nseg_out = nseg;
    starts_out[0] = start_true;
    for (int j = 1; j < kCkptSegs; j++) starts_out[j] = NAN;
    double xe, d;
    int v;
    if (!carrier_fixup(start_true, c, p, xe, &v, &d)) return 0;
    for (int j = first_derived_segment(p, nseg, nruns, run_samples); j < nseg; j++)
        starts_out[j] = seg[v * (kCkptSegs - 1) + j - 1] + d;
    return 1;
}

int gpsb200_carrier_probe_host(double guess, double f_carr, int64_t nsamples, int run_samples, int mode, void *probe_out,
                               double *seg_out) {
    if (!probe_out || nsamples < 0 || nsamples >= ((int64_t) 1 << 31) || (mode != 0 && mode != 1) || run_samples < 0 ||
        (run_samples > 0 && nsamples % run_samples != 0))
        return GPSB200_ERR_ARG;
    const double c = f_carr * (1.0 / (double) GPSB200_SAMPLERATE);
    const int nruns = run_samples > 0 ? (int) (nsamples / run_samples) : 0;
    double *seg = run_samples > 0 ? seg_out : nullptr;
    if (seg)                                 // states a walk does not record stay NaN
        for (int k = 0; k < kSegStates; k++) seg[k] = NAN;
    CarrierProbe p{};
    if (mode == 0) {
        for (int v = 0; v < 2; v++)
            carrier_probe_walk(guess, c, nsamples, v, p.n_w, p.x_w, p.x_end[v], p.m_pos[v], p.m_neg[v],
                               seg ? seg + v * (kCkptSegs - 1) : nullptr, nruns, run_samples);
    } else {
        carrier_probe_walk2(guess, c, nsamples, p, seg, nruns, run_samples);
    }
    memcpy(probe_out, &p, sizeof p);
    return GPSB200_OK;
}

int gpsb200_carrier_chain(const gpsb200_chan_t *chans, int nblk, int nchan, const double *phase_in,
                          double *phase_out, int threads) {
    if (!chans || !phase_out || nblk < 0 || nchan < 1) return GPSB200_ERR_ARG;
    const double delt = 1.0 / (double) GPSB200_SAMPLERATE;
    auto work = [&](int lo, int hi) {
        for (int c = lo; c < hi; c++) {
            int prn = 0;
            double ph = phase_in ? phase_in[c] : 0.0;
            for (int b = 0; b < nblk; b++) {
                const gpsb200_chan_t &in = chans[(size_t) b * nchan + c];
                if (in.prn <= 0) {
                    prn = 0;
                    continue;
                }
                if ((b == 0 && !phase_in) || in.prn != prn) {
                    if (!(b == 0 && phase_in)) ph = in.carr_phase;
                    prn = in.prn;
                }
                int64_t dummy = 0;
                nco_advance<NCO_CARRIER>(ph, in.f_carr * delt, GPSB200_BLOCK_SAMPLES, dummy);
            }
            phase_out[c] = prn > 0 ? ph : 0.0;
        }
    };
    threads = std::max(1, std::min(threads, nchan));
    std::vector<std::thread> th;
    const int per = (nchan + threads - 1) / threads;
    for (int t = 0; t < threads; t++) {
        const int lo = t * per, hi = std::min(nchan, lo + per);
        if (lo < hi) th.emplace_back(work, lo, hi);
    }
    for (auto &t : th) t.join();
    return GPSB200_OK;
}

int gpsb200_create(const gpsb200_config_t *cfg, gpsb200_ctx_t **out) {
    if (!cfg || !out) return GPSB200_ERR_ARG;
    gpsb200_ctx *ctx = new gpsb200_ctx();
    ctx->cfg = *cfg;
    gpsb200_config_t &c = ctx->cfg;
    if (c.run_samples == 0) c.run_samples = 2400;
    if (c.host_threads <= 0) c.host_threads = (int) std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    if (c.max_nav_frames <= 0) c.max_nav_frames = 1;
    if (c.max_chan < 1 || c.max_chan > GPSB200_MAX_CHAN || c.max_blocks < 1 || c.run_samples < 32 ||
        c.run_samples % 32 != 0 || GPSB200_BLOCK_SAMPLES % c.run_samples != 0) {
        delete ctx;
        return GPSB200_ERR_ARG;
    }
    ctx->nruns = GPSB200_BLOCK_SAMPLES / c.run_samples;
    ctx->pool.reset(new WorkerPool(std::min(c.host_threads, c.max_chan)));
    *out = ctx;   // from here on errors are reported through the context
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(ctx, GPSB200_ERR_CUDA, "no CUDA device: gpsb200 has no CPU fallback");
    CU(cudaSetDevice(c.device));
    CU(cudaStreamCreateWithFlags(&ctx->s_compute, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&ctx->s_copy, cudaStreamNonBlocking));
    {   // the pre-phase (latency-bound walk kernels, the lead-in of everything) outranks the synthesis
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU(cudaStreamCreateWithPriority(&ctx->s_pre, cudaStreamNonBlocking, hi));
        CU(cudaStreamCreateWithPriority(&ctx->s_ck, cudaStreamNonBlocking, hi));
    }
    for (auto &e : ctx->ev) CU(cudaEventCreate(&e));
    const int nchunk = (c.max_blocks + kSynthChunk - 1) / kSynthChunk + (c.max_blocks + kSegBlocks - 1) / kSegBlocks + 5;
    ctx->ev_done.resize(nchunk);
    for (auto &e : ctx->ev_done) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    const size_t max_segs = segments_of(c.max_blocks).size();     // every call's segments have their rows and events
    ctx->ev_seg.resize(max_segs);
    for (auto &e : ctx->ev_seg) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(ctx->h_seg_end.grow(max_segs * c.max_chan, cudaHostAllocMapped));
    ctx->seg_expect.assign(max_segs * c.max_chan, -1.0);
    const size_t nbc = (size_t) c.max_blocks * c.max_chan;
    CU(ctx->d_bc.grow(nbc));
    CU(ctx->h_bc.grow(nbc));
    CU(ctx->d_ck.grow(nbc * ctx->nruns));
    CU(ctx->h_ck.grow((size_t) std::min(c.max_blocks, kHostChainBlocks) * c.max_chan * ctx->nruns));
    CU(ctx->d_carr_end.grow(nbc));
    CU(ctx->d_atab.grow((size_t) c.max_blocks * kAtabRows * 32));
    CU(ctx->d_chain_errors.grow(1));
    CU(ctx->h_chain_errors.grow(1));
    CU(ctx->d_guess.grow(nbc));
    CU(ctx->h_guess.grow(nbc));
    ctx->h_guess_abs.assign(nbc, 1);
    ctx->h_span_flags.assign((size_t) ((c.max_blocks + kSpanBlocks - 1) / kSpanBlocks + 1) * c.max_chan, 0);
    CU(ctx->d_carr0.grow(nbc));
    CU(ctx->h_carr0.grow(nbc));
    // block probes: one copy in HBM (k_chain reads it), one written by the kernel straight into mapped
    // pinned host memory for the host's block-by-block fallback; span summaries only in mapped host memory
    // (a copy-engine download would queue behind the large result downloads of earlier segments)
    CU(ctx->d_probe.grow(nbc));
    CU(ctx->h_probe.grow(nbc, cudaHostAllocMapped));
    CU(ctx->d_seg.grow(nbc * kSegStates));      // only k_checkpoints reads them: HBM only
    ctx->max_spans = (c.max_blocks + kSpanBlocks - 1) / kSpanBlocks + 1;
    const size_t nsc = (size_t) ctx->max_spans * c.max_chan;
    CU(ctx->h_span_sum.grow(nsc, cudaHostAllocMapped));
    CU(ctx->d_spec.grow(nbc));
    if (const char *ev = getenv("GPSB200_TRACE")) ctx->trace_on = atoi(ev) != 0;
    if (const char *ev = getenv("GPSB200_LANES")) ctx->lanes_on = atoi(ev) != 0;
    CU(ctx->d_span_res.grow(nsc));
    CU(ctx->h_span_res.grow(nsc));
    const size_t navw = (size_t) c.max_nav_frames * c.max_chan * GPSB200_NAV_WORDS;
    CU(ctx->d_nav.grow(navw));
    CU(ctx->h_nav.grow(navw));
    memset(ctx->h_nav.get(), 0, navw * sizeof(uint32_t));
    // packed C/A chips (ca[], gps.c:2817), periodically extended so that any 32-chip window
    // starting at chip 0..1022 is two consecutive words; row = prn
    std::vector<uint32_t> chips((size_t) 33 * kChipWords, 0);
    for (int prn = 1; prn <= 32; prn++) {
        uint8_t ca[GPSB200_CA_LEN];
        ca_code(prn, ca);
        for (int n = 0; n < kChipWords * 32; n++)
            if (ca[n % GPSB200_CA_LEN]) chips[(size_t) prn * kChipWords + (n >> 5)] |= 1u << (n & 31);
    }
    CU(ctx->d_chips.grow(chips.size()));
    CU(cudaMemcpy(ctx->d_chips.get(), chips.data(), chips.size() * 4, cudaMemcpyHostToDevice));
    return GPSB200_OK;
}

void gpsb200_destroy(gpsb200_ctx_t *ctx) {
    if (!ctx) return;
    if (ctx->s_compute) cudaSetDevice(ctx->cfg.device);
    if (ctx->s_compute) cudaStreamSynchronize(ctx->s_compute);
    if (ctx->s_copy) cudaStreamSynchronize(ctx->s_copy);
    if (ctx->s_pre) cudaStreamSynchronize(ctx->s_pre);
    if (ctx->s_ck) cudaStreamSynchronize(ctx->s_ck);
    for (auto &e : ctx->ev)
        if (e) cudaEventDestroy(e);
    for (auto &e : ctx->ev_done)
        if (e) cudaEventDestroy(e);
    for (auto &e : ctx->ev_seg)
        if (e) cudaEventDestroy(e);
    if (ctx->s_compute) cudaStreamDestroy(ctx->s_compute);
    if (ctx->s_copy) cudaStreamDestroy(ctx->s_copy);
    if (ctx->s_pre) cudaStreamDestroy(ctx->s_pre);
    if (ctx->s_ck) cudaStreamDestroy(ctx->s_ck);
    delete ctx;   // frees the buffers, on the device selected above
}

int gpsb200_set_nav(gpsb200_ctx_t *ctx, int frame, int chan, const uint32_t dwrd[GPSB200_NAV_WORDS]) {
    if (!ctx || !dwrd) return GPSB200_ERR_ARG;
    if (frame < 0 || frame >= ctx->cfg.max_nav_frames || chan < 0 || chan >= ctx->cfg.max_chan)
        return fail(ctx, GPSB200_ERR_ARG, "gpsb200_set_nav: frame/channel out of range");
    memcpy(&ctx->h_nav[((size_t) frame * ctx->cfg.max_chan + chan) * GPSB200_NAV_WORDS], dwrd, GPSB200_NAV_WORDS * 4);
    ctx->nav_dirty = true;
    return GPSB200_OK;
}

int gpsb200_synth_blocks_device(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                                int sample_size, void *dst_device, void *stream_, double *carr_phase_out,
                                gpsb200_stats_t *stats) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    int rc = check_call(ctx, chans, nblk, nchan, sample_size, dst_device);
    if (!rc) rc = check_aligned(ctx, dst_device, "gpsb200_synth_blocks_device", "dst_device");
    if (!rc) {
        Call call(chans, nblk, nchan, sample_size, dst_device, nullptr, nullptr, s);
        rc = run_pipeline(ctx, call, carr_phase_out, stats);
    }
    return settle(ctx, s, rc);
}

// ---- time-slice hand-over: one call in three steps (see include/gpsb200.h) --------------------------
int gpsb200_slice_prepare(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size,
                          void *dst_device, void *dst_host, void *stream_, gpsb200_slice_link_t *link) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, slice_prepare(ctx, chans, nblk, nchan, sample_size, dst_device, dst_host, s, link));
}

int gpsb200_slice_probe(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_guess_in, int eager) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = ctx->call.active ? ctx->call.stream : nullptr;
    return settle(ctx, s, slice_probe(ctx, prn_in, phase_guess_in, eager));
}

int gpsb200_slice_finish_cb(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_in, int32_t *prn_out,
                            double *phase_out, gpsb200_stats_t *stats, gpsb200_handoff_fn handoff, void *user) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = ctx->call.active ? ctx->call.stream : nullptr;
    return settle(ctx, s, slice_finish(ctx, prn_in, phase_in, prn_out, phase_out, stats, handoff, user));
}

int gpsb200_slice_finish(gpsb200_ctx_t *ctx, const int32_t *prn_in, const double *phase_in, int32_t *prn_out,
                         double *phase_out, gpsb200_stats_t *stats) {
    return gpsb200_slice_finish_cb(ctx, prn_in, phase_in, prn_out, phase_out, stats, nullptr, nullptr);
}

int gpsb200_slice_wait(gpsb200_ctx_t *ctx) {
    if (!ctx || !ctx->s_compute) return GPSB200_ERR_ARG;
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaStreamSynchronize(ctx->s_pre));
    CU(cudaStreamSynchronize(ctx->s_ck));
    if (ctx->call.stream) CU(cudaStreamSynchronize(ctx->call.stream));
    CU(cudaStreamSynchronize(ctx->s_copy));
    if (ctx->call.finished) {
        ctx->call.finished = false;
        return call_verdict(ctx, ctx->call);
    }
    return GPSB200_OK;
}

int gpsb200_slice_link_host(const gpsb200_chan_t *chans, int nblk, int nchan, gpsb200_slice_link_t *link) {
    // the link of a slice from its parameters alone (what prepare_blocks fills in relative mode); no device involved
    if (!chans || !link || nblk < 1 || nchan < 1 || nchan > GPSB200_MAX_CHAN) return GPSB200_ERR_ARG;
    const double delt = 1.0 / (double) GPSB200_SAMPLERATE;
    memset(link, 0, sizeof *link);
    for (int c = 0; c < nchan; c++) {
        uint64_t acc = 0;
        int prev = chans[c].prn;
        bool absolute = false;
        link->prn_first[c] = prev;
        link->first_phase[c] = prev > 0 ? chans[c].carr_phase : 0.0;
        for (int b = 0; b < nblk; b++) {
            const gpsb200_chan_t &in = chans[(size_t) b * nchan + c];
            if (in.prn <= 0) {
                prev = 0;
                absolute = true;
                continue;
            }
            if (in.prn != prev) {
                acc = phase_to_fix(in.carr_phase);
                absolute = true;
            }
            prev = in.prn;
            acc = guess_block(acc, in.f_carr * delt);
        }
        link->prn_last[c] = prev > 0 ? prev : 0;
        link->reset_inside[c] = absolute ? 1 : 0;
        link->value[c] = fix_to_phase(acc);
    }
    return GPSB200_OK;
}

int gpsb200_link_apply(const gpsb200_slice_link_t *link, int nchan, const int32_t *prn_in, const double *phase_in,
                       int32_t *prn_out, double *phase_out) {
    if (!link || !prn_out || !phase_out || nchan < 1 || nchan > GPSB200_MAX_CHAN) return GPSB200_ERR_ARG;
    for (int c = 0; c < nchan; c++) {
        if (link->prn_last[c] <= 0) {
            prn_out[c] = 0;
            phase_out[c] = 0.0;
            continue;
        }
        double ph = link->value[c];
        if (!link->reset_inside[c]) {
            const bool cont = prn_in && phase_in && prn_in[c] > 0 && prn_in[c] == link->prn_first[c];
            ph += cont ? phase_in[c] : link->first_phase[c];
            if (ph >= 1.0) ph -= 1.0;
        }
        prn_out[c] = link->prn_last[c];
        phase_out[c] = (ph >= 0.0 && ph < 1.0) ? ph : 0.0;
    }
    return GPSB200_OK;
}

const char *gpsb200_synth_kernel_name(const gpsb200_ctx_t *ctx, int nchan) {
    if (!ctx) return "";
    SynthArgs a{};
    a.nchan = nchan;
    a.run_samples = ctx->cfg.run_samples;
    a.lanes = ctx->lanes_on && !ctx->lanes_veto ? 1 : 0;
    return synth_lanes_applicable(a) ? "k_synth_lanes" : "k_synth";
}

int gpsb200_debug_corrupt_chain(gpsb200_ctx_t *ctx, int on) {
    if (!ctx || on < 0 || on > 2) return GPSB200_ERR_ARG;
    ctx->fault_inject_chain = on;
    return GPSB200_OK;
}

int gpsb200_debug_run_checkpoints(gpsb200_ctx_t *ctx, int nblk, int nchan, void *out) {
    if (!ctx || !out || nblk < 1 || nblk > ctx->cfg.max_blocks || nchan < 1 || nchan > ctx->cfg.max_chan)
        return GPSB200_ERR_ARG;
    if (!ctx->s_compute) return fail(ctx, GPSB200_ERR_CUDA, "context has no CUDA device");
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaDeviceSynchronize());             // the call's streams may be the caller's
    CU(cudaMemcpy(out, ctx->d_ck.get(), (size_t) nblk * ctx->nruns * nchan * sizeof(RunCkpt), cudaMemcpyDeviceToHost));
    return GPSB200_OK;
}

int gpsb200_debug_block_probes(gpsb200_ctx_t *ctx, int nblk, int nchan, void *probes_out, double *seg_out,
                               double *guess_out) {
    if (!ctx || !probes_out || nblk < 1 || nblk > ctx->cfg.max_blocks || nchan < 1 || nchan > ctx->cfg.max_chan)
        return GPSB200_ERR_ARG;
    if (!ctx->s_compute) return fail(ctx, GPSB200_ERR_CUDA, "context has no CUDA device");
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaDeviceSynchronize());             // the call's streams may be the caller's
    const size_t cnt = (size_t) nblk * nchan;
    CU(cudaMemcpy(probes_out, ctx->d_probe.get(), cnt * sizeof(CarrierProbe), cudaMemcpyDeviceToHost));
    if (seg_out) CU(cudaMemcpy(seg_out, ctx->d_seg.get(), cnt * kSegStates * sizeof(double), cudaMemcpyDeviceToHost));
    if (guess_out) CU(cudaMemcpy(guess_out, ctx->d_guess.get(), cnt * sizeof(double), cudaMemcpyDeviceToHost));
    return GPSB200_OK;
}

int gpsb200_debug_synth_shape(gpsb200_ctx_t *ctx, int nblk, int nchan, int sample_size, const char **kernel,
                              int *ctas_per_block, int *runs_per_cta) {
    if (!ctx || !kernel || !ctas_per_block || !runs_per_cta || nblk < 1 || nchan < 1 || nchan > ctx->cfg.max_chan ||
        (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16))
        return GPSB200_ERR_ARG;
    if (!ctx->s_compute) return fail(ctx, GPSB200_ERR_CUDA, "context has no CUDA device");
    CU(cudaSetDevice(ctx->cfg.device));      // the shape depends on the SM count of the context's device
    const SynthArgs a = make_args(ctx, 0, nblk, nchan, sample_size, nullptr);   // the arguments of such a launch
    int ctas = 0, threads = 0;
    size_t smem = 0;
    synth_launch_shape(a, &ctas, &threads, &smem, ctas_per_block, runs_per_cta);
    *kernel = synth_lanes_applicable(a) ? "k_synth_lanes" : "k_synth";
    return GPSB200_OK;
}

int gpsb200_carrier_chain_device(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan,
                                 const double *phase_in, double *phase_out) {
    if (!ctx || !chans || !phase_out || nblk < 0 || nchan < 1 || nchan > ctx->cfg.max_chan) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, carrier_chain_device(ctx, chans, nblk, nchan, phase_in, phase_out));
}

int gpsb200_replay_device(gpsb200_ctx_t *ctx, void *dst_device, void *stream_, int kernel_mask) {
    if (!ctx || !ctx->have_last) return GPSB200_ERR_ARG;
    const int rc = check_aligned(ctx, dst_device, "gpsb200_replay_device", "dst_device");
    if (rc) return rc;
    CU(cudaSetDevice(ctx->cfg.device));
    cudaStream_t s = caller_stream(ctx, stream_);
    SynthArgs a = ctx->last;
    if (dst_device) a.out = dst_device;
    if (kernel_mask & 8) CU(launch_tables(a, s));
    if (kernel_mask & 4) {
        CU(launch_probe(a, s));
        CU(launch_chain(a, s));
    }
    if (kernel_mask & 1) CU(launch_checkpoints(a, s));
    if (kernel_mask & 2) CU(launch_synth(a, s));
    return GPSB200_OK;
}

int gpsb200_synth_blocks_scatter(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size,
                                 void *const *dst_blocks, double *carr_phase_out, gpsb200_stats_t *stats) {
    if (!ctx || !dst_blocks) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, synth_host(ctx, chans, nblk, nchan, sample_size, nullptr, dst_blocks, carr_phase_out, stats));
}

int gpsb200_synth_blocks(gpsb200_ctx_t *ctx, const gpsb200_chan_t *chans, int nblk, int nchan, int sample_size,
                         void *dst, double *carr_phase_out, gpsb200_stats_t *stats) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, synth_host(ctx, chans, nblk, nchan, sample_size, dst, nullptr, carr_phase_out, stats));
}

int gpsb200_acquire(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, const gpsb200_acq_config_t *cfg,
                    gpsb200_acq_result_t *res, uint64_t *grid) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, acquire(ctx, iq, nsamples, sample_size, cfg, false, nullptr, res, grid, false,
                                        ctx->s_compute));
}

int gpsb200_acquire_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                           const gpsb200_acq_config_t *cfg, gpsb200_acq_result_t *res, uint64_t *grid, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, acquire(ctx, iq_device, nsamples, sample_size, cfg, false, nullptr, res, grid, true, s));
}

int gpsb200_acquire_windows(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                            const gpsb200_acq_config_t *cfg, const double *f_lo_prn, gpsb200_acq_result_t *res,
                            uint64_t *grid) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, acquire(ctx, iq, nsamples, sample_size, cfg, true, f_lo_prn, res, grid, false,
                                        ctx->s_compute));
}

int gpsb200_acquire_windows_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                   const gpsb200_acq_config_t *cfg, const double *f_lo_prn, gpsb200_acq_result_t *res,
                                   uint64_t *grid, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, acquire(ctx, iq_device, nsamples, sample_size, cfg, true, f_lo_prn, res, grid, true, s));
}

int gpsb200_debug_acq_split(gpsb200_ctx_t *ctx, int force, int nprn, int nbins) {
    if (!ctx || !(force == -1 || force == 0 || acq::split_allowed(force)) || nprn < 1 || nprn > 32 || nbins < 1 ||
        nbins > GPSB200_ACQ_MAX_BINS)
        return GPSB200_ERR_ARG;
    if (force >= 0) ctx->acq.force_split = force;
    if (!ctx->acq.sms) {
        if (!ctx->s_compute) return fail(ctx, GPSB200_ERR_CUDA, "context has no CUDA device");
        CU(cudaDeviceGetAttribute(&ctx->acq.sms, cudaDevAttrMultiProcessorCount, ctx->cfg.device));
    }
    return acq::split_of(ctx->acq, nprn, nbins);
}

int gpsb200_track_start(int prn, double doppler_hz, int64_t sample, gpsb200_track_state_t *st) {
    if (!st || prn < 1 || prn > 32 || !(std::fabs(doppler_hz) <= 10000.0) || sample < 0) return GPSB200_ERR_ARG;
    memset(st, 0, sizeof *st);
    st->prn = prn;
    st->sample = sample;
    trk::start_steps(doppler_hz, st->carr_step, st->code_step);
    st->carr_freq = (int64_t) st->carr_step * 1024;
    return GPSB200_OK;
}

int gpsb200_track(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base,
                  gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                  int32_t *nepochs) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, track(ctx, iq, nsamples, sample_size, base, state, nchan, max_epochs, epochs, nepochs,
                                      false, ctx->s_compute));
}

int gpsb200_track_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size, int64_t base,
                         gpsb200_track_state_t *state, int nchan, int max_epochs, gpsb200_track_epoch_t *epochs,
                         int32_t *nepochs, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, track(ctx, iq_device, nsamples, sample_size, base, state, nchan, max_epochs, epochs, nepochs,
                                true, s));
}

void gpsb200_vtrack_config_default(gpsb200_vtrack_config_t *cfg) {
    if (!cfg) return;
    memset(cfg, 0, sizeof *cfg);
    cfg->periods = 20;
    cfg->sigma_code_m = 50.0;
    cfg->sigma_rate_mps = 10.0;
    cfg->q_min = 1.2;
    cfg->accel_psd = 1.0;
    cfg->bias_psd = 0.1;
    cfg->drift_psd = 0.01;
    cfg->sigma_pos = 100.0;
    cfg->sigma_vel = 1.0;
    cfg->sigma_bias = 10.0;
    cfg->sigma_drift = 1.0;
}

int gpsb200_vtrack_seed(const gpsb200_vtrack_config_t *cfg, const double *x8, double t_rx, int64_t s0,
                        const int32_t *prn, int nchan, gpsb200_vtrack_state_t *st) {
    if (!x8 || !prn || !st || nchan < 1 || nchan > GPSB200_TRK_MAX_CHAN || s0 < 0 || !(t_rx >= 0.0 && t_rx < 604800.0))
        return GPSB200_ERR_ARG;
    if (!vtk::check_config(cfg).empty()) return GPSB200_ERR_ARG;
    for (int i = 0; i < 8; i++)
        if (!std::isfinite(x8[i])) return GPSB200_ERR_ARG;
    uint32_t seen = 0;
    for (int c = 0; c < nchan; c++) {
        if (prn[c] < 1 || prn[c] > 32 || (seen >> (prn[c] - 1) & 1u)) return GPSB200_ERR_ARG;
        seen |= 1u << (prn[c] - 1);
    }
    memset(st, 0, sizeof *st);
    st->s0 = s0;
    st->t_f = s0;
    st->nchan = nchan;
    st->t0 = t_rx + x8[6] / 2.99792458e8;
    for (int i = 0; i < 8; i++) st->x[i] = x8[i];
    const double sd[8] = {cfg->sigma_pos, cfg->sigma_pos, cfg->sigma_pos, cfg->sigma_vel,
                          cfg->sigma_vel, cfg->sigma_vel, cfg->sigma_bias, cfg->sigma_drift};
    for (int i = 0; i < 8; i++) st->P[i * 9] = sd[i] * sd[i];
    for (int c = 0; c < nchan; c++) st->ch[c].nco.prn = prn[c];
    return GPSB200_OK;
}

int gpsb200_vtrack(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size, int64_t base,
                   const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg, gpsb200_vtrack_state_t *state,
                   int max_updates, gpsb200_fix_t *fixes, gpsb200_vtrack_chan_t *out, int32_t *nupdates,
                   gpsb200_track_epoch_t *epochs, int max_epochs, int32_t *nepochs) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, vtrack(ctx, iq, nsamples, sample_size, base, chans, cfg, state, max_updates, fixes, out,
                                       nupdates, epochs, max_epochs, nepochs, false, ctx->s_compute));
}

int gpsb200_vtrack_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size, int64_t base,
                          const gpsb200_pvt_chan_t *chans, const gpsb200_vtrack_config_t *cfg,
                          gpsb200_vtrack_state_t *state, int max_updates, gpsb200_fix_t *fixes,
                          gpsb200_vtrack_chan_t *out, int32_t *nupdates, gpsb200_track_epoch_t *epochs, int max_epochs,
                          int32_t *nepochs, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, vtrack(ctx, iq_device, nsamples, sample_size, base, chans, cfg, state, max_updates, fixes, out,
                                 nupdates, epochs, max_epochs, nepochs, true, s));
}

int gpsb200_debug_vtrack_cluster(gpsb200_ctx_t *ctx, int ctas) {
    if (!ctx || ctas < 0 || ctas > vtk::kMaxCluster) return GPSB200_ERR_ARG;
    ctx->vtk_ctas = ctas;
    return GPSB200_OK;
}

int gpsb200_pvt(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg, gpsb200_fix_t *fixes,
                double *residuals) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt", chans, nchan, epochs, nepochs, max_epochs, cfg, fixes,
                                        residuals, pvt::Stage()));
}

int gpsb200_pvt_raim(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                     const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
                     const gpsb200_raim_config_t *raim, gpsb200_fix_t *fixes, double *residuals, gpsb200_raim_t *out) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!raim || !out) return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_raim: NULL raim or out"));
    pvt::Stage st;
    st.raim = raim;
    st.raim_out = out;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_raim", chans, nchan, epochs, nepochs, max_epochs, cfg, fixes,
                                        residuals, st));
}

int gpsb200_pvt_araim(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_track_epoch_t *epochs,
                      const int32_t *nepochs, int max_epochs, const gpsb200_pvt_config_t *cfg,
                      const gpsb200_araim_config_t *araim, gpsb200_fix_t *fixes, double *residuals,
                      gpsb200_araim_t *out) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!araim || !out) return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_araim: NULL araim or out"));
    pvt::Stage st;
    st.araim = araim;
    st.araim_out = out;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_araim", chans, nchan, epochs, nepochs, max_epochs, cfg, fixes,
                                        residuals, st));
}

int gpsb200_pvt_coarse(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                       const gpsb200_track_epoch_t *epochs, const int32_t *nepochs, int max_epochs,
                       const gpsb200_pvt_config_t *cfg, const gpsb200_coarse_config_t *apriori, gpsb200_fix_t *fixes,
                       double *residuals, gpsb200_coarse_t *out, int64_t *ms) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!apriori || !out)
        return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_coarse: NULL apriori or out"));
    pvt::Stage st;
    st.coarse = apriori;
    st.coarse_out = out;
    st.ms = ms;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_coarse", chans, nchan, epochs, nepochs, max_epochs, cfg, fixes,
                                        residuals, st));
}

int gpsb200_pvt_search(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                       const gpsb200_track_epoch_t *epochs, const int32_t *nepochs, int max_epochs,
                       const gpsb200_pvt_config_t *cfg, const gpsb200_search_config_t *search, gpsb200_fix_t *fixes,
                       double *residuals, gpsb200_search_t *out, int64_t *ms, double *node_rms) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!search || !out)
        return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_search: NULL search or out"));
    pvt::Stage st;
    st.search = search;
    st.search_out = out;
    st.ms = ms;
    st.node_rms = node_rms;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_search", chans, nchan, epochs, nepochs, max_epochs, cfg, fixes,
                                        residuals, st));
}

int gpsb200_snapshot_measure(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                             const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res,
                             const gpsb200_snapshot_config_t *cfg, gpsb200_snapshot_t *out) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, snapshot_measure(ctx, iq, nsamples, sample_size, acq, res, cfg, out, false,
                                                 ctx->s_compute));
}

int gpsb200_snapshot_measure_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                    const gpsb200_acq_config_t *acq, const gpsb200_acq_result_t *res,
                                    const gpsb200_snapshot_config_t *cfg, gpsb200_snapshot_t *out, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, snapshot_measure(ctx, iq_device, nsamples, sample_size, acq, res, cfg, out, true, s));
}

int gpsb200_snapshot_batch(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                           const gpsb200_acq_config_t *acq, int nwin, const int64_t *s0, const double *f_lo,
                           const gpsb200_snapshot_config_t *cfg, gpsb200_acq_result_t *res, gpsb200_snapshot_t *out) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, snapshot_batch(ctx, iq, nsamples, sample_size, acq, nwin, s0, f_lo, cfg, res, out, false,
                                               ctx->s_compute));
}

int gpsb200_snapshot_batch_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                                  const gpsb200_acq_config_t *acq, int nwin, const int64_t *s0, const double *f_lo,
                                  const gpsb200_snapshot_config_t *cfg, gpsb200_acq_result_t *res,
                                  gpsb200_snapshot_t *out, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, snapshot_batch(ctx, iq_device, nsamples, sample_size, acq, nwin, s0, f_lo, cfg, res, out, true,
                                         s));
}

int gpsb200_collective(gpsb200_ctx_t *ctx, const void *iq, int64_t nsamples, int sample_size,
                       const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                       const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                       gpsb200_acq_result_t *res, gpsb200_acq_result_t *seed, gpsb200_collective_t *out,
                       gpsb200_cd_score_t *scores, gpsb200_cd_cell_t *table) {
    if (!ctx) return GPSB200_ERR_ARG;
    return settle(ctx, nullptr, collective(ctx, iq, nsamples, sample_size, acq, f_lo_prn, eph, ap, cfg, res, seed, out,
                                           scores, table, false, ctx->s_compute));
}

int gpsb200_collective_device(gpsb200_ctx_t *ctx, const void *iq_device, int64_t nsamples, int sample_size,
                              const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                              const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                              gpsb200_acq_result_t *res, gpsb200_acq_result_t *seed, gpsb200_collective_t *out,
                              gpsb200_cd_score_t *scores, gpsb200_cd_cell_t *table, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, collective(ctx, iq_device, nsamples, sample_size, acq, f_lo_prn, eph, ap, cfg, res, seed, out,
                                     scores, table, true, s));
}

int gpsb200_pvt_snapshot(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan, const gpsb200_snapshot_t *meas,
                         const gpsb200_pvt_config_t *cfg, const gpsb200_coarse_config_t *apriori, gpsb200_fix_t *fixes,
                         double *residuals, gpsb200_coarse_t *out, int64_t *ms) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!apriori || !out || !meas)
        return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_snapshot: NULL meas, apriori or out"));
    pvt::Stage st;
    st.coarse = apriori;
    st.coarse_out = out;
    st.ms = ms;
    st.meas = meas;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_snapshot", chans, nchan, nullptr, nullptr, 1, cfg, fixes,
                                        residuals, st));
}

int gpsb200_pvt_snapshot_search(gpsb200_ctx_t *ctx, const gpsb200_pvt_chan_t *chans, int nchan,
                                const gpsb200_snapshot_t *meas, const gpsb200_pvt_config_t *cfg,
                                const gpsb200_search_config_t *search, gpsb200_fix_t *fixes, double *residuals,
                                gpsb200_search_t *out, int64_t *ms, double *node_rms) {
    if (!ctx) return GPSB200_ERR_ARG;
    if (!search || !out || !meas)
        return settle(ctx, nullptr, fail(ctx, GPSB200_ERR_ARG, "gpsb200_pvt_snapshot_search: NULL meas, search or out"));
    pvt::Stage st;
    st.search = search;
    st.search_out = out;
    st.ms = ms;
    st.node_rms = node_rms;
    st.meas = meas;
    return settle(ctx, nullptr, pvt_fix(ctx, "gpsb200_pvt_snapshot_search", chans, nchan, nullptr, nullptr, 1, cfg, fixes,
                                        residuals, st));
}

int gpsb200_search_nodes(int n, double *xyz) {
    if (!xyz || n < GPSB200_SEARCH_MIN_NODES || n > GPSB200_SEARCH_MAX_NODES) return GPSB200_ERR_ARG;
    pvt::search_nodes(n, xyz);
    return GPSB200_OK;
}

int gpsb200_araim_kfa(double p_fa_vert, double p_fa_horz, double *kfa_h, double *kfa_v) {
    if (!kfa_h || !kfa_v) return GPSB200_ERR_ARG;
    return pvt::araim_kfa(p_fa_vert, p_fa_horz, kfa_h, kfa_v) ? GPSB200_OK : GPSB200_ERR_ARG;
}

int gpsb200_raim_thresholds(double p_fa, double p_md, double *T, double *lambda) {
    if (!T || !lambda) return GPSB200_ERR_ARG;
    return pvt::raim_thresholds(p_fa, p_md, T, lambda) ? GPSB200_OK : GPSB200_ERR_ARG;
}

int gpsb200_pvt_replay(gpsb200_ctx_t *ctx, void *stream_) {
    if (!ctx) return GPSB200_ERR_ARG;
    cudaStream_t s = caller_stream(ctx, stream_);
    return settle(ctx, s, pvt_replay(ctx, s));
}

}  // extern "C"
