// k_synth_lanes: the per-sample synthesis (gps.c:2767-2857) with LANE = SAMPLE.
//
// k_synth (synth_kernels.cu) puts the channels on the lanes and pays a warp reduction per sample (and FP64 additions for
// both NCOs of every channel-sample); with 12 channels a quarter of its lanes idle and the reduction is a shuffle
// butterfly. Here a lane owns three samples of a 96-sample window and loops over the channels of the call, accumulating
// in registers: integer work only, proportional to the channel count.
// What makes that possible is synth_lanes.h: from the exact run anchors of k_checkpoints both NCO phases of any sample are
// integer arithmetic on certified fixed-point linear phases; the rare samples a band test cannot certify are repaired
// from the exact FP64 walk of nco_exact.h. The algorithm is the one the host model (lanes_model.cpp) runs against the
// oracle in the CPU tests; this file only distributes it over a warp:
//
//   channel side  up to 16 channels: lane = (half h, channel c), state of channel c at window w + h of the warp's run,
//                 every trip produces the chip-sign words and the 32-bit phase base of TWO windows into shared memory;
//                 17..32 channels: lane = channel, one window per trip
//   sample side   lane i: samples i, 32 + i, 64 + i of each window of the trip: per channel one broadcast read of the
//                 window record, three table look-ups at the unsigned phase (32 consecutive samples per look-up: at
//                 most 27 entries at 5 kHz, in distinct banks or broadcast), the chip x data-bit sign applied after
//                 the look-up through a second, predicated accumulator
//   output        quantise + pack (gps.c:2833-2845), staged per warp, written with 16-byte stores
#include <cuda_runtime.h>
#include <stdint.h>

#include "nco_exact.h"
#include "synth_kernels.h"
#include "synth_lanes.h"

namespace gpsb200 {

namespace {

// 16 warps per CTA, 2 CTAs per SM at 64 registers. Fewer resident warps with the registers to hold all of the window
// state (1 CTA of 16, 20 or 24 warps at 93 / 93 / 80 registers, no spills on the common path) measured slower: the
// kernel is bound by integer issue and needs the warps more than it loses to the spills.
constexpr int kLaneWarps = 16;
constexpr int kLaneCtas = 2;
constexpr int kLaneChipWords = 36;      // 1023 chips periodically extended to 1152 bits (window_signs reads word j0/32 + 2)

struct LaneWin {
    uint32_t s0, s1, s2;                // sign words of samples 0..31, 32..63, 64..95 (bit lanes::sign_pos(i): sample 32 j + i)
    uint32_t base;                      // 32-bit carrier phase of sample 0, biased by -1 (fast_base)
};

// The per-(block, channel) constants of the channel side's window state (lanes::init_steps). They are read from shared
// memory at every trip rather than kept in registers across the sample side.
struct LaneSteps {
    uint64_t D96, E96;
    uint32_t inv32, e22;
};

// CH = channel capacity of the variant (16 or 32). The channel side uses all 32 lanes: with CH = 16 the two half-warps
// prepare two consecutive windows per trip, with CH = 32 the warp prepares one.
// The carrier tables ([channel][k]: I + (Q << 16), gain-scaled, gps.c:2781-2782; 2 KB per channel) sit in front of this
// struct at the start of the dynamic shared memory. The look-ups address an entry as slot * 4 + table base (table_at),
// which needs no alignment of the base, so the layout has no alignment slack and the kernel no rounded-up base to
// rebuild or keep. Entry k of
// channel c is stored at (k + swz(c)) mod 512 (swz(c) = c * 32 / CH): the transposing fill from k_tables' [k][channel]
// layout is then free of bank conflicts, and the look-ups take the rotation from the phase itself: the channel side adds
// swz(c) << 23 to the window's phase base, so that the top 9 bits of a sample's phase are its stored slot. Channel c's
// table base is then a compile-time offset from the loop's base in the unrolled channel loop.
template <int CH>
struct LanesSmem {
    static constexpr int kWins = 32 / CH;
    uint32_t chips[CH][kLaneChipWords];                 // packed C/A chips, bit n = ca[n mod 1023]
    uint32_t nav[CH][kNavWords];                        // NAV words of this block's frame
    alignas(16) LaneWin win[kLaneWarps][kWins][CH];     // per warp: the window(s) in flight
    alignas(16) uint32_t step[CH];                      // 32-bit carrier increment per sample (fast_step)
    LaneSteps steps[CH];
    alignas(16) uint32_t stage[kLaneWarps][kWins * lanes::kWindow];   // packed output of the window(s)
    uint32_t band[CH][lanes::kBandList + 1];            // band_residues() of each channel's step; rows skewed by one bank
};
template <int CH>
constexpr size_t lanes_smem_bytes() { return sizeof(LanesSmem<CH>) + (size_t) CH * 2048; }

// Entry of the carrier table at byte address ta + OFF for the 32-bit phase p: the stored slot is p >> 23,
// its address slot * 4 + ta. Written as a shift and a multiply-add so that the address takes one ALU and one FMA-pipe
// instruction: the shift-and-mask form ((p >> 21) & 0x7FC) | ta puts both on the integer ALU pipe, which the sign tests
// and sums of the loop already keep close to saturation.
template <int OFF>
__device__ __forceinline__ int table_at(uint32_t p, uint32_t ta) {
    int e;
    asm volatile("{\n\t.reg .b32 i, ad;\n\tshr.b32 i, %1, 23;\n\tmad.lo.u32 ad, i, 4, %2;\n\tld.shared.b32 %0, [ad+%3];\n\t}"
                 : "=r"(e)
                 : "r"(p), "r"(ta), "n"(OFF));
    return e;
}

// The rare paths that walk from the exact run anchor (nco_exact.h), out of line: inlined, their FP64 walks raise the
// register pressure of the whole run loop, and at 64 registers more of the window state is then kept in local memory on
// the common path as well.
template <class ChipFn, class NavFn>
__device__ __noinline__ uint3 exact_signs_call(lanes::Anchor an, int w, ChipFn chips, NavFn nav) {
    uint32_t W[3];
    lanes::exact_signs(an, w, chips, nav, W);
    return make_uint3(W[0], W[1], W[2]);
}

// Certain carrier table index of sample n of window w of the run.
__device__ __noinline__ int exact_index_call(lanes::Anchor an, int w, int n) {
    // linear carrier phase at the window start, as init_run() + advance_window() make it (sums modulo 2^64: exact)
    const uint64_t D = lanes::carr_step_fix(an.c);
    const uint64_t P = lanes::carr_fix(an.x0) + (uint64_t) w * ((uint64_t) lanes::kWindow * D);
    return lanes::exact_index(P, D, an, w, n);
}

// acc += e if (w & bit) != 0, as one logic instruction that sets a predicate and one predicated add: written as C++ the
// compiler selects (SEL) and then adds, one instruction more per channel-sample.
__device__ __forceinline__ void add_if(int &acc, uint32_t w, uint32_t bit, int e) {
    asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tand.b32 t, %1, %2;\n\tsetp.ne.u32 p, t, 0;\n\t@p add.s32 %0, %0, %3;\n\t}"
        : "+r"(acc)
        : "r"(w), "r"(bit), "r"(e));
}

// The sums over the channels of one window for this lane's samples n0, n0 + 32, n0 + 64. NC > 0: the call has NC
// channels, known at compile time (the full-capacity case), so the loop has a fixed trip count and no remainder; NC = 0:
// nchan channels. all_j: every channel's entry at the unsigned phase; neg_j: those of the channels whose chip x data bit
// is negative. The sample is all_j - 2 neg_j: table[k ^ 256] = -table[k] entry by entry, and the packed I + (Q << 16)
// sums are linear modulo 2^32. Two channels per trip (an odd count is padded with the next slot, which is all zeros).
template <int NC>
__device__ __forceinline__ void window_sums(const LaneWin *wp, const uint32_t *sp, uint32_t ta, int nchan, uint32_t n0,
                                            uint32_t sbit, int accs[3]) {
    const int nc = NC > 0 ? NC : nchan;
    const uint32_t n1 = n0 + 32u, n2 = n0 + 64u;
    int all0 = 0, all1 = 0, all2 = 0, neg0 = 0, neg1 = 0, neg2 = 0;
#pragma unroll 4
    for (int c = 0; c < nc; c += 2, wp += 2, sp += 2, ta += 2 * 2048u) {     // table of channel c; c + 1 at + 2048
        const uint4 wa = *reinterpret_cast<const uint4 *>(&wp[0]);           // broadcast
        const uint4 wb = *reinterpret_cast<const uint4 *>(&wp[1]);
        const uint2 st = *reinterpret_cast<const uint2 *>(sp);
        const uint32_t a0 = wa.w + n0 * st.x, a1 = wa.w + n1 * st.x, a2 = wa.w + n2 * st.x;
        const uint32_t b0 = wb.w + n0 * st.y, b1 = wb.w + n1 * st.y, b2 = wb.w + n2 * st.y;
        const int ea0 = table_at<0>(a0, ta), eb0 = table_at<2048>(b0, ta);
        const int ea1 = table_at<0>(a1, ta), eb1 = table_at<2048>(b1, ta);
        const int ea2 = table_at<0>(a2, ta), eb2 = table_at<2048>(b2, ta);
        all0 += ea0 + eb0;
        all1 += ea1 + eb1;
        all2 += ea2 + eb2;
        add_if(neg0, wa.x, sbit, ea0);
        add_if(neg0, wb.x, sbit, eb0);
        add_if(neg1, wa.y, sbit, ea1);
        add_if(neg1, wb.y, sbit, eb1);
        add_if(neg2, wa.z, sbit, ea2);
        add_if(neg2, wb.z, sbit, eb2);
    }
    accs[0] = (int) ((uint32_t) all0 - 2u * (uint32_t) neg0);
    accs[1] = (int) ((uint32_t) all1 - 2u * (uint32_t) neg1);
    accs[2] = (int) ((uint32_t) all2 - 2u * (uint32_t) neg2);
}

template <bool IQ16, int CH>
__global__ void __launch_bounds__(kLaneWarps * 32, kLaneCtas) k_synth_lanes(SynthArgs a) {
    constexpr int WINS = 32 / CH;                     // windows per trip
    constexpr int SWZ = 32 / CH;                      // swz(c) = c * SWZ
    constexpr int BYTES = IQ16 ? 4 : 2;               // output bytes per sample
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int32_t *tab = reinterpret_cast<int32_t *>(smem_raw);                                            // [channel][512]
    LanesSmem<CH> &sm = *reinterpret_cast<LanesSmem<CH> *>(smem_raw + CH * 2048);
    // 32-bit shared address of the tables, for the look-ups' address arithmetic (table_at)
    const uint32_t tab_base = (uint32_t) __cvta_generic_to_shared(smem_raw);
    constexpr uint32_t kFull = 0xFFFFFFFFu;

    const int b = blockIdx.x / a.ctas_per_block;
    const int g = blockIdx.x - b * a.ctas_per_block;
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int nchan = a.nchan;
    const BlockChanDev *bc = a.bc + (size_t) b * nchan;

    // ---- per-CTA tables ----------------------------------------------------------------------------------
    {
        const int32_t *src = a.atab + (size_t) b * kAtabRows * 32;             // [k][lane], column c = channel c
        for (int i = tid; i < 512 * CH; i += nthr) {
            const int k = i / CH, c = i - k * CH;
            tab[c * 512 + ((k + c * SWZ) & 511)] = c < nchan ? src[k * 32 + c] : 0;
        }
        for (int i = tid; i < CH * kLaneChipWords; i += nthr) {
            const int c = i / kLaneChipWords, w = i - c * kLaneChipWords;
            uint32_t v = 0;
            if (c < nchan && bc[c].prn > 0) {
                const uint32_t *cw = a.chipbits + bc[c].prn * kChipWords;        // 33 words: bits 0 .. 1055
                // bit n of the extension = bit n - 1023 = bit 32 (w - 32) + i + 1 of the stream
                v = w < kChipWords ? cw[w] : __funnelshift_r(cw[w - 32], cw[w - 31], 1);
            }
            sm.chips[c][w] = v;
        }
        for (int i = tid; i < CH * kNavWords; i += nthr) {
            const int c = i / kNavWords, w = i - c * kNavWords;
            uint32_t v = 0;
            if (c < nchan && bc[c].prn > 0) v = a.nav[((size_t) bc[c].frame * a.nav_stride + c) * kNavWords + w];
            sm.nav[c][w] = v;
        }
        // step constants and residue lists of the channels' steps, one lane per channel of the last warp
        if (warp == kLaneWarps - 1 && lane < CH) {
            const bool ok = lane < nchan && bc[lane].prn > 0;
            lanes::ChanRun k;
            lanes::init_steps(k, ok, ok ? bc[lane].c_carr : 0.0, ok ? bc[lane].c_code : 0.0);
            sm.steps[lane] = LaneSteps{k.D96, k.E96, k.inv32, k.e22};
            sm.step[lane] = lanes::fast_step(k);
            lanes::band_residues(lanes::fast_step(k), &sm.band[lane][0]);
        }
    }
    __syncthreads();

    // ---- roles of this lane -----------------------------------------------------------------------------------
    const int ch = lane & (CH - 1), half = lane / CH;                            // channel side
    const bool chan_ok = ch < nchan && bc[ch < nchan ? ch : 0].prn > 0;
    const uint32_t *nav_row = &sm.nav[ch][0];
    const uint32_t *chip_row = &sm.chips[ch][0];
    const uint32_t *band_row = &sm.band[ch][0];
    auto navf = [nav_row](int iw) { return nav_row[iw]; };
    auto chipf = [chip_row](int i) { return chip_row[i]; };
    const uint32_t n0 = (uint32_t) lane, n1 = n0 + 32u, n2 = n0 + 64u;              // sample side: this lane's samples
    const uint32_t sbit = 1u << lanes::sign_pos(lane);                            // and sign bit
    const int nwin = a.run_samples / lanes::kWindow;
    uint32_t *stage = &sm.stage[warp][0];

    const int run_first = g * a.runs_per_cta;
    const int run_last = min(run_first + a.runs_per_cta, a.nruns);
#pragma unroll 1
    for (int r = run_first + warp; r < run_last; r += kLaneWarps) {
        // ---- channel side: exact anchor of (run, channel), window state of window 0 + half -------------------------
        // The anchor is read again from global memory (L1/L2-resident) on the rare paths that walk from it rather than
        // held in registers across the sample side, where at 64 registers it pushed the window state to local memory.
        auto anchor = [&](int c) {
            const RunCkpt k0 = a.ck[((size_t) b * a.nruns + r) * nchan + c];
            return lanes::Anchor{k0.x, k0.y, bc[c].c_carr, bc[c].c_code, k0.nav};
        };
        lanes::ChanRun s;
        auto load_steps = [&]() {
            const LaneSteps k = sm.steps[ch];
            s.D96 = k.D96;
            s.E96 = k.E96;
            s.inv32 = k.inv32;
            s.e22 = k.e22;
        };
        {
            const lanes::Anchor an = chan_ok ? anchor(ch) : lanes::Anchor{0.0, 0.0, 0.0, 0.0, 0u};
            lanes::init_run(s, chan_ok, an.x0, an.y0, an.navpos, an.c, an.d, navf);     // all zero when !chan_ok
        }
        if (WINS == 2 && chan_ok && half == 1) {
            load_steps();
            lanes::advance_window(s, navf);
        }
        // output of the trip's first window: derived once per run, advanced per trip
        uint4 *dst = reinterpret_cast<uint4 *>(reinterpret_cast<char *>(a.out) +
                                               ((size_t) b * kBlockSamples + (size_t) r * a.run_samples) * BYTES);

#pragma unroll 1
        for (int w = 0; w < nwin; w += WINS) {
            uint32_t flagged;                           // bit half * CH + c: channel c has a fast_risky sample in window w + half
            {
                uint32_t S[3] = {0u, 0u, 0u};
                uint32_t base = (uint32_t) (ch * SWZ) << 23;                        // rotation of the channel's table
                bool band = false;
                if (chan_ok) load_steps();
                if (chan_ok && w > 0) {
#pragma unroll
                    for (int i = 0; i < WINS; i++) lanes::advance_window(s, navf);
                }
                if (chan_ok && w + half < nwin) {
                    base += lanes::fast_base(s);
                    band = lanes::window_band_risky(band_row, base);                 // the rotation keeps the low 23 bits
                    if (!lanes::window_signs(s, chipf, navf, S)) {
                        const uint3 e = exact_signs_call(anchor(ch), w + half, chipf, navf);
                        S[0] = e.x;
                        S[1] = e.y;
                        S[2] = e.z;
                    }
                }
                *reinterpret_cast<uint4 *>(&sm.win[warp][half][ch]) = make_uint4(S[0], S[1], S[2], base);
                flagged = __ballot_sync(kFull, band);
            }
            __syncwarp();

            // ---- sample side ------------------------------------------------------------------------------------
#pragma unroll
            for (int hh = 0; hh < WINS; hh++) {
                if (w + hh >= nwin) break;
                const LaneWin *wrow = &sm.win[warp][hh][0];
                int accs[3];
                // The fixed-count loop for the full 32-channel call only: in the 16-channel variant the sample side
                // runs once per window of the trip, and a second copy of the loop for each was slower at 12 channels.
                if (CH == 32 && nchan == CH)                                      // warp-uniform
                    window_sums<CH>(wrow, &sm.step[0], tab_base, nchan, n0, sbit, accs);
                else
                    window_sums<0>(wrow, &sm.step[0], tab_base, nchan, n0, sbit, accs);
                // ---- repair: the channel side flagged the channels with a sample of this window within 2^-25 cycles below
                // an index boundary (warp-uniform). Take the certain index of exactly those (channel, sample) pairs (64-bit
                // linear phase; exact walk from the run anchor inside the 2^-41 band) and patch the sums.
                for (uint32_t m = WINS == 1 ? flagged : (flagged >> (hh * CH)) & 0xFFFFu; m != 0u; m &= m - 1u) {
                    const int c = __ffs((int) m) - 1;
                    const uint4 wv = *reinterpret_cast<const uint4 *>(&wrow[c]);
                    const uint32_t st = sm.step[c];
                    const uint32_t p0 = wv.w + n0 * st, p1 = wv.w + n1 * st, p2 = wv.w + n2 * st;
                    const bool risky = lanes::fast_risky(p0) | lanes::fast_risky(p1) | lanes::fast_risky(p2);
                    if (!risky) continue;
                    const lanes::Anchor ac = anchor(c);
                    const uint32_t ps[3] = {p0, p1, p2}, sw[3] = {wv.x, wv.y, wv.z};
#pragma unroll
                    for (int j = 0; j < 3; j++) {
                        if (!lanes::fast_risky(ps[j])) continue;
                        const int kf = (int) (ps[j] >> 23);                          // stored slot (rotated)
                        const int k = exact_index_call(ac, w + hh, 32 * j + lane);
                        const int fix = tab[c * 512 + ((k + c * SWZ) & 511)] - tab[c * 512 + kf];
                        accs[j] += (sw[j] & sbit) ? -fix : fix;
                    }
                }
                // ---- quantise + pack (gps.c:2833-2845) ---------------------------------------------------------------
                // i = (short) i_acc is the low half of the packed sum p, q = (short) q_acc its high half after the
                // borrow that sign-extending i took (gps.c:2834-2835): q << 16 = p - i = the high half of
                // x = p + ((p & 0x8000) << 1). So x is the int16 pair (i, q) as stored, and the int8 pair
                // (i >> 4, q >> 4) (gps.c:2844) is bits 4..11 of p and bits 20..27 of x.
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    const uint32_t p = (uint32_t) accs[j];
                    const uint32_t x = p + ((p & 0x8000u) << 1);
                    const int n = hh * lanes::kWindow + 32 * j + lane;
                    if (IQ16)
                        stage[n] = x;
                    else
                        reinterpret_cast<uint16_t *>(stage)[n] = (uint16_t) (((p >> 4) & 0xFFu) | ((x >> 12) & 0xFF00u));
                }
            }
            __syncwarp();
            // ---- 16-byte stores of the window(s) of this trip ------------------------------------------------------------
            {
                constexpr int kVec = WINS * lanes::kWindow * BYTES / 16;       // 16-byte vectors of a full trip
                const int nvec = WINS == 1 || nwin - w >= WINS ? kVec : kVec / WINS;
                const uint4 *srcv = reinterpret_cast<const uint4 *>(stage);
#pragma unroll
                for (int i = lane; i < ((kVec + 31) & ~31); i += 32)
                    if (i < nvec) dst[i] = srcv[i];
                dst += kVec;
            }
        }
    }
}

}  // namespace

bool synth_lanes_applicable(const SynthArgs &a) {
    return a.lanes && a.nchan <= 32 && a.run_samples % lanes::kWindow == 0 && a.run_samples <= lanes::kMaxRun;
}

static int device_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return 132;                                                             // H100 SXM
    return n;
}

static void lanes_shape(const SynthArgs &a, int *ctas_per_block, int *runs_per_cta) {
    // CTAs all take about the same time and 2 per SM are resident (2 x 132 on an H100 SXM): aim at 40 or more waves so
    // that the last, partly filled one costs little (2999 blocks as ONE CTA each are 11.4 waves -> 12: 5 % lost), in
    // steps of one run per warp of a CTA
    int per_block = (40 * kLaneCtas * device_sms() + a.nblk - 1) / a.nblk;
    if (per_block > 16) per_block = 16;
    if (per_block < 1) per_block = 1;
    int per_cta = (a.nruns + per_block - 1) / per_block;
    per_cta = (per_cta + kLaneWarps - 1) / kLaneWarps * kLaneWarps;
    per_block = (a.nruns + per_cta - 1) / per_cta;
    *ctas_per_block = per_block;
    *runs_per_cta = per_cta;
}

template <bool IQ16, int CH>
static cudaError_t launch_lanes_t(const SynthArgs &a, cudaStream_t s) {
    const size_t smem = lanes_smem_bytes<CH>();
    cudaError_t e = cudaFuncSetAttribute(k_synth_lanes<IQ16, CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    if (e != cudaSuccess) return e;
    k_synth_lanes<IQ16, CH><<<a.nblk * a.ctas_per_block, kLaneWarps * 32, smem, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_synth_lanes(const SynthArgs &a_in, cudaStream_t s) {
    SynthArgs a = a_in;
    lanes_shape(a, &a.ctas_per_block, &a.runs_per_cta);
    if (a.nchan <= 16) return a.iq16 ? launch_lanes_t<true, 16>(a, s) : launch_lanes_t<false, 16>(a, s);
    return a.iq16 ? launch_lanes_t<true, 32>(a, s) : launch_lanes_t<false, 32>(a, s);
}

void synth_lanes_launch_shape(const SynthArgs &a, int *ctas, int *threads, size_t *smem, int *ctas_per_block,
                              int *runs_per_cta) {
    int per_block, per_cta;
    lanes_shape(a, &per_block, &per_cta);
    *ctas = a.nblk * per_block;
    *threads = kLaneWarps * 32;
    *smem = a.nchan <= 16 ? lanes_smem_bytes<16>() : lanes_smem_bytes<32>();
    *ctas_per_block = per_block;
    *runs_per_cta = per_cta;
}

}  // namespace gpsb200
