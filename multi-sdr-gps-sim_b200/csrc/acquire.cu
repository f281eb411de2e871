// GPS L1 C/A acquisition search (include/gpsb200.h: gpsb200_acquire; DESIGN §9).
//
// k_acq_grid: one CTA per (Doppler bin, PRN), 256 threads, each thread 12 code delays (tau = tid + 256 r). Per coherent
// period k the CTA wipes the carrier off the 5999 samples the period's 3000 delays read and keeps their int32 prefix sums
// S (I and Q) in shared memory. The replica is +-1 and constant between its sign changes q_0 < q_1 < ... (about 510 of
// them), so with S[i] = sum_{m<i} x[m]:
//     C(tau) = +-( 2 * sum_i (-1)^i S[tau + q_i] - S[tau] + S[tau + 3000] )
// (an odd number of changes is padded with q = 3000, further padding comes in pairs (0, 0) that cancel; the sign is
// irrelevant to C^2). One shared-memory load and one 3-input add per (delay, sign change, component) instead of 3000
// multiply-adds. Powers accumulate over the K periods in registers; the CTA then reduces its row: P1, the lowest tau at
// P1, and P2 outside +-3 samples of that tau. k_acq_pick takes per PRN the row with the largest P1 (lowest j on ties) --
// the global argmax with the contract's tie rule, since each row's argmax is its lowest-tau maximum.
//
// Per-PRN Doppler windows (gpsb200_acquire_windows; DESIGN §9.1) run the same two kernels: k_acq_grid<T, true> reads
// its phase steps from a [nprn][nbins] table instead of [nbins], and k_acq_pick reports each PRN's own f_lo. The
// standard instantiation k_acq_grid<T, false, 1> compiles to the code it had before windows existed (an index with a
// run-time row stride of 0 instead made it spill 24 more bytes).
//
// A search of fewer rows than a wave (a warm start: 12 PRNs x 5 bins is 60 CTAs on 132 SMs) leaves SMs idle. It splits
// each row's 3072 delays over kSplit CTAs (grid z): each slice builds the prefix sums its delays read and writes its
// powers to device scratch, and k_acq_reduce applies the row's argmax, tie and P2 rules, with no atomics. The split
// comes from nprn x nbins and the SM count (split_for), never from the caller; the results are the same bits either way.
// A batch (DESIGN §11.6) splits only a pass of fewer rows than one full wave (batch_split): on 8 windows of the standard
// grid split_for picks 3 slices, whose prefix sums cost twice a row's, and the pass ran 17 % slower than unsplit.
#include <cmath>
#include <cstring>
#include <vector>

#include "acquire.h"
#include "device_buffer.h"
#include "rx_samples.cuh"
#include "synth_tables.h"

namespace gpsb200 {
namespace acq {

namespace {

using rx::load_iq;

struct Best {
    uint64_t v;
    int t;
};
__device__ __forceinline__ Best better(Best a, Best b) {   // larger power, then lower delay
    return (b.v > a.v || (b.v == a.v && b.t < a.t)) ? b : a;
}

constexpr int kWarps = kThreads / 32;

// The delays of one CTA of a search split kSplit ways: slice z takes tau = tau0 + tid + 256 r, r < kR, tau0 = z kSpan; its
// kSpan delays read kNeed samples from tau0 on, kPer per thread. kSplit = 1 is the whole row (kPer = 24, as ever).
template <int kSplit>
struct Slice {
    static constexpr int kR = kTausPerThread / kSplit;
    static constexpr int kSpan = kThreads * kR;
    static constexpr int kNeed = kSpan + kCode - 1;
    static constexpr int kPer = (kNeed + kThreads - 1) / kThreads;
    static_assert(kR * kSplit == kTausPerThread && kPer * kThreads <= kPrefix, "slice shape");
};
static_assert(Slice<1>::kPer * kThreads == kPrefix, "prefix split");

struct Smem {
    alignas(16) int16_t edges[kMaxEdges];   // read 8 at a time
    int2 tab[512];                       // (cos, sin)
    int2 S[kPrefix + 1];                 // S[i] = (sum_{m<i} I_d, sum_{m<i} Q_d) of the current period, from tau0 on
    int2 wsum[kWarps];
    uint64_t rv[kWarps];
    int rt[kWarps];
};

// The reduction of row `idx`'s powers pw (delay tid + 256 r): its grid row (grid NULL: not wanted), argmax (lowest tau
// on ties), P2 outside +-kExclude samples of it; rows[idx] = (P1, P2, tau1). rv / rt: kWarps entries of shared memory.
__device__ __forceinline__ void reduce_row(const uint64_t (&pw)[kTausPerThread], uint64_t *grid, size_t idx,
                                           uint64_t *rv, int *rt, uint64_t *rows) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t *g = grid ? grid + idx * kCode : nullptr;
    Best b{pw[0], tid};
#pragma unroll
    for (int r = 0; r < kTausPerThread; r++) {
        const int t = tid + kThreads * r;
        if (t < kCode) {
            if (g) g[t] = pw[r];
            if (pw[r] > b.v) b = Best{pw[r], t};
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best c{__shfl_xor_sync(0xffffffffu, b.v, o), __shfl_xor_sync(0xffffffffu, b.t, o)};
        b = better(b, c);
    }
    if (lane == 0) {
        rv[warp] = b.v;
        rt[warp] = b.t;
    }
    __syncthreads();
    b = Best{rv[0], rt[0]};
    for (int w = 1; w < kWarps; w++) b = better(b, Best{rv[w], rt[w]});
    const int t1 = b.t;
    __syncthreads();
    uint64_t p2 = 0;
#pragma unroll
    for (int r = 0; r < kTausPerThread; r++) {
        const int t = tid + kThreads * r;
        int d = abs(t - t1);
        d = min(d, kCode - d);
        if (t < kCode && d > kExclude && pw[r] > p2) p2 = pw[r];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t c = __shfl_xor_sync(0xffffffffu, p2, o);
        p2 = c > p2 ? c : p2;
    }
    if (lane == 0) rv[warp] = p2;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kWarps; w++) p2 = rv[w] > p2 ? rv[w] : p2;
        uint64_t *row = rows + idx * 3;
        row[0] = b.v;
        row[1] = p2;
        row[2] = (uint64_t) t1;
    }
}

// kWindows: phase steps from a [nprn][nbins] table. kSplit > 1: CTA (j, p, z) computes slice z of row (p, j) and writes
// its powers to grid (scratch of [nprn][nbins][3000], required); k_acq_reduce reduces the rows. The prefix sums start at
// tau0 instead of 0: C takes differences of S only (its coefficients sum to zero), so C is the same integer.
// The body of k_acq_grid and k_acq_batch, which differ only in where a CTA's samples start.
template <typename T, bool kWindows, int kSplit>
__device__ __forceinline__ void grid_row(const T *__restrict__ iq, const int16_t *__restrict__ edges_all,
                                         const int32_t *__restrict__ nedges_all, const int32_t *__restrict__ prns,
                                         const uint32_t *__restrict__ u_bins, int K, int nbins,
                                         uint64_t *__restrict__ grid, uint64_t *__restrict__ rows) {
    using Sh = Slice<kSplit>;
    constexpr int kPer = Sh::kPer, kR = Sh::kR;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j = blockIdx.x, p = blockIdx.y;
    const int tau0 = kSplit == 1 ? 0 : (int) blockIdx.z * Sh::kSpan;
    const int prn = prns[p];
    const int ne = nedges_all[prn];
    const uint32_t u = u_bins[kWindows ? p * nbins + j : j];
    rx::fill_carrier_table(sm.tab, kThreads);
    for (int i = tid; i < ne; i += kThreads) sm.edges[i] = edges_all[prn * kMaxEdges + i];
    if (tid == 0) sm.S[0] = make_int2(0, 0);

    uint64_t pw[kR];
#pragma unroll
    for (int r = 0; r < kR; r++) pw[r] = 0;

    for (int k = 0; k < K; k++) {
        __syncthreads();   // tables/edges written; the previous period's S fully read
        // wipe-off of samples tau0 + m, m = kPer * tid .. + kPer - 1 of the period, local inclusive sums into S[m + 1]
        const int m0 = kPer * tid;
        const int64_t base = (int64_t) kCode * k + tau0;
        int sI = 0, sQ = 0;
#pragma unroll 4
        for (int i = 0; i < kPer; i++) {
            const int m = m0 + i;
            int dI = 0, dQ = 0;
            if (tau0 + m < 2 * kCode - 1) {   // the window's 3000 K + 2999 samples; beyond: zeros (delays >= 3000 only)
                int I, Q;
                load_iq<T>(iq, base + m, I, Q);
                const int2 d = rx::wipe_off(sm.tab, (uint32_t) (base + m) * u, I, Q);
                dI = d.x;
                dQ = d.y;
            }
            sI += dI;
            sQ += dQ;
            sm.S[m + 1] = make_int2(sI, sQ);
        }
        // exclusive scan of the thread totals
        int xI = sI, xQ = sQ;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int yI = __shfl_up_sync(0xffffffffu, xI, o), yQ = __shfl_up_sync(0xffffffffu, xQ, o);
            if (lane >= o) {
                xI += yI;
                xQ += yQ;
            }
        }
        if (lane == 31) sm.wsum[warp] = make_int2(xI, xQ);
        __syncthreads();
        int oI = xI - sI, oQ = xQ - sQ;
        for (int w = 0; w < warp; w++) {
            oI += sm.wsum[w].x;
            oQ += sm.wsum[w].y;
        }
#pragma unroll 4
        for (int i = 0; i < kPer; i++) {
            int2 v = sm.S[m0 + i + 1];
            v.x += oI;
            v.y += oQ;
            sm.S[m0 + i + 1] = v;
        }
        __syncthreads();

        // correlation: sum over the replica's sign changes
        int aI[kR], aQ[kR];
#pragma unroll
        for (int r = 0; r < kR; r++) aI[r] = aQ[r] = 0;
        const int2 *Sb = sm.S + tid;
        for (int e = 0; e < ne; e += 8) {
            const int4 w4 = *reinterpret_cast<const int4 *>(&sm.edges[e]);
            const int wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int h = 0; h < 4; h++) {
                const int2 *pa = Sb + (wv[h] & 0xffff), *pb = Sb + ((uint32_t) wv[h] >> 16);
#pragma unroll
                for (int r = 0; r < kR; r++) {
                    const int2 a = pa[kThreads * r], b = pb[kThreads * r];
                    aI[r] += a.x - b.x;
                    aQ[r] += a.y - b.y;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int2 s0 = Sb[kThreads * r], s1 = Sb[kThreads * r + kCode];
            const int cI = 2 * aI[r] - s0.x + s1.x, cQ = 2 * aQ[r] - s0.y + s1.y;
            pw[r] += (uint64_t) ((int64_t) cI * cI + (int64_t) cQ * cQ);
        }
    }

    if constexpr (kSplit == 1) {
        reduce_row(pw, grid, (size_t) p * nbins + j, sm.rv, sm.rt, rows);
    } else {
        uint64_t *g = grid + ((size_t) p * nbins + j) * kCode;
#pragma unroll
        for (int r = 0; r < kR; r++) {
            const int t = tau0 + tid + kThreads * r;
            if (t < kCode) g[t] = pw[r];
        }
    }
}

template <typename T, bool kWindows, int kSplit>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
k_acq_grid(const T *__restrict__ iq, const int16_t *__restrict__ edges_all, const int32_t *__restrict__ nedges_all,
           const int32_t *__restrict__ prns, const uint32_t *__restrict__ u_bins, int K, int nbins,
           uint64_t *__restrict__ grid, uint64_t *__restrict__ rows) {
    grid_row<T, kWindows, kSplit>(iq, edges_all, nedges_all, prns, u_bins, K, nbins, grid, rows);
}

// A batch of windows (gpsb200_snapshot_batch; DESIGN §11.6): the per-PRN window search with row p = w nprn + q of grid
// y the (window w, PRN q) pair. prns and u_bins hold one row per pair; window w's samples start win_off[w] samples
// from iq.
template <typename T, int kSplit>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
k_acq_batch(const T *__restrict__ iq, const int64_t *__restrict__ win_off, int nprn,
            const int16_t *__restrict__ edges_all, const int32_t *__restrict__ nedges_all,
            const int32_t *__restrict__ prns, const uint32_t *__restrict__ u_bins, int K, int nbins,
            uint64_t *__restrict__ grid, uint64_t *__restrict__ rows) {
    const T *w = iq + 2 * win_off[blockIdx.y / nprn];
    grid_row<T, true, kSplit>(w, edges_all, nedges_all, prns, u_bins, K, nbins, grid, rows);
}

// The rows of a split search: one CTA per (bin, PRN) reduces the powers its slices wrote to grid, as k_acq_grid does.
__global__ void __launch_bounds__(kThreads) k_acq_reduce(const uint64_t *__restrict__ grid, int nbins,
                                                         uint64_t *__restrict__ rows) {
    __shared__ uint64_t rv[kWarps];
    __shared__ int rt[kWarps];
    const size_t row = (size_t) blockIdx.y * nbins + blockIdx.x;
    const uint64_t *g = grid + row * kCode;
    uint64_t pw[kTausPerThread];
#pragma unroll
    for (int r = 0; r < kTausPerThread; r++) {
        const int t = threadIdx.x + kThreads * r;
        pw[r] = t < kCode ? g[t] : 0;
    }
    reduce_row(pw, nullptr, row, rv, rt, rows);
}

// One warp per PRN: the row with the largest P1, lowest j on ties. f_lo_prn (NULL: f_lo for every PRN): per-PRN first bins.
__global__ void k_acq_pick(const uint64_t *__restrict__ rows, const int32_t *__restrict__ prns, int nbins, double f_lo,
                           const double *__restrict__ f_lo_prn, double step, gpsb200_acq_result_t *__restrict__ res) {
    const int p = blockIdx.x, lane = threadIdx.x;
    Best b{0, 0x7fffffff};
    // lanes without a bin keep (0, INT_MAX): any real row wins against them, ties going to the lower j
    for (int j = lane; j < nbins; j += 32) b = better(b, Best{rows[((size_t) p * nbins + j) * 3], j});
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best c{__shfl_xor_sync(0xffffffffu, b.v, o), __shfl_xor_sync(0xffffffffu, b.t, o)};
        b = better(b, c);
    }
    if (lane == 0) {
        const uint64_t *row = rows + ((size_t) p * nbins + b.t) * 3;
        gpsb200_acq_result_t r;
        r.prn = prns[p];
        r.bin = b.t;
        r.delay = (int32_t) row[2];
        r.reserved = 0;
        r.doppler_hz = (f_lo_prn ? f_lo_prn[p] : f_lo) + (double) b.t * step;
        r.delay_chips = (double) r.delay * 1023.0 / 3000.0;
        r.p1 = row[0];
        r.p2 = row[1];
        r.ratio = r.p2 ? (double) r.p1 / (double) r.p2 : INFINITY;
        res[p] = r;
    }
}

// Sign changes of PRN prn's sampled replica c[n] = 2 ca[(n * 1023) / 3000] - 1: chip c starts at sample
// ceil(3000 c / 1023); an odd count is padded with 3000, the rest up to a multiple of 8 with (0, 0) pairs.
int replica_edges(int prn, int16_t *out) {
    uint8_t ca[GPSB200_CA_LEN];
    ca_code(prn, ca);
    int n = 0;
    for (int c = 1; c < GPSB200_CA_LEN; c++)
        if (ca[c] != ca[c - 1]) out[n++] = (int16_t) ((3000 * c + 1022) / 1023);
    if (n & 1) out[n++] = kCode;
    while (n & 7) out[n++] = 0;
    return n;
}

// The kernels of every (sample type, windows, split): a table, so that launch and the attribute set-up name them once.
using GridKernel = const void *;
template <typename T, bool kWin>
const GridKernel kGrid[] = {(GridKernel) k_acq_grid<T, kWin, 1>, (GridKernel) k_acq_grid<T, kWin, 2>,
                                (GridKernel) k_acq_grid<T, kWin, 3>, (GridKernel) k_acq_grid<T, kWin, 4>,
                                (GridKernel) k_acq_grid<T, kWin, 6>};
template <typename T>
const GridKernel kBatch[] = {(GridKernel) k_acq_batch<T, 1>, (GridKernel) k_acq_batch<T, 2>,
                             (GridKernel) k_acq_batch<T, 3>, (GridKernel) k_acq_batch<T, 4>,
                             (GridKernel) k_acq_batch<T, 6>};
constexpr int kSplits[] = {1, 2, 3, 4, 6};
constexpr int kNumSplits = sizeof(kSplits) / sizeof(kSplits[0]);

GridKernel grid_kernel(int sample_size, bool windows, int split) {
    int i = 0;
    while (kSplits[i] != split) i++;
    if (sample_size == GPSB200_SC08) return windows ? kGrid<int8_t, true>[i] : kGrid<int8_t, false>[i];
    return windows ? kGrid<int16_t, true>[i] : kGrid<int16_t, false>[i];
}

GridKernel batch_kernel(int sample_size, int split) {
    int i = 0;
    while (kSplits[i] != split) i++;
    return sample_size == GPSB200_SC08 ? kBatch<int8_t>[i] : kBatch<int16_t>[i];
}

// The phase steps of rows p < nrow from their first bins f_lo[p] (NULL: cfg->f_lo_hz for one row), [nrow][nbins].
std::vector<uint32_t> phase_steps(const gpsb200_acq_config_t *cfg, int nrow, const double *f_lo) {
    std::vector<uint32_t> u((size_t) nrow * cfg->nbins);
    for (int p = 0; p < nrow; p++)
        for (int j = 0; j < cfg->nbins; j++)
            u[(size_t) p * cfg->nbins + j] = phase_step((f_lo ? f_lo[p] : cfg->f_lo_hz) + (double) j * cfg->step_hz);
    return u;
}

}  // namespace

bool split_allowed(int split) {
    for (int s : kSplits)
        if (s == split) return true;
    return false;
}

int split_for(int rows, int sms) {
    // per-SM work in rows, when the rows x split CTAs spread evenly: ceil(rows split / sms) / split; the least wins,
    // the smallest split on ties (so a search of a wave or more, like the standard one, is never split)
    int best = 1;
    int64_t num = (rows + sms - 1) / sms, den = 1;   // ceil(rows / sms) / 1
    for (int s : kSplits) {
        const int64_t n = ((int64_t) rows * s + sms - 1) / sms;
        if (n * den < num * s) {
            best = s;
            num = n;
            den = s;
        }
    }
    return best;
}

int split_of(const Scratch &sc, int nprn, int nbins) {
    return sc.force_split ? sc.force_split : split_for(nprn * nbins, sc.sms);
}

int batch_split(const Scratch &sc, int npair, int nbins) {
    const int64_t rows = (int64_t) npair * nbins;
    if (sc.force_split || rows < (int64_t) kCtasPerSm * sc.sms) return split_of(sc, npair, nbins);
    return 1;
}

int64_t window_samples(const gpsb200_acq_config_t *cfg) { return (int64_t) kCode * cfg->ms + (kCode - 1); }

uint32_t phase_step(double f_hz) { return (uint32_t) (int64_t) llround(f_hz * 4294967296.0 / 3e6); }

namespace {
bool bins_inside(double f_lo, const gpsb200_acq_config_t *cfg) {
    const double f_hi = f_lo + (double) (cfg->nbins - 1) * cfg->step_hz;
    return std::isfinite(f_lo) && std::isfinite(cfg->step_hz) && (cfg->nbins == 1 || cfg->step_hz > 0.0) &&
           std::fabs(f_lo) <= 1.5e6 && std::fabs(f_hi) <= 1.5e6;
}
}  // namespace

std::string check(const gpsb200_acq_config_t *cfg, int64_t nsamples, int sample_size, bool windows,
                  const double *f_lo_prn) {
    if (!cfg) return "config is NULL";
    if (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16) return "sample_size must be GPSB200_SC08 or GPSB200_SC16";
    if (cfg->ms < 1 || cfg->ms > GPSB200_ACQ_MAX_MS) return "ms (K) must be 1..100";
    if (cfg->nprn < 1 || cfg->nprn > 32) return "nprn must be 1..32";
    for (int i = 0; i < cfg->nprn; i++)
        if (cfg->prn[i] < 1 || cfg->prn[i] > 32) return "PRN " + std::to_string(cfg->prn[i]) + " outside 1..32";
    if (cfg->nbins < 1 || cfg->nbins > GPSB200_ACQ_MAX_BINS) return "nbins must be 1..1024";
    if (!windows && !bins_inside(cfg->f_lo_hz, cfg)) return "Doppler bins must lie within +-1.5 MHz with step_hz > 0";
    if (windows) {
        if (!f_lo_prn) return "f_lo_prn is NULL";
        for (int i = 0; i < cfg->nprn; i++)
            if (!bins_inside(f_lo_prn[i], cfg))
                return "Doppler bins of PRN " + std::to_string(cfg->prn[i]) +
                       " must lie within +-1.5 MHz with step_hz > 0";
    }
    if (cfg->s0 < 0 || nsamples < 0 || cfg->s0 > nsamples || nsamples - cfg->s0 < window_samples(cfg))
        return "the window s0 .. s0 + 3000 K + 2998 is not inside the buffer of " + std::to_string(nsamples) + " samples";
    return std::string();
}

cudaError_t scratch_reserve(Scratch &sc, const gpsb200_acq_config_t *cfg, bool windows, bool want_grid) {
    CU_RET(sc.d_edges.grow((size_t) 33 * kMaxEdges));
    CU_RET(sc.d_nedges.grow(33));
    CU_RET(sc.d_res.grow(32));
    CU_RET(sc.h_res.grow(32));
    CU_RET(sc.d_prn.grow(32));
    CU_RET(sc.d_flo.grow(32));
    if (!sc.ready) {
        std::vector<int16_t> e((size_t) 33 * kMaxEdges, 0);
        std::vector<int32_t> n(33, 0);
        for (int prn = 1; prn <= 32; prn++) n[prn] = replica_edges(prn, e.data() + (size_t) prn * kMaxEdges);
        CU_RET(cudaMemcpy(sc.d_edges.get(), e.data(), e.size() * sizeof(int16_t), cudaMemcpyHostToDevice));
        CU_RET(cudaMemcpy(sc.d_nedges.get(), n.data(), n.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
        for (int i = 0; i < kNumSplits; i++)
            for (GridKernel k : {kGrid<int8_t, false>[i], kGrid<int16_t, false>[i], kGrid<int8_t, true>[i],
                                 kGrid<int16_t, true>[i], kBatch<int8_t>[i], kBatch<int16_t>[i]})
                CU_RET(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, sizeof(Smem)));
        int dev = 0;
        CU_RET(cudaGetDevice(&dev));
        CU_RET(cudaDeviceGetAttribute(&sc.sms, cudaDevAttrMultiProcessorCount, dev));
        sc.ready = true;
    }
    CU_RET(sc.d_rows.grow((size_t) 32 * cfg->nbins * 3));
    CU_RET(sc.d_u.grow((size_t) (windows ? cfg->nprn : 1) * cfg->nbins));
    if (want_grid || split_of(sc, cfg->nprn, cfg->nbins) > 1)
        CU_RET(sc.d_grid.grow((size_t) cfg->nprn * cfg->nbins * kCode));
    return cudaSuccess;
}

cudaError_t batch_reserve(Scratch &sc, const gpsb200_acq_config_t *cfg, int nwin) {
    const size_t npair = (size_t) nwin * cfg->nprn;
    CU_RET(scratch_reserve(sc, cfg, true, false));
    CU_RET(sc.d_rows.grow(npair * cfg->nbins * 3));
    CU_RET(sc.d_u.grow(npair * cfg->nbins));
    CU_RET(sc.d_boff.grow((size_t) nwin));
    CU_RET(sc.d_bprn.grow(npair));
    CU_RET(sc.d_bflo.grow(npair));
    CU_RET(sc.d_bres.grow(npair));
    if (batch_split(sc, (int) npair, cfg->nbins) > 1) CU_RET(sc.d_grid.grow(npair * cfg->nbins * kCode));
    return cudaSuccess;
}

cudaError_t launch(Scratch &sc, const void *window, int sample_size, const gpsb200_acq_config_t *cfg,
                   const double *f_lo_prn, bool want_grid, cudaStream_t s) {
    // the small parameter arrays go up by value in the stream order (the host copies are on this call's stack)
    const std::vector<uint32_t> u = phase_steps(cfg, f_lo_prn ? cfg->nprn : 1, f_lo_prn);
    CU_RET(cudaMemcpyAsync(sc.d_u.get(), u.data(), u.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_prn.get(), cfg->prn, cfg->nprn * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (f_lo_prn)
        CU_RET(cudaMemcpyAsync(sc.d_flo.get(), f_lo_prn, cfg->nprn * sizeof(double), cudaMemcpyHostToDevice, s));
    const int split = split_of(sc, cfg->nprn, cfg->nbins);
    const dim3 grid(cfg->nbins, cfg->nprn, split);
    uint64_t *g = want_grid || split > 1 ? sc.d_grid.get() : nullptr;
    const GridKernel kernel = grid_kernel(sample_size, f_lo_prn != nullptr, split);
    // cudaLaunchKernel reads each argument at the address given: these local pointer copies, never an owning array
    const void *src = window;   // either sample type: the kernels take the pointer as is
    const int16_t *edges = sc.d_edges.get();
    const int32_t *nedges = sc.d_nedges.get(), *prn = sc.d_prn.get();
    const uint32_t *u_dev = sc.d_u.get();
    uint64_t *rows = sc.d_rows.get();
    void *args[] = {(void *) &src, (void *) &edges, (void *) &nedges, (void *) &prn, (void *) &u_dev,
                    (void *) &cfg->ms, (void *) &cfg->nbins, (void *) &g, (void *) &rows};
    CU_RET(cudaLaunchKernel(kernel, grid, dim3(kThreads), args, sizeof(Smem), s));
    if (split > 1) {
        k_acq_reduce<<<dim3(cfg->nbins, cfg->nprn), kThreads, 0, s>>>(sc.d_grid.get(), cfg->nbins, rows);
        CU_RET(cudaGetLastError());
    }
    k_acq_pick<<<cfg->nprn, 32, 0, s>>>(rows, sc.d_prn.get(), cfg->nbins, cfg->f_lo_hz,
                                        f_lo_prn ? sc.d_flo.get() : nullptr, cfg->step_hz, sc.d_res.get());
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(sc.h_res.get(), sc.d_res.get(), cfg->nprn * sizeof(gpsb200_acq_result_t),
                           cudaMemcpyDeviceToHost, s));
    // pageable sources of the two uploads must outlive them: wait here (the search is blocking anyway)
    return cudaStreamSynchronize(s);
}

cudaError_t launch_batch(Scratch &sc, const void *src, int sample_size, const gpsb200_acq_config_t *cfg, int nwin,
                         const int64_t *win_off, const double *f_lo, gpsb200_acq_result_t *res, cudaStream_t s) {
    const int npair = nwin * cfg->nprn;
    std::vector<int32_t> prn((size_t) npair);
    for (int i = 0; i < npair; i++) prn[i] = cfg->prn[i % cfg->nprn];
    const std::vector<uint32_t> u = phase_steps(cfg, npair, f_lo);
    CU_RET(cudaMemcpyAsync(sc.d_u.get(), u.data(), u.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_bprn.get(), prn.data(), prn.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_bflo.get(), f_lo, npair * sizeof(double), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_boff.get(), win_off, nwin * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    const int split = batch_split(sc, npair, cfg->nbins);
    uint64_t *g = split > 1 ? sc.d_grid.get() : nullptr;
    // the arguments by address, of local pointer copies as in launch
    const void *p = src;
    int nprn = cfg->nprn;
    const int64_t *boff = sc.d_boff.get();
    const int16_t *edges = sc.d_edges.get();
    const int32_t *nedges = sc.d_nedges.get(), *bprn = sc.d_bprn.get();
    const uint32_t *u_dev = sc.d_u.get();
    uint64_t *rows = sc.d_rows.get();
    void *args[] = {(void *) &p, (void *) &boff, (void *) &nprn, (void *) &edges, (void *) &nedges,
                    (void *) &bprn, (void *) &u_dev, (void *) &cfg->ms, (void *) &cfg->nbins, (void *) &g,
                    (void *) &rows};
    CU_RET(cudaLaunchKernel(batch_kernel(sample_size, split), dim3(cfg->nbins, npair, split), dim3(kThreads), args,
                            sizeof(Smem), s));
    if (split > 1) {
        k_acq_reduce<<<dim3(cfg->nbins, npair), kThreads, 0, s>>>(sc.d_grid.get(), cfg->nbins, rows);
        CU_RET(cudaGetLastError());
    }
    k_acq_pick<<<npair, 32, 0, s>>>(rows, bprn, cfg->nbins, cfg->f_lo_hz, sc.d_bflo.get(), cfg->step_hz,
                                    sc.d_bres.get());
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(res, sc.d_bres.get(), npair * sizeof(gpsb200_acq_result_t), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

}  // namespace acq
}  // namespace gpsb200
