// Collective detection (include/gpsb200.h: gpsb200_collective; DESIGN §11.7).
//
// The search leaves every PRN's power grid P[nprn][nbins][3000] on the device. k_cd_rowsum sums each row exactly in 128
// bits, k_cd_q turns each row into uint16 q by its PRN's mean, stored twice over (kRow entries) so that a cyclic read
// (d + b) mod 3000 is a plain read at d + b. k_cd_setup (one warp) tests which PRNs are used, once per call, and sets up
// the lattice frame. k_cd_score takes kTile hypotheses per CTA: all its threads predict the (hypothesis, used PRN)
// cells in FP64 into shared memory, then each warp sweeps the 3000 clock shifts of its hypotheses, lane = shift mod 32,
// over coalesced reads of the q rows, and reduces to the best shift with a shuffle argmax. k_cd_pick (one CTA) finds
// the winner and the runner-up, and k_cd_seed (one CTA per PRN) forms the seeds at the winner's cells. Every sum is an
// integer and every tie rule fixed, so nothing depends on the order the device runs in.
#include <cmath>
#include <cstring>
#include <vector>

#include "collective.h"
#include "device_buffer.h"
#include "orbit.cuh"

namespace gpsb200 {
namespace cd {

struct Setup {
    double E[3], N[3], U[3];   // the frame at x_a
    double t0;                 // ap.t_a + (s0 - ap.s_a) / 3e6
    int nused;
    uint32_t used;
    int idx[32];               // the used PRNs' indices into acq->prn, in order
    uint64_t mu[32];
};

namespace {

using pvt::Geo;
using pvt::predict;
using pvt::predict_steps;
using pvt::round_half_up;
using pvt::wrap_half_week;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTile = 16;          // hypotheses per CTA of k_cd_score
constexpr int kCode = 3000;
constexpr int kChunks = 12;        // shifts b = 256 c + lane + 32 r, c < 12, r < 8: 3072 >= 3000
constexpr unsigned kFull = 0xffffffffu;

struct Args {
    const uint64_t *grid;
    uint64_t *rowsum;
    uint16_t *q;
    const gpsb200_ephemeris_t *eph;
    Setup *setup;
    gpsb200_cd_score_t *scores;
    gpsb200_cd_cell_t *table;
    gpsb200_collective_t *rec;
    const gpsb200_acq_result_t *res;
    gpsb200_acq_result_t *seed;
    int64_t s0;
    int nprn, nbins, nhyp;
    double step_hz;
    int prn[32];
    double flo[32];
    gpsb200_coarse_config_t ap;
    gpsb200_collective_config_t cfg;
};

struct U128 {
    uint64_t lo, hi;
};
__device__ __forceinline__ void add(U128 &a, uint64_t lo, uint64_t hi) {
    a.lo += lo;
    a.hi += hi + (a.lo < lo);
}
// The sum of every thread's a over the CTA, on every thread. sh: kWarps entries of shared memory.
__device__ U128 block_sum(U128 a, U128 *sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) add(a, __shfl_xor_sync(kFull, a.lo, o), __shfl_xor_sync(kFull, a.hi, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
    __syncthreads();
    U128 s{0, 0};
    for (int w = 0; w < kWarps; w++) add(s, sh[w].lo, sh[w].hi);
    return s;
}

// min(floor(2^GPSB200_CD_Q_SHIFT P / mu), GPSB200_CD_Q_CAP) for mu > 0, 0 for mu = 0: P / mu (capped at once when the
// quotient alone reaches 2^(16 - shift)), then GPSB200_CD_Q_SHIFT steps of long division (the remainder stays below
// mu < 2^63, so doubling it never overflows).
__device__ __forceinline__ uint16_t qval(uint64_t P, uint64_t mu) {
    if (mu == 0) return 0;
    const uint64_t a = P / mu;
    if (a >= (1u << (16 - GPSB200_CD_Q_SHIFT))) return GPSB200_CD_Q_CAP;
    uint64_t r = P - a * mu;
    uint32_t v = (uint32_t) a;
#pragma unroll
    for (int i = 0; i < GPSB200_CD_Q_SHIFT; i++) {
        r <<= 1;
        v <<= 1;
        if (r >= mu) {
            r -= mu;
            v |= 1;
        }
    }
    return (uint16_t) min(v, (uint32_t) GPSB200_CD_Q_CAP);
}

// Row (p, j) of the grid: its 128-bit sum.
__global__ void __launch_bounds__(kThreads) k_cd_rowsum(const Args a) {
    __shared__ U128 sh[kWarps];
    const size_t row = (size_t) blockIdx.y * a.nbins + blockIdx.x;
    const uint64_t *g = a.grid + row * kCode;
    U128 s{0, 0};
    for (int t = threadIdx.x; t < kCode; t += kThreads) add(s, g[t], 0);
    s = block_sum(s, sh);
    if (threadIdx.x == 0) {
        a.rowsum[row * 2] = s.lo;
        a.rowsum[row * 2 + 1] = s.hi;
    }
}

// Row (p, j): mu_p from PRN p's row sums, then the row's q, twice over.
__global__ void __launch_bounds__(kThreads) k_cd_q(const Args a) {
    __shared__ U128 sh[kWarps];
    const int p = blockIdx.y;
    U128 s{0, 0};
    for (int j = threadIdx.x; j < a.nbins; j += kThreads) {
        const uint64_t *r = a.rowsum + ((size_t) p * a.nbins + j) * 2;
        add(s, r[0], r[1]);
    }
    s = block_sum(s, sh);
    const unsigned __int128 sum = ((unsigned __int128) s.hi << 64) | s.lo;
    const uint64_t mu = (uint64_t) (sum / (unsigned __int128) ((uint64_t) a.nbins * kCode));
    if (blockIdx.x == 0 && threadIdx.x == 0) a.setup->mu[p] = mu;
    const size_t row = (size_t) p * a.nbins + blockIdx.x;
    const uint64_t *g = a.grid + row * kCode;
    uint16_t *q = a.q + row * kRow;
    for (int i = threadIdx.x; i < kRow; i += kThreads) q[i] = qval(g[i < kCode ? i : (i < 2 * kCode ? i - kCode : i - 2 * kCode)], mu);
}

// Step 2 and the frame: one warp, lane = searched PRN. The record starts as a record without a winner.
__global__ void k_cd_setup(const Args a) {
    const int lane = threadIdx.x;
    Setup &st = *a.setup;
    Geo g;
    g.set(a.ap.x_a);
    const double U[3] = {g.cla * g.clo, g.cla * g.slo, g.sla};
    const double t0 = a.ap.t_a + (double) (a.s0 - a.ap.s_a) / 3e6;
    bool use = false;
    if (lane < a.nprn) {
        const gpsb200_ephemeris_t &e = a.eph[a.prn[lane] - 1];
        if (e.valid && e.health == 0 && fabs(wrap_half_week(t0 - e.toe)) <= 7200.0 && st.mu[lane] > 0) {
            double sel;
            predict(e, a.ap.x_a, t0, U, sel);
            use = sel >= sin(a.cfg.mask_deg * kPi / 180.0);
        }
    }
    const uint32_t used = __ballot_sync(kFull, use);
    if (use) st.idx[__popc(used & ((1u << lane) - 1))] = lane;
    if (lane == 0) {
        const double E[3] = {-g.slo, g.clo, 0.0}, N[3] = {-g.sla * g.clo, -g.sla * g.slo, g.cla};
        for (int i = 0; i < 3; i++) {
            st.E[i] = E[i];
            st.N[i] = N[i];
            st.U[i] = U[i];
        }
        st.t0 = t0;
        st.nused = __popc(used);
        st.used = used;
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        gpsb200_collective_t r;
        r.status = __popc(used) < GPSB200_CD_MIN_USED ? GPSB200_CD_FEW : GPSB200_CD_OK;
        r.nused = __popc(used);
        r.used = used;
        r.shift = r.winner = r.runner = -1;
        r.score = r.runner_score = 0;
        r.o_t = r.x[0] = r.x[1] = r.x[2] = r.lat_deg = r.lon_deg = r.height = r.runner_dist = nan;
        *a.rec = r;
    }
}

// The offsets (o_e, o_n, o_u, o_t) of hypothesis h.
__device__ __forceinline__ void offsets(const Args &a, int h, double *o) {
#pragma unroll
    for (int ax = 0; ax < 4; ax++) {
        const int n = a.cfg.n[ax];
        const int i = h % n;
        h /= n;
        o[ax] = n > 1 ? ((double) i - (double) (n - 1) * 0.5) * a.cfg.step[ax] : 0.0;
    }
}
__device__ __forceinline__ void position(const Setup &st, const double *xa, const double *o, double *x) {
#pragma unroll
    for (int i = 0; i < 3; i++) x[i] = xa[i] + o[0] * st.E[i] + o[1] * st.N[i] + o[2] * st.U[i];
}

// Step 5 for hypothesis h and searched PRN p: its bin (-1 outside the grid) and delay.
__device__ __forceinline__ void cell(const Args &a, const Setup &st, int h, int p, int &j, int &d) {
    double o[4], x[3], sel, rate, drift;
    offsets(a, h, o);
    position(st, a.ap.x_a, o, x);
    const double pred = predict_steps<true>(a.eph[a.prn[p] - 1], x, st.t0 + o[3], st.U, sel, &rate, &drift);
    d = (int) round_half_up(3000.0 * (1.0 - (pred - floor(pred)))) % kCode;
    const double f = -(rate - kC * drift) / kLambda;
    const double jj = a.nbins == 1 ? 0.0 : round_half_up((f - a.flo[p]) / a.step_hz);
    j = jj >= 0.0 && jj < (double) a.nbins ? (int) jj : -1;
}

// Steps 5 and 6 for kTile hypotheses.
__global__ void __launch_bounds__(kThreads) k_cd_score(const Args a) {
    __shared__ const uint16_t *rows[kTile][32];
    __shared__ int nrow[kTile];
    const Setup &st = *a.setup;
    const int nu = st.nused, h0 = blockIdx.x * kTile;
    if (threadIdx.x < kTile) nrow[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < kTile * nu; i += kThreads) {
        const int t = i / nu, k = i - t * nu, h = h0 + t;
        if (h >= a.nhyp) continue;
        const int p = st.idx[k];
        int j, d;
        cell(a, st, h, p, j, d);
        if (a.table) a.table[(size_t) h * a.nprn + p] = gpsb200_cd_cell_t{j, d};
        if (j >= 0) rows[t][atomicAdd(&nrow[t], 1)] = a.q + ((size_t) p * a.nbins + j) * kRow + d;
    }
    if (a.table)
        for (int i = threadIdx.x; i < kTile * a.nprn; i += kThreads) {
            const int t = i / a.nprn, p = i - t * a.nprn, h = h0 + t;
            if (h < a.nhyp && !((st.used >> p) & 1)) a.table[(size_t) h * a.nprn + p] = gpsb200_cd_cell_t{-1, -1};
        }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int t = warp; t < kTile; t += kWarps) {
        const int h = h0 + t;
        if (h >= a.nhyp) break;
        const int n = nrow[t];   // the rows' order is the atomics': a sum of integers does not depend on it
        uint32_t best = 0;
        int bb = lane;
#pragma unroll 1
        for (int c = 0; c < kChunks; c++) {
            uint32_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll 2
            for (int k = 0; k < n; k++) {
                const uint16_t *r = rows[t][k] + c * 256 + lane;
#pragma unroll
                for (int u = 0; u < 8; u++) acc[u] += r[32 * u];
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int b = c * 256 + lane + 32 * u;
                if (b < kCode && (acc[u] > best || (c == 0 && u == 0))) {
                    best = acc[u];
                    bb = b;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const uint32_t ov = __shfl_xor_sync(kFull, best, o);
            const int ob = __shfl_xor_sync(kFull, bb, o);
            if (ov > best || (ov == best && ob < bb)) {
                best = ov;
                bb = ob;
            }
        }
        if (lane == 0) a.scores[h] = gpsb200_cd_score_t{best, bb};
    }
}

constexpr int kPickThreads = 1024;
// The largest score and its lowest h over the CTA, on every thread. sv / sh: kPickThreads / 32 entries.
__device__ void block_argmax(uint32_t &v, int &h, uint32_t *sv, int *sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint32_t ov = __shfl_xor_sync(kFull, v, o);
        const int oh = __shfl_xor_sync(kFull, h, o);
        if (ov > v || (ov == v && oh < h)) {
            v = ov;
            h = oh;
        }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = v;
        sh[threadIdx.x >> 5] = h;
    }
    __syncthreads();
    v = sv[0];
    h = sh[0];
    for (int w = 1; w < kPickThreads / 32; w++)
        if (sv[w] > v || (sv[w] == v && sh[w] < h)) {
            v = sv[w];
            h = sh[w];
        }
}

// Step 7 and the record: one CTA. Hypotheses without a score yet (none here: every h is scored) would lose to any.
__global__ void __launch_bounds__(kPickThreads) k_cd_pick(const Args a) {
    __shared__ uint32_t sv[kPickThreads / 32];
    __shared__ int sh[kPickThreads / 32];
    uint32_t v = 0;
    int w = 0x7fffffff;
    for (int h = threadIdx.x; h < a.nhyp; h += kPickThreads) {
        const uint32_t s = a.scores[h].score;
        if (w == 0x7fffffff || s > v) {   // h rises, so the first of equal scores stays
            v = s;
            w = h;
        }
    }
    block_argmax(v, w, sv, sh);
    const uint32_t wv = v;
    const int win = w;
    double ow[4];
    offsets(a, win, ow);
    v = 0;
    int r = 0x7fffffff;
    for (int h = threadIdx.x; h < a.nhyp; h += kPickThreads) {
        double o[4];
        offsets(a, h, o);
        const double de = o[0] - ow[0], dn = o[1] - ow[1], du = o[2] - ow[2];
        if (!(sqrt(de * de + dn * dn + du * du) > a.cfg.distinct_m)) continue;
        const uint32_t s = a.scores[h].score;
        if (r == 0x7fffffff || s > v) {
            v = s;
            r = h;
        }
    }
    block_argmax(v, r, sv, sh);
    if (threadIdx.x == 0) {
        const Setup &st = *a.setup;
        gpsb200_collective_t &o = *a.rec;
        o.winner = win;
        o.score = wv;
        o.shift = a.scores[win].shift;
        o.o_t = ow[3];
        position(st, a.ap.x_a, ow, o.x);
        double lat, lon, hgt;
        pvt::ecef_llh(o.x, lat, lon, hgt);
        o.lat_deg = lat * (180.0 / M_PI);
        o.lon_deg = lon * (180.0 / M_PI);
        o.height = hgt;
        o.status = GPSB200_CD_OK;
        if (r != 0x7fffffff) {
            double orr[4];
            offsets(a, r, orr);
            const double de = orr[0] - ow[0], dn = orr[1] - ow[1], du = orr[2] - ow[2];
            o.runner = r;
            o.runner_score = v;
            o.runner_dist = sqrt(de * de + dn * dn + du * du);
            if ((uint64_t) 100 * v >= (uint64_t) GPSB200_CD_AMBIGUOUS_PCT * wv) o.status = GPSB200_CD_AMBIGUOUS;
        }
    }
}

// Step 8: one CTA per searched PRN.
__global__ void __launch_bounds__(kThreads) k_cd_seed(const Args a) {
    __shared__ int jd[2];
    __shared__ uint64_t sv[kWarps];
    const int p = blockIdx.x;
    const Setup &st = *a.setup;
    const gpsb200_collective_t &rec = *a.rec;
    if (threadIdx.x == 0) {
        int j = -1, d = 0;
        if (rec.winner >= 0 && ((st.used >> p) & 1)) {
            cell(a, st, rec.winner, p, j, d);
            d = (d + rec.shift) % kCode;
        }
        jd[0] = j;
        jd[1] = d;
    }
    __syncthreads();
    const int j = jd[0], d = jd[1];
    gpsb200_acq_result_t r = a.res[p];
    if (j < 0) {
        if (threadIdx.x == 0) {
            r.ratio = -1.0;
            a.seed[p] = r;
        }
        return;
    }
    const uint64_t *g = a.grid + ((size_t) p * a.nbins + j) * kCode;
    uint64_t p2 = 0;
    for (int t = threadIdx.x; t < kCode; t += kThreads) {
        int dd = abs(t - d);
        dd = min(dd, kCode - dd);
        if (dd > 3 && g[t] > p2) p2 = g[t];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t c = __shfl_xor_sync(kFull, p2, o);
        p2 = c > p2 ? c : p2;
    }
    if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = p2;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kWarps; w++) p2 = sv[w] > p2 ? sv[w] : p2;
        r.bin = j;
        r.delay = d;
        r.doppler_hz = a.flo[p] + (double) j * a.step_hz;
        r.delay_chips = (double) d * 1023.0 / 3000.0;
        r.p1 = g[d];
        r.p2 = p2;
        r.ratio = p2 ? (double) r.p1 / (double) p2 : INFINITY;
        a.seed[p] = r;
    }
}

}  // namespace

std::string check(const gpsb200_collective_config_t *cfg) {
    int64_t n = 1;
    for (int a = 0; a < 4; a++) {
        if (cfg->n[a] < 1) return "every lattice size n must be >= 1";
        n *= cfg->n[a];
        if (n > GPSB200_CD_MAX_HYP) return "the lattice holds more than GPSB200_CD_MAX_HYP hypotheses";
        if (cfg->n[a] > 1 && !(std::isfinite(cfg->step[a]) && cfg->step[a] > 0.0))
            return "a lattice step must be finite and > 0 where n > 1";
    }
    if (!std::isfinite(cfg->mask_deg)) return "mask_deg must be finite";
    if (!std::isfinite(cfg->distinct_m)) return "distinct_m must be finite";
    if (cfg->reserved != 0) return "reserved must be 0";
    return std::string();
}

int64_t hypotheses(const gpsb200_collective_config_t *cfg) {
    return (int64_t) cfg->n[0] * cfg->n[1] * cfg->n[2] * cfg->n[3];
}

cudaError_t launch(Scratch &sc, const uint64_t *d_grid, const gpsb200_acq_result_t *d_res,
                   const gpsb200_acq_config_t *acq, const double *f_lo_prn, const gpsb200_ephemeris_t *eph,
                   const gpsb200_coarse_config_t *ap, const gpsb200_collective_config_t *cfg,
                   gpsb200_acq_result_t *seed, gpsb200_collective_t *out, gpsb200_cd_score_t *scores,
                   gpsb200_cd_cell_t *table, cudaStream_t s) {
    const int nprn = acq->nprn, nbins = acq->nbins;
    const int64_t nhyp = hypotheses(cfg);
    CU_RET(sc.d_eph.grow(32));
    CU_RET(sc.d_setup.grow(1));
    CU_RET(sc.d_rec.grow(1));
    CU_RET(sc.d_seed.grow(32));
    CU_RET(sc.d_rowsum.grow((size_t) nprn * nbins * 2));
    CU_RET(sc.d_q.grow((size_t) nprn * nbins * kRow));
    CU_RET(sc.d_scores.grow((size_t) nhyp));
    if (table) CU_RET(sc.d_table.grow((size_t) nhyp * nprn));
    Args a{};
    a.grid = d_grid;
    a.rowsum = sc.d_rowsum.get();
    a.q = sc.d_q.get();
    a.eph = sc.d_eph.get();
    a.setup = sc.d_setup.get();
    a.scores = sc.d_scores.get();
    a.table = table ? sc.d_table.get() : nullptr;
    a.rec = sc.d_rec.get();
    a.res = d_res;
    a.seed = sc.d_seed.get();
    a.s0 = acq->s0;
    a.nprn = nprn;
    a.nbins = nbins;
    a.nhyp = (int) nhyp;
    a.step_hz = acq->step_hz;
    for (int p = 0; p < nprn; p++) {
        a.prn[p] = acq->prn[p];
        a.flo[p] = f_lo_prn ? f_lo_prn[p] : acq->f_lo_hz;
    }
    a.ap = *ap;
    a.cfg = *cfg;
    // eph is the caller's memory: wait for the copy before returning (every path below synchronizes s)
    CU_RET(cudaMemcpyAsync(sc.d_eph.get(), eph, 32 * sizeof(gpsb200_ephemeris_t), cudaMemcpyHostToDevice, s));
    k_cd_rowsum<<<dim3(nbins, nprn), kThreads, 0, s>>>(a);
    CU_RET(cudaGetLastError());
    k_cd_q<<<dim3(nbins, nprn), kThreads, 0, s>>>(a);
    CU_RET(cudaGetLastError());
    k_cd_setup<<<1, 32, 0, s>>>(a);
    CU_RET(cudaGetLastError());
    int nused = 0;
    CU_RET(cudaMemcpyAsync(&nused, &sc.d_setup.get()->nused, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaStreamSynchronize(s));
    const bool scored = nused >= GPSB200_CD_MIN_USED;
    if (scored) {
        k_cd_score<<<(unsigned) ((nhyp + kTile - 1) / kTile), kThreads, 0, s>>>(a);
        CU_RET(cudaGetLastError());
        k_cd_pick<<<1, kPickThreads, 0, s>>>(a);
        CU_RET(cudaGetLastError());
    }
    k_cd_seed<<<nprn, kThreads, 0, s>>>(a);
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(out, sc.d_rec.get(), sizeof(gpsb200_collective_t), cudaMemcpyDeviceToHost, s));
    CU_RET(cudaMemcpyAsync(seed, sc.d_seed.get(), nprn * sizeof(gpsb200_acq_result_t), cudaMemcpyDeviceToHost, s));
    if (scores) {
        if (scored)
            CU_RET(cudaMemcpyAsync(scores, sc.d_scores.get(), nhyp * sizeof(gpsb200_cd_score_t), cudaMemcpyDeviceToHost,
                                   s));
        else
            memset(scores, 0, nhyp * sizeof(gpsb200_cd_score_t));
    }
    if (table) {
        if (scored)
            CU_RET(cudaMemcpyAsync(table, sc.d_table.get(), nhyp * nprn * sizeof(gpsb200_cd_cell_t),
                                   cudaMemcpyDeviceToHost, s));
        else
            memset(table, 0xff, nhyp * nprn * sizeof(gpsb200_cd_cell_t));
    }
    return cudaStreamSynchronize(s);
}

}  // namespace cd
}  // namespace gpsb200
