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
using rx::sine512;

struct Best {
    uint64_t v;
    int t;
};
__device__ __forceinline__ Best better(Best a, Best b) {   // larger power, then lower delay
    return (b.v > a.v || (b.v == a.v && b.t < a.t)) ? b : a;
}

constexpr int kPer = kPrefix / kThreads;   // 24 prefix entries per thread
static_assert(kPer * kThreads == kPrefix, "prefix split");
constexpr int kWarps = kThreads / 32;

struct Smem {
    alignas(16) int16_t edges[kMaxEdges];   // read 8 at a time
    int2 tab[512];                       // (cos, sin)
    int2 S[kPrefix + 1];                 // S[i] = (sum_{m<i} I_d, sum_{m<i} Q_d) of the current period
    int2 wsum[kWarps];
    uint64_t rv[kWarps];
    int rt[kWarps];
};

template <typename T>
__global__ void __launch_bounds__(kThreads, 3)
k_acq_grid(const T *__restrict__ iq, const int16_t *__restrict__ edges_all, const int32_t *__restrict__ nedges_all,
           const int32_t *__restrict__ prns, const uint32_t *__restrict__ u_bins, int K, int nbins,
           uint64_t *__restrict__ grid, uint64_t *__restrict__ rows) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j = blockIdx.x, p = blockIdx.y;
    const int prn = prns[p];
    const int ne = nedges_all[prn];
    const uint32_t u = u_bins[j];
    for (int i = tid; i < 512; i += kThreads) sm.tab[i] = make_int2(sine512(i + 128), sine512(i));
    for (int i = tid; i < ne; i += kThreads) sm.edges[i] = edges_all[prn * kMaxEdges + i];
    if (tid == 0) sm.S[0] = make_int2(0, 0);

    uint64_t pw[kTausPerThread];
#pragma unroll
    for (int r = 0; r < kTausPerThread; r++) pw[r] = 0;

    for (int k = 0; k < K; k++) {
        __syncthreads();   // tables/edges written; the previous period's S fully read
        // wipe-off of samples m = kPer * tid .. + kPer - 1 of the period, local inclusive sums into S[m + 1]
        const int m0 = kPer * tid;
        const int64_t base = (int64_t) kCode * k;
        int sI = 0, sQ = 0;
#pragma unroll 4
        for (int i = 0; i < kPer; i++) {
            const int m = m0 + i;
            int dI = 0, dQ = 0;
            if (m < 2 * kCode - 1) {   // the window's 3000 K + 2999 samples; beyond: zeros (delays >= 3000 only)
                int I, Q;
                load_iq<T>(iq, base + m, I, Q);
                const uint32_t ph = (uint32_t) (base + m) * u;
                const int2 cs = sm.tab[ph >> 23];
                dI = I * cs.x + Q * cs.y;
                dQ = Q * cs.x - I * cs.y;
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
        int aI[kTausPerThread], aQ[kTausPerThread];
#pragma unroll
        for (int r = 0; r < kTausPerThread; r++) aI[r] = aQ[r] = 0;
        const int2 *Sb = sm.S + tid;
        for (int e = 0; e < ne; e += 8) {
            const int4 w4 = *reinterpret_cast<const int4 *>(&sm.edges[e]);
            const int wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int h = 0; h < 4; h++) {
                const int2 *pa = Sb + (wv[h] & 0xffff), *pb = Sb + ((uint32_t) wv[h] >> 16);
#pragma unroll
                for (int r = 0; r < kTausPerThread; r++) {
                    const int2 a = pa[kThreads * r], b = pb[kThreads * r];
                    aI[r] += a.x - b.x;
                    aQ[r] += a.y - b.y;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kTausPerThread; r++) {
            const int2 s0 = Sb[kThreads * r], s1 = Sb[kThreads * r + kCode];
            const int cI = 2 * aI[r] - s0.x + s1.x, cQ = 2 * aQ[r] - s0.y + s1.y;
            pw[r] += (uint64_t) ((int64_t) cI * cI + (int64_t) cQ * cQ);
        }
    }

    // the row: grid, argmax (lowest tau on ties), P2 outside +-kExclude samples of it
    uint64_t *g = grid ? grid + ((size_t) p * nbins + j) * kCode : nullptr;
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
        sm.rv[warp] = b.v;
        sm.rt[warp] = b.t;
    }
    __syncthreads();
    b = Best{sm.rv[0], sm.rt[0]};
    for (int w = 1; w < kWarps; w++) b = better(b, Best{sm.rv[w], sm.rt[w]});
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
    if (lane == 0) sm.rv[warp] = p2;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kWarps; w++) p2 = sm.rv[w] > p2 ? sm.rv[w] : p2;
        uint64_t *row = rows + ((size_t) p * nbins + j) * 3;
        row[0] = b.v;
        row[1] = p2;
        row[2] = (uint64_t) t1;
    }
}

// One warp per PRN: the row with the largest P1, lowest j on ties.
__global__ void k_acq_pick(const uint64_t *__restrict__ rows, const int32_t *__restrict__ prns, int nbins, double f_lo,
                           double step, gpsb200_acq_result_t *__restrict__ res) {
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
        r.doppler_hz = f_lo + (double) b.t * step;
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

}  // namespace

int64_t window_samples(const gpsb200_acq_config_t *cfg) { return (int64_t) kCode * cfg->ms + (kCode - 1); }

uint32_t phase_step(double f_hz) { return (uint32_t) (int64_t) llround(f_hz * 4294967296.0 / 3e6); }

std::string check(const gpsb200_acq_config_t *cfg, int64_t nsamples, int sample_size) {
    if (!cfg) return "config is NULL";
    if (sample_size != GPSB200_SC08 && sample_size != GPSB200_SC16) return "sample_size must be GPSB200_SC08 or GPSB200_SC16";
    if (cfg->ms < 1 || cfg->ms > GPSB200_ACQ_MAX_MS) return "ms (K) must be 1..100";
    if (cfg->nprn < 1 || cfg->nprn > 32) return "nprn must be 1..32";
    for (int i = 0; i < cfg->nprn; i++)
        if (cfg->prn[i] < 1 || cfg->prn[i] > 32) return "PRN " + std::to_string(cfg->prn[i]) + " outside 1..32";
    if (cfg->nbins < 1 || cfg->nbins > GPSB200_ACQ_MAX_BINS) return "nbins must be 1..1024";
    const double f_hi = cfg->f_lo_hz + (double) (cfg->nbins - 1) * cfg->step_hz;
    if (!std::isfinite(cfg->f_lo_hz) || !std::isfinite(cfg->step_hz) || !(cfg->nbins == 1 || cfg->step_hz > 0.0) ||
        std::fabs(cfg->f_lo_hz) > 1.5e6 || std::fabs(f_hi) > 1.5e6)
        return "Doppler bins must lie within +-1.5 MHz with step_hz > 0";
    if (cfg->s0 < 0 || nsamples < 0 || cfg->s0 > nsamples || nsamples - cfg->s0 < window_samples(cfg))
        return "the window s0 .. s0 + 3000 K + 2998 is not inside the buffer of " + std::to_string(nsamples) + " samples";
    return std::string();
}

cudaError_t scratch_reserve(Scratch &sc, const gpsb200_acq_config_t *cfg, bool want_grid) {
    if (!sc.d_edges) {
        std::vector<int16_t> e((size_t) 33 * kMaxEdges, 0);
        std::vector<int32_t> n(33, 0);
        for (int prn = 1; prn <= 32; prn++) n[prn] = replica_edges(prn, e.data() + (size_t) prn * kMaxEdges);
        CU_RET(cudaMalloc(&sc.d_edges, e.size() * sizeof(int16_t)));
        CU_RET(cudaMemcpy(sc.d_edges, e.data(), e.size() * sizeof(int16_t), cudaMemcpyHostToDevice));
        CU_RET(cudaMalloc(&sc.d_nedges, n.size() * sizeof(int32_t)));
        CU_RET(cudaMemcpy(sc.d_nedges, n.data(), n.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
        CU_RET(cudaMalloc(&sc.d_res, 32 * sizeof(gpsb200_acq_result_t)));
        CU_RET(cudaHostAlloc(&sc.h_res, 32 * sizeof(gpsb200_acq_result_t), cudaHostAllocDefault));
        CU_RET(cudaMalloc(&sc.d_prn, 32 * sizeof(int32_t)));
        CU_RET(cudaFuncSetAttribute(k_acq_grid<int8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, sizeof(Smem)));
        CU_RET(cudaFuncSetAttribute(k_acq_grid<int16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, sizeof(Smem)));
    }
    CU_RET(grow(sc.d_rows, sc.rows_cap, (size_t) 32 * cfg->nbins * 3));
    CU_RET(grow(sc.d_u, sc.u_cap, (size_t) cfg->nbins));
    if (want_grid) CU_RET(grow(sc.d_grid, sc.grid_cap, (size_t) cfg->nprn * cfg->nbins * kCode));
    return cudaSuccess;
}

void scratch_free(Scratch &sc) {
    cudaFree(sc.d_edges);
    cudaFree(sc.d_nedges);
    cudaFree(sc.d_grid);
    cudaFree(sc.d_rows);
    cudaFree(sc.d_res);
    cudaFreeHost(sc.h_res);
    cudaFree(sc.d_u);
    cudaFree(sc.d_prn);
    sc = Scratch();
}

cudaError_t launch(Scratch &sc, const void *window, int sample_size, const gpsb200_acq_config_t *cfg, bool want_grid,
                   cudaStream_t s) {
    // the small parameter arrays go up by value in the stream order (the host copies are on this call's stack)
    std::vector<uint32_t> u(cfg->nbins);
    for (int j = 0; j < cfg->nbins; j++) u[j] = phase_step(cfg->f_lo_hz + (double) j * cfg->step_hz);
    CU_RET(cudaMemcpyAsync(sc.d_u, u.data(), u.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CU_RET(cudaMemcpyAsync(sc.d_prn, cfg->prn, cfg->nprn * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    const dim3 grid(cfg->nbins, cfg->nprn);
    uint64_t *g = want_grid ? sc.d_grid : nullptr;
    if (sample_size == GPSB200_SC08)
        k_acq_grid<int8_t><<<grid, kThreads, sizeof(Smem), s>>>(static_cast<const int8_t *>(window), sc.d_edges, sc.d_nedges,
                                                                sc.d_prn, sc.d_u, cfg->ms, cfg->nbins, g, sc.d_rows);
    else
        k_acq_grid<int16_t><<<grid, kThreads, sizeof(Smem), s>>>(static_cast<const int16_t *>(window), sc.d_edges,
                                                                 sc.d_nedges, sc.d_prn, sc.d_u, cfg->ms, cfg->nbins, g,
                                                                 sc.d_rows);
    CU_RET(cudaGetLastError());
    k_acq_pick<<<cfg->nprn, 32, 0, s>>>(sc.d_rows, sc.d_prn, cfg->nbins, cfg->f_lo_hz, cfg->step_hz, sc.d_res);
    CU_RET(cudaGetLastError());
    CU_RET(cudaMemcpyAsync(sc.h_res, sc.d_res, cfg->nprn * sizeof(gpsb200_acq_result_t), cudaMemcpyDeviceToHost, s));
    // pageable sources of the two uploads must outlive them: wait here (the search is blocking anyway)
    return cudaStreamSynchronize(s);
}

}  // namespace acq
}  // namespace gpsb200
