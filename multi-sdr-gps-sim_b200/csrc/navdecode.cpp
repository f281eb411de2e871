// Bit sync, frame sync and word decoding of the 50 bit/s navigation message from the epochs of one tracked channel
// (include/gpsb200.h: gpsb200_nav_decode; DESIGN §10). Cheap and sequential: host code, shared by the CLI and Python.
#include <stdint.h>

#include <vector>

#include "../../include/gpsb200.h"

namespace {

unsigned parity_of(uint32_t v) { return (unsigned) __builtin_popcount(v) & 1u; }

// IS-GPS-200 parity equations over data bits d1..d24 (word bits 29..6): bit masks of the data bits each parity bit sums.
const uint32_t kParityMask[6] = {0x3B1F3480u, 0x1D8F9A40u, 0x2EC7CD00u, 0x1763E680u, 0x2BB1F340u, 0x0B7A89C0u};

uint32_t parity6(uint32_t data24, unsigned d29, unsigned d30) {
    const uint32_t d = (data24 & 0xFFFFFFu) << 6;
    const unsigned star[6] = {d29, d30, d29, d30, d30, d29};
    uint32_t p = 0;
    for (int k = 0; k < 6; k++) p = (p << 1) | ((star[k] + parity_of(kParityMask[k] & d)) & 1u);
    return p;
}

int word_check(uint32_t word, uint32_t prev, uint32_t *data) {
    const unsigned d29 = (prev >> 1) & 1u, d30 = prev & 1u;
    uint32_t dat = (word >> 6) & 0xFFFFFFu;
    if (d30) dat ^= 0xFFFFFFu;
    if (data) *data = dat;
    return parity6(dat, d29, d30) == (word & 0x3Fu) ? 1 : 0;
}

const uint32_t kPreamble = 0x8Bu;   // 10001011

uint32_t bits_word(const std::vector<int> &v, int64_t i, int n) {
    uint32_t w = 0;
    for (int k = 0; k < n; k++) w = (w << 1) | (uint32_t) v[i + k];
    return w;
}

}  // namespace

extern "C" {

uint32_t gpsb200_nav_parity(uint32_t data24, int d29, int d30) { return parity6(data24, d29 & 1, d30 & 1); }

int gpsb200_nav_word_check(uint32_t word, uint32_t prev, uint32_t *data) { return word_check(word, prev, data); }

int gpsb200_nav_decode(const gpsb200_track_epoch_t *ep, int64_t n, gpsb200_nav_bit_t *bits, int64_t max_bits,
                       gpsb200_nav_word_t *words, int64_t max_words, gpsb200_nav_sync_t *sync) {
    if (!sync || n < 0 || (n > 0 && !ep) || max_bits < n / 20 || max_words < n / 600 || (max_bits > 0 && !bits) ||
        (max_words > 0 && !words))
        return GPSB200_ERR_ARG;
    gpsb200_nav_sync_t sy{-1, 0, -1, 0, 0, 0, 0, -1};
    // bit sync: prompt-I sign changes between consecutive locked epochs, by position mod 20
    int64_t hist[20] = {0};
    for (int64_t i = 1; i < n; i++)
        if (ep[i].lock && ep[i - 1].lock && ((ep[i].p_i > 0) != (ep[i - 1].p_i > 0))) hist[i % 20]++;
    int edge = 0;
    for (int k = 1; k < 20; k++)
        if (hist[k] > hist[edge]) edge = k;
    if (hist[edge] == 0) {
        *sync = sy;
        return GPSB200_OK;
    }
    sy.bit_edge = edge;
    const int64_t nb = (n - edge) / 20;
    std::vector<int> v((size_t) nb);
    for (int64_t k = 0; k < nb; k++) {
        const gpsb200_track_epoch_t *e = ep + edge + 20 * k;
        int64_t sum = 0;
        int locked = 1;
        for (int j = 0; j < 20; j++) {
            sum += e[j].p_i;
            locked &= e[j].lock;
        }
        v[k] = sum > 0 ? 1 : 0;
        bits[k].sample = e[0].sample;
        bits[k].sum = sum;
        bits[k].value = v[k];
        bits[k].locked = locked;
    }
    sy.nbits = (int32_t) nb;
    // frame sync: preamble in either polarity, TLM and HOW parity, subframe id 1..5
    for (int64_t i = 2; i + 60 <= nb && sy.frame_bit < 0; i++) {
        const uint32_t pre = bits_word(v, i, 8);
        if (pre != kPreamble && pre != (~kPreamble & 0xFFu)) continue;
        const uint32_t flip = pre == kPreamble ? 0u : 0x3FFFFFFFu;
        const uint32_t prev = bits_word(v, i - 2, 2) ^ (flip & 3u);
        const uint32_t tlm = bits_word(v, i, 30) ^ flip, how = bits_word(v, i + 30, 30) ^ flip;
        uint32_t hd;
        if (!word_check(tlm, prev, nullptr) || !word_check(how, tlm, &hd)) continue;
        const int sf = (int) ((hd >> 2) & 7u);
        if (sf < 1 || sf > 5) continue;
        sy.frame_bit = (int32_t) i;
        sy.inverted = flip ? 1 : 0;
    }
    if (sy.frame_bit >= 0) {
        if (sy.inverted)
            for (int64_t k = 0; k < nb; k++) {
                v[k] ^= 1;
                bits[k].value = v[k];
            }
        const int64_t i0 = sy.frame_bit;
        uint32_t prev = bits_word(v, i0 - 2, 2);
        for (int64_t w = 0; i0 + 30 * (w + 1) <= nb; w++) {
            const int64_t b = i0 + 30 * w;
            gpsb200_nav_word_t &o = words[w];
            o.sample = bits[b].sample;
            o.raw = bits_word(v, b, 30);
            o.parity_ok = word_check(o.raw, prev, &o.data);
            o.index = (int32_t) w;
            o.subframe = 0;
            o.tow = -1;
            if (w % 10 == 1) {
                o.subframe = (int32_t) ((o.data >> 2) & 7u);
                o.tow = (int32_t) ((o.data >> 7) & 0x1FFFFu);
                if (o.parity_ok) {
                    sy.subframes++;
                    if (sy.first_tow < 0) sy.first_tow = o.tow;
                }
            }
            sy.words_ok += o.parity_ok;
            sy.nwords++;
            prev = o.raw;
        }
    }
    *sync = sy;
    return GPSB200_OK;
}

}  // extern "C"
