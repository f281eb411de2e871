// Bit sync, frame sync and word decoding of the 50 bit/s navigation message from the epochs of one tracked channel
// (include/gpsb200.h: gpsb200_nav_decode; DESIGN §10), and the ephemeris, Klobuchar terms and transmit-time anchor the
// words carry (gpsb200_nav_ephemeris, gpsb200_nav_time_anchor; DESIGN §11), and the almanac of subframes 4 and 5
// (gpsb200_nav_almanac; DESIGN §9.1). Cheap and sequential: host code, shared by
// the CLI and Python.
#include <stdint.h>

#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/gpsb200.h"
#include "synth_tables.h"

namespace {

using gpsb200::kPi;
using gpsb200::parity6;

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

// The low `bits` bits of v as a two's complement integer.
double sext(uint32_t v, int bits) {
    const int64_t m = (int64_t) v & ((1ll << bits) - 1);
    return (double) (m >= (1ll << (bits - 1)) ? m - (1ll << bits) : m);
}

// A 32-bit field split 8 + 24 over two words: the low 8 data bits of `hi`, all 24 of `lo`.
int32_t split32(uint32_t hi, uint32_t lo) { return (int32_t) (((hi & 0xFFu) << 24) | (lo & 0xFFFFFFu)); }

// Subframe starts: a TLM (index a multiple of 10) with its 9 successors in sequence and all 10 with good parity.
// Returns the subframe id of the HOW, 0 when words[i] starts no such subframe.
int subframe_id(const gpsb200_nav_word_t *words, int64_t n, int64_t i) {
    if (i < 0 || i + 10 > n || words[i].index % 10 != 0) return 0;
    for (int j = 0; j < 10; j++)
        if (words[i + j].index != words[i].index + j || !words[i + j].parity_ok) return 0;
    return (int) ((words[i + 1].data >> 2) & 7u);
}

// IS-GPS-200 scale factors; semicircles are turned into radians with the reference's pi (kPi).
const double kP2m5 = 0.03125, kP2m19 = 1.0 / 524288.0, kP2m29 = 1.0 / 536870912.0, kP2m31 = 1.0 / 2147483648.0,
             kP2m33 = 1.0 / 8589934592.0, kP2m43 = 1.0 / 8796093022208.0, kP2m55 = 1.0 / 36028797018963968.0;

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

int gpsb200_nav_ephemeris(const gpsb200_nav_word_t *words, int64_t n, gpsb200_ephemeris_t *eph, gpsb200_iono_t *iono) {
    if (!eph || n < 0 || (n > 0 && !words)) return GPSB200_ERR_ARG;
    memset(eph, 0, sizeof *eph);
    if (iono) memset(iono, 0, sizeof *iono);
    auto good_subframe = [&](int64_t i) { return subframe_id(words, n, i); };
    for (int64_t i = n - 30; i >= 0; i--) {
        if (good_subframe(i) != 1 || good_subframe(i + 10) != 2 || good_subframe(i + 20) != 3) continue;
        const gpsb200_nav_word_t *s1 = words + i, *s2 = words + i + 10, *s3 = words + i + 20;
        const int32_t iodc = (int32_t) (((s1[2].data & 3u) << 8) | ((s1[7].data >> 16) & 0xFFu));
        const int32_t iode2 = (int32_t) ((s2[2].data >> 16) & 0xFFu), iode3 = (int32_t) ((s3[9].data >> 16) & 0xFFu);
        if (iode2 != iode3 || iode2 != (iodc & 0xFF)) continue;
        gpsb200_ephemeris_t &e = *eph;
        e.week = (int32_t) ((s1[2].data >> 14) & 0x3FFu);
        e.ura = (int32_t) ((s1[2].data >> 8) & 0xFu);
        e.health = (int32_t) ((s1[2].data >> 2) & 0x3Fu);
        e.iodc = iodc;
        e.iode = iode2;
        e.tgd = sext(s1[6].data, 8) * kP2m31;
        e.toc = (double) (s1[7].data & 0xFFFFu) * 16.0;
        e.af2 = sext(s1[8].data >> 16, 8) * kP2m55;
        e.af1 = sext(s1[8].data, 16) * kP2m43;
        e.af0 = sext(s1[9].data >> 2, 22) * kP2m31;
        e.crs = sext(s2[2].data, 16) * kP2m5;
        e.deltan = sext(s2[3].data >> 8, 16) * kP2m43 * kPi;
        e.m0 = (double) split32(s2[3].data, s2[4].data) * kP2m31 * kPi;
        e.cuc = sext(s2[5].data >> 8, 16) * kP2m29;
        e.ecc = (double) (uint32_t) split32(s2[5].data, s2[6].data) * kP2m33;
        e.cus = sext(s2[7].data >> 8, 16) * kP2m29;
        e.sqrta = (double) (uint32_t) split32(s2[7].data, s2[8].data) * kP2m19;
        e.toe = (double) ((s2[9].data >> 8) & 0xFFFFu) * 16.0;
        e.cic = sext(s3[2].data >> 8, 16) * kP2m29;
        e.omg0 = (double) split32(s3[2].data, s3[3].data) * kP2m31 * kPi;
        e.cis = sext(s3[4].data >> 8, 16) * kP2m29;
        e.inc0 = (double) split32(s3[4].data, s3[5].data) * kP2m31 * kPi;
        e.crc = sext(s3[6].data >> 8, 16) * kP2m5;
        e.aop = (double) split32(s3[6].data, s3[7].data) * kP2m31 * kPi;
        e.omgdot = sext(s3[8].data, 24) * kP2m43 * kPi;
        e.idot = sext(s3[9].data >> 2, 14) * kP2m43 * kPi;
        e.valid = 1;
        break;
    }
    if (iono)
        for (int64_t i = n - 10; i >= 0; i--) {
            if (good_subframe(i) != 4) continue;
            const gpsb200_nav_word_t *s = words + i;
            if (((s[2].data >> 22) & 3u) != 1u || ((s[2].data >> 16) & 0x3Fu) != 56u) continue;
            iono->alpha[0] = sext(s[2].data >> 8, 8) * std::ldexp(1.0, -30);
            iono->alpha[1] = sext(s[2].data, 8) * std::ldexp(1.0, -27);
            iono->alpha[2] = sext(s[3].data >> 16, 8) * std::ldexp(1.0, -24);
            iono->alpha[3] = sext(s[3].data >> 8, 8) * std::ldexp(1.0, -24);
            iono->beta[0] = sext(s[3].data, 8) * 2048.0;
            iono->beta[1] = sext(s[4].data >> 16, 8) * 16384.0;
            iono->beta[2] = sext(s[4].data >> 8, 8) * 65536.0;
            iono->beta[3] = sext(s[4].data, 8) * 65536.0;
            iono->valid = 1;
            break;
        }
    return GPSB200_OK;
}

int gpsb200_nav_almanac(const gpsb200_nav_word_t *words, int64_t n, int32_t week, gpsb200_almanac_record_t rec[32],
                        int32_t *wna_out) {
    if (!rec || n < 0 || (n > 0 && !words)) return GPSB200_ERR_ARG;
    memset(rec, 0, 32 * sizeof *rec);
    int32_t wna = -1;
    for (int64_t i = 0; i + 10 <= n; i++) {
        const int sf = subframe_id(words, n, i);
        if (sf != 4 && sf != 5) continue;
        const gpsb200_nav_word_t *s = words + i;
        if (((s[2].data >> 22) & 3u) != 1u) continue;
        const int svid = (int) ((s[2].data >> 16) & 0x3Fu);
        if (sf == 5 && svid == 51) {
            wna = (int32_t) (s[2].data & 0xFFu);
            continue;
        }
        if (svid < 1 || svid > 32) continue;
        gpsb200_almanac_record_t &r = rec[svid - 1];
        r.svid = svid;
        r.valid = 1;
        r.e = (double) (s[2].data & 0xFFFFu) * std::ldexp(1.0, -21);
        r.toa_sec = (double) ((s[3].data >> 16) & 0xFFu) * 4096.0;
        r.delta_i = sext(s[3].data, 16) * std::ldexp(1.0, -19);
        r.omegadot = sext(s[4].data >> 8, 16) * std::ldexp(1.0, -38);
        r.health = (int32_t) (s[4].data & 0xFFu);
        r.sqrta = (double) (s[5].data & 0xFFFFFFu) * std::ldexp(1.0, -11);
        r.omega0 = sext(s[6].data, 24) * std::ldexp(1.0, -23);
        r.aop = sext(s[7].data, 24) * std::ldexp(1.0, -23);
        r.m0 = sext(s[8].data, 24) * std::ldexp(1.0, -23);
        r.af0 = sext((((s[9].data >> 16) & 0xFFu) << 3) | ((s[9].data >> 2) & 7u), 11) * std::ldexp(1.0, -20);
        r.af1 = sext(s[9].data >> 5, 11) * std::ldexp(1.0, -38);
    }
    // WNa (8 bits) to the full week nearest the caller's: within -128..127 of it
    const int32_t full = wna < 0 ? -1 : week + (int32_t) ((((wna - week) % 256 + 256 + 128) % 256) - 128);
    for (int sv = 0; sv < 32; sv++)
        if (rec[sv].svid) rec[sv].toa_week = full;
    if (wna_out) *wna_out = wna;
    return GPSB200_OK;
}

int gpsb200_nav_time_anchor(const gpsb200_nav_word_t *words, int64_t n, const gpsb200_nav_sync_t *sync,
                            int32_t *anchor_epoch, int64_t *anchor_ms) {
    if (!sync || !anchor_epoch || !anchor_ms || n < 0 || (n > 0 && !words)) return GPSB200_ERR_ARG;
    *anchor_epoch = -1;
    *anchor_ms = 0;
    if (sync->bit_edge < 0 || sync->frame_bit < 0) return GPSB200_OK;
    for (int64_t i = 0; i < n; i++) {
        const gpsb200_nav_word_t &w = words[i];
        if (w.index % 10 != 1 || !w.parity_ok || w.tow < 0) continue;
        const int64_t ep = (int64_t) sync->bit_edge + 20 * ((int64_t) sync->frame_bit + 30 * (int64_t) w.index);
        if (ep > INT32_MAX) return GPSB200_OK;
        const int64_t week_ms = 604800000;
        *anchor_epoch = (int32_t) ep;
        *anchor_ms = (((6 * (int64_t) w.tow - 6) * 1000 + 600) % week_ms + week_ms) % week_ms;
        return GPSB200_OK;
    }
    return GPSB200_OK;
}

}  // extern "C"
