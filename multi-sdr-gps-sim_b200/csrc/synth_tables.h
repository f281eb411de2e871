// Constant data of the GPS L1 C/A path, shared by host and device code.
#pragma once
#include <stdint.h>

namespace gpsb200 {

// First quadrant of the reference's 512-entry sine table (gps.c:145-178):
// floor(250*sin(2*pi*(k+0.5)/512)+0.5) for k = 0..127, except k = 35 where the
// reference holds 105 (formula: 105.50007). Remaining entries by symmetry:
// sin[255-k] = sin[k], sin[k+256] = -sin[k]; cos[k] = sin[(k+128)&511] (gps.c:180-213).
// tests/test_oracle.py / test_host_api.py check the expansion against the reference arrays.
#define GPSB200_QUARTER_SINE                                                              \
    2, 5, 8, 11, 14, 17, 20, 23, 26, 29, 32, 35, 38, 41, 44, 47,                          \
    50, 53, 56, 59, 62, 65, 68, 71, 74, 77, 80, 83, 86, 89, 91, 94,                       \
    97, 100, 103, 105, 108, 111, 114, 116, 119, 122, 125, 127, 130, 132, 135, 138,        \
    140, 143, 145, 148, 150, 153, 155, 157, 160, 162, 164, 167, 169, 171, 173, 176,       \
    178, 180, 182, 184, 186, 188, 190, 192, 194, 196, 198, 200, 202, 204, 205, 207,       \
    209, 210, 212, 214, 215, 217, 218, 220, 221, 223, 224, 225, 227, 228, 229, 230,       \
    232, 233, 234, 235, 236, 237, 238, 239, 240, 241, 241, 242, 243, 244, 244, 245,       \
    245, 246, 247, 247, 248, 248, 248, 249, 249, 249, 249, 250, 250, 250, 250, 250

// G2 code-phase delay in chips for PRN 1..32 (IS-GPS-200 Table 3-Ia; gps.c:273-278).
#define GPSB200_G2_DELAY                                                                  \
    5, 6, 7, 8, 17, 18, 139, 140, 141, 251, 252, 254, 255, 256, 257, 258,                 \
    469, 470, 471, 472, 473, 474, 509, 512, 513, 514, 515, 516, 859, 860, 861, 862

// C/A Gold code chips (0/1) of one PRN: G1 = x^10+x^3+1, G2 = x^10+x^9+x^8+x^6+x^3+x^2+1,
// both registers all ones, G2 delayed per PRN (gps.c:272-309).
inline int ca_code(int prn, uint8_t *ca /*[1023]*/) {
    static const uint16_t delay[32] = {GPSB200_G2_DELAY};
    if (prn < 1 || prn > 32) return -1;
    uint8_t g1[1023], g2[1023];
    unsigned r1 = 0x3FF, r2 = 0x3FF;
    for (int i = 0; i < 1023; i++) {
        g1[i] = (r1 >> 9) & 1;
        g2[i] = (r2 >> 9) & 1;
        unsigned f1 = ((r1 >> 2) ^ (r1 >> 9)) & 1;
        unsigned f2 = ((r2 >> 1) ^ (r2 >> 2) ^ (r2 >> 5) ^ (r2 >> 7) ^ (r2 >> 8) ^ (r2 >> 9)) & 1;
        r1 = ((r1 << 1) | f1) & 0x3FF;
        r2 = ((r2 << 1) | f2) & 0x3FF;
    }
    const int d = delay[prn - 1];
    for (int i = 0; i < 1023; i++) ca[i] = g1[i] ^ g2[(i + 1023 - d) % 1023];
    return 0;
}

// Physical constants of the reference, spelled as gps.h:87-102 spells them: the scenario, the NAV decoder and k_pvt
// all compute with these doubles.
constexpr double kGM = 3.986005e14;               // GM_EARTH
constexpr double kOmegaE = 7.2921151467e-5;       // OMEGA_EARTH
constexpr double kPi = 3.1415926535898;           // PI
constexpr double kWgsA = 6378137.0;               // WGS84_RADIUS
constexpr double kWgsE = 0.0818191908426;         // WGS84_ECCENTRICITY
constexpr double kC = 2.99792458e8;               // SPEED_OF_LIGHT
constexpr double kLambda = 0.190293672798365;     // LAMBDA_L1

inline unsigned parity_of(uint32_t v) { return (unsigned) __builtin_popcount(v) & 1u; }

// IS-GPS-200 parity equations over data bits d1..d24 (word bits 29..6): bit masks of the data bits each parity bit sums.
constexpr uint32_t kParityMask[6] = {0x3B1F3480u, 0x1D8F9A40u, 0x2EC7CD00u, 0x1763E680u, 0x2BB1F340u, 0x0B7A89C0u};

// The six parity bits D25..D30 (D25 in bit 5) of data bits d1..d24 (bits 23..0, before the D30* complement), given
// D29*, D30* of the previous word (computeChecksum, gps.c:1008-1072).
inline uint32_t parity6(uint32_t data24, unsigned d29, unsigned d30) {
    const uint32_t d = (data24 & 0xFFFFFFu) << 6;
    const unsigned star[6] = {d29, d30, d29, d30, d30, d29};
    uint32_t p = 0;
    for (int k = 0; k < 6; k++) p = (p << 1) | ((star[k] + parity_of(kParityMask[k] & d)) & 1u);
    return p;
}

}  // namespace gpsb200
