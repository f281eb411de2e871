// Input of the receiver command-line programs (gpsb200-acq, gpsb200-track): PRN lists, 3 Msps I/Q files, the context
// their receiver calls run in, and the a-priori position and time of assisted runs.
#pragma once
#include <sys/stat.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../include/gpsb200.h"

// A PRN list such as "1-32" or "3,7,12-15" into cfg->prn / cfg->nprn; false unless it names 1 to 32 PRNs, all in 1..32.
inline bool parse_prns(const char *s, gpsb200_acq_config_t *cfg) {
    cfg->nprn = 0;
    std::string t(s);
    size_t pos = 0;
    while (pos <= t.size()) {
        size_t end = t.find(',', pos);
        if (end == std::string::npos) end = t.size();
        const std::string item = t.substr(pos, end - pos);
        int a = 0, b = 0;
        if (sscanf(item.c_str(), "%d-%d", &a, &b) == 2) {
        } else if (sscanf(item.c_str(), "%d", &a) == 1) {
            b = a;
        } else {
            return false;
        }
        for (int p = a; p <= b; p++) {
            if (cfg->nprn >= 32 || p < 1 || p > 32) return false;
            cfg->prn[cfg->nprn++] = p;
        }
        pos = end + 1;
    }
    return cfg->nprn > 0;
}

// Whole I,Q samples in the file at path, elem bytes per component; -1 when the file cannot be opened.
inline long long file_samples(const char *path, size_t elem) {
    struct stat st;
    if (stat(path, &st) != 0) return -1;
    return (long long) st.st_size / (long long) (2 * elem);
}

// Samples s0 .. s0 + n - 1 of an open I/Q file into buf; false when they cannot all be read.
inline bool read_at(FILE *f, long long s0, long long n, size_t elem, std::vector<char> &buf) {
    buf.resize((size_t) n * 2 * elem);
    return fseeko(f, (off_t) (s0 * 2 * (long long) elem), SEEK_SET) == 0 && fread(buf.data(), 1, buf.size(), f) == buf.size();
}

// A context on CUDA device `device` for receiver calls only: one channel and one block, the least synthesis can take.
inline int create_rx_context(int device, gpsb200_ctx_t **ctx) {
    gpsb200_config_t cc;
    memset(&cc, 0, sizeof cc);
    cc.device = device;
    cc.max_chan = 1;
    cc.max_blocks = 1;
    return gpsb200_create(&cc, ctx);
}

// GPS week and second of a calendar date and time "YYYY/MM/DD,hh:mm:ss[.s]" (GPS time, no leap seconds): days since
// 1980-01-06.
inline bool gps_of_date(const char *text, int32_t &week, double &sow) {
    int y, mo, d, hh, mm;
    double sec;
    if (sscanf(text, "%d/%d/%d,%d:%d:%lf", &y, &mo, &d, &hh, &mm, &sec) != 6 || y < 1980 || mo < 1 || mo > 12 || d < 1 ||
        d > 31 || hh < 0 || hh > 23 || mm < 0 || mm > 59 || !(sec >= 0.0 && sec < 60.0))
        return false;
    const int a = (14 - mo) / 12, yy = y + 4800 - a, m = mo + 12 * a - 3;
    const long jdn = d + (153 * m + 2) / 5 + 365L * yy + yy / 4 - yy / 100 + yy / 400 - 32045;
    const long days = jdn - 2444245;                // 1980-01-06
    if (days < 0) return false;
    week = (int32_t) (days / 7);
    sow = (double) (days % 7) * 86400.0 + hh * 3600.0 + mm * 60.0 + sec;
    return true;
}

// ECEF (m) of a WGS-84 "LAT,LON,H" (degrees, degrees, m); false unless three numbers are given.
inline bool ecef_of_llh(const char *text, double x[3]) {
    double llh[3];
    if (sscanf(text, "%lf,%lf,%lf", &llh[0], &llh[1], &llh[2]) != 3) return false;
    const double kA = 6378137.0, kE2 = 0.0818191908426 * 0.0818191908426;   // WGS-84
    const double la = llh[0] * M_PI / 180.0, lo = llh[1] * M_PI / 180.0;
    const double N = kA / sqrt(1.0 - kE2 * sin(la) * sin(la));
    x[0] = (N + llh[2]) * cos(la) * cos(lo);
    x[1] = (N + llh[2]) * cos(la) * sin(lo);
    x[2] = (N * (1.0 - kE2) + llh[2]) * sin(la);
    return true;
}
