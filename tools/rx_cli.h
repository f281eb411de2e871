// Input of the receiver command-line programs (gpsb200-acq, gpsb200-track): PRN lists, 3 Msps I/Q files, and the
// context their receiver calls run in.
#pragma once
#include <sys/stat.h>

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
