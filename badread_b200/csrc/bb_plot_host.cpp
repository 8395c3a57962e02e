// bb_plot_host.cpp — the text of `badread_b200 plot --windows`: one line per window, "name\tposition\tidentity" and
// "\tmean qscore" with qualities, the values as printf's "%.4f" writes them (std::to_chars with a precision is specified
// as printf's conversion, so the digits are exact), formatted by several host threads into one buffer.
#include <algorithm>
#include <charconv>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/badread_b200.h"

namespace {

// Lines of points [lo, hi) into out (room for them is the caller's): returns the bytes written.
int64_t format_points(int32_t n_aln, const char *names, const int64_t *name_off, const int64_t *pos0, const int64_t *point_off,
                      const double *identity, const double *qual, int64_t lo, int64_t hi, char *out) {
    char *o = out;
    int32_t a = (int32_t)(std::upper_bound(point_off, point_off + n_aln + 1, lo) - point_off) - 1;
    for (int64_t p = lo; p < hi; p++) {
        while (p >= point_off[a + 1]) a++;
        const int64_t nl = name_off[a + 1] - name_off[a];
        std::memcpy(o, names + name_off[a], (size_t)nl);
        o += nl;
        *o++ = '\t';
        o = std::to_chars(o, o + 24, pos0[a] + (p - point_off[a])).ptr;
        *o++ = '\t';
        o = std::to_chars(o, o + 40, identity[p], std::chars_format::fixed, 4).ptr;
        if (qual) {
            *o++ = '\t';
            o = std::to_chars(o, o + 40, qual[p], std::chars_format::fixed, 4).ptr;
        }
        *o++ = '\n';
    }
    return o - out;
}

}  // namespace

extern "C" int64_t bb_window_line_bound(int64_t name_len) { return name_len + 1 + 24 + 1 + 40 + 1 + 40 + 1; }

extern "C" int bb_window_format(int32_t n_aln, const char *names, const int64_t *name_off, const int64_t *pos0,
                                const int64_t *point_off, const double *identity, const double *qual, int64_t lo, int64_t hi,
                                char *out, int64_t cap, int64_t *out_len) {
    if (n_aln < 0 || !name_off || !point_off || !out_len || lo < 0 || hi < lo || hi > point_off[n_aln] ||
        (hi > lo && (!names || !pos0 || !identity || !out)))
        return BB_ERR_ARG;
    *out_len = 0;
    int64_t longest = 0;
    for (int32_t a = 0; a < n_aln; a++) longest = std::max(longest, name_off[a + 1] - name_off[a]);
    const int64_t line = bb_window_line_bound(longest), n = hi - lo;
    if (n * line > cap) return BB_ERR_CAPACITY;
    const int64_t n_threads = std::max<int64_t>(1, std::min<int64_t>({(int64_t)std::thread::hardware_concurrency(), 32,
                                                                       (n + 65535) / 65536}));
    // each thread formats a contiguous share into its own part of out; the parts are then closed up in order
    std::vector<int64_t> len((size_t)n_threads);
    std::vector<std::thread> pool;
    auto share = [&](int64_t t) { return lo + n * t / n_threads; };
    for (int64_t t = 0; t < n_threads; t++)
        pool.emplace_back([&, t]() {
            len[(size_t)t] = format_points(n_aln, names, name_off, pos0, point_off, identity, qual, share(t), share(t + 1),
                                           out + (share(t) - lo) * line);
        });
    for (auto &th : pool) th.join();
    int64_t at = len[0];
    for (int64_t t = 1; t < n_threads; t++) {
        std::memmove(out + at, out + (share(t) - lo) * line, (size_t)len[(size_t)t]);
        at += len[(size_t)t];
    }
    *out_len = at;
    return BB_OK;
}
