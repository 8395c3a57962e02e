// emu_em_load.cpp — the error model loader (badread_b200/csrc/bb_em_load.cuh) under the warp emulator, CTA by CTA, in the
// order bbl_em_load (bb_tu_em_load.cu) runs its passes, with the text tile size as an argument so that tests can put tile
// edges anywhere (TEST INFRASTRUCTURE).  Built with fewer threads per tile CTA than the device (EML_THREADS,
// EML_SUMS_THREADS below) to keep the emulator fast; the code paths are the same.
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_em_load.cuh"

namespace {

struct RowInfo {   // BBRowInfo's fields (bb_kernels.cuh)
    double cum_last, cum0;
    int32_t e0, ne, first_is_identity, pad;
};

struct Tables {
    int64_t k = 0, n_rows = 0, n_entries = 0, n_alts = 0, pool_bytes = 0, fallback = 0;
    std::vector<int32_t> k2r, row_off;
    std::vector<int64_t> codes;
    std::vector<double> cum, probs;
    std::vector<uint8_t> flags, pool;
    std::vector<uint32_t> slots;
    std::vector<RowInfo> info;
} g;

template <typename F> void grid(int64_t n_blocks, int threads, F &&f) {
    gridDim.x = (unsigned)n_blocks;
    for (int64_t b = 0; b < n_blocks; b++) {
        blockIdx.x = (unsigned)b;
        emu::run_block(threads, f);
    }
    gridDim.x = 1;
    blockIdx.x = 0;
}

int64_t blocks(int64_t n, int t) { return (n + t - 1) / t; }

void scan_counts(const int32_t *c, int64_t n, int64_t *out) {
    const int64_t tiles = blocks(n, EML_CNT_TILE);
    std::vector<int64_t> sums((size_t)tiles + 1);
    grid(tiles, EML_THREADS, [&]() { eml_k_cnt_sums(c, n, sums.data()); });
    grid(1, EML_SUMS_THREADS, [&]() { eml_k_scan_sums(sums.data(), tiles); });
    if (tiles) grid(tiles, EML_THREADS, [&]() { eml_k_cnt_scan(c, n, sums.data(), out); });
    else out[0] = 0;
}

}  // namespace

// Runs the loader over text[0..n); counts[] = k, rows, entries, alternatives, pool bytes, fallback bits, pool overflow.
// The tables stay here for emu_em_fetch.  dense: build kmer_to_row (k <= 12).
extern "C" __attribute__((visibility("default")))
int emu_em_load(const uint8_t *text_in, int64_t n, int32_t tile, int dense, int64_t *counts) {
    g = Tables{};
    for (int i = 0; i < 7; i++) counts[i] = 0;
    std::vector<uint8_t> text(text_in, text_in + n);
    int k = 0;
    while (k < n && k < EML_MAX_K + 2 && text[(size_t)k] != ',') k++;
    if (n == 0) { counts[5] = BB_EM_FALLBACK_EMPTY_LINE; return 0; }
    if (k == n || k == EML_MAX_K + 2 || k < 3 || k > EML_MAX_K) { counts[5] = BB_EM_FALLBACK_K; return 0; }
    g.k = k;
    const int64_t text_tiles = blocks(n, tile);
    std::vector<int64_t> tsum((size_t)text_tiles + 1);
    grid(text_tiles, EML_THREADS, [&]() { eml_k_nl_count(text.data(), n, tile, tsum.data()); });
    grid(1, EML_SUMS_THREADS, [&]() { eml_k_scan_sums(tsum.data(), text_tiles); });
    const int64_t n_lines = tsum[(size_t)text_tiles] + (text[(size_t)n - 1] != '\n' ? 1 : 0);
    std::vector<int64_t> starts((size_t)n_lines + 1, -7);
    grid(text_tiles, EML_THREADS, [&]() { eml_k_nl_emit(text.data(), n, tile, tsum.data(), starts.data()); });
    for (int64_t v : starts) if (v < 0) return -3;   // a line start never written

    int fb[2] = {0, 0};
    std::vector<int32_t> n_alt((size_t)n_lines);
    std::vector<int64_t> alt_base((size_t)n_lines + 1);
    g.codes.assign((size_t)n_lines, 0);
    grid(blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS,
         [&]() { eml_k_lines(text.data(), starts.data(), n_lines, k, n_alt.data(), g.codes.data(), fb); });
    counts[0] = k;
    counts[1] = g.n_rows = n_lines;
    if (fb[0]) { counts[5] = fb[0]; return 0; }
    scan_counts(n_alt.data(), n_lines, alt_base.data());
    const int64_t n_alts = alt_base[(size_t)n_lines];
    counts[3] = n_alts;

    std::vector<int64_t> alt_pos((size_t)n_alts), row_off64((size_t)n_lines + 1);
    std::vector<uint8_t> alt_len((size_t)n_alts);
    std::vector<int32_t> alt_row((size_t)n_alts), n_ent((size_t)n_lines);
    std::vector<double> alt_prob((size_t)n_alts), rem((size_t)n_lines);
    grid(blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, [&]() {
        eml_k_alts(text.data(), starts.data(), n_lines, k, alt_base.data(), alt_pos.data(), alt_len.data(), alt_row.data(),
                   alt_prob.data(), n_ent.data(), rem.data());
    });
    scan_counts(n_ent.data(), n_lines, row_off64.data());
    const int64_t ne = row_off64[(size_t)n_lines];
    counts[2] = ne;

    std::vector<int32_t> pooled((size_t)n_alts);
    std::vector<int64_t> pool_off((size_t)n_alts + 1);
    grid(blocks(n_alts, EML_ALIGN_THREADS), EML_ALIGN_THREADS, [&]() {
        eml_k_align<false>(text.data(), n_alts, k, starts.data(), alt_pos.data(), alt_len.data(), alt_row.data(),
                           alt_base.data(), row_off64.data(), pooled.data(), nullptr, nullptr, nullptr, nullptr, nullptr);
    });
    scan_counts(pooled.data(), n_alts, pool_off.data());
    const int64_t pool_len = pool_off[(size_t)n_alts];
    counts[4] = pool_len;
    g.slots.assign((size_t)(ne * k), 0xdeadbeefu);
    g.flags.assign((size_t)ne, 0xee);
    g.pool.assign((size_t)std::max<int64_t>(pool_len, 1), 0);
    grid(blocks(n_alts, EML_ALIGN_THREADS), EML_ALIGN_THREADS, [&]() {
        eml_k_align<true>(text.data(), n_alts, k, starts.data(), alt_pos.data(), alt_len.data(), alt_row.data(),
                          alt_base.data(), row_off64.data(), nullptr, pool_off.data(), g.slots.data(), g.flags.data(),
                          g.pool.data(), fb + 1);
    });
    counts[6] = fb[1];
    if (fb[1]) return 0;

    g.row_off.assign((size_t)n_lines + 1, -7);
    g.cum.assign((size_t)ne, -1.0);
    g.probs.assign((size_t)ne, -1.0);
    g.info.assign((size_t)n_lines, RowInfo{});
    if (dense && k <= 12) g.k2r.assign((size_t)1 << (2 * k), -1);
    grid(blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, [&]() {
        eml_k_rows<RowInfo>(n_lines, k, alt_base.data(), alt_prob.data(), rem.data(), row_off64.data(), g.codes.data(),
                            g.row_off.data(), g.cum.data(), g.probs.data(), g.flags.data(), g.slots.data(), g.info.data(),
                            g.k2r.empty() ? nullptr : g.k2r.data(), fb);
    });
    counts[5] = fb[0];
    g.n_entries = ne;
    return 0;
}

// The tables of the last emu_em_load; rowinfo[5 * n_rows] = cum_last, cum0, e0, ne, first_is_identity of each row
extern "C" __attribute__((visibility("default")))
int emu_em_fetch(int32_t *k2r, int64_t *codes, int32_t *row_off, double *cum, double *probs, uint8_t *flags, uint32_t *slots,
                 uint8_t *pool, double *rowinfo) {
    if (k2r) std::copy(g.k2r.begin(), g.k2r.end(), k2r);
    std::copy(g.codes.begin(), g.codes.end(), codes);
    std::copy(g.row_off.begin(), g.row_off.end(), row_off);
    std::copy(g.cum.begin(), g.cum.end(), cum);
    std::copy(g.probs.begin(), g.probs.end(), probs);
    std::copy(g.flags.begin(), g.flags.end(), flags);
    std::copy(g.slots.begin(), g.slots.end(), slots);
    std::copy(g.pool.begin(), g.pool.end(), pool);
    for (size_t r = 0; r < g.info.size(); r++) {
        const RowInfo &ri = g.info[r];
        const double v[5] = {ri.cum_last, ri.cum0, (double)ri.e0, (double)ri.ne, (double)ri.first_is_identity};
        std::copy(v, v + 5, rowinfo + 5 * r);
    }
    return 0;
}

// eml_parse_prob on one string: 1 and *out on the fast path, 0 off it (p must then be anything)
extern "C" __attribute__((visibility("default")))
int emu_em_parse_prob(const uint8_t *s, int64_t n, double *out, int64_t *end) {
    int64_t p = 0;
    const bool ok = eml_parse_prob(s, p, n, *out);
    *end = p;
    return ok ? 1 : 0;
}

// EmlPySum over x[0..n): CPython 3.12's sum(x)
extern "C" __attribute__((visibility("default")))
double emu_em_pysum(const double *x, int64_t n) {
    EmlPySum s;
    for (int64_t i = 0; i < n; i++) s.add(x[i], i == 0);
    return n ? s.result() : 0.0;
}
