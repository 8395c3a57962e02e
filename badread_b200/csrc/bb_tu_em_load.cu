// bb_tu_em_load.cu — compiles the error model loader (bb_em_load.cuh) and runs its passes over a model file's text in
// device memory (bbl_em_load, declared in bb_call.h).
#include <algorithm>
#include <chrono>

#include "bb_call.h"
#include "bb_em_load.cuh"
#include "bb_kernels.cuh"

namespace {

double ms_since(std::chrono::steady_clock::time_point &t) {
    const auto now = std::chrono::steady_clock::now();
    const double ms = std::chrono::duration<double, std::milli>(now - t).count();
    t = now;
    return ms;
}

unsigned blocks(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// out[0..n] = the exclusive scan of the counts c[0..n) (out[n] their total), through tile sums in `sums`
void scan_counts(cudaStream_t st, const int32_t *c, int64_t n, int64_t *sums, int64_t *out) {
    const int64_t tiles = (n + EML_CNT_TILE - 1) / EML_CNT_TILE;
    if (tiles) eml_k_cnt_sums<<<(unsigned)tiles, EML_THREADS, 0, st>>>(c, n, sums);
    eml_k_scan_sums<<<1, EML_SUMS_THREADS, 0, st>>>(sums, tiles);
    if (tiles) eml_k_cnt_scan<<<(unsigned)tiles, EML_THREADS, 0, st>>>(c, n, sums, out);
    else cudaMemsetAsync(out, 0, sizeof(int64_t), st);
}

}  // namespace

// (a CUDA failure is reported as "error model load: <what>: <error>")
void bbl_em_load(cudaStream_t st, const uint8_t *text, int64_t n, bool dense, bb_em_load_info *info, BBEmLoadOut *out) {
    *out = BBEmLoadOut{};
    const char *what = "error model load";
    auto t = std::chrono::steady_clock::now();
    // k: the length of the first line's first token
    uint8_t head[EML_MAX_K + 2] = {};
    const int64_t nh = std::min<int64_t>(n, (int64_t)sizeof(head));
    d2h(head, text, nh);
    int k = 0;
    while (k < nh && head[k] != ',') k++;
    if (n == 0) { info->fallback |= BB_EM_FALLBACK_EMPTY_LINE; return; }
    if (k == nh || k < 3 || k > EML_MAX_K) { info->fallback |= BB_EM_FALLBACK_K; return; }
    info->k = k;

    // 1. line starts
    Scratch S;
    const int64_t text_tiles = (n + EML_TEXT_TILE - 1) / EML_TEXT_TILE;
    int64_t *tsum = S.get<int64_t>(text_tiles + 1, what);
    int *flag = S.get<int>(2, what);
    check(cudaMemsetAsync(flag, 0, 2 * sizeof(int), st), "error model load: cudaMemsetAsync");
    eml_k_nl_count<<<(unsigned)text_tiles, EML_THREADS, 0, st>>>(text, n, EML_TEXT_TILE, tsum);
    eml_k_scan_sums<<<1, EML_SUMS_THREADS, 0, st>>>(tsum, text_tiles);
    int64_t n_nl = 0;
    uint8_t last = 0;
    check(cudaMemcpyAsync(&last, text + n - 1, 1, cudaMemcpyDeviceToHost, st), "error model load: cudaMemcpyAsync");
    d2h(&n_nl, tsum + text_tiles, 1, st);
    const int64_t n_lines = n_nl + (last != '\n' ? 1 : 0);
    if (n_lines > INT32_MAX) { info->fallback |= BB_EM_FALLBACK_SIZE; return; }
    int64_t *starts = S.get<int64_t>(n_lines + 1, what);
    eml_k_nl_emit<<<(unsigned)text_tiles, EML_THREADS, 0, st>>>(text, n, EML_TEXT_TILE, tsum, starts);

    // 2. lines checked, alternatives counted
    out->codes = S.result((size_t)n_lines * sizeof(int64_t), what);
    int32_t *n_alt = S.get<int32_t>(n_lines, what);
    int64_t *alt_base = S.get<int64_t>(n_lines + 1, what);
    int64_t *csum = S.get<int64_t>((n_lines + EML_CNT_TILE - 1) / EML_CNT_TILE + 1, what);
    eml_k_lines<<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(text, starts, n_lines, k, n_alt,
                                                                               out->codes.as<int64_t>(), flag);
    int fb = 0;
    d2h(&fb, flag, 1, st);
    info->ms_parse = ms_since(t);
    info->n_rows = n_lines;
    if (fb) { info->fallback |= (uint32_t)fb; return; }
    scan_counts(st, n_alt, n_lines, csum, alt_base);
    int64_t n_alts = 0;
    d2h(&n_alts, alt_base + n_lines, 1, st);
    info->n_alts = n_alts;

    // 3. alternatives placed, remainders
    int64_t *alt_pos = S.get<int64_t>(n_alts, what);
    uint8_t *alt_len = S.get<uint8_t>(n_alts, what);
    int32_t *alt_row = S.get<int32_t>(n_alts, what);
    double *alt_prob = S.get<double>(n_alts, what);
    int32_t *n_ent = S.get<int32_t>(n_lines, what);
    double *rem = S.get<double>(n_lines, what);
    int64_t *row_off64 = S.get<int64_t>(n_lines + 1, what);
    eml_k_alts<<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(text, starts, n_lines, k, alt_base, alt_pos,
                                                                              alt_len, alt_row, alt_prob, n_ent, rem);
    scan_counts(st, n_ent, n_lines, csum, row_off64);
    int64_t n_entries = 0;
    d2h(&n_entries, row_off64 + n_lines, 1, st);
    info->n_entries = n_entries;
    if (n_entries > INT32_MAX) { info->fallback |= BB_EM_FALLBACK_SIZE; return; }
    info->ms_parse += ms_since(t);

    // 4. alignments: pooled bytes, their scan, then slots, flags and pool
    int32_t *pooled = S.get<int32_t>(n_alts, what);
    int64_t *pool_off = S.get<int64_t>(n_alts + 1, what);
    int64_t *asum = S.get<int64_t>((n_alts + EML_CNT_TILE - 1) / EML_CNT_TILE + 1, what);
    const unsigned ab = blocks(n_alts, EML_ALIGN_THREADS);
    if (ab) eml_k_align<false><<<ab, EML_ALIGN_THREADS, 0, st>>>(text, n_alts, k, starts, alt_pos, alt_len, alt_row, alt_base,
                                                                 row_off64, pooled, nullptr, nullptr, nullptr, nullptr, nullptr);
    scan_counts(st, pooled, n_alts, asum, pool_off);
    int64_t pool_len = 0;
    d2h(&pool_len, pool_off + n_alts, 1, st);
    info->pool_bytes = pool_len;
    out->slots = S.result((size_t)n_entries * k * sizeof(uint32_t), what);
    out->flags = S.result((size_t)n_entries, what);
    out->pool = S.result((size_t)pool_len, what);
    if (!pool_len) check(cudaMemsetAsync(out->pool.p, 0, 1, st), "error model load: cudaMemsetAsync");   // (the host tables keep one byte of an empty pool)
    if (ab) eml_k_align<true><<<ab, EML_ALIGN_THREADS, 0, st>>>(text, n_alts, k, starts, alt_pos, alt_len, alt_row, alt_base,
                                                                row_off64, nullptr, pool_off, out->slots.as<uint32_t>(),
                                                                out->flags.as<uint8_t>(), out->pool.as<uint8_t>(), flag + 1);
    int cap = 0;
    d2h(&cap, flag + 1, 1, st);
    info->ms_align = ms_since(t);
    if (cap) throw Fail{BB_ERR_CAPACITY, "error model: the slot pool outgrows " + std::to_string(EML_POOL_LIMIT) + " bytes"};

    // 5. rows and the dense index
    out->row_off = S.result((size_t)(n_lines + 1) * sizeof(int32_t), what);
    out->cum = S.result((size_t)n_entries * sizeof(double), what);
    out->probs = S.result((size_t)n_entries * sizeof(double), what);
    out->rowinfo = S.result((size_t)n_lines * sizeof(BBRowInfo), what);
    if (dense && k <= 12) {
        out->kmer_to_row = S.result(((size_t)1 << (2 * k)) * sizeof(int32_t), what);
        check(cudaMemsetAsync(out->kmer_to_row.p, 0xff, ((size_t)1 << (2 * k)) * sizeof(int32_t), st), "error model load: cudaMemsetAsync");
    }
    eml_k_rows<BBRowInfo><<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(
        n_lines, k, alt_base, alt_prob, rem, row_off64, out->codes.as<int64_t>(), out->row_off.as<int32_t>(), out->cum.as<double>(),
        out->probs.as<double>(), out->flags.as<uint8_t>(), out->slots.as<uint32_t>(), out->rowinfo.as<BBRowInfo>(),
        out->kmer_to_row.as<int32_t>(), flag);
    check(cudaGetLastError(), "error model load: eml_k_rows");
    d2h(&fb, flag, 1, st);
    info->ms_tables = ms_since(t);
    info->fallback |= (uint32_t)fb;
}
