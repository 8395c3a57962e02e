// bb_tu_em_load.cu — compiles the error model loader (bb_em_load.cuh) and runs its passes over a model file's text in
// device memory (bbl_em_load, declared in bb_launch.h).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <vector>

#include "bb_em_load.cuh"
#include "bb_launch.h"

namespace {

double ms_since(std::chrono::steady_clock::time_point &t) {
    const auto now = std::chrono::steady_clock::now();
    const double ms = std::chrono::duration<double, std::milli>(now - t).count();
    t = now;
    return ms;
}

unsigned blocks(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

struct Scratch {   // device buffers of one load, freed when it returns
    std::vector<void *> ptrs;
    ~Scratch() { for (void *p : ptrs) cudaFree(p); }
    template <typename T> cudaError_t alloc(T **p, int64_t count) {
        void *v = nullptr;
        const cudaError_t e = cudaMalloc(&v, (size_t)std::max<int64_t>(count, 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(v);
        *p = reinterpret_cast<T *>(v);
        return e;
    }
};

// out[0..n] = the exclusive scan of the counts c[0..n) (out[n] their total), through tile sums in `sums`
void scan_counts(cudaStream_t st, const int32_t *c, int64_t n, int64_t *sums, int64_t *out) {
    const int64_t tiles = (n + EML_CNT_TILE - 1) / EML_CNT_TILE;
    if (tiles) eml_k_cnt_sums<<<(unsigned)tiles, EML_THREADS, 0, st>>>(c, n, sums);
    eml_k_scan_sums<<<1, EML_SUMS_THREADS, 0, st>>>(sums, tiles);
    if (tiles) eml_k_cnt_scan<<<(unsigned)tiles, EML_THREADS, 0, st>>>(c, n, sums, out);
    else cudaMemsetAsync(out, 0, sizeof(int64_t), st);
}

template <typename T> cudaError_t fetch(cudaStream_t st, T *h, const T *d) {
    cudaError_t e = cudaMemcpyAsync(h, d, sizeof(T), cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
}

}  // namespace

#define EML_CUDA(call)                                                                            \
    do {                                                                                          \
        const cudaError_t e_ = (call);                                                            \
        if (e_ != cudaSuccess) {                                                                  \
            std::snprintf(msg, msg_len, "error model load: %s: %s", #call, cudaGetErrorString(e_)); \
            return BB_ERR_CUDA;                                                                   \
        }                                                                                         \
    } while (0)

int bbl_em_load(cudaStream_t st, const uint8_t *text, int64_t n, bool dense, bb_em_load_info *info, BBEmLoadOut *out,
                char *msg, size_t msg_len) {
    msg[0] = 0;
    *out = BBEmLoadOut{};
    auto t = std::chrono::steady_clock::now();
    // k: the length of the first line's first token
    uint8_t head[EML_MAX_K + 2] = {};
    const int64_t nh = std::min<int64_t>(n, (int64_t)sizeof(head));
    if (nh) EML_CUDA(cudaMemcpy(head, text, (size_t)nh, cudaMemcpyDeviceToHost));
    int k = 0;
    while (k < nh && head[k] != ',') k++;
    if (n == 0) { info->fallback |= BB_EM_FALLBACK_EMPTY_LINE; return BB_OK; }
    if (k == nh || k < 3 || k > EML_MAX_K) { info->fallback |= BB_EM_FALLBACK_K; return BB_OK; }
    info->k = k;

    // 1. line starts
    Scratch S;
    const int64_t text_tiles = (n + EML_TEXT_TILE - 1) / EML_TEXT_TILE;
    int64_t *tsum, *starts;
    int *flag;
    EML_CUDA(S.alloc(&tsum, text_tiles + 1));
    EML_CUDA(S.alloc(&flag, 2));
    EML_CUDA(cudaMemsetAsync(flag, 0, 2 * sizeof(int), st));
    eml_k_nl_count<<<(unsigned)text_tiles, EML_THREADS, 0, st>>>(text, n, EML_TEXT_TILE, tsum);
    eml_k_scan_sums<<<1, EML_SUMS_THREADS, 0, st>>>(tsum, text_tiles);
    int64_t n_nl = 0;
    uint8_t last = 0;
    EML_CUDA(cudaMemcpyAsync(&last, text + n - 1, 1, cudaMemcpyDeviceToHost, st));
    EML_CUDA(fetch(st, &n_nl, tsum + text_tiles));
    const int64_t n_lines = n_nl + (last != '\n' ? 1 : 0);
    if (n_lines > INT32_MAX) { info->fallback |= BB_EM_FALLBACK_SIZE; return BB_OK; }
    EML_CUDA(S.alloc(&starts, n_lines + 1));
    eml_k_nl_emit<<<(unsigned)text_tiles, EML_THREADS, 0, st>>>(text, n, EML_TEXT_TILE, tsum, starts);

    // 2. lines checked, alternatives counted
    int32_t *n_alt;
    int64_t *alt_base, *csum;
    EML_CUDA(cudaMalloc(&out->codes, (size_t)n_lines * sizeof(int64_t)));
    EML_CUDA(S.alloc(&n_alt, n_lines));
    EML_CUDA(S.alloc(&alt_base, n_lines + 1));
    EML_CUDA(S.alloc(&csum, (n_lines + EML_CNT_TILE - 1) / EML_CNT_TILE + 1));
    eml_k_lines<<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(text, starts, n_lines, k, n_alt, out->codes, flag);
    int fb = 0;
    EML_CUDA(fetch(st, &fb, flag));
    info->ms_parse = ms_since(t);
    info->n_rows = n_lines;
    if (fb) { info->fallback |= (uint32_t)fb; return BB_OK; }
    scan_counts(st, n_alt, n_lines, csum, alt_base);
    int64_t n_alts = 0;
    EML_CUDA(fetch(st, &n_alts, alt_base + n_lines));
    info->n_alts = n_alts;

    // 3. alternatives placed, remainders
    int64_t *alt_pos, *row_off64;
    uint8_t *alt_len;
    int32_t *alt_row, *n_ent;
    double *alt_prob, *rem;
    EML_CUDA(S.alloc(&alt_pos, n_alts));
    EML_CUDA(S.alloc(&alt_len, n_alts));
    EML_CUDA(S.alloc(&alt_row, n_alts));
    EML_CUDA(S.alloc(&alt_prob, n_alts));
    EML_CUDA(S.alloc(&n_ent, n_lines));
    EML_CUDA(S.alloc(&rem, n_lines));
    EML_CUDA(S.alloc(&row_off64, n_lines + 1));
    eml_k_alts<<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(text, starts, n_lines, k, alt_base, alt_pos,
                                                                              alt_len, alt_row, alt_prob, n_ent, rem);
    scan_counts(st, n_ent, n_lines, csum, row_off64);
    int64_t n_entries = 0;
    EML_CUDA(fetch(st, &n_entries, row_off64 + n_lines));
    info->n_entries = n_entries;
    if (n_entries > INT32_MAX) { info->fallback |= BB_EM_FALLBACK_SIZE; return BB_OK; }
    info->ms_parse += ms_since(t);

    // 4. alignments: pooled bytes, their scan, then slots, flags and pool
    int32_t *pooled;
    int64_t *pool_off, *asum;
    EML_CUDA(S.alloc(&pooled, n_alts));
    EML_CUDA(S.alloc(&pool_off, n_alts + 1));
    EML_CUDA(S.alloc(&asum, (n_alts + EML_CNT_TILE - 1) / EML_CNT_TILE + 1));
    const unsigned ab = blocks(n_alts, EML_ALIGN_THREADS);
    if (ab) eml_k_align<false><<<ab, EML_ALIGN_THREADS, 0, st>>>(text, n_alts, k, starts, alt_pos, alt_len, alt_row, alt_base,
                                                                 row_off64, pooled, nullptr, nullptr, nullptr, nullptr, nullptr);
    scan_counts(st, pooled, n_alts, asum, pool_off);
    int64_t pool_len = 0;
    EML_CUDA(fetch(st, &pool_len, pool_off + n_alts));
    info->pool_bytes = pool_len;
    EML_CUDA(cudaMalloc(&out->slots, (size_t)std::max<int64_t>(n_entries * k, 1) * sizeof(uint32_t)));
    EML_CUDA(cudaMalloc(&out->flags, (size_t)std::max<int64_t>(n_entries, 1)));
    EML_CUDA(cudaMalloc(&out->pool, (size_t)std::max<int64_t>(pool_len, 1)));
    if (!pool_len) EML_CUDA(cudaMemsetAsync(out->pool, 0, 1, st));   // (the host tables keep one byte of an empty pool)
    if (ab) eml_k_align<true><<<ab, EML_ALIGN_THREADS, 0, st>>>(text, n_alts, k, starts, alt_pos, alt_len, alt_row, alt_base,
                                                                row_off64, nullptr, pool_off, out->slots, out->flags, out->pool,
                                                                flag + 1);
    int cap = 0;
    EML_CUDA(fetch(st, &cap, flag + 1));
    info->ms_align = ms_since(t);
    if (cap) {
        std::snprintf(msg, msg_len, "error model: the slot pool outgrows %lld bytes", (long long)EML_POOL_LIMIT);
        return BB_ERR_CAPACITY;
    }

    // 5. rows and the dense index
    EML_CUDA(cudaMalloc(&out->row_off, (size_t)(n_lines + 1) * sizeof(int32_t)));
    EML_CUDA(cudaMalloc(&out->cum, (size_t)n_entries * sizeof(double)));
    EML_CUDA(cudaMalloc(&out->probs, (size_t)n_entries * sizeof(double)));
    EML_CUDA(cudaMalloc(&out->rowinfo, (size_t)n_lines * sizeof(BBRowInfo)));
    if (dense && k <= 12) {
        EML_CUDA(cudaMalloc(&out->kmer_to_row, ((size_t)1 << (2 * k)) * sizeof(int32_t)));
        EML_CUDA(cudaMemsetAsync(out->kmer_to_row, 0xff, ((size_t)1 << (2 * k)) * sizeof(int32_t), st));
    }
    eml_k_rows<BBRowInfo><<<blocks(n_lines, EML_LINE_THREADS), EML_LINE_THREADS, 0, st>>>(
        n_lines, k, alt_base, alt_prob, rem, row_off64, out->codes, out->row_off, out->cum, out->probs, out->flags, out->slots,
        out->rowinfo, out->kmer_to_row, flag);
    EML_CUDA(cudaGetLastError());
    EML_CUDA(fetch(st, &fb, flag));
    info->ms_tables = ms_since(t);
    info->fallback |= (uint32_t)fb;
    return BB_OK;
}

void bbl_em_load_free(BBEmLoadOut *out) {
    for (void *p : {(void *)out->kmer_to_row, (void *)out->codes, (void *)out->row_off, (void *)out->cum, (void *)out->probs,
                    (void *)out->flags, (void *)out->slots, (void *)out->pool, (void *)out->rowinfo})
        if (p) cudaFree(p);
    *out = BBEmLoadOut{};
}
