// bb_em_load.cuh — an error model file (its text, inflated if it was gzip) parsed into the simulate tables on the device,
// with the semantics of ErrorModel.load_from_file + _build_tables (error_model.py) on the files the builders write:
//   line      kmer,p;alt,p;...;   (the trailing ';' optional), one line per k-mer, '\n' line ends
//   row       one per line, in file order; its entries are the line's alternatives, then the "random change" remainder
//             entry (flags 2, slots BB_SLOT_NONE) when 1.0 - sum(probs) > 0, with CPython 3.12's compensated sum()
//   slots     align_kmers (bb_host.cpp small_nw_path + bb_host_align_kmers): a slot of up to 3 bases inline, a longer
//             one in the pool, pool bytes appended in file order
// Anything off that fast path (another number form, a duplicate k-mer, mixed k, a non-ACGT base, an empty line, a stray
// separator, '\r', an alternative of more than EML_MAX_ALT bases) sets a BB_EM_FALLBACK_* bit instead: the caller then
// loads the file with the host loader, which keeps its messages and assertions.
//
// Passes (every offset 64-bit):
//  1. eml_k_nl_count / eml_k_scan_sums / eml_k_nl_emit: newlines per tile of text, their scan, each line's start
//  2. eml_k_lines: one thread per line checks it and counts its alternatives; eml_k_cnt_* scan the counts
//  3. eml_k_alts: one thread per line places its alternatives and their probabilities, and its remainder
//  4. eml_k_align<false> / <true>: one thread per alternative aligns it to its k-mer, first for its pooled bytes (scanned
//     into pool offsets), then to write its slots, flags and pool bytes
//  5. eml_k_rows: one thread per row writes probs, cum, the remainder entry, the row summaries and the dense index
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>

#include "../../include/badread_b200.h"

#ifndef EML_THREADS
#define EML_THREADS 256          // threads of the tile kernels (text and count tiles)
#endif
#ifndef EML_SUMS_THREADS
#define EML_SUMS_THREADS 1024    // threads of the one CTA of eml_k_scan_sums
#endif
#define EML_ITEMS 8                          // counts per thread of a count tile
#define EML_CNT_TILE (EML_THREADS * EML_ITEMS)
#define EML_TEXT_TILE 16384                  // bytes per text tile; any value in 1 .. 2^30 parses the same
#define EML_LINE_THREADS 128                 // threads of the per-line and per-row kernels
#define EML_ALIGN_THREADS 64                 // threads of eml_k_align (its traceback rows live in shared memory)
#define EML_MAX_K 16
#define EML_MAX_ALT 64                       // longest alternative on the fast path
#define EML_POOL_LIMIT (1ll << 24)           // a pooled slot's offset fits 24 bits (bb_host_align_kmers)
#define EML_SLOT_NONE 0xFFFFFFFFu

// ---- scans
// Exclusive block scan of the threads' values in thread order; *total = the block's sum.  Every thread must call it.
__device__ __forceinline__ int64_t eml_block_exscan(int64_t v, int64_t *total) {
    __shared__ int64_t s_warp[EML_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = v;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    int64_t before = 0, all = 0;
    for (int k = 0; k < EML_THREADS / 32; k++) {
        if (k == w) before = all;
        all += s_warp[k];
    }
    __syncthreads();   // (s_warp is reused by the next call)
    *total = all;
    return before + inc - v;
}

// One CTA: v[0..n) becomes its exclusive prefix sums, v[n] the total (v has n + 1 entries)
__global__ void __launch_bounds__(EML_SUMS_THREADS) eml_k_scan_sums(int64_t *__restrict__ v, int64_t n) {
    __shared__ int64_t s[EML_SUMS_THREADS];
    const int64_t per = (n + EML_SUMS_THREADS - 1) / EML_SUMS_THREADS;
    const int64_t c0 = (int64_t)threadIdx.x * per < n ? (int64_t)threadIdx.x * per : n;
    const int64_t c1 = c0 + per < n ? c0 + per : n;
    int64_t sum = 0;
    for (int64_t t = c0; t < c1; t++) sum += v[t];
    s[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t run = 0;
        for (int r = 0; r < EML_SUMS_THREADS; r++) {
            const int64_t x = s[r];
            s[r] = run;
            run += x;
        }
        v[n] = run;
    }
    __syncthreads();
    int64_t run = s[threadIdx.x];
    for (int64_t t = c0; t < c1; t++) {
        const int64_t x = v[t];
        v[t] = run;
        run += x;
    }
}

// The counts c[0..n) in tiles of EML_CNT_TILE: sums[t] = tile t's sum
__global__ void __launch_bounds__(EML_THREADS)
eml_k_cnt_sums(const int32_t *__restrict__ c, int64_t n, int64_t *__restrict__ sums) {
    const int64_t i0 = (int64_t)blockIdx.x * EML_CNT_TILE + (int64_t)threadIdx.x * EML_ITEMS;
    int64_t s = 0;
    for (int j = 0; j < EML_ITEMS; j++)
        if (i0 + j < n) s += c[i0 + j];
    int64_t total;
    eml_block_exscan(s, &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// out[i] = c[0] + .. + c[i - 1] for i <= n, from the scanned tile sums
__global__ void __launch_bounds__(EML_THREADS)
eml_k_cnt_scan(const int32_t *__restrict__ c, int64_t n, const int64_t *__restrict__ tile_off, int64_t *__restrict__ out) {
    const int64_t i0 = (int64_t)blockIdx.x * EML_CNT_TILE + (int64_t)threadIdx.x * EML_ITEMS;
    int64_t s = 0;
    for (int j = 0; j < EML_ITEMS; j++)
        if (i0 + j < n) s += c[i0 + j];
    int64_t total;
    int64_t run = tile_off[blockIdx.x] + eml_block_exscan(s, &total);
    for (int j = 0; j < EML_ITEMS && i0 + j < n; j++) {
        out[i0 + j] = run;
        run += c[i0 + j];
        if (i0 + j == n - 1) out[n] = run;
    }
}

// ---- lines
// Thread threadIdx.x's bytes [a, b) of the tile of `tile` bytes
__device__ __forceinline__ void eml_tile_range(int64_t n, int32_t tile, int64_t &a, int64_t &b) {
    const int64_t t0 = (int64_t)blockIdx.x * tile, t1 = t0 + tile < n ? t0 + tile : n;
    const int32_t per = (tile + EML_THREADS - 1) / EML_THREADS;
    a = t0 + (int64_t)threadIdx.x * per < t1 ? t0 + (int64_t)threadIdx.x * per : t1;
    b = a + per < t1 ? a + per : t1;
}

// f(c, i) for the bytes text[a..b) in order, 16 at a time where they are aligned
template <typename F>
__device__ __forceinline__ void eml_each_byte(const uint8_t *__restrict__ text, int64_t a, int64_t b, F &&f) {
    int64_t i = a;
    for (; i < b && (i & 15); i++) f((uint32_t)text[i], i);
    for (; i + 16 <= b; i += 16) {
        const uint4 v = *reinterpret_cast<const uint4 *>(text + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 16; j++) f((w[j >> 2] >> (8 * (j & 3))) & 0xffu, i + j);
    }
    for (; i < b; i++) f((uint32_t)text[i], i);
}

__device__ __forceinline__ int64_t eml_newlines(const uint8_t *__restrict__ text, int64_t a, int64_t b) {
    int64_t c = 0;
    eml_each_byte(text, a, b, [&](uint32_t x, int64_t) { c += x == '\n'; });
    return c;
}

// sums[t] = newlines in tile t
__global__ void __launch_bounds__(EML_THREADS)
eml_k_nl_count(const uint8_t *__restrict__ text, int64_t n, int32_t tile, int64_t *__restrict__ sums) {
    int64_t a, b, total;
    eml_tile_range(n, tile, a, b);
    eml_block_exscan(eml_newlines(text, a, b), &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// starts[0] = 0 and starts[l + 1] = the byte after the l-th newline; when the text does not end in a newline, the last
// line's entry after it is n + 1.  So line l is text[starts[l] .. starts[l + 1] - 1) without its newline.
__global__ void __launch_bounds__(EML_THREADS)
eml_k_nl_emit(const uint8_t *__restrict__ text, int64_t n, int32_t tile, const int64_t *__restrict__ tile_off,
              int64_t *__restrict__ starts) {
    int64_t a, b, total;
    eml_tile_range(n, tile, a, b);
    int64_t p = tile_off[blockIdx.x] + eml_block_exscan(eml_newlines(text, a, b), &total);
    if (blockIdx.x == 0 && threadIdx.x == 0) starts[0] = 0;
    eml_each_byte(text, a, b, [&](uint32_t c, int64_t i) {
        if (c == '\n') starts[++p] = i + 1;
    });
    if (a < b && b == n && text[n - 1] != '\n') starts[p + 1] = n + 1;
}

// ---- one line
__device__ __forceinline__ int eml_base(uint32_t c) {
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}

// float(text[p..)) for a probability on Clinger's fast path: digits with an optional '.' and fraction, the significand
// m below 2^53 and at most 22 fraction digits d, so that m and 10^d are exact doubles and m / 10^d, one correctly rounded
// division, is what float() gives.  p ends at the first byte after the number; false off the fast path.
__device__ __forceinline__ bool eml_parse_prob(const uint8_t *__restrict__ text, int64_t &p, int64_t e, double &out) {
    uint64_t m = 0;
    int digits = 0, frac = -1;
    for (; p < e; p++) {
        const uint32_t c = text[p];
        if (c >= '0' && c <= '9') {
            m = m * 10u + (c - '0');
            if (m >= (1ull << 53)) return false;
            digits++;
            if (frac >= 0) frac++;
        } else if (c == '.' && frac < 0) {
            frac = 0;
        } else {
            break;
        }
    }
    if (digits == 0 || frac > 22) return false;
    double p10 = 1.0;
    for (int i = 0; i < frac; i++) p10 = __dmul_rn(p10, 10.0);   // exact: 10^22 < 2^53 * 2^22
    out = __ddiv_rn((double)m, p10);
    return true;
}

// CPython 3.12's sum() of floats (Neumaier's compensated sum, Python/bltinmodule.c): the int start 0 plus the first item,
// then every item with its compensation, the compensation added at the end when it is non-zero and finite.
struct EmlPySum {
    double f = 0.0, c = 0.0;
    __device__ __forceinline__ void add(double x, bool first) {
        if (first) { f = __dadd_rn(0.0, x); return; }
        const double t = __dadd_rn(f, x);
        const double af = f < 0.0 ? -f : f, ax = x < 0.0 ? -x : x;
        c = __dadd_rn(c, af >= ax ? __dadd_rn(__dsub_rn(f, t), x) : __dadd_rn(__dsub_rn(x, t), f));
        f = t;
    }
    __device__ __forceinline__ double result() const { return (c != 0.0 && c - c == 0.0) ? __dadd_rn(f, c) : f; }
};

// Why the byte c (or the end of the line, c < 0) cannot follow a token or a number
__device__ __forceinline__ uint32_t eml_stray(int c, bool in_number) {
    if (c == '\r') return BB_EM_FALLBACK_CR;
    if (in_number && (c == '+' || c == '-' || c == '_' || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z')))
        return BB_EM_FALLBACK_NUMBER;
    if (!in_number && c > ' ' && c != ',' && c != ';') return BB_EM_FALLBACK_BASE;
    return BB_EM_FALLBACK_SYNTAX;
}

// Walks line text[s..e) (without its newline): f(j, first byte, length, probability) for its alternatives in order (the
// k-mer itself is alternative 0) and *code = the k-mer's 2-bit code.  Returns the fallback bits, 0 on the fast path.
template <typename F>
__device__ __forceinline__ uint32_t eml_walk_line(const uint8_t *__restrict__ text, int64_t s, int64_t e, int k, uint32_t *code,
                                                  F &&f) {
    if (s >= e) return BB_EM_FALLBACK_EMPTY_LINE;
    uint32_t first = 0, last = 0, cd = 0;
    int64_t p = s;
    for (int j = 0;; j++) {
        const int64_t t0 = p;
        for (; p < e; p++) {
            const int b = eml_base(text[p]);
            if (b < 0) break;
            if (j == 0 && p - t0 < EML_MAX_K) cd = cd * 4u + (uint32_t)b;
        }
        const int64_t len = p - t0;
        if (p == e || text[p] != ',' || len == 0) return eml_stray(p == e ? -1 : (int)text[p], false);
        if (j == 0) {
            if (len != k) return BB_EM_FALLBACK_K;
            first = text[t0];
            last = text[t0 + k - 1];
        } else if (len > EML_MAX_ALT) {
            return BB_EM_FALLBACK_LONG_ALT;
        } else if (len < 2 || text[t0] != first || text[p - 1] != last) {
            return BB_EM_FALLBACK_ALT_ENDS;
        }
        p++;
        double v;
        if (!eml_parse_prob(text, p, e, v)) return p < e && text[p] == '\r' ? BB_EM_FALLBACK_CR : BB_EM_FALLBACK_NUMBER;
        if (p < e && text[p] != ';') return eml_stray((int)text[p], true);
        f(j, t0, (int)len, v);
        if (p == e || ++p == e) break;   // (a ';' may end the line)
    }
    *code = cd;
    return 0;
}

// Pass 2, one thread per line: n_alt[l] = its alternatives, codes[l] its k-mer's code; *fallback |= its fallback bits
__global__ void __launch_bounds__(EML_LINE_THREADS)
eml_k_lines(const uint8_t *__restrict__ text, const int64_t *__restrict__ starts, int64_t n_lines, int k,
            int32_t *__restrict__ n_alt, int64_t *__restrict__ codes, int *__restrict__ fallback) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_lines) return;
    int32_t cnt = 0;
    uint32_t code = 0;
    const uint32_t fb = eml_walk_line(text, starts[l], starts[l + 1] - 1, k, &code, [&](int, int64_t, int, double) { cnt++; });
    n_alt[l] = fb ? 0 : cnt;
    codes[l] = code;
    if (fb) atomicOr(fallback, (int)fb);
}

// Pass 3, one thread per line: alternative alt_base[l] + j's first byte, length, row and probability; the row's remainder
// 1.0 - sum(probs) and its entries (the alternatives, and the remainder entry when the remainder is > 0)
__global__ void __launch_bounds__(EML_LINE_THREADS)
eml_k_alts(const uint8_t *__restrict__ text, const int64_t *__restrict__ starts, int64_t n_lines, int k,
           const int64_t *__restrict__ alt_base, int64_t *__restrict__ alt_pos, uint8_t *__restrict__ alt_len,
           int32_t *__restrict__ alt_row, double *__restrict__ alt_prob, int32_t *__restrict__ n_ent, double *__restrict__ rem) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_lines) return;
    const int64_t a0 = alt_base[l];
    EmlPySum sum;
    int32_t cnt = 0;
    uint32_t code;
    eml_walk_line(text, starts[l], starts[l + 1] - 1, k, &code, [&](int j, int64_t pos, int len, double v) {
        alt_pos[a0 + j] = pos;
        alt_len[a0 + j] = (uint8_t)len;
        alt_row[a0 + j] = (int32_t)l;
        alt_prob[a0 + j] = v;
        sum.add(v, j == 0);
        cnt++;
    });
    const double r = __dsub_rn(1.0, sum.result());
    rem[l] = r;
    n_ent[l] = cnt + (r > 0.0 ? 1 : 0);
}

// ---- alignment
// Slot lengths of one alternative, 8 bits each (a slot holds at most EML_MAX_ALT bytes), kept in registers
struct EmlSlotLens {
    uint64_t lo = 0, hi = 0;
    __device__ __forceinline__ void set(int s, uint32_t v) {
        if (s < 8) lo = (lo & ~(0xffull << (8 * s))) | ((uint64_t)v << (8 * s));
        else hi = (hi & ~(0xffull << (8 * (s - 8)))) | ((uint64_t)v << (8 * (s - 8)));
    }
    __device__ __forceinline__ uint32_t get(int s) const {
        return (uint32_t)((s < 8 ? lo >> (8 * s) : hi >> (8 * (s - 8))) & 0xffu);
    }
};

// align_kmers (bb_host_align_kmers) of alternative alt[0..L) to its k-mer: the lengths of its k slots.  The slots are
// consecutive pieces of the alternative: slot 0 is its first base and the bases inserted before the inner k-mer's first
// base, slot s its base aligned to k-mer base s (or none where that base is deleted) and the bases inserted after it, slot
// k - 1 its last base.  The edit path is small_nw_path's (bb_host.cpp): edit distance of the inner alternative (query) to
// the inner k-mer (target), traced back from the bottom-right cell preferring I, then D, then the diagonal.  tb: this
// thread's column of traceback rows, one 2-bit direction per cell (0 diagonal, 1 I, 2 D) of query row i at tb[i * stride].
__device__ __forceinline__ EmlSlotLens eml_align_slots(const uint8_t *__restrict__ kmer, int k, const uint8_t *__restrict__ alt,
                                                       int L, uint32_t *tb, int stride) {
    const int m = k - 2, n = L - 2;
    uint32_t t[EML_MAX_K - 2];
#pragma unroll
    for (int j = 0; j < EML_MAX_K - 2; j++) t[j] = j < m ? kmer[1 + j] : 0u;
    int prev[EML_MAX_K - 1];
#pragma unroll
    for (int j = 0; j <= EML_MAX_K - 2; j++) prev[j] = j;
    for (int i = 1; i <= n; i++) {
        const uint32_t q = alt[i];
        int diag = prev[0], left = i;
        prev[0] = i;
        uint32_t bits = 0;
#pragma unroll
        for (int j = 1; j <= EML_MAX_K - 2; j++) {
            if (j <= m) {
                const int up = prev[j];
                int c = diag + (q != t[j - 1] ? 1 : 0);
                c = c < up + 1 ? c : up + 1;
                c = c < left + 1 ? c : left + 1;
                const uint32_t dir = up + 1 == c ? 1u : left + 1 == c ? 2u : 0u;
                bits |= dir << (2 * (j - 1));
                diag = up;
                prev[j] = c;
                left = c;
            }
        }
        tb[i * stride] = bits;
    }
    EmlSlotLens s;
    int i = n, j = m;
    uint32_t pend = 0;   // bases inserted after the slot the walk reaches next
    while (i > 0 && j > 0) {
        const uint32_t dir = (tb[i * stride] >> (2 * (j - 1))) & 3u;
        if (dir == 1u) { pend++; i--; }
        else if (dir == 2u) { s.set(j, pend); pend = 0; j--; }
        else { s.set(j, 1 + pend); pend = 0; i--; j--; }
    }
    pend += (uint32_t)i;
    for (; j > 0; j--) { s.set(j, pend); pend = 0; }
    if (pend == 1) {   // a single leading insertion moves into slot 1 (error_model.py:225-228)
        s.set(0, 1);
        s.set(1, s.get(1) + 1);
    } else {
        s.set(0, 1 + pend);
    }
    s.set(k - 1, 1);
    return s;
}

// Pass 4, one thread per alternative.  FILL false: pooled[a] = the bytes its slots longer than 3 put in the pool.  FILL
// true: with pool_off[a] the scan of those, its entry's k slots (len | bases << 8, or len | pool offset << 8), its flags
// (1 when the alternative is the k-mer) and its pool bytes; *capacity = 1 when a pooled slot starts at or beyond
// EML_POOL_LIMIT.
template <bool FILL>
__global__ void __launch_bounds__(EML_ALIGN_THREADS)
eml_k_align(const uint8_t *__restrict__ text, int64_t n_alts, int k, const int64_t *__restrict__ starts,
            const int64_t *__restrict__ alt_pos, const uint8_t *__restrict__ alt_len, const int32_t *__restrict__ alt_row,
            const int64_t *__restrict__ alt_base, const int64_t *__restrict__ row_off, int32_t *__restrict__ pooled,
            const int64_t *__restrict__ pool_off, uint32_t *__restrict__ slots, uint8_t *__restrict__ flags,
            uint8_t *__restrict__ pool, int *__restrict__ capacity) {
    __shared__ uint32_t s_tb[(EML_MAX_ALT - 1) * EML_ALIGN_THREADS];
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_alts) return;
    const int32_t r = alt_row[a];
    const uint8_t *kmer = text + starts[r], *alt = text + alt_pos[a];
    const int L = alt_len[a];
    const EmlSlotLens s = eml_align_slots(kmer, k, alt, L, s_tb + threadIdx.x, EML_ALIGN_THREADS);
    if (!FILL) {
        int32_t bytes = 0;
        for (int j = 0; j < k; j++) {
            const uint32_t len = s.get(j);
            if (len > 3) bytes += (int32_t)len;
        }
        pooled[a] = bytes;
        return;
    }
    const int64_t e = row_off[r] + (a - alt_base[r]);
    int64_t off = pool_off[a];
    int start = 0;
    for (int j = 0; j < k; j++) {
        const uint32_t len = s.get(j);
        uint32_t enc = len;
        if (len <= 3) {
            for (uint32_t c = 0; c < len; c++) enc |= (uint32_t)alt[start + (int)c] << (8 * (c + 1));
        } else {
            if (off >= EML_POOL_LIMIT) {
                *capacity = 1;
                return;
            }
            enc |= (uint32_t)off << 8;
            for (uint32_t c = 0; c < len; c++) pool[off + c] = alt[start + (int)c];
            off += len;
        }
        slots[e * k + j] = enc;
        start += (int)len;
    }
    bool same = L == k;
    for (int j = 0; same && j < k; j++) same = alt[j] == kmer[j];
    flags[e] = same ? 1 : 0;
}

// ---- rows
// Pass 5, one thread per row: probs and cum (itertools.accumulate: a plain running sum) of its entries, its remainder
// entry, its summary (RowInfo is BBRowInfo, bb_kernels.cuh) and, with a dense index, kmer_to_row[code] = row (a k-mer
// two rows share sets BB_EM_FALLBACK_DUPLICATE in *fallback).  Runs after eml_k_align<true> (it reads the first flags).
template <typename RowInfo>
__global__ void __launch_bounds__(EML_LINE_THREADS)
eml_k_rows(int64_t n_rows, int k, const int64_t *__restrict__ alt_base, const double *__restrict__ alt_prob,
           const double *__restrict__ rem, const int64_t *__restrict__ row_off64, const int64_t *__restrict__ codes,
           int32_t *__restrict__ row_off, double *__restrict__ cum, double *__restrict__ probs, uint8_t *__restrict__ flags,
           uint32_t *__restrict__ slots, RowInfo *__restrict__ info, int32_t *__restrict__ kmer_to_row,
           int *__restrict__ fallback) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const int64_t e0 = row_off64[r], e1 = row_off64[r + 1], a0 = alt_base[r], na = alt_base[r + 1] - a0;
    double run = 0.0;
    for (int64_t j = 0; j < na; j++) {
        const double p = alt_prob[a0 + j];
        run = j == 0 ? p : __dadd_rn(run, p);
        probs[e0 + j] = p;
        cum[e0 + j] = run;
    }
    if (e1 - e0 > na) {
        const int64_t e = e0 + na;
        run = __dadd_rn(run, rem[r]);
        probs[e] = rem[r];
        cum[e] = run;
        flags[e] = 2;
        for (int j = 0; j < k; j++) slots[e * k + j] = EML_SLOT_NONE;
    }
    row_off[r] = (int32_t)e0;
    if (r == n_rows - 1) row_off[n_rows] = (int32_t)e1;
    RowInfo ri;
    ri.cum_last = run;
    ri.cum0 = cum[e0];
    ri.e0 = (int32_t)e0;
    ri.ne = (int32_t)(e1 - e0);
    ri.first_is_identity = flags[e0] == 1 ? 1 : 0;
    ri.pad = 0;
    info[r] = ri;
    if (kmer_to_row && atomicExch(&kmer_to_row[codes[r]], (int32_t)r) != -1) atomicOr(fallback, BB_EM_FALLBACK_DUPLICATE);
}
