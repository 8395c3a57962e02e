// bb_fastq.cuh — FASTQ parsing and the model builders' aligned slices on the device.
//
// The parse has the semantics of model_builders.load_fastq (binary mode):
//  - lines are split on '\n' only; a final line without '\n' is a line;
//  - between records a line is a header when it is not blank and its first byte after the leading whitespace (space,
//    '\t', '\n', '\r', '\v', '\f') is '@'; every other line there is skipped;
//  - the three lines after a header are taken whatever they hold: sequence, '+' line, qualities;
//  - the name is the first whitespace-separated token after the '@'; sequence and qualities are stripped of whitespace
//    (the sequence is upper-cased when it is gathered).
// Passes, every offset 64-bit:
//  1. fq_k_count_nl / fq_k_scan64 / fq_k_emit_nl: the positions of the newlines, in order (a block scan per tile of
//     FQ_TILE bytes, one CTA scanning the tiles' counts).
//  2. fq_k_line_maps / fq_k_scan_maps / fq_k_records: over lines, the 4-state machine (0 between records, 1 sequence next,
//     2 '+' line next, 3 qualities next) as maps of the state before a stretch of lines to the state after it and the
//     records it starts; one CTA applies the tiles' maps in order, then each tile writes its records' header lines.
//  3. fq_k_fields: one thread per record finds the name, sequence and quality spans from its four lines.
// fq_k_gather then writes the builders' flat read / qual / ref arrays (model_builders.FlatAlignments) from the parsed text.
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../include/badread_b200.h"

#ifndef FQ_THREADS
#define FQ_THREADS 256               // threads of every tile kernel
#endif
#ifndef FQ_SCAN_THREADS
#define FQ_SCAN_THREADS 1024         // threads of the one CTA of the scans
#endif
// The tiles are kernel arguments, so that tests can put tile edges anywhere; any tile >= 1 and any lines per thread >= 1
// parse the same.
#define FQ_TILE 16384                // bytes per tile of pass 1 (64 per thread)
#define FQ_LINES_PER_THREAD 16       // lines per thread of pass 2 (4096 lines per tile)

struct FastqRec {   // spans of one record in the text: [lo, hi)
    int64_t name_lo, name_hi, seq_lo, seq_hi, qual_lo, qual_hi;
};

// One chosen alignment for fq_k_gather: the FASTQ record, the raw slice bounds of the read (Python slice semantics on
// the record's sequence and, separately, on its qualities), the reference slice bounds on its contig (at contig_at of the
// uploaded contigs, contig_len bytes) and the strand.
struct FastqAln {
    int64_t rec, read_start, read_end, ref_start, ref_end, contig_at, contig_len;
    int32_t reverse, pad;
};

__device__ __forceinline__ bool fq_space(uint32_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

// Python's seq[a:b] on a sequence of n: *lo and the length
__host__ __device__ __forceinline__ int64_t fq_slice(int64_t n, int64_t a, int64_t b, int64_t *lo) {
    if (a < 0) a = a + n < 0 ? 0 : a + n;
    if (a > n) a = n;
    if (b < 0) b = b + n < 0 ? 0 : b + n;
    if (b > n) b = n;
    *lo = a;
    return b > a ? b - a : 0;
}

// ------------------------------------------------------------------------------------------------ newlines
// Exclusive block scan of one value per thread (FQ_THREADS threads); *total = the block's sum.  Every thread calls it.
__device__ __forceinline__ int64_t fq_block_scan(int64_t v, int64_t *total) {
    __shared__ int64_t s_warp[FQ_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = v;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    int64_t before = 0, all = 0;
    for (int k = 0; k < FQ_THREADS / 32; k++) {
        if (k == w) before = all;
        all += s_warp[k];
    }
    __syncthreads();
    *total = all;
    return before + inc - v;
}

__device__ __forceinline__ void fq_thread_bytes(int64_t n, int32_t tile, int64_t *a, int64_t *b) {
    const int64_t t0 = (int64_t)blockIdx.x * tile, t1 = t0 + tile < n ? t0 + tile : n;
    const int32_t per = (tile + FQ_THREADS - 1) / FQ_THREADS;
    *a = t0 + (int64_t)threadIdx.x * per < t1 ? t0 + (int64_t)threadIdx.x * per : t1;
    *b = *a + per < t1 ? *a + per : t1;
}

__device__ __forceinline__ int64_t fq_count_nl(const uint8_t *__restrict__ text, int64_t a, int64_t b) {
    int64_t c = 0;
    int64_t i = a;
    for (; i < b && (i & 15); i++) c += text[i] == '\n';
    for (; i + 16 <= b; i += 16) {
        const uint4 v = *reinterpret_cast<const uint4 *>(text + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 16; j++) c += ((w[j >> 2] >> (8 * (j & 3))) & 0xffu) == '\n';
    }
    for (; i < b; i++) c += text[i] == '\n';
    return c;
}

// counts[t] = the newlines of tile t
__global__ void __launch_bounds__(FQ_THREADS) fq_k_count_nl(const uint8_t *__restrict__ text, int64_t n, int32_t tile, int64_t *__restrict__ counts) {
    int64_t a, b, total;
    fq_thread_bytes(n, tile, &a, &b);
    fq_block_scan(fq_count_nl(text, a, b), &total);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// One CTA: v[0..n) replaced by its exclusive prefix sums; *total = the sum
__global__ void __launch_bounds__(FQ_SCAN_THREADS) fq_k_scan64(int64_t *__restrict__ v, int64_t n, int64_t *__restrict__ total) {
    __shared__ int64_t s[FQ_SCAN_THREADS];
    const int64_t per = (n + FQ_SCAN_THREADS - 1) / FQ_SCAN_THREADS;
    const int64_t c0 = (int64_t)threadIdx.x * per < n ? (int64_t)threadIdx.x * per : n, c1 = c0 + per < n ? c0 + per : n;
    int64_t sum = 0;
    for (int64_t i = c0; i < c1; i++) sum += v[i];
    s[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t run = 0;
        for (int r = 0; r < FQ_SCAN_THREADS; r++) {
            const int64_t x = s[r];
            s[r] = run;
            run += x;
        }
        *total = run;
    }
    __syncthreads();
    int64_t run = s[threadIdx.x];
    for (int64_t i = c0; i < c1; i++) {
        const int64_t x = v[i];
        v[i] = run;
        run += x;
    }
}

// nl[base[t] ..] = the positions of tile t's newlines
__global__ void __launch_bounds__(FQ_THREADS)
fq_k_emit_nl(const uint8_t *__restrict__ text, int64_t n, int32_t tile, const int64_t *__restrict__ base, int64_t *__restrict__ nl) {
    int64_t a, b, total;
    fq_thread_bytes(n, tile, &a, &b);
    int64_t at = base[blockIdx.x] + fq_block_scan(fq_count_nl(text, a, b), &total);
    for (int64_t i = a; i < b; i++)
        if (text[i] == '\n') nl[at++] = i;
}

// ------------------------------------------------------------------------------------------------ the record machine
// A stretch of lines as a map of the state before it: bits 2s..2s+1 of `next` the state after it from state s, cnt[s]
// the records it starts from state s.
struct FqMap {
    uint32_t next;
    uint32_t cnt[4];
};

__device__ __forceinline__ FqMap fq_identity() { return FqMap{0xe4u, {0, 0, 0, 0}}; }

__device__ __forceinline__ uint32_t fq_next(const FqMap &m, uint32_t s) { return (m.next >> (2 * s)) & 3u; }

// a, then b
__device__ __forceinline__ FqMap fq_then(const FqMap &a, const FqMap &b) {
    FqMap r;
    r.next = 0;
#pragma unroll
    for (uint32_t s = 0; s < 4; s++) {
        const uint32_t m = fq_next(a, s);
        r.next |= fq_next(b, m) << (2 * s);
        r.cnt[s] = a.cnt[s] + b.cnt[m];
    }
    return r;
}

__device__ __forceinline__ void fq_line(const int64_t *__restrict__ nl, int64_t n_nl, int64_t n, int64_t i, int64_t *s, int64_t *e) {
    *s = i ? nl[i - 1] + 1 : 0;
    *e = i < n_nl ? nl[i] : n;
}

// line i is a header between records: not blank, '@' after its leading whitespace
__device__ __forceinline__ bool fq_is_header(const uint8_t *__restrict__ text, const int64_t *__restrict__ nl, int64_t n_nl,
                                             int64_t n, int64_t i) {
    int64_t s, e;
    fq_line(nl, n_nl, n, i, &s, &e);
    while (s < e && fq_space(text[s])) s++;
    return s < e && text[s] == '@';
}

// the map of lines [a, b)
__device__ __forceinline__ FqMap fq_lines_map(const uint8_t *__restrict__ text, const int64_t *__restrict__ nl, int64_t n_nl,
                                              int64_t n, int64_t a, int64_t b) {
    FqMap m = fq_identity();
    for (int64_t i = a; i < b; i++) {
        const uint32_t h = fq_is_header(text, nl, n_nl, n, i);
        // 0 -> 1 on a header (one record), else 0; 1 -> 2 -> 3 -> 0
        FqMap l{(h ? 1u : 0u) | (2u << 2) | (3u << 4), {h, 0, 0, 0}};
        m = fq_then(m, l);
    }
    return m;
}

// Exclusive block scan of the threads' maps in thread order; *total = the block's map.  Every thread calls it.
__device__ __forceinline__ FqMap fq_map_scan(FqMap m, FqMap *total) {
    __shared__ FqMap s_map[2][FQ_THREADS];
    int cur = 0;
    s_map[0][threadIdx.x] = m;
    __syncthreads();
    for (int d = 1; d < FQ_THREADS; d <<= 1) {
        const FqMap x = s_map[cur][threadIdx.x];
        s_map[cur ^ 1][threadIdx.x] = (int)threadIdx.x >= d ? fq_then(s_map[cur][threadIdx.x - d], x) : x;
        cur ^= 1;
        __syncthreads();
    }
    *total = s_map[cur][FQ_THREADS - 1];
    const FqMap before = threadIdx.x ? s_map[cur][threadIdx.x - 1] : fq_identity();
    __syncthreads();   // (s_map is reused by the next call)
    return before;
}

// lines [a, b) of this thread, lpt per thread (a tile of FQ_THREADS * lpt lines)
__device__ __forceinline__ void fq_thread_lines(int64_t n_lines, int32_t lpt, int64_t *a, int64_t *b) {
    const int64_t tile = (int64_t)FQ_THREADS * lpt;
    const int64_t t0 = (int64_t)blockIdx.x * tile, t1 = t0 + tile < n_lines ? t0 + tile : n_lines;
    *a = t0 + (int64_t)threadIdx.x * lpt < t1 ? t0 + (int64_t)threadIdx.x * lpt : t1;
    *b = *a + lpt < t1 ? *a + lpt : t1;
}

// maps[t] = the map of line tile t
__global__ void __launch_bounds__(FQ_THREADS)
fq_k_line_maps(const uint8_t *__restrict__ text, const int64_t *__restrict__ nl, int64_t n_nl, int64_t n, int64_t n_lines,
               int32_t lpt, FqMap *__restrict__ maps) {
    int64_t a, b;
    fq_thread_lines(n_lines, lpt, &a, &b);
    FqMap total;
    fq_map_scan(fq_lines_map(text, nl, n_nl, n, a, b), &total);
    if (threadIdx.x == 0) maps[blockIdx.x] = total;
}

// One CTA: the maps of the line tiles applied in order from state 0: tile t's start state and first record number to
// state[t] / base[t]; *n_rec = the records
__global__ void __launch_bounds__(FQ_SCAN_THREADS)
fq_k_scan_maps(const FqMap *__restrict__ maps, int64_t n_tiles, int32_t *__restrict__ state, int64_t *__restrict__ base,
               int64_t *__restrict__ n_rec) {
    __shared__ int64_t s_base[FQ_SCAN_THREADS][4];
    __shared__ uint8_t s_next[FQ_SCAN_THREADS];
    __shared__ uint8_t s_start[FQ_SCAN_THREADS];
    const int64_t per = (n_tiles + FQ_SCAN_THREADS - 1) / FQ_SCAN_THREADS;
    const int64_t c0 = (int64_t)threadIdx.x * per < n_tiles ? (int64_t)threadIdx.x * per : n_tiles;
    const int64_t c1 = c0 + per < n_tiles ? c0 + per : n_tiles;
    uint32_t next = 0xe4u;
    int64_t cnt[4] = {0, 0, 0, 0};
    for (int64_t t = c0; t < c1; t++) {   // this thread's run of tiles from each start state
        uint32_t nn = 0;
        for (uint32_t s = 0; s < 4; s++) {
            const uint32_t m = (next >> (2 * s)) & 3u;
            cnt[s] += maps[t].cnt[m];
            nn |= fq_next(maps[t], m) << (2 * s);
        }
        next = nn;
    }
    for (int s = 0; s < 4; s++) s_base[threadIdx.x][s] = cnt[s];
    s_next[threadIdx.x] = (uint8_t)next;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t st = 0;
        int64_t run = 0;
        for (int r = 0; r < FQ_SCAN_THREADS; r++) {
            const int64_t c = s_base[r][st];
            const uint32_t nx = (s_next[r] >> (2 * st)) & 3u;
            s_base[r][0] = run;
            s_start[r] = (uint8_t)st;
            run += c;
            st = nx;
        }
        *n_rec = run;
    }
    __syncthreads();
    uint32_t st = s_start[threadIdx.x];
    int64_t run = s_base[threadIdx.x][0];
    for (int64_t t = c0; t < c1; t++) {
        state[t] = (int32_t)st;
        base[t] = run;
        run += maps[t].cnt[st];
        st = fq_next(maps[t], st);
    }
}

// rec_line[r] = the header line of record r
__global__ void __launch_bounds__(FQ_THREADS)
fq_k_records(const uint8_t *__restrict__ text, const int64_t *__restrict__ nl, int64_t n_nl, int64_t n, int64_t n_lines,
             int32_t lpt, const int32_t *__restrict__ state, const int64_t *__restrict__ base, int64_t *__restrict__ rec_line) {
    int64_t a, b;
    fq_thread_lines(n_lines, lpt, &a, &b);
    FqMap total;
    const FqMap before = fq_map_scan(fq_lines_map(text, nl, n_nl, n, a, b), &total);
    const uint32_t s0 = (uint32_t)state[blockIdx.x];
    uint32_t st = fq_next(before, s0);
    int64_t r = base[blockIdx.x] + before.cnt[s0];
    for (int64_t i = a; i < b; i++) {
        if (st == 0) {
            if (fq_is_header(text, nl, n_nl, n, i)) {
                rec_line[r++] = i;
                st = 1;
            }
        } else {
            st = (st + 1) & 3u;
        }
    }
}

// One thread per record: its spans.  *err = the least (record << 1 | kind) of a failing record: kind 0 a header without
// a name, kind 1 a record the file ends in (fewer than three lines after its header).
__global__ void __launch_bounds__(FQ_THREADS)
fq_k_fields(const uint8_t *__restrict__ text, const int64_t *__restrict__ nl, int64_t n_nl, int64_t n, int64_t n_lines,
            const int64_t *__restrict__ rec_line, int64_t n_rec, FastqRec *__restrict__ recs, unsigned long long *__restrict__ err) {
    const int64_t r = (int64_t)blockIdx.x * FQ_THREADS + threadIdx.x;
    if (r >= n_rec) return;
    const int64_t h = rec_line[r];
    int64_t s, e;
    fq_line(nl, n_nl, n, h, &s, &e);
    while (s < e && fq_space(text[s])) s++;
    s++;   // (the '@')
    while (s < e && fq_space(text[s])) s++;
    int64_t t = s;
    while (t < e && !fq_space(text[t])) t++;
    FastqRec R{s, t, 0, 0, 0, 0};
    if (t == s) atomicMin(err, (unsigned long long)r << 1);
    if (h + 3 >= n_lines) {
        atomicMin(err, ((unsigned long long)r << 1) | 1ull);
    } else {
        for (int k = 1; k <= 3; k += 2) {
            fq_line(nl, n_nl, n, h + k, &s, &e);
            while (s < e && fq_space(text[s])) s++;
            while (e > s && fq_space(text[e - 1])) e--;
            if (k == 1) { R.seq_lo = s; R.seq_hi = e; } else { R.qual_lo = s; R.qual_hi = e; }
        }
    }
    recs[r] = R;
}

// ------------------------------------------------------------------------------------------------ the aligned slices
// One CTA per alignment a: read[read_off[a] ..] / qual[..] the read slice (upper-cased) and the quality slice, each padded
// with NUL to read_off[a + 1]; ref[ref_off[a] ..] the reference slice, reverse-complemented (comp) on '-', padded to
// ref_off[a + 1].  *bad = the least alignment whose read holds a byte >= 0x80 in its sequence or qualities.
__global__ void __launch_bounds__(FQ_THREADS)
fq_k_gather(const uint8_t *__restrict__ text, const FastqRec *__restrict__ recs, const FastqAln *__restrict__ alns,
            const int64_t *__restrict__ read_off, const int64_t *__restrict__ ref_off, const uint8_t *__restrict__ contigs,
            const uint8_t *__restrict__ comp, uint8_t *__restrict__ read, uint8_t *__restrict__ qual, uint8_t *__restrict__ ref,
            unsigned long long *__restrict__ bad) {
    const int64_t a = blockIdx.x;
    const FastqAln A = alns[a];
    const FastqRec R = recs[A.rec];
    __shared__ int s_odd;
    if (threadIdx.x == 0) s_odd = 0;
    __syncthreads();
    bool odd = false;
    for (int64_t i = R.seq_lo + threadIdx.x; i < R.seq_hi; i += FQ_THREADS) odd |= text[i] >= 0x80;
    for (int64_t i = R.qual_lo + threadIdx.x; i < R.qual_hi; i += FQ_THREADS) odd |= text[i] >= 0x80;
    if (odd) s_odd = 1;   // (every writer stores the same value)
    __syncthreads();
    if (s_odd) {
        if (threadIdx.x == 0) atomicMin(bad, (unsigned long long)a);
        return;
    }
    int64_t s_lo, q_lo, f_lo;
    const int64_t s_n = fq_slice(R.seq_hi - R.seq_lo, A.read_start, A.read_end, &s_lo);
    const int64_t q_n = fq_slice(R.qual_hi - R.qual_lo, A.read_start, A.read_end, &q_lo);
    const int64_t f_n = fq_slice(A.contig_len, A.ref_start, A.ref_end, &f_lo);
    const uint8_t *seq = text + R.seq_lo + s_lo, *qs = text + R.qual_lo + q_lo, *fr = contigs + A.contig_at + f_lo;
    const int64_t r0 = read_off[a], rp = read_off[a + 1] - r0;
    for (int64_t i = threadIdx.x; i < rp; i += FQ_THREADS) {
        const uint32_t c = i < s_n ? seq[i] : 0u;
        read[r0 + i] = (uint8_t)(c - ((c >= 'a' && c <= 'z') ? 32u : 0u));
        qual[r0 + i] = i < q_n ? qs[i] : (uint8_t)0;
    }
    const int64_t f0 = ref_off[a], fp = ref_off[a + 1] - f0;
    for (int64_t i = threadIdx.x; i < fp; i += FQ_THREADS)
        ref[f0 + i] = i >= f_n ? (uint8_t)0 : A.reverse ? comp[fr[f_n - 1 - i]] : fr[i];
}

// ------------------------------------------------------------------------------------------------ host side of the gather
// What bb_flat_build hands fq_k_gather: per alignment its descriptor and offsets, and the M / I / D runs in read
// orientation (length << 2 | 0 M, 1 I, 2 D) with the read and reference offsets each starts at.
struct FqPlan {
    std::vector<FastqAln> alns;
    std::vector<uint32_t> ops;
    std::vector<int32_t> p0, r0;
    std::vector<int64_t> read_off{0}, ref_off{0}, ops_off{0};
};

// The plan of alignments records[0..n_aln) of the PAF view v against the FASTQ records whose names are
// names[name_off[r] .. name_off[r + 1]) (a repeated name: its last record; the join hashes only the names the alignments
// need) and the contigs at contig_at[ref id] (-1: not loaded).  Returns 0, or with failed[0] = the alignment: 1 its read
// is missing, 2 its reference is (checked in that order per alignment, FlatAlignments' order), 4 its CIGAR spans more
// than 2^31 - 1 bases.
inline int fq_plan(const char *names, const int64_t *name_off, int64_t n_rec, const bb_aln_view *v, int32_t n_aln,
                   const int64_t *records, const int64_t *contig_at, const int64_t *contig_len, FqPlan &P, int64_t *failed) {
    failed[0] = -1;
    failed[1] = 0;
    auto name_of = [&](int64_t j) {
        const int32_t id = v->read_id[j];
        return std::string_view(v->read_names + v->read_name_off[id], (size_t)(v->read_name_off[id + 1] - v->read_name_off[id]));
    };
    std::unordered_map<std::string_view, int64_t> rec_of;
    for (int32_t i = 0; i < n_aln; i++) rec_of.emplace(name_of(records[i]), -1);
    for (int64_t r = 0; r < n_rec; r++) {
        auto it = rec_of.find(std::string_view(names + name_off[r], (size_t)(name_off[r + 1] - name_off[r])));
        if (it != rec_of.end()) it->second = r;
    }
    P.alns.resize((size_t)n_aln);
    for (int32_t i = 0; i < n_aln; i++) {
        const int64_t j = records[i], rec = rec_of[name_of(j)], at = contig_at[v->ref_id[j]];
        if (rec < 0 || at < 0) {
            failed[0] = i;
            failed[1] = rec < 0 ? 1 : 2;
            return (int)failed[1];
        }
        const bool reverse = (v->flag[j] & 16) != 0;
        const int64_t c0 = v->cigar_off[j], c1 = v->cigar_off[j + 1];
        int64_t rp = 0, fp = 0;
        for (int64_t c = 0; c < c1 - c0; c++) {
            const uint32_t run = v->cigar[reverse ? c1 - 1 - c : c0 + c], code = run & 15u, count = run >> 4;
            if (code > 2) continue;   // (FlatAlignments uses M, I and D only)
            P.ops.push_back((count << 2) | code);
            P.p0.push_back((int32_t)rp);
            P.r0.push_back((int32_t)fp);
            rp += code != 2 ? count : 0;
            fp += code != 1 ? count : 0;
            if (rp > INT32_MAX || fp > INT32_MAX) {
                failed[0] = i;
                failed[1] = 4;
                return 4;
            }
        }
        P.alns[(size_t)i] = FastqAln{rec, v->read_start[j], v->read_end[j], v->ref_start[j], v->ref_end[j], at,
                                     contig_len[v->ref_id[j]], reverse, 0};
        P.read_off.push_back(P.read_off.back() + rp);
        P.ref_off.push_back(P.ref_off.back() + fp);
        P.ops_off.push_back((int64_t)P.ops.size());
    }
    return 0;
}
