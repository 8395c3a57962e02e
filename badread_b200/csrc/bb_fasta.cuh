// bb_fasta.cuh — FASTA parsing on the device: the bytes of a FASTA file (or of its inflated BGZF) in device memory to the
// upper-cased bases of its contigs and a table of its header lines, with the semantics of misc.load_fasta_arrays:
//  - a line is the bytes between newlines; it is a header line when its first byte is '>' ('>' anywhere else is data);
//  - every byte outside header lines is kept except '\n', '\r', ' ' and '\t' ('\v', '\f' and bytes >= 0x80 are kept),
//    and 'a'-'z' are upper-cased;
//  - header line k has its start (the '>'), its end (its newline, or the end of the file) and the number of bytes kept
//    before it.  So contig k's bases are kept bytes [kept[k], kept[k + 1]) (the last contig's run to the end) and kept
//    bytes [0, kept[0]) lie before the first header.  The host turns the header lines into names, depths and flags and
//    picks the contigs (misc.fasta_contigs), then fasta_k_gather forms the reference.
//
// Three passes over fixed tiles of `tile` bytes, every offset 64-bit.  The state a byte depends on is whether its line is
// a header line.  A tile knows whether it starts a line (the byte before it is a newline), so only a line that began in an
// earlier tile leaves its start state open: each tile is a map from that state (0 or 1) to (bytes kept, state at its end).
//  1. fasta_k_summarize: each tile's map and its number of header lines, from a block scan of its threads' maps.
//  2. fasta_k_scan: one CTA applies the tiles' maps in order: each tile's start state, kept offset and first header.
//  3. fasta_k_emit: each tile again with its start state known: a block scan of the threads' maps places every thread's
//     kept bytes, which it writes upper-cased, and its header lines' starts, ends and kept offsets.
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>

#ifndef FASTA_THREADS
#define FASTA_THREADS 256            // threads of a tile (passes 1 and 3)
#endif
#ifndef FASTA_SCAN_THREADS
#define FASTA_SCAN_THREADS 1024      // threads of the one CTA of pass 2
#endif
#define FASTA_TILE 16384             // bytes per tile (64 per thread); any value in 1 .. 2^30 parses the same
#define FASTA_GATHER 16              // output bytes per thread of fasta_k_gather

// A stretch of text as a map of the header state at its start: kept bytes from state 0 (low 32 bits) and from state 1
// (high 32 bits); bit 0 / bit 1 of meta the state at its end from state 0 / 1; meta >> 2 the header lines starting in it.
// A stretch that starts a line, or holds a newline, ends in the same state from both.
struct FastaMap {
    uint64_t kept;
    uint32_t meta;
    uint32_t pad;
};

struct FastaTileStart {   // pass 2's result for one tile
    int64_t kept;         // bytes kept before the tile
    int64_t hdr;          // header lines before the tile
    int32_t state;        // header state at its first byte (when that byte does not start a line)
    int32_t pad;
};

__device__ __forceinline__ FastaMap fasta_identity() { return FastaMap{0, 2u, 0}; }

// a, then b (every half of kept stays below 2^32: a tile has at most 2^30 bytes)
__device__ __forceinline__ FastaMap fasta_then(FastaMap a, FastaMap b) {
    const uint32_t a0 = a.meta & 1u, a1 = (a.meta >> 1) & 1u;
    const uint64_t b0 = a0 ? (b.kept >> 32) : (b.kept & 0xffffffffu), b1 = a1 ? (b.kept >> 32) : (b.kept & 0xffffffffu);
    FastaMap r;
    r.kept = a.kept + (b0 | (b1 << 32));
    r.meta = ((b.meta >> a0) & 1u) | (((b.meta >> a1) & 1u) << 1) | ((a.meta & ~3u) + (b.meta & ~3u));
    r.pad = 0;
    return r;
}

__device__ __forceinline__ bool fasta_keep(uint32_t c) { return c != '\n' && c != '\r' && c != ' ' && c != '\t'; }

// f(c, i) for the bytes text[a..b) in order, 16 at a time where they are aligned
template <typename F>
__device__ __forceinline__ void fasta_each_byte(const uint8_t *__restrict__ text, int64_t a, int64_t b, F &&f) {
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

// The map of text[a..b) (the identity when empty)
__device__ __forceinline__ FastaMap fasta_stretch_map(const uint8_t *__restrict__ text, int64_t a, int64_t b) {
    if (a >= b) return fasta_identity();
    bool ls = a == 0 || text[a - 1] == '\n';
    uint32_t h0 = 0, h1 = 1, k0 = 0, k1 = 0, hdr = 0;
    fasta_each_byte(text, a, b, [&](uint32_t c, int64_t) {
        if (ls) { h0 = h1 = (c == '>'); hdr += h0; }
        const bool keep = fasta_keep(c);
        k0 += keep && !h0;
        k1 += keep && !h1;
        ls = c == '\n';
    });
    return FastaMap{(uint64_t)k0 | ((uint64_t)k1 << 32), h0 | (h1 << 1) | (hdr << 2), 0};
}

// Exclusive block scan of the threads' maps in thread order; *total = the whole block's map.  Every thread must call it.
__device__ __forceinline__ FastaMap fasta_block_scan(FastaMap m, FastaMap *total) {
    __shared__ FastaMap s_warp[FASTA_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    FastaMap inc = m;
    for (int d = 1; d < 32; d <<= 1) {
        FastaMap o;
        o.kept = __shfl_up_sync(0xffffffffu, inc.kept, d);
        o.meta = __shfl_up_sync(0xffffffffu, inc.meta, d);
        o.pad = 0;
        if (lane >= d) inc = fasta_then(o, inc);
    }
    FastaMap exc;
    exc.kept = __shfl_up_sync(0xffffffffu, inc.kept, 1);
    exc.meta = __shfl_up_sync(0xffffffffu, inc.meta, 1);
    exc.pad = 0;
    if (lane == 0) exc = fasta_identity();
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    FastaMap before = fasta_identity(), all = fasta_identity();
    for (int k = 0; k < FASTA_THREADS / 32; k++) {
        if (k == w) before = all;
        all = fasta_then(all, s_warp[k]);
    }
    __syncthreads();   // (s_warp is reused by the next call)
    *total = all;
    return fasta_then(before, exc);
}

// Pass 1: maps[t] = the map of tile t
__global__ void __launch_bounds__(FASTA_THREADS)
fasta_k_summarize(const uint8_t *__restrict__ text, int64_t n, int32_t tile, FastaMap *__restrict__ maps) {
    const int64_t t0 = (int64_t)blockIdx.x * tile, t1 = t0 + tile < n ? t0 + tile : n;
    const int32_t per = (tile + FASTA_THREADS - 1) / FASTA_THREADS;
    const int64_t a = t0 + (int64_t)threadIdx.x * per < t1 ? t0 + (int64_t)threadIdx.x * per : t1;
    const int64_t b = a + per < t1 ? a + per : t1;
    FastaMap total;
    fasta_block_scan(fasta_stretch_map(text, a, b), &total);
    if (threadIdx.x == 0) maps[blockIdx.x] = total;
}

// The maps of tiles [c0, c1) applied in order from (state, kept, hdr)
__device__ __forceinline__ void fasta_apply(const FastaMap &m, int32_t &state, int64_t &kept, int64_t &hdr) {
    kept += state ? (int64_t)(m.kept >> 32) : (int64_t)(m.kept & 0xffffffffu);
    hdr += m.meta >> 2;
    state = (m.meta >> state) & 1;
}

// Pass 2 (one CTA): starts[t] for every tile; totals[0] = bytes kept, totals[1] = header lines
__global__ void __launch_bounds__(FASTA_SCAN_THREADS)
fasta_k_scan(const FastaMap *__restrict__ maps, int64_t n_tiles, FastaTileStart *__restrict__ starts, int64_t *__restrict__ totals) {
    __shared__ int64_t s_kept[2][FASTA_SCAN_THREADS], s_hdr[FASTA_SCAN_THREADS];
    __shared__ int32_t s_state[2][FASTA_SCAN_THREADS];
    const int64_t per = (n_tiles + FASTA_SCAN_THREADS - 1) / FASTA_SCAN_THREADS;
    const int64_t c0 = (int64_t)threadIdx.x * per < n_tiles ? (int64_t)threadIdx.x * per : n_tiles;
    const int64_t c1 = c0 + per < n_tiles ? c0 + per : n_tiles;
    // this thread's run of tiles from both start states
    for (int s = 0; s < 2; s++) {
        int32_t state = s;
        int64_t kept = 0, hdr = 0;
        for (int64_t t = c0; t < c1; t++) fasta_apply(maps[t], state, kept, hdr);
        s_kept[s][threadIdx.x] = kept;
        s_state[s][threadIdx.x] = state;
        if (s == 0) s_hdr[threadIdx.x] = hdr;
    }
    __syncthreads();
    if (threadIdx.x == 0) {   // the runs in order: each run's start (in place of its own results)
        int32_t state = 0;
        int64_t kept = 0, hdr = 0;
        for (int r = 0; r < FASTA_SCAN_THREADS; r++) {
            const int64_t k = s_kept[state][r], h = s_hdr[r];
            const int32_t next = s_state[state][r];
            s_kept[0][r] = kept;
            s_hdr[r] = hdr;
            s_state[0][r] = state;
            kept += k;
            hdr += h;
            state = next;
        }
        totals[0] = kept;
        totals[1] = hdr;
    }
    __syncthreads();
    int32_t state = s_state[0][threadIdx.x];
    int64_t kept = s_kept[0][threadIdx.x], hdr = s_hdr[threadIdx.x];
    for (int64_t t = c0; t < c1; t++) {
        starts[t] = FastaTileStart{kept, hdr, state, 0};
        fasta_apply(maps[t], state, kept, hdr);
    }
}

// Pass 3: the kept bytes of tile blockIdx.x, upper-cased, to out[]; for every header line that starts in it
// hdr_start / hdr_kept, and for every one that ends in it hdr_end
__global__ void __launch_bounds__(FASTA_THREADS)
fasta_k_emit(const uint8_t *__restrict__ text, int64_t n, int32_t tile, const FastaTileStart *__restrict__ starts,
             uint8_t *__restrict__ out, int64_t *__restrict__ hdr_start, int64_t *__restrict__ hdr_end,
             int64_t *__restrict__ hdr_kept) {
    const int64_t t0 = (int64_t)blockIdx.x * tile, t1 = t0 + tile < n ? t0 + tile : n;
    const int32_t per = (tile + FASTA_THREADS - 1) / FASTA_THREADS;
    const int64_t a = t0 + (int64_t)threadIdx.x * per < t1 ? t0 + (int64_t)threadIdx.x * per : t1;
    const int64_t b = a + per < t1 ? a + per : t1;
    FastaMap total;
    const FastaMap before = fasta_block_scan(fasta_stretch_map(text, a, b), &total);
    const FastaTileStart S = starts[blockIdx.x];
    int64_t kept = S.kept + (int64_t)(S.state ? before.kept >> 32 : before.kept & 0xffffffffu);
    int64_t hdr = S.hdr + (int64_t)(before.meta >> 2);
    uint32_t h = (before.meta >> S.state) & 1u;
    if (a >= b) return;
    bool ls = a == 0 || text[a - 1] == '\n';
    fasta_each_byte(text, a, b, [&](uint32_t c, int64_t i) {
        if (ls) {
            h = c == '>';
            if (h) { hdr_start[hdr] = i; hdr_kept[hdr] = kept; hdr++; }
        }
        if (c == '\n' && h) { hdr_end[hdr - 1] = i; h = 0; }
        if (fasta_keep(c) && !h) out[kept++] = (uint8_t)(c - ((c >= 'a' && c <= 'z') ? 32u : 0u));
        ls = c == '\n';
    });
    if (b == n && h) hdr_end[hdr - 1] = n;   // a header line the file ends in
}

// dst[dst_off[r] ..  dst_off[r + 1]) = src[src_lo[r] ..] for the n_ranges ranges (dst_off[n_ranges] = the total)
__global__ void __launch_bounds__(256)
fasta_k_gather(const uint8_t *__restrict__ src, const int64_t *__restrict__ src_lo, const int64_t *__restrict__ dst_off,
               int32_t n_ranges, uint8_t *__restrict__ dst) {
    const int64_t total = dst_off[n_ranges];
    const int64_t p0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * FASTA_GATHER;
    if (p0 >= total) return;
    int32_t lo = 0, hi = n_ranges - 1;   // the last range starting at or before p0
    while (lo < hi) {
        const int32_t mid = (lo + hi + 1) >> 1;
        if (dst_off[mid] <= p0) lo = mid; else hi = mid - 1;
    }
    const int64_t p1 = p0 + FASTA_GATHER < total ? p0 + FASTA_GATHER : total;
    for (int64_t p = p0; p < p1; p++) {
        while (dst_off[lo + 1] <= p) lo++;
        dst[p] = src[src_lo[lo] + (p - dst_off[lo])];
    }
}
