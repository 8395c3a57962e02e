// bb_gunzip.cuh — any gzip stream (RFC 1952: one member or many, as gzip, pigz or zlib write them) inflated on the device,
// one deflate stream decoded in parallel chunks: the speculative-chunk scheme of pugz and rapidgzip (PAPERS.md).
//
// The deflate data are cut into chunks of C compressed bytes.  Block boundaries inside a member are not byte-aligned and
// are recorded nowhere, so each chunk first looks for them:
//  - gz_k_find tests every bit offset of a chunk, a cheap prefilter first (non-final, dynamic, HLIT <= 286, HDIST <= 30,
//    a complete code-length code), then infl_dynamic_tables, exactly infl_member's rules, and keeps the first
//    GZ_CANDIDATES offsets that pass (one: a chunk whose first one fails is repaired).  A chunk without any is absorbed by its predecessor.
//  - gz_k_decode runs one decoder per chunk (lane 0 of a warp, as infl_k_members) from its first candidate that decodes
//    without error up to the first block boundary at or past the next chunk's start.  It writes 16-bit symbols: a byte,
//    or GZ_MARK + w for byte w of the unknown 32 KiB window before the chunk.  Crossing a final block it reads the
//    trailer and the next member's header and goes on with an empty window.
//  - Chunk i + 1 is confirmed iff it started where chunk i stopped: both are then the first block boundary at or after
//    chunk i + 1's start, one as seen by a decoder on the true stream, the other as guessed.  Chunk 0 starts at the true
//    start.  A chunk that is not confirmed is decoded again from its predecessor's end (a repair launch, at most
//    GZ_REPAIR_ROUNDS of them); what is left after that is decoded by one chain (gz_k_chain), slow but right.
//  - gz_k_windows resolves each chunk's 32 KiB window in chunk order, gz_k_resolve turns every chunk's symbols into
//    bytes at prefix-summed offsets, and gz_k_crc checks every member's CRC-32 over slices combined as bb_crc32.cuh does.
// A chunk's symbols go to a slot sized from a ratio of its input; a decoder past the slot goes on counting.  If a
// confirmed chunk overflowed, every chunk is decoded again from its confirmed start, the ones that overflowed into slots
// of the size they reported (one launch, no search: slots are reallocated as one buffer).
//
// Device memory peaks at the input, plus the symbol slots (2 bytes per symbol, GZ_RATIO * 5/4 symbols per input byte:
// about 10 bytes per input byte, more after a re-run), plus the output, plus 32 KiB of window per chunk.
//
// Every read stays inside the input (bits past its end read as zero and mark the decode truncated), every write inside
// the chunk's slot, and every loop consumes input or produces output, so corrupt input ends with a status, never with a
// fault or a hang.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/badread_b200.h"
#include "bb_inflate.cuh"

#define GZ_WINDOW 32768
#define GZ_MARK 256                  // symbols GZ_MARK + w: byte w of the window before the chunk
#ifndef GZ_CANDIDATES
#define GZ_CANDIDATES 1   // block starts kept per chunk (DESIGN.md §4: 1, 2 and 4 measured)
#endif
#define GZ_FIND_THREADS 128
#ifndef GZ_SPAN   // (the tests build the emulator with other values)
#define GZ_SPAN (1 << 30)
#endif
#ifndef GZ_REBASE   // (the tests build the emulator with other values)
#define GZ_REBASE (1 << 29)
#endif
#define GZ_RESOLVE_THREADS 256
#ifndef GZ_WINDOW_THREADS
#define GZ_WINDOW_THREADS 1024
#endif
#define GZ_SLICE 65536               // output bytes per warp of the CRC-32 check

enum GzStatus {   // after the InflStatus values
    GZ_NOT_GZIP = 11, GZ_BAD_METHOD = 12, GZ_BAD_FLAGS = 13, GZ_TRUNC_HEADER = 14, GZ_BAD_ISIZE = 15
};

enum GzFlags {
    GZ_F_END_MEMBER = 1,   // it stopped at a member's first block
    GZ_F_ENDED = 2,        // it reached the end of the stream (end = 8 n)
    GZ_F_OVER = 4          // more symbols than its slot: len is what it needed
};

struct GzTask {            // one decode
    int64_t start;         // bit offset to start at; -1: the chunk's candidates in turn
    int64_t stop;          // it stops at the first block boundary at or past this bit offset
    int32_t chunk;         // its slot
    int32_t member_start;  // start is a member's first block (an empty window)
};

struct GzRes {             // one chunk's decode
    int64_t start, end;    // bit offsets where it started and where it stopped
    int64_t len;           // symbols
    int64_t member_at;     // input offset of the header of the member it stopped or failed in; -1: the one it started in
    int32_t status;        // InflStatus / GzStatus
    int32_t cand;          // the candidate it started at; -1: a given start
    int32_t n_members;     // member ends it crossed
    int32_t flags;         // GzFlags
};

struct GzMemberEnd {       // a member's end, as a decoder crossed it
    int64_t out;           // symbols of the chunk before the end
    int64_t next;          // input offset of the next member's header (n: none)
    uint32_t crc, isize;   // the trailer
};

struct GzSlice {           // output bytes [at, at + len) of one member, mlen bytes in all, `after` of them after the slice
    int64_t at, len, after, mlen;
    int32_t member, first; // first: the member's first slice (it adds the CRC-32's initial register)
};

// The gzip member header at in[at..n): *data = the offset of its deflate data.  0 or a GzStatus, as Python's gzip
// module reads it: FEXTRA, FNAME, FCOMMENT and FHCRC skipped, another method refused; and, as RFC 1952 asks, a reserved
// flag bit refused.
__host__ __device__ inline int gz_header(const uint8_t *in, int64_t n, int64_t at, int64_t *data) {
    if (n - at < 2 || in[at] != 0x1f || in[at + 1] != 0x8b) return GZ_NOT_GZIP;
    if (n - at < 10) return GZ_TRUNC_HEADER;
    if (in[at + 2] != 8) return GZ_BAD_METHOD;
    const int flg = in[at + 3];
    if (flg & 0xe0) return GZ_BAD_FLAGS;
    int64_t p = at + 10;
    if (flg & 4) {                                        // FEXTRA
        if (n - p < 2) return GZ_TRUNC_HEADER;
        p += 2 + ((int64_t)in[p] | ((int64_t)in[p + 1] << 8));
        if (p > n) return GZ_TRUNC_HEADER;
    }
    for (int f = 8; f <= 16; f <<= 1) {                  // FNAME, FCOMMENT: zero-terminated
        if (!(flg & f)) continue;
        while (p < n && in[p]) p++;
        if (p == n) return GZ_TRUNC_HEADER;
        p++;
    }
    if (flg & 2) {                                        // FHCRC
        if (n - p < 2) return GZ_TRUNC_HEADER;
        p += 2;
    }
    *data = p;
    return 0;
}

// x^(8 n) modulo the CRC-32 polynomial for a 64-bit n (bgzf_x8n for members past 4 GiB)
__device__ __forceinline__ uint32_t gz_x8n(uint64_t n) {
    uint32_t r = 0x80000000u, sq = 1u << 23;
    for (; n; n >>= 1) {
        if (n & 1u) r = bgzf_mulmod(r, sq);
        sq = bgzf_mulmod(sq, sq);
    }
    return r;
}

// a bit reader over in[base..n) at bit `bit` of the input
__device__ __forceinline__ void gz_seek(InflBits &b, int64_t &base, const uint8_t *in, int64_t n, int64_t bit) {
    base = bit >> 3;
    const int64_t left = n - base;
    b = InflBits{in + base, (int32_t)(left < GZ_SPAN ? (left > 0 ? left : 0) : GZ_SPAN), 0, 0, 0};
    infl_get(b, (int)(bit & 7));
}

// moves the reader's window forward once it has read GZ_REBASE bytes, so that a reader covers any length of input
__device__ __forceinline__ void gz_rebase(InflBits &b, int64_t &base, int64_t n) {
    if (b.pos <= GZ_REBASE) return;
    const int32_t k = b.pos - 16;
    b.p += k;
    b.pos -= k;
    base += k;
    const int64_t left = n - base;
    b.n = (int32_t)(left < GZ_SPAN ? left : GZ_SPAN);
}

struct GzDecode {          // what one decode reads and where it writes
    const uint8_t *in;
    int64_t n, stop;       // input bytes; it stops at the first block boundary at or past bit `stop`
    uint16_t *sym;         // the chunk's slot of `cap` symbols
    int64_t cap;
    GzMemberEnd *mend;     // the chunk's m_cap member ends
    int32_t m_cap;
};

// Decodes from bit `start` of in[0..n) to the first block boundary at or past bit `stop` (or the end of the stream),
// symbols to sym[0..cap), member ends to mend[0..m_cap).  One thread.  r.status = INFL_OK or why it failed.
__device__ void gz_decode(const GzDecode &d, int64_t start, bool member_start, InflWarpSmem &s, GzRes &r) {
    const uint8_t *in = d.in;
    const int64_t n = d.n, stop = d.stop, cap = d.cap;
    uint16_t *sym = d.sym;
    GzMemberEnd *mend = d.mend;
    const int m_cap = d.m_cap;
    InflBits b;
    int64_t base;
    gz_seek(b, base, in, n, start);
    int64_t pos = 0, mstart = member_start ? 0 : -GZ_WINDOW;   // symbols before mstart are out of reach
    bool fresh = member_start;
    r.start = start;
    r.len = 0;
    r.member_at = -1;
    r.n_members = 0;
    r.flags = 0;
    r.status = INFL_OK;
#define GZ_FAIL(st) do { r.status = (st); r.end = (base + b.pos) * 8 - b.cnt; r.len = pos; return; } while (0)
    for (;;) {                                            // one block per pass
        gz_rebase(b, base, n);
        const int64_t at = (base + b.pos) * 8 - b.cnt;
        if (at >= stop) {
            r.end = at;
            if (fresh) r.flags |= GZ_F_END_MEMBER;
            break;
        }
        fresh = false;
        const int last = (int)infl_get(b, 1);
        const int type = (int)infl_get(b, 2);
        if (type == 0) {                                  // stored
            infl_drop(b, b.cnt & 7);
            const uint32_t len = infl_get(b, 16), nlen = infl_get(b, 16);
            if (infl_past_end(b)) GZ_FAIL(INFL_TRUNCATED);
            if ((len ^ 0xffffu) != nlen) GZ_FAIL(INFL_BAD_STORED);
            for (uint32_t i = 0; i < len; i++, pos++) {
                const uint16_t v = (uint16_t)infl_get(b, 8);
                if (pos < cap) sym[pos] = v;
            }
            if (infl_past_end(b)) GZ_FAIL(INFL_TRUNCATED);
        } else {
            if (type == 3) GZ_FAIL(INFL_BAD_BLOCK);
            if (type == 1) {
                infl_fixed_tables(s);
            } else {
                const int st = infl_dynamic_tables(b, s);
                if (st != INFL_OK) GZ_FAIL(st);
            }
            for (;;) {
                int c = infl_decode(b, s.lit);
                if (c < 0) GZ_FAIL(INFL_BAD_CODE);
                if (infl_past_end(b)) GZ_FAIL(INFL_TRUNCATED);
                if (c < 256) {
                    if (pos < cap) sym[pos] = (uint16_t)c;
                    pos++;
                    gz_rebase(b, base, n);
                    continue;
                }
                if (c == 256) break;
                c -= 257;
                if (c >= 29) GZ_FAIL(INFL_BAD_CODE);
                const int len = infl_c_len_base[c] + (int)infl_get(b, infl_c_len_extra[c]);
                const int dsym = infl_decode(b, s.dist);
                if (dsym < 0 || dsym >= 30) GZ_FAIL(INFL_BAD_CODE);
                const int dist = infl_c_dist_base[dsym] + (int)infl_get(b, infl_c_dist_extra[dsym]);
                if (infl_past_end(b)) GZ_FAIL(INFL_TRUNCATED);
                if (pos - dist < mstart) GZ_FAIL(INFL_BAD_DISTANCE);
                for (int i = 0; i < len; i++, pos++) {
                    if (pos >= cap) continue;
                    const int64_t from = pos - dist;
                    sym[pos] = from >= 0 ? sym[from] : (uint16_t)(GZ_MARK + GZ_WINDOW + from);
                }
                gz_rebase(b, base, n);
            }
        }
        if (!last) continue;
        // the member's trailer follows the final block's last byte, then NUL padding or the next member
        infl_drop(b, b.cnt & 7);
        const uint32_t crc = infl_get(b, 16) | (infl_get(b, 16) << 16);
        const uint32_t isize = infl_get(b, 16) | (infl_get(b, 16) << 16);
        if (infl_past_end(b)) GZ_FAIL(INFL_TRUNCATED);
        int64_t next = base + b.pos - b.cnt / 8;
        while (next < n && in[next] == 0) next++;
        if (r.n_members < m_cap) mend[r.n_members] = GzMemberEnd{pos, next, crc, isize};
        r.n_members++;
        r.member_at = next;
        if (next == n) {
            r.end = 8 * n;
            r.flags |= GZ_F_ENDED;
            break;
        }
        int64_t data = 0;
        const int st = gz_header(in, n, next, &data);
        if (st) GZ_FAIL(st);
        gz_seek(b, base, in, n, 8 * data);
        mstart = pos;
        fresh = true;
    }
#undef GZ_FAIL
    r.len = pos;
    if (pos > cap) r.flags |= GZ_F_OVER;
}

// up to 64 bits of the input from bit `bit` on (bits past the end read as zero)
__device__ __forceinline__ uint64_t gz_bits(const uint8_t *in, int64_t n, int64_t bit) {
    const int64_t at = bit >> 3;
    uint64_t v = 0;
    for (int k = 0; k < 8; k++) v |= (uint64_t)(at + k < n ? in[at + k] : 0u) << (8 * k);
    return v >> (bit & 7);
}

// Whether bit `bit` may start a non-final dynamic block: a necessary condition of infl_dynamic_tables that reads only
// the first 3 + 14 + 57 bits.
__device__ __forceinline__ bool gz_prefilter(const uint8_t *in, int64_t n, int64_t bit) {
    const uint64_t h = gz_bits(in, n, bit);
    if ((h & 7u) != 4u) return false;                     // BFINAL 0, BTYPE 2
    if (((h >> 3) & 31u) > 29u || ((h >> 8) & 31u) > 29u) return false;
    const int ncode = (int)((h >> 13) & 15u) + 4;
    const uint64_t cl = gz_bits(in, n, bit + 17);
    int kraft = 0;
    for (int i = 0; i < ncode; i++) {
        const int l = (int)((cl >> (3 * i)) & 7u);
        if (l) kraft += 128 >> l;
    }
    return kraft == 128;
}

// Whether bit `bit` starts a non-final dynamic block whose header passes infl_dynamic_tables.  (Not inlined, so that
// the finder's loop keeps little state alive across infl_build's calls.)
__device__ __noinline__ bool gz_candidate_ok(const uint8_t *in, int64_t n, int64_t bit, InflWarpSmem &s) {
    InflBits b;
    int64_t rb;
    gz_seek(b, rb, in, n, bit + 3);
    return infl_dynamic_tables(b, s) == INFL_OK;
}

// Chunk c = blockIdx.x: the first GZ_CANDIDATES bit offsets in [lo[c], hi[c]) where a non-final dynamic block header is
// valid, to cand[c * GZ_CANDIDATES ..] (-1 for each one missing).
__global__ void __launch_bounds__(GZ_FIND_THREADS)
gz_k_find(const uint8_t *__restrict__ in, int64_t n, const int64_t *__restrict__ lo, const int64_t *__restrict__ hi,
          int64_t *__restrict__ cand) {
    __shared__ InflWarpSmem s;
    __shared__ uint8_t pass[GZ_FIND_THREADS];
    __shared__ int found;
    const int64_t c = blockIdx.x, a = lo[c], z = hi[c];
    if (threadIdx.x == 0) found = 0;
    __syncthreads();
    for (int64_t base = a; base < z; base += GZ_FIND_THREADS) {
        const int64_t bit = base + threadIdx.x;
        pass[threadIdx.x] = bit < z && gz_prefilter(in, n, bit);
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int t = 0; t < GZ_FIND_THREADS && found < GZ_CANDIDATES; t++) {
                if (pass[t] && gz_candidate_ok(in, n, base + t, s)) cand[c * GZ_CANDIDATES + found++] = base + t;
            }
        }
        __syncthreads();
        if (found >= GZ_CANDIDATES) break;
    }
    if (threadIdx.x == 0)
        for (int k = found; k < GZ_CANDIDATES; k++) cand[c * GZ_CANDIDATES + k] = -1;
}

// Task t = blockIdx.x * INFL_WARPS + warp, decoded by lane 0 into its chunk's slot sym[off[chunk] .. + cap[chunk]);
// a task without a start tries the chunk's candidates in turn and keeps the first that decodes without error.
__global__ void __launch_bounds__(INFL_THREADS, 8)   // (8 CTAs per SM: up to 64 registers, and no spill)
gz_k_decode(const uint8_t *__restrict__ in, int64_t n, const GzTask *__restrict__ tasks, int n_tasks,
            const int64_t *__restrict__ cand, uint16_t *__restrict__ sym, const int64_t *__restrict__ off,
            const int64_t *__restrict__ cap, GzMemberEnd *__restrict__ mend, int m_cap, GzRes *__restrict__ res) {
    __shared__ InflWarpSmem s_warp[INFL_WARPS];
    const int w = threadIdx.x >> 5;
    const int64_t t = (int64_t)blockIdx.x * INFL_WARPS + w;
    if (t >= n_tasks || (threadIdx.x & 31)) return;
    const GzTask T = tasks[t];
    const int c = T.chunk;
    const GzDecode d{in, n, T.stop, sym + off[c], cap[c], mend + (int64_t)c * m_cap, m_cap};
    GzRes r;
    r.status = INFL_BAD_BLOCK;   // (no candidate at all)
    r.start = r.end = r.member_at = -1;
    r.len = 0;
    r.n_members = r.flags = 0;
    r.cand = -1;
    for (int k = T.start >= 0 ? -1 : 0; k < GZ_CANDIDATES; k++) {   // k = -1: the given start
        const int64_t bit = k < 0 ? T.start : cand[(int64_t)c * GZ_CANDIDATES + k];
        if (bit < 0) break;
        gz_decode(d, bit, k < 0 && T.member_start != 0, s_warp[w], r);
        r.cand = k;
        if (k < 0 || r.status == INFL_OK) break;
    }
    res[c] = r;
}

// One thread: chunks a0 .. n_chunks - 1 in order, each one whose start is not its predecessor's end decoded again from
// there; a failure ends the chain (its chunk keeps the status).  *n_decoded = the decodes it ran.
__global__ void __launch_bounds__(32)
gz_k_chain(const uint8_t *__restrict__ in, int64_t n, const GzTask *__restrict__ tasks, int a0, int n_chunks,
           uint16_t *__restrict__ sym, const int64_t *__restrict__ off, const int64_t *__restrict__ cap,
           GzMemberEnd *__restrict__ mend, int m_cap, GzRes *__restrict__ res, int *__restrict__ n_decoded) {
    __shared__ InflWarpSmem s;
    if (threadIdx.x) return;
    int done = 0;
    for (int a = a0; a < n_chunks; a++) {
        const GzRes p = res[a - 1];
        if (p.status != INFL_OK) break;
        if (p.flags & GZ_F_ENDED) {                       // nothing after the stream's end
            res[a] = GzRes{p.end, p.end, 0, -1, INFL_OK, -1, 0, GZ_F_ENDED};
            continue;
        }
        if (res[a].status == INFL_OK && res[a].start == p.end) continue;
        GzRes r;
        const GzDecode d{in, n, tasks[a].stop, sym + off[a], cap[a], mend + (int64_t)a * m_cap, m_cap};
        gz_decode(d, p.end, (p.flags & GZ_F_END_MEMBER) != 0, s, r);
        r.cand = -1;
        res[a] = r;
        done++;
        if (r.status != INFL_OK) break;
    }
    *n_decoded = done;
}

// One CTA, chunks in order: win[k] = the 32 KiB of output before chunk k (out_at[k]), from chunk k - 1's symbols and
// window.  Bytes before the stream read as zero (a symbol that reaches them is refused by gz_k_resolve).
__global__ void __launch_bounds__(GZ_WINDOW_THREADS)
gz_k_windows(const uint16_t *__restrict__ sym, const int64_t *__restrict__ off, const int64_t *__restrict__ out_at,
             int n_chunks, uint8_t *__restrict__ win) {
    for (int k = 1; k < n_chunks; k++) {
        const int64_t p0 = out_at[k - 1], w0 = p0 - GZ_WINDOW, me = out_at[k] - GZ_WINDOW;
        const uint16_t *ps = sym + off[k - 1];
        const uint8_t *pw = win + (int64_t)(k - 1) * GZ_WINDOW;
        uint8_t *dst = win + (int64_t)k * GZ_WINDOW;
        for (int t = threadIdx.x; t < GZ_WINDOW; t += GZ_WINDOW_THREADS) {
            const int64_t g = me + t;
            uint8_t v = 0;
            if (g >= p0) {
                const uint16_t x = ps[g - p0];
                v = x < GZ_MARK ? (uint8_t)x : pw[x - GZ_MARK];
            } else if (g >= 0) {
                v = pw[g - w0];
            }
            dst[t] = v;
        }
        __syncthreads();
    }
}

// Chunk k = blockIdx.x: out[out_at[k] + i] = its symbol i, a window symbol read from win[k].  A symbol reaching before
// lo[k], the start of the member the chunk starts in, puts its output offset into *bad (the least one is kept).
__global__ void __launch_bounds__(GZ_RESOLVE_THREADS)
gz_k_resolve(const uint16_t *__restrict__ sym, const int64_t *__restrict__ off, const int64_t *__restrict__ out_at,
             const int64_t *__restrict__ lo, const uint8_t *__restrict__ win, uint8_t *__restrict__ out,
             unsigned long long *__restrict__ bad) {
    const int64_t k = blockIdx.x, at = out_at[k], len = out_at[k + 1] - at, first = lo[k] - (at - GZ_WINDOW);
    const uint16_t *src = sym + off[k];
    const uint8_t *w = win + k * GZ_WINDOW;
    for (int64_t i = threadIdx.x; i < len; i += GZ_RESOLVE_THREADS) {
        const uint16_t x = src[i];
        uint8_t v = (uint8_t)x;
        if (x >= GZ_MARK) {
            if ((int64_t)(x - GZ_MARK) < first) {
                atomicMin(bad, (unsigned long long)(at + i));
                v = 0;
            } else {
                v = w[x - GZ_MARK];
            }
        }
        out[at + i] = v;
    }
}

// Slice s = blockIdx.x * INFL_WARPS + warp: the CRC-32 register of its bytes moved past the rest of its member, XORed
// into acc[member] (the member's first slice also adds the initial register's term): acc[m] ends as ~CRC-32.
__global__ void __launch_bounds__(INFL_THREADS)
gz_k_crc(const uint8_t *__restrict__ out, const GzSlice *__restrict__ slices, int64_t n_slices, uint32_t *__restrict__ acc) {
    __shared__ uint32_t crc_table[256];
    for (int i = threadIdx.x; i < 256; i += INFL_THREADS) crc_table[i] = bgzf_crc_entry((uint32_t)i);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t si = (int64_t)blockIdx.x * INFL_WARPS + (threadIdx.x >> 5);
    if (si >= n_slices) return;
    const GzSlice S = slices[si];
    const int64_t per = (S.len + 31) / 32;
    const int64_t a0 = lane * per < S.len ? lane * per : S.len, a1 = a0 + per < S.len ? a0 + per : S.len;
    uint32_t crc = 0;
    for (int64_t i = a0; i < a1; i++) crc = crc_table[(crc ^ out[S.at + i]) & 0xffu] ^ (crc >> 8);
    uint32_t term = a1 > a0 ? bgzf_mulmod(crc, gz_x8n((uint64_t)(S.len - a1 + S.after))) : 0u;
    for (int d = 16; d > 0; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
    if (lane == 0) {
        if (S.first) term ^= bgzf_mulmod(0xffffffffu, gz_x8n((uint64_t)S.mlen));
        atomicXor(acc + S.member, term);
    }
}

// ---------------------------------------------------------------------------------------------------- host side
// The driver, over a device backend Dev (CUDA in bb_tu_gunzip.cu, the warp emulator in the tests) that provides
// alloc / release / h2d / d2h / fill / sync (0 or an error code), fail(what, code, msg, msg_len) -> BB_ERR_CUDA, and one
// launcher per kernel with the kernel's grid and arguments.

#define GZ_DEFAULT_CHUNK (1 << 17)   // compressed bytes per chunk (DESIGN.md §4: 16 to 256 KiB measured)
#define GZ_REPAIR_ROUNDS 4
#define GZ_RATIO 4                   // symbol slots: this many per input byte of the chunk's span, plus a quarter

inline int gz_fail(char *msg, size_t msg_len, int64_t idx, int64_t at, int st) {
    const char *why;
    switch (st) {
        case GZ_NOT_GZIP: why = idx ? "bytes after the last member that are neither NUL padding nor a gzip member"
                                    : "not a gzip stream (no gzip magic)"; break;
        case GZ_BAD_METHOD: why = "compression method other than deflate"; break;
        case GZ_BAD_FLAGS: why = "reserved header flag set"; break;
        case GZ_TRUNC_HEADER: why = "truncated header"; break;
        case GZ_BAD_ISIZE: why = "ISIZE does not match the inflated length"; break;
        default: why = infl_status_text(st);
    }
    std::snprintf(msg, msg_len, "bb_gzip_decompress: member %lld (offset %lld): %s", (long long)idx, (long long)at, why);
    return BB_ERR_ARG;
}

template <class Dev> struct GzBuf {   // a device buffer released on every exit path
    Dev &dev;
    void *p = nullptr;
    explicit GzBuf(Dev &d) : dev(d) {}
    ~GzBuf() { release(); }
    void release() { if (p) dev.release(p); p = nullptr; }
    int alloc(size_t bytes) { release(); return dev.alloc(&p, bytes < 16 ? 16 : bytes); }
    template <class T> int upload(const std::vector<T> &v) {
        int e = alloc(v.size() * sizeof(T));
        if (!e && !v.empty()) e = dev.h2d(p, v.data(), v.size() * sizeof(T));
        return e;
    }
    template <class T> T *as() const { return (T *)p; }
};

#define GZ_TRY(call) do { const int e_ = (call); if (e_) return dev.fail(#call, e_, msg, msg_len); } while (0)

// The chunked inflater on in[0..n) (host memory): on success *out is a device buffer of *total bytes (at least 16
// allocated) that the caller releases; otherwise BB_ERR_ARG with msg naming the member (index and input offset).
template <class Dev>
int gz_inflate(Dev &dev, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out, int64_t *total,
               bb_gzip_stats *stats, char *msg, size_t msg_len) {
    GzBuf<Dev> d_out(dev), d_in(dev), d_lo(dev), d_hi(dev), d_cand(dev), d_tasks(dev), d_sym(dev), d_off(dev), d_cap(dev),
        d_mend(dev), d_res(dev), d_count(dev);
    if (n == 0) {   // an empty file holds no members
        GZ_TRY(d_out.alloc(16));
        *out = d_out.template as<uint8_t>();
        d_out.p = nullptr;
        *total = 0;
        return BB_OK;
    }
    int64_t data0 = 0;
    if (const int e = gz_header(in, n, 0, &data0)) return gz_fail(msg, msg_len, 0, 0, e);
    const int64_t C = chunk_bytes > 0 ? chunk_bytes : GZ_DEFAULT_CHUNK;
    const int64_t n_chunks = std::max<int64_t>(1, (n - data0 + C - 1) / C);
    GZ_TRY(d_in.alloc((size_t)n));
    GZ_TRY(dev.h2d(d_in.p, in, (size_t)n));
    const uint8_t *din = d_in.template as<uint8_t>();

    // block starts of every chunk but the first
    std::vector<int64_t> lo(n_chunks), hi(n_chunks), cand((size_t)n_chunks * GZ_CANDIDATES, -1);
    for (int64_t j = 0; j < n_chunks; j++) {
        lo[j] = 8 * (data0 + j * C);
        hi[j] = 8 * std::min(data0 + (j + 1) * C, n);
    }
    if (n_chunks > 1) {
        GZ_TRY(d_lo.upload(lo));
        GZ_TRY(d_hi.upload(hi));
        GZ_TRY(d_cand.alloc(cand.size() * sizeof(int64_t)));
        dev.find((unsigned)(n_chunks - 1), din, n, d_lo.template as<int64_t>() + 1, d_hi.template as<int64_t>() + 1,
                 d_cand.template as<int64_t>() + GZ_CANDIDATES);
        GZ_TRY(dev.d2h(cand.data() + GZ_CANDIDATES, d_cand.template as<int64_t>() + GZ_CANDIDATES,
                       (cand.size() - GZ_CANDIDATES) * sizeof(int64_t)));
        GZ_TRY(dev.sync());
    }
    // the chunks with a candidate (and the first): a chunk without one is absorbed by its predecessor
    std::vector<int64_t> act{0};
    for (int64_t j = 1; j < n_chunks; j++)
        if (cand[(size_t)j * GZ_CANDIDATES] >= 0) act.push_back(j);
    const int na = (int)act.size();
    std::vector<GzTask> tasks(na);
    std::vector<int64_t> acand((size_t)na * GZ_CANDIDATES), cap(na), off(na + 1);
    for (int a = 0; a < na; a++) {
        const int64_t from = lo[act[a]] / 8, to = a + 1 < na ? lo[act[a + 1]] / 8 : n;
        tasks[a] = GzTask{a ? -1 : 8 * data0, a + 1 < na ? lo[act[a + 1]] : INT64_MAX, a, a ? 0 : 1};
        std::copy_n(cand.begin() + act[a] * GZ_CANDIDATES, GZ_CANDIDATES, acand.begin() + (size_t)a * GZ_CANDIDATES);
        cap[a] = GZ_RATIO * ((to - from) + (to - from) / 4) + 4096;
    }
    stats->chunks = n_chunks;
    stats->absorbed = n_chunks - na;
    GZ_TRY(d_cand.upload(acand));
    int m_cap = 4;
    std::vector<GzRes> res(na);
    auto alloc_slots = [&]() -> int {
        d_sym.release();
        d_mend.release();
        off[0] = 0;
        for (int a = 0; a < na; a++) off[a + 1] = off[a] + cap[a];
        int e = d_off.upload(off);
        if (!e) e = d_cap.upload(cap);
        if (!e) e = d_sym.alloc((size_t)off[na] * sizeof(uint16_t));
        if (!e) e = d_mend.alloc((size_t)na * m_cap * sizeof(GzMemberEnd));
        return e;
    };
    auto decode = [&](const std::vector<GzTask> &ts) -> int {
        int e = d_tasks.upload(ts);
        if (e || ts.empty()) return e;
        const int nt = (int)ts.size();
        dev.decode((unsigned)((nt + INFL_WARPS - 1) / INFL_WARPS), din, n, d_tasks.template as<GzTask>(), nt,
                   d_cand.template as<int64_t>(), d_sym.template as<uint16_t>(), d_off.template as<int64_t>(),
                   d_cap.template as<int64_t>(), d_mend.template as<GzMemberEnd>(), m_cap, d_res.template as<GzRes>());
        if ((e = dev.d2h(res.data(), d_res.p, res.size() * sizeof(GzRes)))) return e;
        return dev.sync();
    };
    // the member a failing chunk's decode failed in: (index, input offset)
    auto fail_at = [&](int a) {
        int64_t idx = 0, at = 0;
        for (int b = 0; b < a; b++) {
            idx += res[b].n_members;
            if (res[b].member_at >= 0) at = res[b].member_at;
        }
        return gz_fail(msg, msg_len, idx + res[a].n_members, res[a].member_at >= 0 ? res[a].member_at : at, res[a].status);
    };
    GZ_TRY(alloc_slots());
    GZ_TRY(d_res.alloc(res.size() * sizeof(GzRes)));
    GZ_TRY(decode(tasks));
    if (res[0].status != INFL_OK) return fail_at(0);

    // stitching: res[0 .. P) are confirmed, each one starting where its predecessor stopped
    int P = 1;
    auto extend = [&]() {
        for (; P < na; P++) {
            const GzRes &p = res[P - 1];
            if (p.flags & GZ_F_ENDED) res[P] = GzRes{p.end, p.end, 0, -1, INFL_OK, -1, 0, GZ_F_ENDED};
            else if (res[P].status != INFL_OK || res[P].start != p.end) break;
        }
    };
    extend();
    for (int round = 0; round < GZ_REPAIR_ROUNDS && P < na; round++) {
        std::vector<GzTask> rep;   // every chunk whose start is not where its (possibly unconfirmed) predecessor stopped
        for (int a = P; a < na; a++) {
            const GzRes &p = res[a - 1];
            if (p.status != INFL_OK || (p.flags & GZ_F_ENDED)) continue;
            if (a > P && res[a].status == INFL_OK && res[a].start == p.end) continue;
            rep.push_back(GzTask{p.end, tasks[a].stop, a, (p.flags & GZ_F_END_MEMBER) ? 1 : 0});
        }
        GZ_TRY(decode(rep));
        stats->repaired += (int64_t)rep.size();
        if (res[P].status != INFL_OK) return fail_at(P);   // (it started where a confirmed decode stopped)
        extend();
    }
    if (P < na) {   // what is left: one chain on the device
        int chained = 0;
        GZ_TRY(dev.h2d(d_res.p, res.data(), res.size() * sizeof(GzRes)));
        GZ_TRY(d_count.alloc(sizeof(int)));
        GZ_TRY(d_tasks.upload(tasks));
        dev.chain(din, n, d_tasks.template as<GzTask>(), P, na, d_sym.template as<uint16_t>(), d_off.template as<int64_t>(),
                  d_cap.template as<int64_t>(), d_mend.template as<GzMemberEnd>(), m_cap, d_res.template as<GzRes>(),
                  d_count.template as<int>());
        GZ_TRY(dev.d2h(res.data(), d_res.p, res.size() * sizeof(GzRes)));
        GZ_TRY(dev.d2h(&chained, d_count.p, sizeof(int)));
        GZ_TRY(dev.sync());
        stats->chained = chained;
        extend();
        if (P < na) return fail_at(P);
    }
    for (int a = 1; a < na; a++) stats->first_candidate += res[a].cand == 0;

    // slots or member records too small: every chunk decoded again from its confirmed start
    int need_m = m_cap;
    bool over = false;
    for (int a = 0; a < na; a++) {
        need_m = std::max(need_m, res[a].n_members);
        if (res[a].flags & GZ_F_OVER) {
            cap[a] = res[a].len;
            over = true;
        }
    }
    if (over || need_m > m_cap) {
        stats->reruns++;
        m_cap = need_m;
        GZ_TRY(alloc_slots());
        std::vector<GzTask> again;
        for (int a = 0; a < na; a++)
            if (res[a].start < 8 * n)   // (not an empty chunk after the stream's end)
                again.push_back(GzTask{res[a].start, tasks[a].stop, a, (!a || (res[a - 1].flags & GZ_F_END_MEMBER)) ? 1 : 0});
        const std::vector<GzRes> before = res;
        GZ_TRY(decode(again));
        for (const GzTask &t : again)
            if (res[t.chunk].status != INFL_OK || res[t.chunk].end != before[t.chunk].end || (res[t.chunk].flags & GZ_F_OVER))
                return fail_at(t.chunk);
        for (int a = 0; a < na; a++)
            if (before[a].start >= 8 * n) res[a] = before[a];
    }

    // the chunks' places in the output and the members
    std::vector<int64_t> out_at(na + 1), mlo(na);
    out_at[0] = 0;
    for (int a = 0; a < na; a++) out_at[a + 1] = out_at[a] + res[a].len;
    const int64_t len = out_at[na];
    std::vector<GzMemberEnd> mend((size_t)na * m_cap);
    GZ_TRY(dev.d2h(mend.data(), d_mend.p, mend.size() * sizeof(GzMemberEnd)));
    GZ_TRY(dev.sync());
    struct Member { int64_t lo, hi, at; uint32_t crc, isize; };
    std::vector<Member> members;
    int64_t m_lo = 0, m_at = 0;
    for (int a = 0; a < na; a++) {
        mlo[a] = m_lo;
        for (int k = 0; k < res[a].n_members; k++) {
            const GzMemberEnd &e = mend[(size_t)a * m_cap + k];
            members.push_back(Member{m_lo, out_at[a] + e.out, m_at, e.crc, e.isize});
            m_lo = out_at[a] + e.out;
            m_at = e.next;
        }
    }
    stats->members = (int64_t)members.size();

    // windows, then symbols to bytes
    GzBuf<Dev> d_at(dev), d_mlo(dev), d_win(dev), d_bad(dev), d_slices(dev), d_acc(dev);
    GZ_TRY(d_out.alloc((size_t)len));
    GZ_TRY(d_at.upload(out_at));
    GZ_TRY(d_mlo.upload(mlo));
    GZ_TRY(d_win.alloc((size_t)na * GZ_WINDOW));
    GZ_TRY(d_bad.alloc(sizeof(unsigned long long)));
    GZ_TRY(dev.fill(d_bad.p, 0xff, sizeof(unsigned long long)));
    if (na > 1)
        dev.windows(d_sym.template as<uint16_t>(), d_off.template as<int64_t>(), d_at.template as<int64_t>(), na,
                    d_win.template as<uint8_t>());
    dev.resolve((unsigned)na, d_sym.template as<uint16_t>(), d_off.template as<int64_t>(), d_at.template as<int64_t>(),
                d_mlo.template as<int64_t>(), d_win.template as<uint8_t>(), d_out.template as<uint8_t>(),
                d_bad.template as<unsigned long long>());
    unsigned long long bad = 0;
    GZ_TRY(dev.d2h(&bad, d_bad.p, sizeof(bad)));
    GZ_TRY(dev.sync());
    if (bad != ~0ull) {
        size_t m = 0;
        while (m + 1 < members.size() && members[m].hi <= (int64_t)bad) m++;
        return gz_fail(msg, msg_len, (int64_t)m, members[m].at, INFL_BAD_DISTANCE);
    }
    d_sym.release();
    d_win.release();

    // CRC-32 and ISIZE of every member
    std::vector<GzSlice> slices;
    for (size_t m = 0; m < members.size(); m++) {
        const int64_t mlen = members[m].hi - members[m].lo;
        int64_t at = 0;
        do {
            const int64_t l = std::min<int64_t>(GZ_SLICE, mlen - at);
            slices.push_back(GzSlice{members[m].lo + at, l, mlen - at - l, mlen, (int32_t)m, at == 0});
            at += l;
        } while (at < mlen);
    }
    std::vector<uint32_t> acc(members.size());
    if (!slices.empty()) {
        GZ_TRY(d_slices.upload(slices));
        GZ_TRY(d_acc.alloc(acc.size() * sizeof(uint32_t)));
        GZ_TRY(dev.fill(d_acc.p, 0, acc.size() * sizeof(uint32_t)));
        const int64_t ns = (int64_t)slices.size();
        dev.crc((unsigned)((ns + INFL_WARPS - 1) / INFL_WARPS), d_out.template as<uint8_t>(), d_slices.template as<GzSlice>(), ns,
                d_acc.template as<uint32_t>());
        GZ_TRY(dev.d2h(acc.data(), d_acc.p, acc.size() * sizeof(uint32_t)));
        GZ_TRY(dev.sync());
    }
    for (size_t m = 0; m < members.size(); m++) {
        if (~acc[m] != members[m].crc) return gz_fail(msg, msg_len, (int64_t)m, members[m].at, INFL_BAD_CRC);
        if ((uint32_t)(members[m].hi - members[m].lo) != members[m].isize)
            return gz_fail(msg, msg_len, (int64_t)m, members[m].at, GZ_BAD_ISIZE);
    }
    *out = d_out.template as<uint8_t>();
    d_out.p = nullptr;
    *total = len;
    return BB_OK;
}
#undef GZ_TRY
