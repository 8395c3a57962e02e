// bb_inflate.cuh — BGZF decompression (SAM specification §4.1) on the device: the reader side of bb_bgzf.cuh.
//
// A BGZF file is a series of independent gzip members of at most 64 KiB each, every one with its compressed size in a
// "BC" extra field, its CRC-32 and its inflated size (ISIZE) in the trailer.  The host walks the headers (infl_walk
// below), so every member's input range and, from the ISIZEs, its place in the output are known before any inflating;
// then one warp inflates one member.  Deflate decoding is serial within a member, so lane 0 decodes (stored, fixed and
// dynamic Huffman blocks, back-references anywhere in what the member has produced) straight into the output, and the
// whole warp then checks the CRC-32 over slices of the member, combined as bb_bgzf.cuh combines them.
//
// Every read stays inside the member's deflate data (bits past its end read as zero and mark the member truncated),
// every write inside the member's ISIZE bytes, and every loop consumes input or produces output, so malformed input
// ends with a status per member, never with a fault or a hang.
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>
#include <cstdio>
#include <vector>

#include "bb_crc32.cuh"

#define INFL_WARPS 4                 // members per CTA
#define INFL_THREADS (32 * INFL_WARPS)
#define INFL_MAX_ISIZE 65536         // the largest member BGZF allows, inflated
#define INFL_FAST 9                  // bits resolved by one lookup of the decode tables

enum InflStatus {
    INFL_OK = 0, INFL_TRUNCATED = 1, INFL_BAD_BLOCK = 2, INFL_BAD_STORED = 3, INFL_BAD_TABLE = 4, INFL_BAD_CODE = 5,
    INFL_BAD_DISTANCE = 6, INFL_OVERRUN = 7, INFL_SHORT = 8, INFL_BAD_CRC = 9, INFL_TRAILING = 10
};

struct InflMember {      // one member, from the host walk
    int64_t at;          // offset of the member in the input
    int64_t data;        // offset of its deflate data in the input
    int64_t out;         // offset of its bytes in the output
    int32_t n_data;      // bytes of deflate data
    int32_t isize;       // inflated size (trailer)
    uint32_t crc;        // CRC-32 of the inflated bytes (trailer)
    int32_t pad;
};

struct InflHuff {                       // canonical Huffman code (RFC 1951 §3.2.2)
    uint16_t count[16];                 // codes of each length
    uint16_t sym[288];                  // symbols by code
    uint16_t fast[1 << INFL_FAST];      // (symbol << 4) | length of the code the next INFL_FAST bits start with; 0: longer
};

struct InflWarpSmem {
    InflHuff lit, dist;
    uint8_t lens[320];
};

__constant__ uint8_t infl_c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ uint16_t infl_c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83,
                                             99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t infl_c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t infl_c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                              1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t infl_c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                              12, 12, 13, 13};

// LSB-first bit reader over one member's deflate data
struct InflBits {
    const uint8_t *p;
    int32_t n, pos;      // bytes, next byte to load (may run past n: those bytes read as zero)
    uint64_t buf;
    int cnt;             // bits in buf
};

__device__ __forceinline__ void infl_fill(InflBits &b) {
    while (b.cnt <= 56) {
        const uint64_t byte = b.pos < b.n ? b.p[b.pos] : 0u;
        b.pos++;
        b.buf |= byte << b.cnt;
        b.cnt += 8;
    }
}
__device__ __forceinline__ uint32_t infl_peek(InflBits &b, int n) {
    if (b.cnt < n) infl_fill(b);
    return (uint32_t)(b.buf & ((1ull << n) - 1));
}
__device__ __forceinline__ void infl_drop(InflBits &b, int n) { b.buf >>= n; b.cnt -= n; }
__device__ __forceinline__ uint32_t infl_get(InflBits &b, int n) {
    const uint32_t v = infl_peek(b, n);
    infl_drop(b, n);
    return v;
}
// more bits consumed than the member holds
__device__ __forceinline__ bool infl_past_end(const InflBits &b) { return (int64_t)b.pos * 8 - b.cnt > (int64_t)b.n * 8; }

// Code of the lengths len[0..n): > 0 incomplete, < 0 over-subscribed, 0 complete (or no codes at all).  One thread.
__device__ int infl_build(InflHuff &h, const uint8_t *len, int n) {
    for (int l = 0; l < 16; l++) h.count[l] = 0;
    for (int s = 0; s < n; s++) h.count[len[s]]++;
    int left = 1;
    for (int l = 1; l < 16; l++) {
        left = (left << 1) - h.count[l];
        if (left < 0) return left;
    }
    if (h.count[0] == n) left = 0;
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = (uint16_t)(offs[l] + h.count[l]);
    for (int s = 0; s < n; s++)
        if (len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
    for (int i = 0; i < (1 << INFL_FAST); i++) h.fast[i] = 0;
    uint32_t code = 0;
    int k = 0;
    for (int l = 1; l <= INFL_FAST; l++) {
        for (int c = 0; c < h.count[l]; c++, k++, code++) {
            const uint32_t rev = __brev(code) >> (32 - l);
            for (uint32_t f = rev; f < (1u << INFL_FAST); f += 1u << l) h.fast[f] = (uint16_t)((h.sym[k] << 4) | l);
        }
        code <<= 1;
    }
    return left;
}

// The next symbol of code h, or -1 if the bits are no code of it.
__device__ __forceinline__ int infl_decode(InflBits &b, const InflHuff &h) {
    const uint32_t bits = infl_peek(b, 15);
    const uint16_t e = h.fast[bits & ((1u << INFL_FAST) - 1)];
    if (e) {
        infl_drop(b, e & 15);
        return e >> 4;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; l++) {
        code |= (int)((bits >> (l - 1)) & 1u);
        const int count = h.count[l];
        if (code - count < first) {
            infl_drop(b, l);
            return h.sym[index + (code - first)];
        }
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

// zlib's rule for a literal / length or distance code: complete, or a single code of one bit, or (distances) none.
__device__ __forceinline__ bool infl_code_ok(const InflHuff &h, int err, int n) {
    if (err < 0) return false;
    if (err == 0) return true;
    return h.count[1] == 1 && n - h.count[0] == 1;
}

// The header of a dynamic Huffman block after its 3 type bits: the code-length code, the run-length coded code lengths
// and the literal / length and distance codes built into s.lit and s.dist.  One thread.  Returns an InflStatus.  The
// block finder of bb_gunzip.cuh holds candidate block starts to these same rules.
__device__ __forceinline__ int infl_dynamic_tables(InflBits &b, InflWarpSmem &s) {
    const int nlen = (int)infl_get(b, 5) + 257, ndist = (int)infl_get(b, 5) + 1, ncode = (int)infl_get(b, 4) + 4;
    if (nlen > 286 || ndist > 30) return INFL_BAD_TABLE;
    for (int i = 0; i < 19; i++) s.lens[infl_c_cl_order[i]] = i < ncode ? (uint8_t)infl_get(b, 3) : 0;
    if (infl_past_end(b)) return INFL_TRUNCATED;
    if (infl_build(s.lit, s.lens, 19) != 0) return INFL_BAD_TABLE;   // (the code-length code, complete)
    for (int i = 0; i < nlen + ndist;) {
        const int sym = infl_decode(b, s.lit);
        if (sym < 0) return INFL_BAD_TABLE;
        if (infl_past_end(b)) return INFL_TRUNCATED;
        if (sym < 16) {
            s.lens[i++] = (uint8_t)sym;
            continue;
        }
        uint8_t v = 0;
        int rep;
        if (sym == 16) {
            if (i == 0) return INFL_BAD_TABLE;
            v = s.lens[i - 1];
            rep = 3 + (int)infl_get(b, 2);
        } else if (sym == 17) {
            rep = 3 + (int)infl_get(b, 3);
        } else {
            rep = 11 + (int)infl_get(b, 7);
        }
        if (i + rep > nlen + ndist) return INFL_BAD_TABLE;
        while (rep--) s.lens[i++] = v;
    }
    if (s.lens[256] == 0) return INFL_BAD_TABLE;  // no end-of-block code
    int err = infl_build(s.lit, s.lens, nlen);
    if (!infl_code_ok(s.lit, err, nlen)) return INFL_BAD_TABLE;
    err = infl_build(s.dist, s.lens + nlen, ndist);
    if (!infl_code_ok(s.dist, err, ndist)) return INFL_BAD_TABLE;   // (no distance codes at all: accepted)
    return INFL_OK;
}

// The fixed Huffman codes (RFC 1951 §3.2.6) built into s.lit and s.dist.  One thread.
__device__ __forceinline__ void infl_fixed_tables(InflWarpSmem &s) {
    for (int i = 0; i < 288; i++) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
    infl_build(s.lit, s.lens, 288);
    for (int i = 0; i < 30; i++) s.lens[i] = 5;
    infl_build(s.dist, s.lens, 30);
}

// Inflates one member's deflate data in[0..n) into out[0..isize).  One thread.  Returns an InflStatus.
__device__ int infl_member(const uint8_t *in, int32_t n, uint8_t *out, int32_t isize, InflWarpSmem &s) {
    InflBits b{in, n, 0, 0, 0};
    int32_t pos = 0;
    int last;
    do {
        last = (int)infl_get(b, 1);
        const int type = (int)infl_get(b, 2);
        if (type == 0) {                                  // stored
            infl_drop(b, b.cnt & 7);
            const uint32_t len = infl_get(b, 16), nlen = infl_get(b, 16);
            if (infl_past_end(b)) return INFL_TRUNCATED;
            if ((len ^ 0xffffu) != nlen) return INFL_BAD_STORED;
            if ((int64_t)pos + len > isize) return INFL_OVERRUN;
            for (uint32_t i = 0; i < len; i++) out[pos++] = (uint8_t)infl_get(b, 8);
            if (infl_past_end(b)) return INFL_TRUNCATED;
            continue;
        }
        if (type == 3) return INFL_BAD_BLOCK;
        if (type == 1) {                                  // fixed Huffman codes
            infl_fixed_tables(s);
        } else {                                          // dynamic Huffman codes
            const int st = infl_dynamic_tables(b, s);
            if (st != INFL_OK) return st;
        }
        for (;;) {
            int sym = infl_decode(b, s.lit);
            if (sym < 0) return INFL_BAD_CODE;
            if (infl_past_end(b)) return INFL_TRUNCATED;
            if (sym < 256) {
                if (pos >= isize) return INFL_OVERRUN;
                out[pos++] = (uint8_t)sym;
                continue;
            }
            if (sym == 256) break;
            sym -= 257;
            if (sym >= 29) return INFL_BAD_CODE;
            const int len = infl_c_len_base[sym] + (int)infl_get(b, infl_c_len_extra[sym]);
            const int dsym = infl_decode(b, s.dist);
            if (dsym < 0 || dsym >= 30) return INFL_BAD_CODE;
            const int dist = infl_c_dist_base[dsym] + (int)infl_get(b, infl_c_dist_extra[dsym]);
            if (infl_past_end(b)) return INFL_TRUNCATED;
            if (dist > pos) return INFL_BAD_DISTANCE;
            if (pos + len > isize) return INFL_OVERRUN;
            for (int i = 0; i < len; i++, pos++) out[pos] = out[pos - dist];
        }
    } while (!last);
    // the trailer follows the final block's last byte: zlib and gzip refuse bytes in between (they read them as CRC-32)
    if (((int64_t)b.pos * 8 - b.cnt + 7) / 8 < n) return INFL_TRAILING;
    return pos == isize ? INFL_OK : INFL_SHORT;
}

#ifndef INFL_NO_MEMBER_KERNEL   // (bb_tu_gunzip.cu uses the decoder, not this kernel)
// Member m = blockIdx.x * INFL_WARPS + warp: its deflate data in[members[m].data ..] inflated to out[members[m].out ..],
// then its CRC-32 checked; status[m] = InflStatus.
__global__ void __launch_bounds__(INFL_THREADS)
infl_k_members(const uint8_t *__restrict__ in, const InflMember *__restrict__ members, int64_t n_members,
               uint8_t *__restrict__ out, int32_t *__restrict__ status) {
    __shared__ uint32_t crc_table[256];
    __shared__ InflWarpSmem s_warp[INFL_WARPS];
    for (int i = threadIdx.x; i < 256; i += INFL_THREADS) crc_table[i] = bgzf_crc_entry((uint32_t)i);
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t m = (int64_t)blockIdx.x * INFL_WARPS + w;
    if (m >= n_members) return;
    const InflMember M = members[m];
    uint8_t *dst = out + M.out;
    int st = INFL_OK;
    if (lane == 0) st = infl_member(in + M.data, M.n_data, dst, M.isize, s_warp[w]);
    __syncwarp();
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == INFL_OK) {
        const int len = M.isize, per = (len + 31) / 32;
        const int a0 = lane * per < len ? lane * per : len, a1 = a0 + per < len ? a0 + per : len;
        uint32_t crc = 0;
        for (int i = a0; i < a1; i++) crc = crc_table[(crc ^ dst[i]) & 0xffu] ^ (crc >> 8);
        uint32_t term = a1 > a0 ? bgzf_mulmod(crc, bgzf_x8n((uint32_t)(len - a1))) : 0u;
        for (int d = 16; d > 0; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
        if (lane == 0 && ~(bgzf_mulmod(0xffffffffu, bgzf_x8n((uint32_t)len)) ^ term) != M.crc) st = INFL_BAD_CRC;
    }
    if (lane == 0) status[m] = st;
}
#endif

// ---------------------------------------------------------------------------------------------------- host side
inline const char *infl_status_text(int st) {
    switch (st) {
        case INFL_TRUNCATED: return "truncated deflate data";
        case INFL_BAD_BLOCK: return "invalid block type";
        case INFL_BAD_STORED: return "stored block length does not match its complement";
        case INFL_BAD_TABLE: return "invalid Huffman table";
        case INFL_BAD_CODE: return "invalid Huffman code";
        case INFL_BAD_DISTANCE: return "back-reference before the start of the member";
        case INFL_OVERRUN: return "more data than the ISIZE of the trailer";
        case INFL_SHORT: return "less data than the ISIZE of the trailer";
        case INFL_BAD_CRC: return "CRC-32 mismatch";
        case INFL_TRAILING: return "bytes between the final deflate block and the trailer";
        default: return "ok";
    }
}

inline void infl_message(char *msg, size_t msg_len, int64_t idx, int64_t at, const char *why) {
    std::snprintf(msg, msg_len, "bb_bgzf_decompress: member %lld (offset %lld): %s", (long long)idx, (long long)at, why);
}

// Walks the members of the BGZF stream in[0..n): every member's deflate data, output offset, ISIZE and CRC-32, and
// *total = the inflated size of the stream.  Returns false with a message naming the member for input that is not BGZF
// (no gzip magic, another method, a gzip member without the BC field), a member that runs past the end, or an ISIZE
// beyond 64 KiB.
inline bool infl_walk(const uint8_t *in, int64_t n, std::vector<InflMember> &members, int64_t *total, char *msg, size_t msg_len) {
    auto le16 = [&](int64_t at) { return (uint32_t)in[at] | ((uint32_t)in[at + 1] << 8); };
    auto le32 = [&](int64_t at) { return le16(at) | (le16(at + 2) << 16); };
    members.clear();
    int64_t pos = 0, out = 0;
    for (int64_t idx = 0; pos < n; idx++) {
        const char *why = nullptr;
        uint32_t bsize = 0;
        int64_t xlen = 0;
        if (n - pos < 12) {
            why = "truncated header";
        } else if (in[pos] != 0x1f || in[pos + 1] != 0x8b || in[pos + 2] != 8) {
            why = "not a gzip member with deflate data: the input is not BGZF";
        } else if (in[pos + 3] != 4) {
            why = "gzip member without the BC extra field of BGZF (or with other header fields)";
        } else {
            xlen = le16(pos + 10);
            if (pos + 12 + xlen > n) {
                why = "truncated header";
            } else {
                bool found = false;
                for (int64_t f = pos + 12; f + 4 <= pos + 12 + xlen;) {
                    const int64_t slen = le16(f + 2);
                    if (in[f] == 'B' && in[f + 1] == 'C' && slen == 2 && f + 6 <= pos + 12 + xlen) {
                        bsize = le16(f + 4);
                        found = true;
                    }
                    f += 4 + slen;
                }
                if (!found) why = "gzip member without the BC extra field of BGZF";
                else if ((int64_t)bsize + 1 < 12 + xlen + 8) why = "BSIZE smaller than the member's header and trailer";
                else if (pos + (int64_t)bsize + 1 > n) why = "truncated member";
            }
        }
        if (!why) {
            const int64_t end = pos + (int64_t)bsize + 1;
            InflMember m{};
            m.at = pos;
            m.data = pos + 12 + xlen;
            m.n_data = (int32_t)(end - 8 - m.data);
            m.crc = le32(end - 8);
            const uint32_t isize = le32(end - 4);
            if (isize > INFL_MAX_ISIZE) {
                why = "ISIZE beyond the 64 KiB of a BGZF member";
            } else {
                m.isize = (int32_t)isize;
                m.out = out;
                out += isize;
                members.push_back(m);
                pos = end;
                continue;
            }
        }
        infl_message(msg, msg_len, idx, pos, why);
        return false;
    }
    *total = out;
    return true;
}

// The message of the first member whose status[] is not INFL_OK; false if there is none.
inline bool infl_first_failure(const std::vector<InflMember> &members, const int32_t *status, char *msg, size_t msg_len) {
    for (size_t m = 0; m < members.size(); m++) {
        if (status[m] == INFL_OK) continue;
        infl_message(msg, msg_len, (int64_t)m, members[m].at, infl_status_text(status[m]));
        return true;
    }
    return false;
}
