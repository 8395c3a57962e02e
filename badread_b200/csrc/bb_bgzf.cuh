// bb_bgzf.cuh — BGZF compression of FASTQ text (SAM specification §4.1): a series of independent gzip members, each
// holding at most BGZF_CHUNK bytes of input, with the block size in a "BC" extra field.  A CTA compresses one chunk.
//
// FASTQ as Badread writes it leaves little for LZ77 to find (reads from a genome, random UUIDs in the headers,
// independent quality draws), so there is no string matching here: every chunk is entropy coded with dynamic Huffman
// tables, one deflate block per segment of the chunk.  A segment starts at every sequence or quality line that holds at
// least BGZF_MIN_SEG bytes of the chunk; header and '+' lines, short lines and a chunk's first partial line stay in the
// block before them.  Sequence and quality lines so get their own tables (4-5 symbols against 40-90), and no block
// header (about 60 bytes) pays for fewer than BGZF_MIN_SEG bytes.  A chunk that does not code smaller than its stored
// form becomes one stored block, so a member never exceeds 65 536 bytes.
//
// Chunks sit at fixed offsets of the whole stream (the caller carries the tail between calls), so the compressed
// bytes do not depend on where the caller's buffers end.  Everything a CTA computes is a function of its chunk and
// the index mod 4 of the FASTQ line its first byte belongs to: the output is deterministic.
//
// BAM records (bgzf_k_compress_bam) are segmented the same way without a newline scan: a block starts at every seq or
// qual field (bb_bam_out.cuh) that starts after the chunk's first byte and has at least BGZF_MIN_SEG bytes in the chunk;
// the fixed fields, name and CO tag of a record stay in the block of the qual field before them.
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>

#include "bb_crc32.cuh"

#define BGZF_CHUNK 65280           // input bytes per member (htslib's BGZF_BLOCK_SIZE)
#define BGZF_SLOT 65536            // bytes of a member's slot in the scratch, and the largest member BGZF allows
#define BGZF_THREADS 256
#define BGZF_MIN_SEG 1024          // shortest line that starts its own deflate block (see DESIGN.md §4)
#define BGZF_MAX_BLOCKS (BGZF_CHUNK / BGZF_MIN_SEG + 2)
#define BGZF_HEADER 18             // gzip header with the BC extra field
#define BGZF_TRAILER 8             // CRC32, ISIZE
#define BGZF_NLIT 257              // literals and end-of-block (no lengths: there are no matches)
#define BGZF_NCL 19                // code-length alphabet
#define BGZF_RLE_CAP (BGZF_NLIT + 2)

struct BGZFSmem {
    uint8_t in[BGZF_CHUNK];
    uint32_t out[BGZF_SLOT / 4];               // the member: header, deflate data, trailer
    uint32_t crc_table[256];
    uint32_t freq[BGZF_NLIT];                  // histogram of the current block (and then of its code-length symbols)
    uint8_t lens[BGZF_NLIT];                   // code lengths of the literal / end-of-block code
    uint16_t codes[BGZF_NLIT];                 // its codes, bit-reversed for LSB-first packing
    uint8_t cl_lens[BGZF_NCL];
    uint16_t cl_codes[BGZF_NCL];
    uint8_t rle_sym[BGZF_RLE_CAP], rle_extra[BGZF_RLE_CAP];  // the code lengths run-length coded
    // Huffman construction: leaves in ascending (frequency, symbol) order, internal nodes in creation order
    uint16_t leaf_sym[BGZF_NLIT];
    uint32_t leaf_w[BGZF_NLIT], node_w[BGZF_NLIT];
    uint16_t leaf_parent[BGZF_NLIT], node_parent[BGZF_NLIT];
    uint8_t node_depth[BGZF_NLIT];
    uint8_t all_lens[BGZF_NLIT + 2];
    int bl_count[16], next_code[16];
    int blk_start[BGZF_MAX_BLOCKS + 1];
    uint32_t wsum[BGZF_THREADS / 32];
    uint32_t crc_part[BGZF_THREADS / 32];
    int n_blocks, n_rle, hbits, hclen, too_big;
};
#define BGZF_SMEM_BYTES ((int)sizeof(BGZFSmem))

// order in which a dynamic block header lists the code lengths of the code-length code
__constant__ uint8_t bgzf_c_cl_order[BGZF_NCL] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Exclusive prefix sum over the CTA; *total = the sum of all threads' values.  Every thread must call it.
__device__ __forceinline__ uint32_t bgzf_scan(BGZFSmem &s, uint32_t v, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) s.wsum[warp] = x;
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (int w = 0; w < BGZF_THREADS / 32; w++) {
        if (w < warp) before += s.wsum[w];
        all += s.wsum[w];
    }
    __syncthreads();
    *total = all;
    return before + x - v;
}

// ORs the n_bits low bits of v (n_bits <= 25) into the bit stream at bit position pos (LSB first, as deflate packs).
__device__ __forceinline__ void bgzf_put(uint32_t *out, uint32_t pos, uint32_t v, int n_bits) {
    if (!n_bits) return;
    const uint32_t w = pos >> 5, sh = pos & 31;
    atomicOr((int *)&out[w], (int)(v << sh));
    if (sh + (uint32_t)n_bits > 32) atomicOr((int *)&out[w + 1], (int)(v >> (32 - sh)));
}

// Huffman code lengths of at most max_len bits for the n symbols of freq[] (at least two of them non-zero): the
// lengths of a Huffman tree, lengths beyond max_len cut and the overflow of the Kraft sum paid back by lengthening the
// longest shorter codes, then handed out again by rank, leaves ranked by (frequency, symbol) and the longest lengths
// to the lowest ranks: a less frequent symbol never gets a shorter code, and of two equally frequent symbols the lower
// one never gets the shorter code.  Every thread calls it; one thread builds the tree.
__device__ void bgzf_code_lengths(BGZFSmem &s, const uint32_t *freq, int n, int max_len, uint8_t *lens) {
    for (int i = threadIdx.x; i < n; i += BGZF_THREADS) {
        const uint32_t f = freq[i];
        if (!f) continue;
        int r = 0;
        for (int j = 0; j < n; j++) {
            const uint32_t g = freq[j];
            r += (g != 0u) & ((g < f) | ((g == f) & (j < i)));
        }
        s.leaf_sym[r] = (uint16_t)i;
        s.leaf_w[r] = f;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int m = 0;
        for (int i = 0; i < n; i++) {
            lens[i] = 0;
            m += freq[i] != 0u;
        }
        // two queues: the leaves in order, the internal nodes in the order they are made (their weights never fall)
        int li = 0, ni = 0;
        for (int k = 0; k < m - 1; k++) {
            uint32_t w = 0;
            for (int pick = 0; pick < 2; pick++) {
                if (li < m && (ni >= k || s.leaf_w[li] <= s.node_w[ni])) {
                    w += s.leaf_w[li];
                    s.leaf_parent[li++] = (uint16_t)k;
                } else {
                    w += s.node_w[ni];
                    s.node_parent[ni++] = (uint16_t)k;
                }
            }
            s.node_w[k] = w;
        }
        int *count = s.bl_count;
        for (int l = 0; l < 16; l++) count[l] = 0;
        s.node_depth[m > 1 ? m - 2 : 0] = 0;   // the root (m >= 2: the callers make sure of it)
        for (int k = m - 3; k >= 0; k--) {
            const int d = s.node_depth[s.node_parent[k]] + 1;
            s.node_depth[k] = (uint8_t)(d < 255 ? d : 255);
        }
        for (int r = 0; r < m; r++) {
            const int d = s.node_depth[s.leaf_parent[r]] + 1;
            count[d < max_len ? d : max_len]++;
        }
        uint32_t kraft = 0;
        for (int l = 1; l <= max_len; l++) kraft += (uint32_t)count[l] << (max_len - l);
        while (kraft > (1u << max_len)) {
            count[max_len]--;
            for (int l = max_len - 1; l > 0; l--)
                if (count[l]) {
                    count[l]--;
                    count[l + 1] += 2;
                    break;
                }
            kraft--;
        }
        int r = 0;
        for (int l = max_len; l > 0; l--)
            for (int c = 0; c < count[l]; c++) lens[s.leaf_sym[r++]] = (uint8_t)l;
    }
    __syncthreads();
}

// Canonical codes (RFC 1951 §3.2.2) of lens[0..n), bit-reversed.  One thread.
__device__ void bgzf_canonical(BGZFSmem &s, const uint8_t *lens, int n, uint16_t *codes) {
    int *count = s.bl_count, *next = s.next_code;
    for (int l = 0; l < 16; l++) count[l] = 0;
    for (int i = 0; i < n; i++) count[lens[i]]++;
    count[0] = 0;
    int code = 0;
    for (int l = 1; l < 16; l++) {
        code = (code + count[l - 1]) << 1;
        next[l] = code;
    }
    for (int i = 0; i < n; i++) {
        const int l = lens[i];
        codes[i] = l ? (uint16_t)(__brev((unsigned)next[l]++) >> (32 - l)) : (uint16_t)0;
    }
}

// The header of a dynamic block whose literal code is s.lens: the code lengths of its 257 literal / end-of-block codes
// and of two distance codes of one bit each (there are no matches, but every inflater is given two distance codes, as
// zlib sends them), run-length coded with symbols 16, 17 and 18, and the code-length code itself (at most 7 bits).
// Sets s.hbits.  Every thread calls it.
__device__ void bgzf_block_header(BGZFSmem &s) {
    if (threadIdx.x == 0) {
        uint8_t *all = s.all_lens;
        for (int i = 0; i < BGZF_NLIT; i++) all[i] = s.lens[i];
        all[BGZF_NLIT] = all[BGZF_NLIT + 1] = 1;
        const int total = BGZF_NLIT + 2;
        int n = 0;
        for (int i = 0; i < BGZF_NCL; i++) s.freq[i] = 0;
        for (int i = 0; i < total;) {
            const int v = all[i];
            int run = 1;
            while (i + run < total && all[i + run] == v) run++;
            i += run;
            if (v == 0) {
                while (run >= 11) {
                    const int r = run < 138 ? run : 138;
                    s.rle_sym[n] = 18; s.rle_extra[n++] = (uint8_t)(r - 11);
                    run -= r;
                }
                if (run >= 3) {
                    s.rle_sym[n] = 17; s.rle_extra[n++] = (uint8_t)(run - 3);
                    run = 0;
                }
            } else {
                s.rle_sym[n] = (uint8_t)v; s.rle_extra[n++] = 0;
                run--;
                while (run >= 3) {
                    const int r = run < 6 ? run : 6;
                    s.rle_sym[n] = 16; s.rle_extra[n++] = (uint8_t)(r - 3);
                    run -= r;
                }
            }
            for (; run > 0; run--) { s.rle_sym[n] = (uint8_t)v; s.rle_extra[n++] = 0; }
        }
        s.n_rle = n;
        for (int k = 0; k < n; k++) s.freq[s.rle_sym[k]]++;
        int used = 0;   // zlib's rule: at least two codes of non-zero frequency
        for (int i = 0; i < BGZF_NCL; i++) used += s.freq[i] != 0u;
        for (int i = 0; i < BGZF_NCL && used < 2; i++)
            if (!s.freq[i]) { s.freq[i] = 1; used++; }
    }
    __syncthreads();
    bgzf_code_lengths(s, s.freq, BGZF_NCL, 7, s.cl_lens);
    if (threadIdx.x == 0) {
        bgzf_canonical(s, s.cl_lens, BGZF_NCL, s.cl_codes);
        int hclen = BGZF_NCL;
        while (hclen > 4 && !s.cl_lens[bgzf_c_cl_order[hclen - 1]]) hclen--;
        int bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (int k = 0; k < s.n_rle; k++) {
            const int sym = s.rle_sym[k];
            bits += s.cl_lens[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
        }
        s.hbits = bits;
        s.hclen = hclen;
    }
    __syncthreads();
}

// Writes the block header sized by bgzf_block_header at bit position pos.  One thread.
__device__ void bgzf_write_header(BGZFSmem &s, uint32_t pos, int final, int hclen) {
    bgzf_put(s.out, pos, (uint32_t)(final | (2 << 1)), 3); pos += 3;       // BFINAL, BTYPE = 10 (dynamic)
    bgzf_put(s.out, pos, BGZF_NLIT - 257, 5); pos += 5;                    // HLIT
    bgzf_put(s.out, pos, 2 - 1, 5); pos += 5;                              // HDIST
    bgzf_put(s.out, pos, (uint32_t)(hclen - 4), 4); pos += 4;              // HCLEN
    for (int k = 0; k < hclen; k++) { bgzf_put(s.out, pos, s.cl_lens[bgzf_c_cl_order[k]], 3); pos += 3; }
    for (int k = 0; k < s.n_rle; k++) {
        const int sym = s.rle_sym[k];
        bgzf_put(s.out, pos, s.cl_codes[sym], s.cl_lens[sym]); pos += s.cl_lens[sym];
        const int xb = sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0;
        bgzf_put(s.out, pos, s.rle_extra[k], xb); pos += xb;
    }
}

// Chunk c of in[0..n) into its member; the body of both compressor kernels.  kBam selects where the deflate blocks start:
// FASTQ lines found by a newline scan (line_pref), or the seq and qual fields of BAM records (fields, stream_base).
template <bool kBam>
__device__ __forceinline__ void bgzf_compress_chunk(const uint8_t *__restrict__ in, int64_t n, const int64_t *__restrict__ line_pref,
                                                    const int64_t *__restrict__ fields, int64_t n_fields, int64_t stream_base,
                                                    uint8_t *__restrict__ slots, int32_t *__restrict__ sizes) {
#ifdef BB_EMULATOR
    static BGZFSmem s_mem;
    BGZFSmem &s = s_mem;
#else
    extern __shared__ __align__(16) uint8_t bgzf_smem[];
    BGZFSmem &s = *reinterpret_cast<BGZFSmem *>(bgzf_smem);
#endif
    const int t = threadIdx.x;
    const int64_t c = blockIdx.x;
    const int64_t base = c * BGZF_CHUNK;
    const int len = (int)(n - base < BGZF_CHUNK ? n - base : BGZF_CHUNK);
    int mod4 = 0;
    if constexpr (!kBam) mod4 = (int)(line_pref[c] & 3);
    const uint8_t *src = in + base;
    {   // chunk and CRC table into shared memory, member buffer cleared
        const int n16 = len >> 4;
        for (int i = t; i < n16; i += BGZF_THREADS) reinterpret_cast<uint4 *>(s.in)[i] = reinterpret_cast<const uint4 *>(src)[i];
        for (int i = (n16 << 4) + t; i < len; i += BGZF_THREADS) s.in[i] = src[i];
        for (int i = t; i < BGZF_SLOT / 4; i += BGZF_THREADS) s.out[i] = 0;
        s.crc_table[t] = bgzf_crc_entry((uint32_t)t);
    }
    __syncthreads();

    // each thread's slice of the chunk: newlines before it, and the CRC register of the slice alone
    const int per = (len + BGZF_THREADS - 1) / BGZF_THREADS;
    const int a0 = t * per < len ? t * per : len, a1 = a0 + per < len ? a0 + per : len;
    uint32_t nl = 0, crc = 0;
    for (int i = a0; i < a1; i++) {
        const uint8_t b = s.in[i];
        if constexpr (!kBam) nl += b == '\n';
        crc = s.crc_table[(crc ^ b) & 0xffu] ^ (crc >> 8);
    }
    uint32_t nl_before = 0;
    if constexpr (!kBam) {
        uint32_t nl_all;
        nl_before = bgzf_scan(s, nl, &nl_all);
    }
    // CRC-32 of the chunk = the slices' registers moved past the bytes after them, and the initial register past all
    uint32_t term = a1 > a0 ? bgzf_mulmod(crc, bgzf_x8n((uint32_t)(len - a1))) : 0u;
    for (int d = 16; d > 0; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
    if ((t & 31) == 0) s.crc_part[t >> 5] = term;

    if constexpr (kBam) {
        // block starts: seq and qual fields that start after the chunk's first byte with BGZF_MIN_SEG bytes in the chunk
        // (fields: (stream offset, length) pairs in stream order; in[0] is byte stream_base of the record stream)
        const int64_t cs = stream_base + base, last = cs + len - BGZF_MIN_SEG;
        int64_t lo = 0, hi = n_fields;
        while (lo < hi) {   // first field that starts after cs
            const int64_t mid = (lo + hi) >> 1;
            if (fields[2 * mid] > cs) hi = mid; else lo = mid + 1;
        }
        const int64_t f0 = lo;
        hi = n_fields;
        while (lo < hi) {   // first field that starts after last
            const int64_t mid = (lo + hi) >> 1;
            if (fields[2 * mid] > last) hi = mid; else lo = mid + 1;
        }
        const int64_t nf = lo - f0, fper = (nf + BGZF_THREADS - 1) / BGZF_THREADS;
        const int64_t g0 = f0 + min((int64_t)t * fper, nf), g1 = f0 + min((int64_t)t * fper + fper, nf);
        uint32_t n_starts = 0;
        for (int pass = 0; pass < 2; pass++) {
            uint32_t at = 0;
            if (pass) {
                uint32_t all;
                at = 1 + bgzf_scan(s, n_starts, &all);
                if (t == 0) { s.blk_start[0] = 0; s.n_blocks = 1 + (int)all; s.blk_start[1 + all] = len; }
            }
            for (int64_t g = g0; g < g1; g++)
                if (fields[2 * g + 1] >= BGZF_MIN_SEG) {
                    if (pass) s.blk_start[at++] = (int)(fields[2 * g] - cs);
                    else n_starts++;
                }
        }
    } else {
        // block starts: sequence (line index 1 mod 4) and quality (3 mod 4) lines with BGZF_MIN_SEG bytes in the chunk
        uint32_t n_starts = 0;
        for (int pass = 0; pass < 2; pass++) {
            uint32_t at = 0;
            if (pass) {
                uint32_t all;
                at = 1 + bgzf_scan(s, n_starts, &all);
                if (t == 0) { s.blk_start[0] = 0; s.n_blocks = 1 + (int)all; s.blk_start[1 + all] = len; }
            }
            uint32_t line = (uint32_t)mod4 + nl_before;
            for (int i = a0; i < a1; i++) {
                if (i > a0 && s.in[i - 1] == '\n') line++;
                if (i > 0 && s.in[i - 1] == '\n') {
                    if ((line & 1u) && i + BGZF_MIN_SEG <= len) {
                        int j = i;
                        while (j < i + BGZF_MIN_SEG - 1 && s.in[j] != '\n') j++;
                        if (j == i + BGZF_MIN_SEG - 1) {
                            if (pass) s.blk_start[at++] = i;
                            else n_starts++;
                        }
                    }
                }
            }
        }
    }
    __syncthreads();

    // dynamic blocks, until the data no longer codes smaller than it is stored
    const uint32_t limit = (uint32_t)(BGZF_HEADER + 4 + len) * 8;   // deflate data of fewer bytes than a stored block
    uint32_t pos = BGZF_HEADER * 8;
    if (t == 0) s.too_big = 0;
    for (int b = 0; b < s.n_blocks; b++) {
        const int b0 = s.blk_start[b], b1 = s.blk_start[b + 1];
        for (int i = t; i < BGZF_NLIT; i += BGZF_THREADS) s.freq[i] = 0;
        __syncthreads();
        for (int i = b0 + t; i < b1; i += BGZF_THREADS) atomicAdd(&s.freq[s.in[i]], 1u);
        if (t == 0) s.freq[256] = 1;
        __syncthreads();
        bgzf_code_lengths(s, s.freq, BGZF_NLIT, 15, s.lens);
        if (t == 0) bgzf_canonical(s, s.lens, BGZF_NLIT, s.codes);
        bgzf_block_header(s);
        const int hclen = s.hclen, hbits = s.hbits;
        const int bper = (b1 - b0 + BGZF_THREADS - 1) / BGZF_THREADS;
        const int d0 = b0 + t * bper < b1 ? b0 + t * bper : b1, d1 = d0 + bper < b1 ? d0 + bper : b1;
        uint32_t bits = 0;
        for (int i = d0; i < d1; i++) bits += s.lens[s.in[i]];
        uint32_t data_bits;
        const uint32_t off = bgzf_scan(s, bits, &data_bits);
        const uint32_t end = pos + (uint32_t)hbits + data_bits + s.lens[256];
        if (end > limit) {
            if (t == 0) s.too_big = 1;
            break;
        }
        if (t == 0) {
            bgzf_write_header(s, pos, b == s.n_blocks - 1, hclen);
            bgzf_put(s.out, end - s.lens[256], s.codes[256], s.lens[256]);
        }
        uint32_t w = (pos + (uint32_t)hbits + off) >> 5;
        uint64_t acc = 0;
        int n_acc = (int)((pos + (uint32_t)hbits + off) & 31);
        for (int i = d0; i < d1; i++) {
            const int sym = s.in[i];
            acc |= (uint64_t)s.codes[sym] << n_acc;
            n_acc += s.lens[sym];
            if (n_acc >= 32) {
                atomicOr((int *)&s.out[w++], (int)(uint32_t)acc);
                acc >>= 32;
                n_acc -= 32;
            }
        }
        if (n_acc > 0) atomicOr((int *)&s.out[w], (int)(uint32_t)acc);
        pos = end;
        __syncthreads();
    }
    __syncthreads();
    uint32_t dlen;
    uint8_t *ob = reinterpret_cast<uint8_t *>(s.out);
    if (s.too_big) {   // one stored block (BFINAL = 1, BTYPE = 00)
        for (int i = BGZF_HEADER / 4 + t; i < BGZF_SLOT / 4; i += BGZF_THREADS) s.out[i] = 0;
        __syncthreads();
        for (int i = t; i < len; i += BGZF_THREADS) ob[BGZF_HEADER + 5 + i] = s.in[i];
        dlen = 5 + (uint32_t)len;
    } else {
        dlen = (pos - BGZF_HEADER * 8 + 7) >> 3;
    }
    const uint32_t size = BGZF_HEADER + dlen + BGZF_TRAILER;
    if (t == 0) {
        uint32_t crc_all = bgzf_mulmod(0xffffffffu, bgzf_x8n((uint32_t)len));
        for (int w = 0; w < BGZF_THREADS / 32; w++) crc_all ^= s.crc_part[w];
        crc_all = ~crc_all;
        // ID1 ID2 CM=8 FLG=FEXTRA MTIME=0 XFL=0 OS=255 XLEN=6, subfield 'B' 'C' SLEN=2 BSIZE = member size - 1
        s.out[0] = 0x04088b1fu;
        s.out[1] = 0u;
        s.out[2] = 0x0006ff00u;
        s.out[3] = 0x00024342u;
        ob[16] = (uint8_t)((size - 1) & 0xff);
        ob[17] = (uint8_t)((size - 1) >> 8);
        if (s.too_big) {
            ob[BGZF_HEADER] = 1;
            ob[BGZF_HEADER + 1] = (uint8_t)(len & 0xff); ob[BGZF_HEADER + 2] = (uint8_t)(len >> 8);
            ob[BGZF_HEADER + 3] = (uint8_t)(~len & 0xff); ob[BGZF_HEADER + 4] = (uint8_t)((~len >> 8) & 0xff);
        }
        for (int k = 0; k < 4; k++) {
            ob[BGZF_HEADER + dlen + k] = (uint8_t)(crc_all >> (8 * k));
            ob[BGZF_HEADER + dlen + 4 + k] = (uint8_t)((uint32_t)len >> (8 * k));
        }
        sizes[c] = (int32_t)size;
    }
    __syncthreads();
    uint32_t *dst = reinterpret_cast<uint32_t *>(slots + c * BGZF_SLOT);
    for (uint32_t i = t; i < (size + 3) / 4; i += BGZF_THREADS) dst[i] = s.out[i];
}

// One CTA per chunk: chunk c is in[c * BGZF_CHUNK .. min(n, (c + 1) * BGZF_CHUNK)), its first byte on a line whose
// index mod 4 is line_pref[c] & 3.  Writes the member to slots[c * BGZF_SLOT ..] (whole words) and its size to sizes[c].
// Dynamic shared memory: BGZF_SMEM_BYTES.
__global__ void __launch_bounds__(BGZF_THREADS, 1)
bgzf_k_compress(const uint8_t *__restrict__ in, int64_t n, const int64_t *__restrict__ line_pref, uint8_t *__restrict__ slots,
                int32_t *__restrict__ sizes) {
    bgzf_compress_chunk<false>(in, n, line_pref, nullptr, 0, 0, slots, sizes);
}

// The same for a stream of BAM records whose byte in[0] is byte stream_base of the stream: deflate blocks start at the
// seq and qual fields listed in fields[2 * n_fields] as (stream offset, length) pairs in stream order (bb_bam_out.cuh).
__global__ void __launch_bounds__(BGZF_THREADS, 1)
bgzf_k_compress_bam(const uint8_t *__restrict__ in, int64_t n, const int64_t *__restrict__ fields, int64_t n_fields,
                    int64_t stream_base, uint8_t *__restrict__ slots, int32_t *__restrict__ sizes) {
    bgzf_compress_chunk<true>(in, n, nullptr, fields, n_fields, stream_base, slots, sizes);
}

// Newlines of every chunk (one CTA each) -> counts[c].
__global__ void __launch_bounds__(BGZF_THREADS) bgzf_k_lines(const uint8_t *__restrict__ in, int64_t n, int32_t *__restrict__ counts) {
    __shared__ uint32_t s_count;
    const int64_t base = (int64_t)blockIdx.x * BGZF_CHUNK;
    const int len = (int)(n - base < BGZF_CHUNK ? n - base : BGZF_CHUNK);
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    uint32_t k = 0;
    for (int i = threadIdx.x; i < len; i += BGZF_THREADS) k += in[base + i] == '\n';
    atomicAdd(&s_count, k);
    __syncthreads();
    if (threadIdx.x == 0) counts[blockIdx.x] = (int32_t)s_count;
}

// out[i] = init + v[0] + ... + v[i-1] for i = 0 .. n (one CTA).
__global__ void __launch_bounds__(BGZF_THREADS) bgzf_k_scan(const int32_t *__restrict__ v, int n, int64_t init,
                                                           int64_t *__restrict__ out) {
    __shared__ int64_t s_warp[BGZF_THREADS / 32];
    __shared__ int64_t s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = init;
    for (int tile = 0; tile <= n; tile += BGZF_THREADS) {
        const int i = tile + (int)threadIdx.x;
        const int64_t x0 = i < n ? v[i] : 0;
        int64_t x = x0;
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        int64_t before = s_carry, all = 0;
        for (int w = 0; w < BGZF_THREADS / 32; w++) {
            if (w < warp) before += s_warp[w];
            all += s_warp[w];
        }
        if (i <= n) out[i] = before + x - x0;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += all;
    }
}

// Member c from its slot to out[offsets[c] ..] (one CTA per member).
__global__ void __launch_bounds__(BGZF_THREADS) bgzf_k_pack(const uint8_t *__restrict__ slots, const int32_t *__restrict__ sizes,
                                                           const int64_t *__restrict__ offsets, uint8_t *__restrict__ out) {
    const uint8_t *src = slots + (int64_t)blockIdx.x * BGZF_SLOT;
    uint8_t *dst = out + offsets[blockIdx.x];
    const int size = sizes[blockIdx.x];
    for (int i = threadIdx.x; i < size; i += BGZF_THREADS) dst[i] = src[i];
}
