// bb_models.cuh — device code of the model builders' counting passes (SURVEY.md 8f row f4); host side and C ABI:
// bb_tu_models.cu.  Compiled for the host by the warp emulator as well (tests/emu).
//   bbm_k_kmer_alternatives   badread error_model   (error_model.py:45-66: which read k-mers each reference k-mer became)
//   bbm_k_cigar_qscores       badread qscore_model  (qscore_model.py:104-141: quality of the middle base per CIGAR window)
// An alignment is a CTA, a window is a thread and a window's content is a 64-bit key (128 bits for error-model k-mers
// longer than 12: BBMTableWide) in an open-addressing table: count,
// first occurrence (the reference's dicts keep insertion order, and its stable sorts break ties by it) and, for the qscore
// model, a histogram of the 94 quality values.  Windows whose content does not fit a key go to an overflow list that the
// host evaluates exactly.
#pragma once
#include <cstdint>

#define BBM_EMPTY 0xffffffffffffffffull
#define BBM_WIDE_MAX_LEN 32   // read k-mer bases in the low word of a 128-bit key
#define BBM_NQ 94   // quality characters '!' .. '~'

struct BBMAln {
    const uint8_t *read, *qual, *ref;
    const int64_t *read_off, *ref_off, *ops_off;
    const uint32_t *ops;       // (len << 2) | type, type 0 = M, 1 = I, 2 = D
    const int32_t *op_read0;   // read offset (within the alignment) at which the run starts
    const int32_t *op_ref0;    // reference offset at which the run starts
};

struct BBMTable {
    unsigned long long *keys, *first;
    unsigned int *counts;      // error model: one per slot; qscore model: BBM_NQ per slot
    long long cap;             // power of two
    int *status;               // [0]: table full, [1]: overflow list full
    int *ovf_aln, *ovf_pos, *ovf_k;
    unsigned long long *n_ovf;
    long long ovf_cap;
    static constexpr bool wide = false;
};

// Error-model key for 12 < k <= 16 (sm_90's 16-byte atomicCAS claims a slot): lo = read k-mer (2 bits a base from bit 0
// up), hi = (reference k-mer << 6) | read k-mer length.  Empty: both words all ones (hi never is: the reference k-mer has
// at most 32 bits).
struct __align__(16) BBMKey128 { unsigned long long lo, hi; };

struct BBMTableWide {   // BBMTable with 128-bit keys
    BBMKey128 *keys;
    unsigned long long *first;
    unsigned int *counts;
    long long cap;
    int *status;
    int *ovf_aln, *ovf_pos, *ovf_k;
    unsigned long long *n_ovf;
    long long ovf_cap;
    static constexpr bool wide = true;
};

__device__ __forceinline__ bool bbm_is_empty(unsigned long long key) { return key == BBM_EMPTY; }
__device__ __forceinline__ bool bbm_is_empty(const BBMKey128 &key) { return key.lo == BBM_EMPTY && key.hi == BBM_EMPTY; }

__device__ __forceinline__ unsigned long long bbm_mix64(unsigned long long x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// Slot of `key` (claimed if new), or -1 if the table is (as good as) full: a probe sequence of 1024 slots does not
// happen below a load of ~0.95, and once one thread has given up the others stop at their next key instead of walking the
// whole table each - the caller doubles the table and counts again.
__device__ long long bbm_table_slot(const BBMTable &T, unsigned long long key) {
    if (*(volatile int *)&T.status[0]) return -1;
    unsigned long long h = bbm_mix64(key) & (unsigned long long)(T.cap - 1);
    const long long limit = T.cap < 1024 ? T.cap : 1024;
    for (long long probe = 0; probe < limit; probe++) {
        const unsigned long long prev = atomicCAS(&T.keys[h], BBM_EMPTY, key);
        if (prev == BBM_EMPTY || prev == key) return (long long)h;
        h = (h + 1) & (unsigned long long)(T.cap - 1);
    }
    atomicExch(&T.status[0], 1);
    return -1;
}

// The same for a 128-bit key (Table = BBMTableWide).  A template, so that code which never counts wide keys (the warp
// emulator's other harnesses) needs no 16-byte atomicCAS.
template <typename Table>
__device__ long long bbm_table_slot(const Table &T, BBMKey128 key) {
    if (*(volatile int *)&T.status[0]) return -1;
    unsigned long long h = bbm_mix64(key.hi ^ bbm_mix64(key.lo)) & (unsigned long long)(T.cap - 1);
    const long long limit = T.cap < 1024 ? T.cap : 1024;
    const BBMKey128 empty{BBM_EMPTY, BBM_EMPTY};
    for (long long probe = 0; probe < limit; probe++) {
        const BBMKey128 prev = atomicCAS(&T.keys[h], empty, key);
        if (bbm_is_empty(prev) || (prev.lo == key.lo && prev.hi == key.hi)) return (long long)h;
        h = (h + 1) & (unsigned long long)(T.cap - 1);
    }
    atomicExch(&T.status[0], 1);
    return -1;
}

template <typename Table>
__device__ void bbm_overflow(const Table &T, int aln, int pos, int k) {
    const unsigned long long i = atomicAdd(T.n_ovf, 1ull);
    if ((long long)i < T.ovf_cap) { T.ovf_aln[i] = aln; T.ovf_pos[i] = pos; T.ovf_k[i] = k; }
    else atomicExch(&T.status[1], 1);
}

__device__ __forceinline__ int bbm_base_code(uint8_t c) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1; }

// ---------------------------------------------------------------------------------------------- error model
// error_model.py:45-66.  The window of reference base r (r = 0 .. n_ref - k) spans the alignment columns from r's column
// to the column of reference base r + k - 1; its read k-mer is read[rp[r] : rp[r+k-1] + isM[r+k-1]) with rp[x] = read
// bases in front of x's column (the first window starts at column 0, i.e. at read base 0, whatever the alignment starts
// with).  Counted if the read k-mer has more than one base, both k-mers are ACGT only and they agree in their first and
// last base.  Key: reference k-mer (2k bits) | length (6 bits) | read k-mer (2 bits a base); with a BBMTableWide
// (12 < k <= 16) the BBMKey128 of the same three fields.
template <typename Table>
__global__ void __launch_bounds__(256) bbm_k_kmer_alternatives(BBMAln A, int n_aln, int k, int *rp_pool, uint8_t *ism_pool, Table T) {
    const int a = blockIdx.x;
    if (a >= n_aln) return;
    const uint8_t *read = A.read + A.read_off[a], *ref = A.ref + A.ref_off[a];
    const int n_ref = (int)(A.ref_off[a + 1] - A.ref_off[a]);
    int *rp = rp_pool + A.ref_off[a];
    uint8_t *ism = ism_pool + A.ref_off[a];
    for (long long o = A.ops_off[a] + threadIdx.x; o < A.ops_off[a + 1]; o += blockDim.x) {
        const uint32_t op = A.ops[o];
        const int len = (int)(op >> 2), type = (int)(op & 3u), p0 = A.op_read0[o], r0 = A.op_ref0[o];
        if (type == 0) for (int i = 0; i < len; i++) { rp[r0 + i] = p0 + i; ism[r0 + i] = 1; }
        else if (type == 2) for (int i = 0; i < len; i++) { rp[r0 + i] = p0; ism[r0 + i] = 0; }
    }
    __syncthreads();
    const int shift_ref = 64 - 2 * k, shift_len = shift_ref - 6, max_len = Table::wide ? BBM_WIDE_MAX_LEN : shift_len / 2;
    for (int r = threadIdx.x; r + k <= n_ref; r += blockDim.x) {
        const int p_lo = r == 0 ? 0 : rp[r], p_hi = rp[r + k - 1] + ism[r + k - 1];
        const int len = p_hi - p_lo;
        if (len <= 1) continue;
        if (read[p_lo] != ref[r] || read[p_hi - 1] != ref[r + k - 1]) continue;
        unsigned long long key = 0;
        bool ok = true;
        for (int j = 0; j < k; j++) {
            const int c = bbm_base_code(ref[r + j]);
            ok = ok && c >= 0;
            key = (key << 2) | (unsigned long long)(c & 3);
        }
        if (!ok) continue;
        if (!Table::wide) key <<= shift_ref;
        if (len > max_len) {  // (the host checks the read k-mer's alphabet itself)
            bbm_overflow(T, a, r, k);
            continue;
        }
        unsigned long long rb = 0;
        for (int j = 0; j < len; j++) {
            const int c = bbm_base_code(read[p_lo + j]);
            ok = ok && c >= 0;
            rb |= (unsigned long long)(c & 3) << (2 * j);
        }
        if (!ok) continue;
        long long s;
        if constexpr (Table::wide) s = bbm_table_slot(T, BBMKey128{rb, (key << 6) | (unsigned long long)len});
        else {
            key |= ((unsigned long long)len << shift_len) | rb;
            s = bbm_table_slot(T, key);
        }
        if (s < 0) return;
        atomicAdd(&T.counts[s], 1u);
        atomicMin(&T.first[s], ((unsigned long long)a << 32) | (unsigned long long)r);
    }
}

// ---------------------------------------------------------------------------------------------- qscore model
// qscore_model.py:104-141.  Per read base i: sym[i] ('=' 0, 'X' 1, 'I' 2) and dcount[i] = 'D' columns between base i and
// base i + 1.  The window of (k, i) - k = 1, 3, ..., K read bases from base i on - has the CIGAR
// sym[i] D^min(dcount[i], max_del) sym[i+1] ... sym[i+k-1] (the first window of an alignment also takes the 'D' columns in
// front of base 0) and the quality of its middle base.  Key: length (6 bits) | 2 bits a symbol ('D' = 3).
__global__ void __launch_bounds__(256) bbm_k_cigar_qscores(BBMAln A, int n_aln, int K, int max_del, uint8_t *sym_pool, int *dc_pool,
                                                       int *lead_pool, BBMTable T, unsigned long long *overall) {
    const int a = blockIdx.x;
    if (a >= n_aln) return;
    const uint8_t *read = A.read + A.read_off[a], *qual = A.qual + A.read_off[a], *ref = A.ref + A.ref_off[a];
    const int n_read = (int)(A.read_off[a + 1] - A.read_off[a]);
    uint8_t *sym = sym_pool + A.read_off[a];
    int *dc = dc_pool + A.read_off[a];
    for (int i = threadIdx.x; i < n_read; i += blockDim.x) dc[i] = 0;
    if (threadIdx.x == 0) lead_pool[a] = 0;
    __syncthreads();
    for (long long o = A.ops_off[a] + threadIdx.x; o < A.ops_off[a + 1]; o += blockDim.x) {
        const uint32_t op = A.ops[o];
        const int len = (int)(op >> 2), type = (int)(op & 3u), p0 = A.op_read0[o], r0 = A.op_ref0[o];
        if (type == 0) for (int i = 0; i < len; i++) sym[p0 + i] = read[p0 + i] == ref[r0 + i] ? 0 : 1;
        else if (type == 1) for (int i = 0; i < len; i++) sym[p0 + i] = 2;
        else if (p0 > 0) atomicAdd(&dc[p0 - 1], len);   // (two 'D' runs in a row are one run of 'D' columns)
        else atomicAdd(&lead_pool[a], len);
    }
    __syncthreads();
    const int lead = lead_pool[a];
    for (int kk = 1, kidx = 0; kk <= K; kk += 2, kidx++) {
        for (int i = threadIdx.x; i + kk <= n_read; i += blockDim.x) {
            unsigned long long key = 0;
            int len = 0;
            bool fits = true;
            auto push = [&](unsigned long long s, int count) {
                for (int x = 0; x < count; x++) {
                    if (len >= 29) { fits = false; return; }
                    key |= s << (2 * len);
                    len++;
                }
            };
            if (i == 0) push(3ull, lead < max_del ? lead : max_del);
            for (int j = 0; j < kk && fits; j++) {
                push((unsigned long long)sym[i + j], 1);
                if (j + 1 < kk) push(3ull, dc[i + j] < max_del ? dc[i + j] : max_del);
            }
            const int q = (int)qual[i + (kk - 1) / 2] - 33;
            if (q < 0 || q >= BBM_NQ) { bbm_overflow(T, a, i, -kk); continue; }   // not a quality character: the host decides
            if (kk == 1) atomicAdd(&overall[q], 1ull);
            if (!fits) { bbm_overflow(T, a, i, kk); continue; }
            key |= (unsigned long long)len << 58;
            const long long s = bbm_table_slot(T, key);
            if (s < 0) return;
            atomicAdd(&T.counts[s * BBM_NQ + q], 1u);
            atomicMin(&T.first[s], ((unsigned long long)a << 36) | ((unsigned long long)kidx << 32) | (unsigned long long)i);
        }
    }
}

// Occupied slots -> dense output (arbitrary order; the host sorts by first occurrence).
template <typename Table, typename Key>
__global__ void bbm_k_compact(Table T, int per_slot, Key *keys_out, unsigned long long *first_out,
                          unsigned int *counts_out, unsigned long long *n_out, long long out_cap) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= T.cap || bbm_is_empty(T.keys[s])) return;
    const unsigned long long i = atomicAdd(n_out, 1ull);
    if ((long long)i >= out_cap) return;
    keys_out[i] = T.keys[s];
    first_out[i] = T.first[s];
    for (int x = 0; x < per_slot; x++) counts_out[i * per_slot + x] = T.counts[s * per_slot + x];
}

