// bb_em_tables.h — the k-mer index of an error model as an open-addressing hash table (k-mer code -> table row), for
// models whose dense index kmer_to_row[4^k] would be too large (k > 12; up to k = 16, whose codes fill 32 bits).  One
// builder serves bb_upload_error_model_kmers and the emulator tests; bb_k_build_fragments<.., true> probes it once per
// fragment position.
//
//   entry   (code << 32) | row, one 64-bit word; BB_EM_HASH_EMPTY (row bits -1) marks a free slot
//   slot    Fibonacci hashing of the code, linear probing; the table holds at least twice as many slots as rows
#pragma once
#include <cstdint>

#define BB_EM_HASH_EMPTY 0xffffffffffffffffull
#define BB_EM_MAX_K 16   // a k-mer's 2-bit code fits 32 bits

struct BBEmHashDev {
    const unsigned long long *entries;  // nullptr: the model has no hash index (dense kmer_to_row, or the random model)
    uint32_t bits;                      // 2^bits slots
};

__host__ __device__ __forceinline__ uint32_t bb_em_slot(uint32_t code, uint32_t bits) {
    return (uint32_t)(((unsigned long long)code * 0x9E3779B97F4A7C15ull) >> (64 - bits));
}

// Row of the k-mer with 2-bit code `code`, -1 if the model has no line for it.
__host__ __device__ __forceinline__ int bb_em_find(const unsigned long long *entries, uint32_t bits, uint32_t code) {
    const uint32_t mask = (1u << bits) - 1u;
    for (uint32_t h = bb_em_slot(code, bits);; h = (h + 1u) & mask) {
        const unsigned long long e = entries[h];
        if (e == BB_EM_HASH_EMPTY) return -1;
        if ((uint32_t)(e >> 32) == code) return (int)(uint32_t)e;
    }
}

#include <string>
#include <vector>

struct BBEmHashTable {
    uint32_t bits = 6;
    std::vector<unsigned long long> entries;
};

// Row r has the k-mer whose code is kmer_codes[r] (base j of the k-mer in bits 2*(k-1-j), A=0 C=1 G=2 T=3).  Returns
// false with a message for k outside 3..16, a code outside 0..4^k-1 or a code that two rows share.
static inline bool bb_build_em_hash(int k, int32_t n_rows, const int64_t *kmer_codes, BBEmHashTable &t, std::string &err) {
    if (k < 3 || k > BB_EM_MAX_K) {
        err = "error model: k = " + std::to_string(k) + " is not supported (k must be 3.." + std::to_string(BB_EM_MAX_K) + ")";
        return false;
    }
    t.bits = 6;
    while ((1ull << t.bits) < 2ull * (uint64_t)(n_rows > 0 ? n_rows : 0)) t.bits++;
    t.entries.assign((size_t)1 << t.bits, BB_EM_HASH_EMPTY);
    const uint32_t mask = (1u << t.bits) - 1u;
    const int64_t n_codes = 1ll << (2 * k);
    for (int32_t r = 0; r < n_rows; r++) {
        const int64_t c = kmer_codes[r];
        if (c < 0 || c >= n_codes) {
            err = "error model: k-mer code " + std::to_string(c) + " of row " + std::to_string(r) + " is not a " +
                  std::to_string(k) + "-mer";
            return false;
        }
        const uint32_t code = (uint32_t)c;
        uint32_t h = bb_em_slot(code, t.bits);
        for (; t.entries[h] != BB_EM_HASH_EMPTY; h = (h + 1u) & mask)
            if ((uint32_t)(t.entries[h] >> 32) == code) {
                err = "error model: rows " + std::to_string((uint32_t)t.entries[h]) + " and " + std::to_string(r) +
                      " have the same k-mer (code " + std::to_string(c) + ")";
                return false;
            }
        t.entries[h] = ((unsigned long long)code << 32) | (uint32_t)r;
    }
    return true;
}
