// bb_qscore_tables.h — the device lookup tables of a qscore model (QScoreModel.scores, qscore_model.py:178-271),
// built on the host from the model's CIGAR strings.  One builder serves bb_upload_qscore_model_cigars,
// bb_upload_qscore_model (after unpacking its keys) and the emulator tests, so the kernels (bb_qscore_base in
// bb_kernels.cuh) always read tables of one layout:
//
//   keys of <= 31 symbols  packed 2 bits per symbol ('='=0, 'X'=1, 'I'=2, 'D'=3) under a leading 1 bit, in an
//                          open-addressing table of uint64 (0 = empty) with the key's row beside it
//   longer keys            a side table of BBQLongKey {hash, length, row, offset} (length 0 = empty), probed by a hash
//                          of the symbols; the symbols themselves sit in a pool of uint64 words, 32 symbols per word
//                          (symbol j of a key in bits 2*(j%32) of its word j/32), for the exact comparison of a hit
#pragma once
#include <cstdint>

#define BB_QM_SHORT_MAX 31   // symbols a packed uint64 key can hold under its leading 1 bit
#define BB_QM_LONG_HASH_INIT 0xcbf29ce484222325ull

struct BBQLongKey {
    unsigned long long hash;  // bb_qm_long_hash of the symbols
    int32_t len;              // symbols; 0 = empty slot
    int32_t row;              // into row_off
    int64_t off;              // first pool word
};

// FNV-1a over the 2-bit symbol codes: the side table's hash, fed one symbol at a time as the kernel walks a window.
__host__ __device__ __forceinline__ unsigned long long bb_qm_long_hash(unsigned long long h, unsigned int sym) {
    return (h ^ (unsigned long long)(sym + 1u)) * 0x100000001b3ull;
}

// Slot of a hash in a table of 2^bits entries (Fibonacci hashing, the same mixing as the packed table).
__host__ __device__ __forceinline__ uint32_t bb_qm_slot(unsigned long long h, uint32_t bits) {
    return (uint32_t)((h * 0x9E3779B97F4A7C15ull) >> (64 - bits));
}

#include <algorithm>
#include <string>
#include <vector>

struct BBQScoreTables {
    uint32_t hbits = 6;
    std::vector<uint64_t> hkeys;   // packed keys, 0 = empty
    std::vector<int32_t> hvals;
    uint32_t lbits = 6;
    std::vector<BBQLongKey> lkeys;
    std::vector<uint64_t> lpool;
    int long_max_len = 0;          // longest key in the side table, 0 if it is empty
};

static inline int bb_qm_symbol(uint8_t c) {
    switch (c) { case '=': return 0; case 'X': return 1; case 'I': return 2; case 'D': return 3; default: return -1; }
}

// Key i = key_chars[key_off[i], key_off[i+1]) is the CIGAR of row i.  A repeated key keeps its last row, like the
// dict assignment in QScoreModel.load_from_file.  Returns false with a message for an empty key or a symbol outside =XID.
static inline bool bb_build_qscore_tables(int32_t n_keys, const uint8_t *key_chars, const int32_t *key_off,
                                          BBQScoreTables &t, std::string &err) {
    int32_t n_short = 0, n_long = 0;
    int64_t n_words = 0;
    for (int32_t i = 0; i < n_keys; i++) {
        const int32_t len = key_off[i + 1] - key_off[i];
        if (len <= 0) { err = "qscore model: empty CIGAR key (row " + std::to_string(i) + ")"; return false; }
        for (int32_t j = 0; j < len; j++)
            if (bb_qm_symbol(key_chars[key_off[i] + j]) < 0) {
                err = "qscore model: CIGAR key '" + std::string((const char *)key_chars + key_off[i], (size_t)len) +
                      "' holds a symbol other than =XID";
                return false;
            }
        if (len <= BB_QM_SHORT_MAX) n_short++;
        else { n_long++; n_words += (len + 31) / 32; }
    }
    t.hbits = 6;
    while ((1ull << t.hbits) < 2ull * (uint64_t)n_short) t.hbits++;
    t.hkeys.assign((size_t)1 << t.hbits, 0);
    t.hvals.assign((size_t)1 << t.hbits, -1);
    t.lbits = 6;
    while ((1ull << t.lbits) < 2ull * (uint64_t)n_long) t.lbits++;
    t.lkeys.assign((size_t)1 << t.lbits, BBQLongKey{0ull, 0, -1, 0});
    t.lpool.clear();
    t.lpool.reserve((size_t)n_words);
    t.long_max_len = 0;
    std::vector<int32_t> lkey_of((size_t)1 << t.lbits, -1);   // key index behind each side-table slot (repeats)
    for (int32_t i = 0; i < n_keys; i++) {
        const uint8_t *s = key_chars + key_off[i];
        const int32_t len = key_off[i + 1] - key_off[i];
        if (len <= BB_QM_SHORT_MAX) {
            uint64_t key = 1;
            for (int32_t j = 0; j < len; j++) key = (key << 2) | (uint64_t)bb_qm_symbol(s[j]);
            const uint32_t mask = (uint32_t)(t.hkeys.size() - 1);
            uint32_t h = bb_qm_slot(key, t.hbits);
            while (t.hkeys[h] != 0 && t.hkeys[h] != key) h = (h + 1) & mask;
            t.hkeys[h] = key; t.hvals[h] = i;
            continue;
        }
        unsigned long long hash = BB_QM_LONG_HASH_INIT;
        for (int32_t j = 0; j < len; j++) hash = bb_qm_long_hash(hash, (unsigned)bb_qm_symbol(s[j]));
        const uint32_t mask = (uint32_t)(t.lkeys.size() - 1);
        uint32_t h = bb_qm_slot(hash, t.lbits);
        for (;; h = (h + 1) & mask) {
            BBQLongKey &e = t.lkeys[h];
            if (e.len == 0) break;
            const int32_t o = lkey_of[h];
            if (e.hash == hash && e.len == len && std::equal(s, s + len, key_chars + key_off[o])) break;
        }
        BBQLongKey &e = t.lkeys[h];
        if (e.len == 0) {
            e.hash = hash; e.len = len; e.off = (int64_t)t.lpool.size();
            for (int32_t j = 0; j < len; j++) {
                if ((j & 31) == 0) t.lpool.push_back(0);
                t.lpool.back() |= (uint64_t)bb_qm_symbol(s[j]) << (2 * (j & 31));
            }
            if (len > t.long_max_len) t.long_max_len = len;
        }
        e.row = i; lkey_of[h] = i;
    }
    return true;
}

// The packed keys of bb_upload_qscore_model back to CIGAR strings.  Returns false for a value that is not a leading
// 1 bit over an even number of bits (in particular 0..3).
static inline bool bb_unpack_qscore_keys(int32_t n_keys, const uint64_t *keys, std::vector<uint8_t> &chars,
                                         std::vector<int32_t> &off) {
    static const uint8_t sym[4] = {'=', 'X', 'I', 'D'};
    chars.clear();
    off.assign(1, 0);
    for (int32_t i = 0; i < n_keys; i++) {
        const uint64_t k = keys[i];
        if (k < 4) return false;
        const int top = 63 - __builtin_clzll(k);   // position of the leading 1 bit
        if (top & 1) return false;
        for (int j = top / 2 - 1; j >= 0; j--) chars.push_back(sym[(k >> (2 * j)) & 3]);
        off.push_back((int32_t)chars.size());
    }
    return true;
}
