// emu_qscores.cpp — K5 (bb_k_qscores_pair) under the warp emulator with the tables of the shared host builder
// (badread_b200/csrc/bb_qscore_tables.h), for qscore models whose CIGAR keys may be longer than 31 symbols
// (TEST INFRASTRUCTURE).  The per-base ops / deletion counts come from the alignment task pipeline of emu_align.cpp
// (emu_tasks_align), called by the Python front end (emu_qscores.py).
#include "cuda_emu.h"

#include <string>
#include <vector>

#include "../../badread_b200/csrc/bb_kernels.cuh"

// Builds the tables from key i = key_chars[key_off[i] .. key_off[i+1]) as bb_upload_qscore_model_cigars does, then runs
// bb_k_qscores_pair on ops[n] / dcnt[n].  qual_out: n quality characters.  Returns 2 if the builder rejects the keys
// (message in err_out, err_cap bytes).
extern "C" __attribute__((visibility("default")))
int emu_qscores_cigars(const uint8_t *ops, const unsigned int *dcnt, int n, int kmer_size, int32_t n_keys,
                       const uint8_t *key_chars, const int32_t *key_off, const int32_t *row_off, const uint8_t *scores,
                       const double *cum, unsigned long long seed, unsigned long long read_index, uint8_t *qual_out,
                       char *err_out, int err_cap) {
    BBQScoreTables t;
    std::string err;
    if (!bb_build_qscore_tables(n_keys, key_chars, key_off, t, err)) {
        if (err_cap > 0) { std::strncpy(err_out, err.c_str(), (size_t)err_cap - 1); err_out[err_cap - 1] = 0; }
        return 2;
    }
    BBQScoreModelDev qm;
    std::memset(&qm, 0, sizeof(qm));
    qm.kmer_size = kmer_size; qm.hkeys = t.hkeys.data(); qm.hvals = t.hvals.data(); qm.hbits = t.hbits; qm.row_off = row_off;
    qm.scores = scores; qm.cum = cum;
    qm.long_max_len = t.long_max_len; qm.lbits = t.lbits; qm.lkeys = t.lkeys.data(); qm.lpool = t.lpool.data();
    emu::run_block(256, [&]() { bb_k_qscores_pair(ops, dcnt, n, qm, seed, read_index, qual_out); });
    return 0;
}
