// bb_tu_models.cu — the counting passes of the model builders on the GPU (SURVEY.md 8f row f4):
//   bb_count_kmer_alternatives   badread error_model   (error_model.py:31-83: which read k-mers each reference k-mer became)
//   bb_count_kmer_alternatives_wide   the same for 12 < k <= 16, with 128-bit keys
//   bb_count_cigar_qscores       badread qscore_model  (qscore_model.py:78-153: quality of the middle base per CIGAR window)
// The reference walks every alignment column by column in Python, rebuilding a window string per step; here an
// alignment is a CTA, a window is a thread and a (window content) is a 64-bit key in an open-addressing table:
// count, first occurrence (the reference's dicts keep insertion order, and its stable sorts break ties by it) and,
// for the qscore model, a histogram of the 94 quality values.  Windows whose content does not fit a key (read k-mers /
// CIGARs longer than the key holds: a handful per million) go to an overflow list that the host evaluates exactly.
// Input per alignment a (host code: badread_b200/model_builders.py): the aligned slice of the read (and its
// qualities), the aligned slice of the reference already on the read's strand, and the CIGAR runs in read orientation
// with the read / reference offset each run starts at.
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "../../include/badread_b200.h"

#include "bb_call.h"
#include "bb_models.cuh"

namespace {

int count_common(bool qscores, bool wide, int device, int k, int max_del, int32_t n_aln, const uint8_t *read, const uint8_t *qual,
                 const int64_t *read_off, const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                 const int32_t *op_ref0, const int64_t *ops_off, int64_t table_cap, uint64_t *keys_out, uint64_t *first_out,
                 uint32_t *counts_out, int64_t *n_entries, uint64_t *overall_out, int64_t ovf_cap, int32_t *ovf_aln,
                 int32_t *ovf_pos, int32_t *ovf_k, int64_t *n_ovf) {
    if (n_aln <= 0 || !read || !read_off || !ref || !ref_off || !ops || !ops_off || !op_read0 || !op_ref0 || !keys_out ||
        !first_out || !counts_out || !n_entries || !n_ovf || table_cap < 16 || (table_cap & (table_cap - 1)) ||
        (qscores && (!qual || !overall_out || k < 1 || k > 13 || !(k & 1) || max_del < 0)) ||
        (!qscores && !wide && (k < 1 || k > 12)) || (wide && (k <= 12 || k > 16)))
        return bad_argument("bb_count_*");
    return device_call(device, [&] {
        const int64_t n_read = read_off[n_aln], n_ref = ref_off[n_aln], n_ops = ops_off[n_aln];
        const int per_slot = qscores ? BBM_NQ : 1;
        const size_t key_bytes = wide ? sizeof(BBMKey128) : 8;
        const char *what = "bb_count_*";
        Scratch S;   // (an allocation that fails is BB_ERR_CUDA: to the caller BB_ERR_CAPACITY means a larger table)
        auto filled = [&](auto *&p, int64_t count, int v) {
            p = S.get<std::remove_reference_t<decltype(*p)>>(count, what);
            check(cudaMemset(p, v, (size_t)count * sizeof(*p)), "cudaMemset");
        };
        BBMAln A{};
        A.read = S.input(read, n_read, device, what);
        if (qscores) A.qual = S.input(qual, n_read, device, what);
        A.ref = S.input(ref, n_ref, device, what);
        A.read_off = S.upload(read_off, n_aln + 1, what);
        A.ref_off = S.upload(ref_off, n_aln + 1, what);
        A.ops_off = S.upload(ops_off, n_aln + 1, what);
        A.ops = S.input(ops, n_ops, device, what);
        A.op_read0 = S.input(op_read0, n_ops, device, what);
        A.op_ref0 = S.input(op_ref0, n_ops, device, what);
        BBMTable T{};
        T.cap = table_cap; T.ovf_cap = ovf_cap;
        filled(T.keys, wide ? 2 : table_cap, 0xff);   // (wide: unused, the 128-bit keys are TW's)
        filled(T.first, table_cap, 0xff);
        filled(T.counts, table_cap * per_slot, 0);
        filled(T.status, 4, 0);
        filled(T.n_ovf, 2, 0);
        T.ovf_aln = S.get<int32_t>(ovf_cap, what);
        T.ovf_pos = S.get<int32_t>(ovf_cap, what);
        T.ovf_k = S.get<int32_t>(ovf_cap, what);
        BBMTableWide TW{};
        if (wide) {
            TW.first = T.first; TW.counts = T.counts; TW.cap = T.cap; TW.status = T.status;
            TW.ovf_aln = T.ovf_aln; TW.ovf_pos = T.ovf_pos; TW.ovf_k = T.ovf_k; TW.n_ovf = T.n_ovf; TW.ovf_cap = T.ovf_cap;
            filled(TW.keys, table_cap, 0xff);
        }
        unsigned long long *d_overall = nullptr;
        if (qscores) {
            uint8_t *sym = S.get<uint8_t>(n_read, what);
            int *dc = S.get<int>(n_read, what), *lead = S.get<int>(n_aln, what);
            filled(d_overall, BBM_NQ, 0);
            bbm_k_cigar_qscores<<<n_aln, 256>>>(A, n_aln, k, max_del, sym, dc, lead, T, d_overall);
        } else {
            int *rp = S.get<int>(n_ref, what);
            uint8_t *ism = S.get<uint8_t>(n_ref, what);
            if (wide) bbm_k_kmer_alternatives<<<n_aln, 256>>>(A, n_aln, k, rp, ism, TW);
            else bbm_k_kmer_alternatives<<<n_aln, 256>>>(A, n_aln, k, rp, ism, T);
        }
        check(cudaGetLastError(), qscores ? "bbm_k_cigar_qscores" : "bbm_k_kmer_alternatives");
        unsigned long long *d_keys_out = S.get<unsigned long long>(table_cap * (int64_t)key_bytes / 8, what);
        unsigned long long *d_first_out = S.get<unsigned long long>(table_cap, what), *d_n;
        unsigned int *d_counts_out = S.get<unsigned int>(table_cap * per_slot, what);
        filled(d_n, 2, 0);
        const unsigned int n_blocks = (unsigned int)((table_cap + 255) / 256);
        if (wide) bbm_k_compact<<<n_blocks, 256>>>(TW, per_slot, (BBMKey128 *)d_keys_out, d_first_out, d_counts_out, d_n, table_cap);
        else bbm_k_compact<<<n_blocks, 256>>>(T, per_slot, d_keys_out, d_first_out, d_counts_out, d_n, table_cap);
        check(cudaGetLastError(), "bbm_k_compact");
        int status[2] = {0, 0};
        unsigned long long n = 0, novf = 0;
        d2h(status, T.status, 2);   // (synchronizes with the kernels)
        d2h(&n, d_n, 1);
        d2h(&novf, T.n_ovf, 1);
        *n_entries = (int64_t)n; *n_ovf = (int64_t)novf;
        if (status[0] || status[1])
            throw Fail{BB_ERR_CAPACITY, std::string("bb_count_*: ") + (status[0] ? "table" : "overflow list") + " too small"};
        d2h(keys_out, d_keys_out, (int64_t)n * (int64_t)key_bytes / 8);
        d2h(first_out, d_first_out, (int64_t)n);
        d2h(counts_out, d_counts_out, (int64_t)n * per_slot);
        d2h(ovf_aln, T.ovf_aln, (int64_t)novf);
        d2h(ovf_pos, T.ovf_pos, (int64_t)novf);
        d2h(ovf_k, T.ovf_k, (int64_t)novf);
        if (qscores) d2h(overall_out, d_overall, BBM_NQ);
        return BB_OK;
    });
}

}  // namespace

extern "C" int bb_count_kmer_alternatives(int device, int k, int32_t n_aln, const uint8_t *read, const int64_t *read_off,
                                          const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops,
                                          const int32_t *op_read0, const int32_t *op_ref0, const int64_t *ops_off,
                                          int64_t table_cap, uint64_t *keys_out, uint64_t *first_out, uint32_t *counts_out,
                                          int64_t *n_entries, int64_t ovf_cap, int32_t *ovf_aln, int32_t *ovf_pos,
                                          int32_t *ovf_k, int64_t *n_ovf) {
    return count_common(false, false, device, k, 0, n_aln, read, nullptr, read_off, ref, ref_off, ops, op_read0, op_ref0, ops_off,
                        table_cap, keys_out, first_out, counts_out, n_entries, nullptr, ovf_cap, ovf_aln, ovf_pos, ovf_k, n_ovf);
}

extern "C" int bb_count_kmer_alternatives_wide(int device, int k, int32_t n_aln, const uint8_t *read, const int64_t *read_off,
                                               const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops,
                                               const int32_t *op_read0, const int32_t *op_ref0, const int64_t *ops_off,
                                               int64_t table_cap, uint64_t *keys_out, uint64_t *first_out, uint32_t *counts_out,
                                               int64_t *n_entries, int64_t ovf_cap, int32_t *ovf_aln, int32_t *ovf_pos,
                                               int32_t *ovf_k, int64_t *n_ovf) {
    return count_common(false, true, device, k, 0, n_aln, read, nullptr, read_off, ref, ref_off, ops, op_read0, op_ref0, ops_off,
                        table_cap, keys_out, first_out, counts_out, n_entries, nullptr, ovf_cap, ovf_aln, ovf_pos, ovf_k, n_ovf);
}

extern "C" int bb_count_cigar_qscores(int device, int k, int max_del, int32_t n_aln, const uint8_t *read, const uint8_t *qual,
                                      const int64_t *read_off, const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops,
                                      const int32_t *op_read0, const int32_t *op_ref0, const int64_t *ops_off,
                                      int64_t table_cap, uint64_t *keys_out, uint64_t *first_out, uint32_t *counts_out,
                                      int64_t *n_entries, uint64_t *overall_out, int64_t ovf_cap, int32_t *ovf_aln,
                                      int32_t *ovf_pos, int32_t *ovf_k, int64_t *n_ovf) {
    return count_common(true, false, device, k, max_del, n_aln, read, qual, read_off, ref, ref_off, ops, op_read0, op_ref0, ops_off,
                        table_cap, keys_out, first_out, counts_out, n_entries, overall_out, ovf_cap, ovf_aln, ovf_pos, ovf_k,
                        n_ovf);
}
