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
#include <cstdio>

#include "../../include/badread_b200.h"

#include "bb_models.cuh"

namespace {

struct DevMem {   // everything a call allocates, released on every exit path
    void *p[32];
    int n = 0;
    ~DevMem() { for (int i = 0; i < n; i++) cudaFree(p[i]); }
    template <typename X>
    cudaError_t get(X **out, size_t bytes, const void *src = nullptr, int fill = -1) {
        void *q = nullptr;
        cudaError_t e = cudaMalloc(&q, bytes ? bytes : 16);
        if (e != cudaSuccess) return e;
        p[n++] = q;
        *out = (X *)q;
        if (src) e = cudaMemcpy(q, src, bytes, cudaMemcpyHostToDevice);
        else if (fill >= 0) e = cudaMemset(q, fill, bytes ? bytes : 16);
        return e;
    }
    // an input array: used in place when it is device memory of `device`, else copied like get()
    template <typename X>
    cudaError_t input(X **out, size_t bytes, const X *src, int device) {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device == device) {
            *out = const_cast<X *>(src);
            return cudaSuccess;
        }
        (void)cudaGetLastError();
        return get(out, bytes, src);
    }
};

#define BBM_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    std::snprintf(g_model_error, sizeof(g_model_error), "%s: %s", #call, cudaGetErrorString(e_)); return BB_ERR_CUDA; } } while (0)

thread_local char g_model_error[256] = "";

int count_common(bool qscores, bool wide, int device, int k, int max_del, int32_t n_aln, const uint8_t *read, const uint8_t *qual,
                 const int64_t *read_off, const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                 const int32_t *op_ref0, const int64_t *ops_off, int64_t table_cap, uint64_t *keys_out, uint64_t *first_out,
                 uint32_t *counts_out, int64_t *n_entries, uint64_t *overall_out, int64_t ovf_cap, int32_t *ovf_aln,
                 int32_t *ovf_pos, int32_t *ovf_k, int64_t *n_ovf) {
    g_model_error[0] = 0;
    if (n_aln <= 0 || !read || !read_off || !ref || !ref_off || !ops || !ops_off || !op_read0 || !op_ref0 || !keys_out ||
        !first_out || !counts_out || !n_entries || !n_ovf || table_cap < 16 || (table_cap & (table_cap - 1)) ||
        (qscores && (!qual || !overall_out || k < 1 || k > 13 || !(k & 1) || max_del < 0)) ||
        (!qscores && !wide && (k < 1 || k > 12)) || (wide && (k <= 12 || k > 16))) {
        std::snprintf(g_model_error, sizeof(g_model_error), "bb_count_*: invalid argument");
        return BB_ERR_ARG;
    }
    BBM_TRY(cudaSetDevice(device));
    // cudaGetLastError() after the launch below must report this call's launch only: clear whatever an earlier call of
    // this thread left, e.g. an out-of-memory from an engine's scratch allocation when a second context on the same
    // GPU did not fit (the engine reported it already)
    (void)cudaGetLastError();
    const int64_t n_read = read_off[n_aln], n_ref = ref_off[n_aln], n_ops = ops_off[n_aln];
    const int per_slot = qscores ? BBM_NQ : 1;
    const size_t key_bytes = wide ? sizeof(BBMKey128) : 8;
    DevMem mem;
    BBMAln A{};
    uint8_t *d_read, *d_qual = nullptr, *d_ref;
    int64_t *d_read_off, *d_ref_off, *d_ops_off;
    uint32_t *d_ops;
    int32_t *d_p0, *d_r0;
    BBM_TRY(mem.input(&d_read, (size_t)n_read, read, device));
    if (qscores) BBM_TRY(mem.input(&d_qual, (size_t)n_read, qual, device));
    BBM_TRY(mem.input(&d_ref, (size_t)n_ref, ref, device));
    BBM_TRY(mem.get(&d_read_off, (size_t)(n_aln + 1) * 8, read_off));
    BBM_TRY(mem.get(&d_ref_off, (size_t)(n_aln + 1) * 8, ref_off));
    BBM_TRY(mem.get(&d_ops_off, (size_t)(n_aln + 1) * 8, ops_off));
    BBM_TRY(mem.input(&d_ops, (size_t)n_ops * 4, ops, device));
    BBM_TRY(mem.input(&d_p0, (size_t)n_ops * 4, op_read0, device));
    BBM_TRY(mem.input(&d_r0, (size_t)n_ops * 4, op_ref0, device));
    A.read = d_read; A.qual = d_qual; A.ref = d_ref; A.read_off = d_read_off; A.ref_off = d_ref_off; A.ops_off = d_ops_off;
    A.ops = d_ops; A.op_read0 = d_p0; A.op_ref0 = d_r0;
    BBMTable T{};
    T.cap = table_cap; T.ovf_cap = ovf_cap;
    if (wide) BBM_TRY(mem.get(&T.keys, 16, nullptr, 0xff));   // (unused: the 128-bit keys are TW's)
    else BBM_TRY(mem.get(&T.keys, (size_t)table_cap * 8, nullptr, 0xff));
    BBM_TRY(mem.get(&T.first, (size_t)table_cap * 8, nullptr, 0xff));
    BBM_TRY(mem.get(&T.counts, (size_t)table_cap * per_slot * 4, nullptr, 0));
    BBM_TRY(mem.get(&T.status, 16, nullptr, 0));
    BBM_TRY(mem.get(&T.n_ovf, 16, nullptr, 0));
    BBM_TRY(mem.get(&T.ovf_aln, (size_t)ovf_cap * 4));
    BBM_TRY(mem.get(&T.ovf_pos, (size_t)ovf_cap * 4));
    BBM_TRY(mem.get(&T.ovf_k, (size_t)ovf_cap * 4));
    BBMTableWide TW{};
    if (wide) {
        TW.first = T.first; TW.counts = T.counts; TW.cap = T.cap; TW.status = T.status;
        TW.ovf_aln = T.ovf_aln; TW.ovf_pos = T.ovf_pos; TW.ovf_k = T.ovf_k; TW.n_ovf = T.n_ovf; TW.ovf_cap = T.ovf_cap;
        BBM_TRY(mem.get(&TW.keys, (size_t)table_cap * sizeof(BBMKey128), nullptr, 0xff));
    }
    unsigned long long *d_overall = nullptr;
    if (qscores) {
        uint8_t *sym; int *dc, *lead;
        BBM_TRY(mem.get(&sym, (size_t)n_read));
        BBM_TRY(mem.get(&dc, (size_t)n_read * 4));
        BBM_TRY(mem.get(&lead, (size_t)n_aln * 4));
        BBM_TRY(mem.get(&d_overall, BBM_NQ * 8, nullptr, 0));
        bbm_k_cigar_qscores<<<n_aln, 256>>>(A, n_aln, k, max_del, sym, dc, lead, T, d_overall);
    } else {
        int *rp; uint8_t *ism;
        BBM_TRY(mem.get(&rp, (size_t)n_ref * 4));
        BBM_TRY(mem.get(&ism, (size_t)n_ref));
        if (wide) bbm_k_kmer_alternatives<<<n_aln, 256>>>(A, n_aln, k, rp, ism, TW);
        else bbm_k_kmer_alternatives<<<n_aln, 256>>>(A, n_aln, k, rp, ism, T);
    }
    BBM_TRY(cudaGetLastError());
    unsigned long long *d_keys_out, *d_first_out, *d_n;
    unsigned int *d_counts_out;
    BBM_TRY(mem.get(&d_keys_out, (size_t)table_cap * key_bytes));
    BBM_TRY(mem.get(&d_first_out, (size_t)table_cap * 8));
    BBM_TRY(mem.get(&d_counts_out, (size_t)table_cap * per_slot * 4));
    BBM_TRY(mem.get(&d_n, 16, nullptr, 0));
    const unsigned int n_blocks = (unsigned int)((table_cap + 255) / 256);
    if (wide) bbm_k_compact<<<n_blocks, 256>>>(TW, per_slot, (BBMKey128 *)d_keys_out, d_first_out, d_counts_out, d_n, table_cap);
    else bbm_k_compact<<<n_blocks, 256>>>(T, per_slot, d_keys_out, d_first_out, d_counts_out, d_n, table_cap);
    BBM_TRY(cudaGetLastError());
    int status[2] = {0, 0};
    unsigned long long n = 0, novf = 0;
    BBM_TRY(cudaMemcpy(status, T.status, sizeof(status), cudaMemcpyDeviceToHost));   // (synchronizes with the kernels)
    BBM_TRY(cudaMemcpy(&n, d_n, 8, cudaMemcpyDeviceToHost));
    BBM_TRY(cudaMemcpy(&novf, T.n_ovf, 8, cudaMemcpyDeviceToHost));
    *n_entries = (int64_t)n; *n_ovf = (int64_t)novf;
    if (status[0] || status[1]) {
        std::snprintf(g_model_error, sizeof(g_model_error), "bb_count_*: %s too small", status[0] ? "table" : "overflow list");
        return BB_ERR_CAPACITY;
    }
    BBM_TRY(cudaMemcpy(keys_out, d_keys_out, (size_t)n * key_bytes, cudaMemcpyDeviceToHost));
    BBM_TRY(cudaMemcpy(first_out, d_first_out, (size_t)n * 8, cudaMemcpyDeviceToHost));
    BBM_TRY(cudaMemcpy(counts_out, d_counts_out, (size_t)n * per_slot * 4, cudaMemcpyDeviceToHost));
    if (novf) {
        BBM_TRY(cudaMemcpy(ovf_aln, T.ovf_aln, (size_t)novf * 4, cudaMemcpyDeviceToHost));
        BBM_TRY(cudaMemcpy(ovf_pos, T.ovf_pos, (size_t)novf * 4, cudaMemcpyDeviceToHost));
        BBM_TRY(cudaMemcpy(ovf_k, T.ovf_k, (size_t)novf * 4, cudaMemcpyDeviceToHost));
    }
    if (qscores) BBM_TRY(cudaMemcpy(overall_out, d_overall, BBM_NQ * 8, cudaMemcpyDeviceToHost));
    return BB_OK;
}

}  // namespace

// the message of bb_model_error() for the calling thread, set by the other model-builder inputs (BGZF, SAM / BAM)
void bbm_set_error(const char *msg) { std::snprintf(g_model_error, sizeof(g_model_error), "%s", msg); }

extern "C" const char *bb_model_error(void) { return g_model_error; }

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
