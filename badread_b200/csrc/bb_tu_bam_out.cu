// bb_tu_bam_out.cu — compiles the BAM record kernel (bb_bam_out.cuh) and enqueues it.
#include "../../include/badread_b200.h"
#include "bb_bam_out.cuh"
#include "bb_launch.h"

static_assert(sizeof(BamRec) == sizeof(bb_bam_record) && offsetof(BamRec, out_off) == offsetof(bb_bam_record, out_off) &&
              offsetof(BamRec, text_off) == offsetof(bb_bam_record, text_off) &&
              offsetof(BamRec, out_len) == offsetof(bb_bam_record, out_len) &&
              offsetof(BamRec, name_len) == offsetof(bb_bam_record, name_len) &&
              offsetof(BamRec, co_len) == offsetof(bb_bam_record, co_len),
              "BamRec must have the layout of bb_bam_record");

int64_t bbl_bam_record_size(int32_t name_len, int32_t l_seq, int32_t co_len) { return bam_record_size(name_len, l_seq, co_len); }

void bbl_bam_records(cudaStream_t st, int n_records, const bb_bam_record *recs, const int64_t *pos, const uint8_t *text,
                     int n_src, const uint8_t *const *seq, const uint8_t *const *qual, const int64_t *src_base, uint8_t *out,
                     int64_t stream_base, int64_t *fields) {
    if (n_records <= 0) return;
    BamSrc src{};
    src.n = n_src;
    for (int k = 0; k < n_src && k < BAM_MAX_SRC; k++) {
        src.seq[k] = seq[k];
        src.qual[k] = qual[k];
        src.base[k] = src_base[k];
    }
    src.base[n_src] = src_base[n_src];
    bam_k_records<<<n_records, BAM_THREADS, 0, st>>>(reinterpret_cast<const BamRec *>(recs), pos, text, src, out, stream_base,
                                                      fields);
}
