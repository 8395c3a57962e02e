// bb_launch.h — host-side launchers of the heavy kernels.  Every kernel is a template (bb_kernels.cuh), so it is
// compiled only by the translation unit that launches it: the heavy ones live in bb_tu_*.cu, one file each, and
// build in parallel (the wide wavefront instantiations take minutes of ptxas each); bb_api.cu launches the light
// ones itself.  All launchers are asynchronous on `st`; errors surface through cudaGetLastError() in the caller.
#pragma once
#include <cuda_runtime.h>

#include "bb_kernels.cuh"

void bbl_mutate(int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em, unsigned long long seed, int *work_counter,
                const int *order, int n_items, bool chain);  // chain: the low-latency build (bb_k_mutate_chain)
cudaError_t bbl_window_lane_init();
void bbl_window_lane4(int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em, const BBWinTask *tasks, const int *n_tasks,
                      unsigned long long seed, uint32_t *ckpt_pool, uint8_t *tbuf_pool, int *cursor, BBWinTask *fallback,
                      int *fallback_count);
void bbl_window_lane8(int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em, const BBWinTask *tasks, const int *n_tasks,
                      unsigned long long seed, uint32_t *ckpt_pool, uint8_t *tbuf_pool, int *cursor, BBWinTask *fallback,
                      int *fallback_count);
void bbl_window_lane_hist(int words, int ring_t, int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em, const BBWinTask *tasks,
                          const int *n_tasks, unsigned long long seed, uint2 *hist_pool, uint8_t *tbuf_pool, int *cursor,
                          BBWinTask *fallback, int *fallback_count);
void bbl_window_warp(int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em, BBScratchPool pool, const BBWinTask *tasks,
                     const int *n_tasks, unsigned long long seed, int *cursor);
void bbl_node_warp(int words, int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity, int *cursor,
                   int warp_base);  // words per lane: 1, 2 or 4 (class BBQ_NODE_LEAN1 / 2 / 4)
void bbl_node_lane8(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, int parity, int *cursor);
cudaError_t bbl_node_quad_init();
void bbl_node_quad(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity, int *cursor,
                   int warp_base);
cudaError_t bbl_node_pair_init();
void bbl_node_pair(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity, int *cursor,
                   int warp_base);
void bbl_leaf_warp(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, BBScratchPool pool, int *cursor, int warp_base);
void bbl_leaf_lane_hist(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, uint2 *hist_pool, int *cursor);
cudaError_t bbl_leaf_lane_init();
void bbl_leaf_lane(int grid, cudaStream_t st, BBBatchDev B, BBQueues Q, uint32_t *ckpt_pool, int *cursor);
void bbl_align_pair(cudaStream_t st, const uint8_t *q, int n, const uint8_t *t, int m, int k_upper, BBScratchPool pool,
                    uint8_t *ops, unsigned int *dcnt, int *out5);
// BGZF (bb_bgzf.cuh): the n_chunks chunks of in[0..n) -> members packed back to back into out, out[offsets[n_chunks]]
// bytes in all; line_mod4: index mod 4 of the FASTQ line in[0] belongs to; line_pref[n_chunks] = line_mod4 + newlines.
// Scratch: lines[n_chunks], line_pref and offsets[n_chunks + 1], slots[n_chunks * BGZF_SLOT], sizes[n_chunks].
cudaError_t bbl_bgzf_init();
void bbl_bgzf_pass(cudaStream_t st, const uint8_t *in, int64_t n, int n_chunks, int line_mod4, int32_t *lines,
                   int64_t *line_pref, uint8_t *slots, int32_t *sizes, int64_t *offsets, uint8_t *out);
// The same for BAM records: in[0] is byte stream_base of the record stream, fields[2 * n_fields] the (stream offset,
// length) pairs of the seq and qual fields in stream order (no newline scan).
void bbl_bgzf_pass_bam(cudaStream_t st, const uint8_t *in, int64_t n, int n_chunks, const int64_t *fields, int64_t n_fields,
                       int64_t stream_base, uint8_t *slots, int32_t *sizes, int64_t *offsets, uint8_t *out);
// BAM records (bb_bam_out.cuh): record i of recs[n_records] to out[pos[i] ..], its bases and qualities read from the n_src
// output buffers seq[k] / qual[k] holding bytes [src_base[k], src_base[k + 1]) of the batch output; fields[4 i ..] = stream
// offset and length of its seq and its qual field, out[0] being byte stream_base of the record stream.
struct bb_bam_record;
int64_t bbl_bam_record_size(int32_t name_len, int32_t l_seq, int32_t co_len);
void bbl_bam_records(cudaStream_t st, int n_records, const bb_bam_record *recs, const int64_t *pos, const uint8_t *text,
                     int n_src, const uint8_t *const *seq, const uint8_t *const *qual, const int64_t *src_base, uint8_t *out,
                     int64_t stream_base, int64_t *fields);
// FASTA (bb_fasta.cuh) of text[0..n) in device memory.  bbl_fasta_scan runs passes 1 and 2 in `scratch`
// (bbl_fasta_scratch_bytes(n) bytes); then bbl_fasta_totals(scratch, n)[0] = the bytes kept, [1] = the header lines.
// bbl_fasta_emit writes the kept bytes to kept[] and each header line's start, end and kept offset.
size_t bbl_fasta_scratch_bytes(int64_t n);
void bbl_fasta_scan(cudaStream_t st, const uint8_t *text, int64_t n, void *scratch);
const int64_t *bbl_fasta_totals(const void *scratch, int64_t n);
void bbl_fasta_emit(cudaStream_t st, const uint8_t *text, int64_t n, const void *scratch, uint8_t *kept, int64_t *hdr_start,
                    int64_t *hdr_end, int64_t *hdr_kept);
// bb_c_comp's table (misc._COMP_TABLE) into table[256], for every unit that complements on the device
void bbl_comp_table(uint8_t *table);
// dst[dst_off[r] .. dst_off[r + 1]) = src[src_lo[r] ..] for r < n_ranges; total = dst_off[n_ranges] (device arrays)
void bbl_fasta_gather(cudaStream_t st, const uint8_t *src, const int64_t *src_lo, const int64_t *dst_off, int32_t n_ranges,
                      int64_t total, uint8_t *dst);
// BGZF in host memory in[0..n) inflated on `st` into a new device allocation *out of *total bytes (cudaFree it): the
// input goes through a device buffer of its own, released before the call returns.  BB_ERR_ARG with msg naming the member
// (index and offset) for input that is not BGZF or a corrupt member, as bb_bgzf_decompress; BB_ERR_CUDA otherwise.
int bbl_bgzf_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, uint8_t **out, int64_t *total, char *msg,
                            size_t msg_len);
// Any gzip stream in host memory in[0..n) inflated the same way (bb_tu_gunzip.cu): through bbl_bgzf_inflate_device when
// every member is BGZF, else in chunks of chunk_bytes (0: the default); *stats as bb_gzip_decompress reports them.
struct bb_gzip_stats;
// An error model file's text[0..n) in device memory to its tables (bb_em_load.cuh), in new device allocations that
// bbl_em_load_free releases.  kmer_to_row[4^k] only when `dense` and k <= 12.  info->fallback set: nothing to install.
struct BBEmLoadOut {
    int32_t *kmer_to_row = nullptr;
    int64_t *codes = nullptr;
    int32_t *row_off = nullptr;
    double *cum = nullptr, *probs = nullptr;
    uint8_t *flags = nullptr;
    uint32_t *slots = nullptr;
    uint8_t *pool = nullptr;
    BBRowInfo *rowinfo = nullptr;
};
int bbl_em_load(cudaStream_t st, const uint8_t *text, int64_t n, bool dense, bb_em_load_info *info, BBEmLoadOut *out,
                char *msg, size_t msg_len);
void bbl_em_load_free(BBEmLoadOut *out);
int bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out,
                            int64_t *total, bb_gzip_stats *stats, char *msg, size_t msg_len);
