// bb_tu_bgzf.cu — compiles the BGZF compressor (bb_bgzf.cuh) and enqueues one pass of it.
#include "bb_bgzf.cuh"
#include "bb_launch.h"

static_assert(BGZF_CHUNK == BB_BGZF_CHUNK, "chunk size of the C ABI");

cudaError_t bbl_bgzf_init() {
    const cudaError_t e = cudaFuncSetAttribute(bgzf_k_compress, cudaFuncAttributeMaxDynamicSharedMemorySize, BGZF_SMEM_BYTES);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(bgzf_k_compress_bam, cudaFuncAttributeMaxDynamicSharedMemorySize, BGZF_SMEM_BYTES);
}

void bbl_bgzf_pass_bam(cudaStream_t st, const uint8_t *in, int64_t n, int n_chunks, const int64_t *fields, int64_t n_fields,
                       int64_t stream_base, uint8_t *slots, int32_t *sizes, int64_t *offsets, uint8_t *out) {
    bgzf_k_compress_bam<<<n_chunks, BGZF_THREADS, BGZF_SMEM_BYTES, st>>>(in, n, fields, n_fields, stream_base, slots, sizes);
    bgzf_k_scan<<<1, BGZF_THREADS, 0, st>>>(sizes, n_chunks, 0, offsets);
    bgzf_k_pack<<<n_chunks, BGZF_THREADS, 0, st>>>(slots, sizes, offsets, out);
}

void bbl_bgzf_pass(cudaStream_t st, const uint8_t *in, int64_t n, int n_chunks, int line_mod4, int32_t *lines,
                   int64_t *line_pref, uint8_t *slots, int32_t *sizes, int64_t *offsets, uint8_t *out) {
    bgzf_k_lines<<<n_chunks, BGZF_THREADS, 0, st>>>(in, n, lines);
    bgzf_k_scan<<<1, BGZF_THREADS, 0, st>>>(lines, n_chunks, line_mod4, line_pref);
    bgzf_k_compress<<<n_chunks, BGZF_THREADS, BGZF_SMEM_BYTES, st>>>(in, n, line_pref, slots, sizes);
    bgzf_k_scan<<<1, BGZF_THREADS, 0, st>>>(sizes, n_chunks, 0, offsets);
    bgzf_k_pack<<<n_chunks, BGZF_THREADS, 0, st>>>(slots, sizes, offsets, out);
}
