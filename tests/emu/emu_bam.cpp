// emu_bam.cpp — the BAM record kernel (badread_b200/csrc/bb_bam_out.cuh) and the compressor's BAM mode
// (bgzf_k_compress_bam in bb_bgzf.cuh) under the warp emulator, behind the argument rules of bb_bam_build and
// bb_bam_compress (TEST INFRASTRUCTURE).
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_bam_out.cuh"
#include "../../badread_b200/csrc/bb_bgzf.cuh"

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API int64_t emu_bam_record_size(int32_t name_len, int32_t l_seq, int32_t co_len) {
    return bam_record_size(name_len, l_seq, co_len);
}

// bam_k_records over n records, one emulated CTA each: record i to out[pos[i] ..], bases and qualities from the n_src
// buffers seq[k] / qual[k] holding bytes [src_base[k], src_base[k + 1]) of the batch output.
EMU_API int emu_bam_records(int n, const BamRec *recs, const int64_t *pos, const uint8_t *text, int n_src,
                            const uint8_t *const *seq, const uint8_t *const *qual, const int64_t *src_base, uint8_t *out,
                            int64_t stream_base, int64_t *fields) {
    if (n < 0 || n_src < 1 || n_src > BAM_MAX_SRC) return -2;
    BamSrc src{};
    src.n = n_src;
    for (int k = 0; k < n_src; k++) { src.seq[k] = seq[k]; src.qual[k] = qual[k]; src.base[k] = src_base[k]; }
    src.base[n_src] = src_base[n_src];
    gridDim.x = (unsigned)n;
    for (int i = 0; i < n; i++) {
        blockIdx.x = (unsigned)i;
        emu::run_block(BAM_THREADS, [&]() { bam_k_records(recs, pos, text, src, out, stream_base, fields); });
    }
    return 0;
}

// bb_bam_compress without the context (one pass of any length): the fields that start inside the consumed bytes go to
// the kernel, as bb_bam_compress hands them over.  Returns 0, -2 for bad arguments or -4 if out_cap is too small.
EMU_API int emu_bam_compress(const uint8_t *in, int64_t n, int64_t stream_base, const int64_t *fields, int64_t n_fields,
                             int final, uint8_t *out, int64_t out_cap, int64_t *n_out, int64_t *n_consumed) {
    if (n < 0 || stream_base < 0 || n_fields < 0) return -2;
    const int64_t use = final ? n : n / BGZF_CHUNK * BGZF_CHUNK;
    const int nc = (int)((use + BGZF_CHUNK - 1) / BGZF_CHUNK);
    *n_out = 0;
    *n_consumed = 0;
    if (use + (int64_t)nc * 31 > out_cap) return -4;
    int64_t f0 = 0, f1 = n_fields;
    while (f0 < n_fields && fields[2 * f0] < stream_base) f0++;
    while (f1 > f0 && fields[2 * (f1 - 1)] >= stream_base + use) f1--;
    std::vector<uint4> buf((size_t)use / 16 + 1);   // 16-byte aligned, as cudaMalloc's buffers are
    std::memcpy(buf.data(), in, (size_t)use);
    const uint8_t *d_in = reinterpret_cast<const uint8_t *>(buf.data());
    std::vector<int32_t> sizes(nc);
    std::vector<int64_t> off(nc + 1);
    std::vector<uint32_t> slots((size_t)nc * BGZF_SLOT / 4);
    gridDim.x = (unsigned)nc;
    for (int c = 0; c < nc; c++) {
        blockIdx.x = (unsigned)c;
        emu::run_block(BGZF_THREADS, [&]() {
            bgzf_k_compress_bam(d_in, use, fields + 2 * f0, f1 - f0, stream_base, reinterpret_cast<uint8_t *>(slots.data()),
                                sizes.data());
        });
    }
    blockIdx.x = 0;
    emu::run_block(BGZF_THREADS, [&]() { bgzf_k_scan(sizes.data(), nc, 0, off.data()); });
    for (int c = 0; c < nc; c++) {
        blockIdx.x = (unsigned)c;
        emu::run_block(BGZF_THREADS, [&]() { bgzf_k_pack(reinterpret_cast<uint8_t *>(slots.data()), sizes.data(), off.data(), out); });
    }
    *n_out = off[nc];
    *n_consumed = use;
    return 0;
}
