// bb_bam_out.cuh — unaligned BAM records (SAM specification v1.6 §4.2) of simulated reads, built on the device from the
// workers' output buffers.  A CTA writes one record at a stream position the host computed:
//   block_size, refID -1, pos -1, l_read_name, MAPQ 0, bin 4680 (reg2bin(-1, 0)), n_cigar_op 0, FLAG 4 (unmapped),
//   l_seq, next_refID -1, next_pos -1, tlen 0, read_name NUL, seq (4-bit =ACMGRSVTWYHKDBN codes, high nibble first),
//   qual (Phred: the FASTQ character - 33), and one tag CO:Z holding the rest of the FASTQ header line, NUL-terminated.
// The host uploads the read's name and CO text; the bases and qualities are read where the batch left them.  Every
// record also reports where its seq and qual fields sit in the record stream: the compressor starts its deflate blocks
// there (bgzf_k_compress_bam in bb_bgzf.cuh).
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>

#define BAM_THREADS 128
#define BAM_MAX_SRC 8              // output buffers a record may come from (the workers of a context, at most 8)
#define BAM_FIXED 36               // block_size and the 32 bytes of fixed fields
#define BAM_BIN_UNMAPPED 4680      // reg2bin(-1, 0)

// One record to build (the layout of bb_bam_record in include/badread_b200.h).
struct BamRec {
    int64_t out_off;    // the read's out_off in the batch results: offset into the concatenated output buffers
    int64_t text_off;   // its name, then its CO text, in the text pool
    int32_t out_len;    // l_seq
    int32_t name_len;   // bytes of the name (without the NUL)
    int32_t co_len;     // bytes of the CO text (without the NUL)
    int32_t reserved;
};

// The output buffers of a batch: buffer k holds the bytes [base[k], base[k + 1]) of the concatenated output.
struct BamSrc {
    const uint8_t *seq[BAM_MAX_SRC];
    const uint8_t *qual[BAM_MAX_SRC];
    int64_t base[BAM_MAX_SRC + 1];
    int n;
};

// Bytes of a record: fixed fields, name and NUL, packed bases, qualities, "CO" 'Z' text NUL.
__host__ __device__ __forceinline__ int64_t bam_record_size(int32_t name_len, int32_t l_seq, int32_t co_len) {
    return BAM_FIXED + (int64_t)name_len + 1 + ((int64_t)l_seq + 1) / 2 + l_seq + 3 + co_len + 1;
}

// htslib's seq_nt16_table: the 16 codes of "=ACMGRSVTWYHKDBN" for either case, everything else N (15).
__device__ __forceinline__ uint8_t bam_nt16(int c) {
    const char *alpha = "=ACMGRSVTWYHKDBN";
    if (c >= 'a' && c <= 'z') c -= 32;
    for (int k = 0; k < 16; k++)
        if (alpha[k] == c) return (uint8_t)k;
    return 15;
}

__device__ __forceinline__ void bam_put32(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}

// One CTA per record: record r goes to out[pos[r] ..]; out[0] is byte stream_base of the record stream.
// fields[4 r .. 4 r + 4) = stream offset and length of its seq field, then of its qual field.
__global__ void __launch_bounds__(BAM_THREADS)
bam_k_records(const BamRec *__restrict__ recs, const int64_t *__restrict__ pos, const uint8_t *__restrict__ text, BamSrc src,
              uint8_t *__restrict__ out, int64_t stream_base, int64_t *__restrict__ fields) {
    __shared__ uint8_t s_code[256];
    const int t = threadIdx.x;
    for (int c = t; c < 256; c += BAM_THREADS) s_code[c] = bam_nt16(c);
    const BamRec r = recs[blockIdx.x];
    int k = 0;
    while (k + 1 < src.n && r.out_off >= src.base[k + 1]) k++;
    const uint8_t *seq = src.seq[k] + (r.out_off - src.base[k]);
    const uint8_t *qual = src.qual[k] + (r.out_off - src.base[k]);
    const int64_t at = pos[blockIdx.x];
    uint8_t *p = out + at;
    const int l = r.out_len, nb = (l + 1) / 2;
    const int64_t o_name = BAM_FIXED, o_seq = o_name + r.name_len + 1, o_qual = o_seq + nb, o_tag = o_qual + l;
    __syncthreads();
    if (t == 0) {
        const int64_t size = bam_record_size(r.name_len, l, r.co_len);
        bam_put32(p, (uint32_t)(size - 4));                       // block_size
        bam_put32(p + 4, 0xffffffffu);                            // refID
        bam_put32(p + 8, 0xffffffffu);                            // pos
        p[12] = (uint8_t)(r.name_len + 1);                        // l_read_name
        p[13] = 0;                                                // MAPQ
        p[14] = (uint8_t)(BAM_BIN_UNMAPPED & 0xff); p[15] = (uint8_t)(BAM_BIN_UNMAPPED >> 8);
        p[16] = 0; p[17] = 0;                                     // n_cigar_op
        p[18] = 4; p[19] = 0;                                     // FLAG: unmapped
        bam_put32(p + 20, (uint32_t)l);                           // l_seq
        bam_put32(p + 24, 0xffffffffu);                           // next_refID
        bam_put32(p + 28, 0xffffffffu);                           // next_pos
        bam_put32(p + 32, 0u);                                    // tlen
        p[o_seq - 1] = 0;                                         // the name's NUL
        p[o_tag] = 'C'; p[o_tag + 1] = 'O'; p[o_tag + 2] = 'Z';
        p[o_tag + 3 + r.co_len] = 0;
        fields[4 * (int64_t)blockIdx.x] = stream_base + at + o_seq;
        fields[4 * (int64_t)blockIdx.x + 1] = nb;
        fields[4 * (int64_t)blockIdx.x + 2] = stream_base + at + o_qual;
        fields[4 * (int64_t)blockIdx.x + 3] = l;
    }
    const uint8_t *tx = text + r.text_off;
    for (int i = t; i < r.name_len; i += BAM_THREADS) p[o_name + i] = tx[i];
    for (int i = t; i < r.co_len; i += BAM_THREADS) p[o_tag + 3 + i] = tx[r.name_len + i];
    for (int i = t; i < nb; i += BAM_THREADS) {
        const uint8_t hi = s_code[seq[2 * i]];
        const uint8_t lo = 2 * i + 1 < l ? s_code[seq[2 * i + 1]] : 0;
        p[o_seq + i] = (uint8_t)(hi << 4 | lo);
    }
    for (int i = t; i < l; i += BAM_THREADS) p[o_qual + i] = (uint8_t)(qual[i] - 33);
}
