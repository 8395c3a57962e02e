// bb_tu_fasta.cu — compiles the FASTA parser (bb_fasta.cuh) and enqueues its passes.
#include "bb_call.h"
#include "bb_fasta.cuh"
#include "bb_launch.h"

int64_t bbl_fasta_tiles(int64_t n) { return (n + FASTA_TILE - 1) / FASTA_TILE; }

size_t bbl_fasta_scratch_bytes(int64_t n) {
    return (size_t)bbl_fasta_tiles(n) * (sizeof(FastaMap) + sizeof(FastaTileStart)) + 2 * sizeof(int64_t);
}

void bbl_fasta_scan(cudaStream_t st, const uint8_t *text, int64_t n, void *scratch) {
    const int64_t n_tiles = bbl_fasta_tiles(n);
    FastaMap *maps = reinterpret_cast<FastaMap *>(scratch);
    FastaTileStart *starts = reinterpret_cast<FastaTileStart *>(maps + n_tiles);
    int64_t *totals = reinterpret_cast<int64_t *>(starts + n_tiles);
    if (n_tiles > 0) fasta_k_summarize<<<(unsigned)n_tiles, FASTA_THREADS, 0, st>>>(text, n, FASTA_TILE, maps);
    fasta_k_scan<<<1, FASTA_SCAN_THREADS, 0, st>>>(maps, n_tiles, starts, totals);
}

const int64_t *bbl_fasta_totals(const void *scratch, int64_t n) {
    const int64_t n_tiles = bbl_fasta_tiles(n);
    return reinterpret_cast<const int64_t *>(reinterpret_cast<const FastaTileStart *>(
        reinterpret_cast<const FastaMap *>(scratch) + n_tiles) + n_tiles);
}

void bbl_fasta_emit(cudaStream_t st, const uint8_t *text, int64_t n, const void *scratch, uint8_t *kept, int64_t *hdr_start,
                    int64_t *hdr_end, int64_t *hdr_kept) {
    const int64_t n_tiles = bbl_fasta_tiles(n);
    if (n_tiles == 0) return;
    const FastaTileStart *starts = reinterpret_cast<const FastaTileStart *>(reinterpret_cast<const FastaMap *>(scratch) + n_tiles);
    fasta_k_emit<<<(unsigned)n_tiles, FASTA_THREADS, 0, st>>>(text, n, FASTA_TILE, starts, kept, hdr_start, hdr_end, hdr_kept);
}

void bbl_fasta_gather(cudaStream_t st, const uint8_t *src, const int64_t *src_lo, const int64_t *dst_off, int32_t n_ranges,
                      int64_t total, uint8_t *dst) {
    if (total <= 0) return;
    const int64_t threads = (total + FASTA_GATHER - 1) / FASTA_GATHER;
    fasta_k_gather<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(src, src_lo, dst_off, n_ranges, dst);
}
