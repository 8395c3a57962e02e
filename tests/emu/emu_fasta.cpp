// emu_fasta.cpp — the FASTA parser (badread_b200/csrc/bb_fasta.cuh) under the warp emulator, CTA by CTA, with the tile
// size as an argument so that tests can put tile edges anywhere (TEST INFRASTRUCTURE).  Built with fewer threads per CTA
// than the device (FASTA_THREADS, FASTA_SCAN_THREADS below) to keep the emulator fast; the code paths are the same.
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_fasta.cuh"

// Passes 1 to 3 over text[0..n) in tiles of `tile` bytes.  First call with kept == nullptr: totals[0] = bytes kept,
// totals[1] = header lines.  Second call with kept[totals[0]] and hdr[3 * totals[1]] (starts, ends, kept offsets).
extern "C" __attribute__((visibility("default")))
int emu_fasta_parse(const uint8_t *text, int64_t n, int32_t tile, uint8_t *kept, int64_t *hdr, int64_t *totals) {
    if (tile < 1) return -2;
    const int64_t n_tiles = (n + tile - 1) / tile;
    std::vector<uint8_t> in(text, text + n);   // exact size: a read past the end would leave it
    std::vector<FastaMap> maps((size_t)n_tiles);
    std::vector<FastaTileStart> starts((size_t)n_tiles);
    int64_t tot[2] = {-1, -1};
    gridDim.x = (unsigned)n_tiles;
    for (int64_t t = 0; t < n_tiles; t++) {
        blockIdx.x = (unsigned)t;
        emu::run_block(FASTA_THREADS, [&]() { fasta_k_summarize(in.data(), n, tile, maps.data()); });
    }
    gridDim.x = 1;
    blockIdx.x = 0;
    emu::run_block(FASTA_SCAN_THREADS, [&]() { fasta_k_scan(maps.data(), n_tiles, starts.data(), tot); });
    totals[0] = tot[0];
    totals[1] = tot[1];
    if (!kept) return 0;
    // guard bands around the outputs: a write outside them fails the call (-3) instead of landing elsewhere
    constexpr int64_t G = 4096;
    std::vector<uint8_t> out((size_t)(tot[0] + 2 * G), 0xa5);
    std::vector<int64_t> h((size_t)(3 * tot[1] + 2 * G), -7);
    int64_t *h0 = h.data() + G;
    gridDim.x = (unsigned)n_tiles;
    for (int64_t t = 0; t < n_tiles; t++) {
        blockIdx.x = (unsigned)t;
        emu::run_block(FASTA_THREADS, [&]() {
            fasta_k_emit(in.data(), n, tile, starts.data(), out.data() + G, h0, h0 + tot[1], h0 + 2 * tot[1]);
        });
    }
    gridDim.x = 1;
    blockIdx.x = 0;
    for (int64_t i = 0; i < G; i++)
        if (out[(size_t)i] != 0xa5 || out[(size_t)(G + tot[0] + i)] != 0xa5 || h[(size_t)i] != -7 ||
            h[(size_t)(G + 3 * tot[1] + i)] != -7)
            return -3;
    std::copy(out.begin() + G, out.end() - G, kept);
    std::copy(h0, h0 + 3 * tot[1], hdr);
    return 0;
}

// fasta_k_gather: dst[dst_off[r] .. dst_off[r + 1]) = src[src_lo[r] ..] for r < n_ranges
extern "C" __attribute__((visibility("default")))
int emu_fasta_gather(const uint8_t *src, int64_t n_src, const int64_t *src_lo, const int64_t *dst_off, int32_t n_ranges,
                     uint8_t *dst) {
    const int64_t total = dst_off[n_ranges];
    std::vector<uint8_t> in(src, src + n_src), out((size_t)total);
    const int64_t blocks = (total + 256 * FASTA_GATHER - 1) / (256 * FASTA_GATHER);
    gridDim.x = (unsigned)blocks;
    for (int64_t b = 0; b < blocks; b++) {
        blockIdx.x = (unsigned)b;
        emu::run_block(256, [&]() { fasta_k_gather(in.data(), src_lo, dst_off, n_ranges, out.data()); });
    }
    gridDim.x = 1;
    blockIdx.x = 0;
    std::copy(out.begin(), out.end(), dst);
    return 0;
}
