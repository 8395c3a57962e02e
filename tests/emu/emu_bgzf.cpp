// emu_bgzf.cpp — the BGZF compressor (badread_b200/csrc/bb_bgzf.cuh) under the warp emulator, kernel by kernel in the
// order bbl_bgzf_pass enqueues them, behind the argument rules of bb_bgzf_compress (TEST INFRASTRUCTURE).
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_bgzf.cuh"

// Same arguments and results as bb_bgzf_compress without the context (one pass of any length); returns 0, -2 for bad
// arguments or -4 if out_cap is too small.
extern "C" __attribute__((visibility("default")))
int emu_bgzf_compress(const uint8_t *in, int64_t n, int line_mod4, int final, uint8_t *out, int64_t out_cap, int64_t *n_out,
                      int64_t *n_consumed) {
    if (n < 0 || line_mod4 < 0 || line_mod4 > 3) return -2;
    const int64_t use = final ? n : n / BGZF_CHUNK * BGZF_CHUNK;
    const int nc = (int)((use + BGZF_CHUNK - 1) / BGZF_CHUNK);
    *n_out = 0;
    *n_consumed = 0;
    if (use + (int64_t)nc * 31 > out_cap) return -4;
    std::vector<uint4> buf((size_t)use / 16 + 1);   // 16-byte aligned, as cudaMalloc's buffers are
    std::memcpy(buf.data(), in, (size_t)use);
    const uint8_t *d_in = reinterpret_cast<const uint8_t *>(buf.data());
    std::vector<int32_t> lines(nc), sizes(nc);
    std::vector<int64_t> pref(nc + 1), off(nc + 1);
    std::vector<uint32_t> slots((size_t)nc * BGZF_SLOT / 4);
    gridDim.x = (unsigned)nc;
    for (int c = 0; c < nc; c++) {
        blockIdx.x = (unsigned)c;
        emu::run_block(BGZF_THREADS, [&]() { bgzf_k_lines(d_in, use, lines.data()); });
    }
    blockIdx.x = 0;
    emu::run_block(BGZF_THREADS, [&]() { bgzf_k_scan(lines.data(), nc, line_mod4, pref.data()); });
    for (int c = 0; c < nc; c++) {
        blockIdx.x = (unsigned)c;
        emu::run_block(BGZF_THREADS, [&]() {
            bgzf_k_compress(d_in, use, pref.data(), reinterpret_cast<uint8_t *>(slots.data()), sizes.data());
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
