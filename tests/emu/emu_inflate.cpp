// emu_inflate.cpp — the BGZF inflater (badread_b200/csrc/bb_inflate.cuh) under the warp emulator, CTA by CTA, behind the
// same host walk and status messages as bb_bgzf_decompress (TEST INFRASTRUCTURE).
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_inflate.cuh"

// Same arguments and results as bb_bgzf_decompress without the device: 0, -2 (message in msg) or -4 (*n_out = the size
// needed).  The kernel writes into a buffer of exactly the stream's inflated size, so a write outside the members would
// land outside it; in_copy is an exact-size copy of the input for the same reason.
extern "C" __attribute__((visibility("default")))
int emu_bgzf_decompress(const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out, char *msg, int msg_len) {
    msg[0] = 0;
    std::vector<InflMember> members;
    int64_t total = 0;
    if (!infl_walk(in, n, members, &total, msg, (size_t)msg_len)) return -2;
    *n_out = total;
    if (total > out_cap) return -4;
    if (members.empty()) return 0;
    std::vector<uint8_t> in_copy(in, in + n), out_buf((size_t)total);
    const int64_t n_members = (int64_t)members.size();
    std::vector<int32_t> status(members.size(), -1);
    const unsigned grid = (unsigned)((n_members + INFL_WARPS - 1) / INFL_WARPS);
    gridDim.x = grid;
    for (unsigned c = 0; c < grid; c++) {
        blockIdx.x = c;
        emu::run_block(INFL_THREADS, [&]() { infl_k_members(in_copy.data(), members.data(), n_members, out_buf.data(), status.data()); });
    }
    blockIdx.x = 0;
    if (infl_first_failure(members, status.data(), msg, (size_t)msg_len)) return -2;
    std::memcpy(out, out_buf.data(), (size_t)total);
    return 0;
}
