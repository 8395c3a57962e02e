// emu_plot.cpp — the window series kernel (badread_b200/csrc/bb_plot.cuh) under the warp emulator, CTA by CTA, with the
// positions per thread as an argument so that tests can put tile edges anywhere (TEST INFRASTRUCTURE).  Built with fewer
// threads per CTA than the device (WS_THREADS in emu_plot.py); the code paths are the same.
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_plot.cuh"

// All n_aln alignments of the flat arrays in one pass, as bb_window_series runs them: identity / mean_qual get
// sum(max(0, L - window)) values each (mean_qual == nullptr: no qscores).
extern "C" __attribute__((visibility("default")))
int emu_window_series(int32_t n_aln, const uint8_t *read, const uint8_t *qual, const uint8_t *ref, const int64_t *read_off,
                      const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0, const int32_t *op_ref0,
                      const int64_t *ops_off, int64_t window, int items, double *identity, double *mean_qual) {
    if (items < 1 || items > WS_ITEMS || window < 1) return -2;
    std::vector<int64_t> s_off((size_t)n_aln + 1, 0), p_off((size_t)n_aln + 1, 0);
    for (int32_t a = 0; a < n_aln; a++) {
        const int64_t L = read_off[a + 1] - read_off[a];
        s_off[(size_t)a + 1] = s_off[(size_t)a] + L + 1;
        p_off[(size_t)a + 1] = p_off[(size_t)a] + (L > window ? L - window : 0);
    }
    // exact sizes (a read or write past the end would leave them)
    std::vector<uint8_t> rd(read, read + read_off[n_aln]), rf(ref, ref + ref_off[n_aln]);
    std::vector<uint8_t> ql(qual ? qual : read, (qual ? qual : read) + read_off[n_aln]);
    std::vector<uint32_t> op(ops, ops + ops_off[n_aln]);
    std::vector<int32_t> p0(op_read0, op_read0 + ops_off[n_aln]), r0(op_ref0, op_ref0 + ops_off[n_aln]);
    std::vector<int64_t> E((size_t)s_off.back(), -1), Q((size_t)s_off.back(), -1);
    std::vector<double> id((size_t)p_off.back()), mq((size_t)p_off.back());
    gridDim.x = (unsigned)n_aln;
    for (int32_t a = 0; a < n_aln; a++) {
        blockIdx.x = (unsigned)a;
        emu::run_block(WS_THREADS, [&]() {
            ws_k_series(rd.data(), mean_qual ? ql.data() : nullptr, rf.data(), read_off, ref_off, op.data(), p0.data(), r0.data(),
                        ops_off, window, items, s_off.data(), p_off.data(), E.data(), Q.data(), id.data(), mq.data());
        });
    }
    gridDim.x = 1;
    blockIdx.x = 0;
    std::copy(id.begin(), id.end(), identity);
    if (mean_qual) std::copy(mq.begin(), mq.end(), mean_qual);
    return 0;
}
