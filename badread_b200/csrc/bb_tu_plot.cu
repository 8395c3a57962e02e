// bb_tu_plot.cu — compiles the window series of `badread plot` (bb_plot.cuh) and its C ABI entry, bb_window_series.  Like
// the model builders' entries it takes a device instead of a context, reports failures through bb_model_error() and runs
// on the legacy default stream.
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_call.h"
#include "bb_plot.cuh"

extern "C" int bb_window_series(int device, int32_t n_aln, const uint8_t *read, const uint8_t *qual, const uint8_t *ref,
                                const int64_t *read_off, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                                const int32_t *op_ref0, const int64_t *ops_off, int64_t window, int want_qual, int32_t first_aln,
                                int32_t n_pass, double *out_identity, double *out_qual, int64_t *n_points) {
    if (n_aln < 0 || first_aln < 0 || n_pass < 0 || (int64_t)first_aln + n_pass > n_aln || window < 1 || !read_off ||
        !ref_off || !ops_off || !n_points || (n_pass && (!read || !ref || !ops || !op_read0 || !op_ref0 || !out_identity)) ||
        (n_pass && want_qual && (!qual || !out_qual)))
        return bad_argument("bb_window_series");
    // pass-local offsets: alignment k = first_aln + k of the pass
    std::vector<int64_t> r_off((size_t)n_pass + 1), f_off((size_t)n_pass + 1), o_off((size_t)n_pass + 1),
        s_off((size_t)n_pass + 1, 0), p_off((size_t)n_pass + 1, 0);
    const int64_t rb = read_off[first_aln], fb = ref_off[first_aln], ob = ops_off[first_aln];
    for (int32_t k = 0; k <= n_pass; k++) {
        r_off[(size_t)k] = read_off[first_aln + k] - rb;
        f_off[(size_t)k] = ref_off[first_aln + k] - fb;
        o_off[(size_t)k] = ops_off[first_aln + k] - ob;
        if (k < n_pass) {
            const int64_t L = read_off[first_aln + k + 1] - read_off[first_aln + k];
            s_off[(size_t)k + 1] = s_off[(size_t)k] + L + 1;
            p_off[(size_t)k + 1] = p_off[(size_t)k] + (L > window ? L - window : 0);
        }
    }
    *n_points = p_off[(size_t)n_pass];
    if (n_pass == 0) {
        bbm_set_error("");
        return BB_OK;
    }
    const int64_t n_read = r_off.back(), n_ref = f_off.back(), n_ops = o_off.back(), n_pts = p_off.back(), n_sums = s_off.back();
    return device_call(device, [&] {
        Scratch S(BB_ERR_CAPACITY);
        const uint8_t *d_read = S.input(read + rb, n_read, device, "the read slices");
        const uint8_t *d_qual = want_qual ? S.input(qual + rb, n_read, device, "the quality slices") : nullptr;
        const uint8_t *d_ref = S.input(ref + fb, n_ref, device, "the reference slices");
        const uint32_t *d_ops = S.input(ops + ob, n_ops, device, "the CIGAR runs");
        const int32_t *d_p0 = S.input(op_read0 + ob, n_ops, device, "the CIGAR runs");
        const int32_t *d_r0 = S.input(op_ref0 + ob, n_ops, device, "the CIGAR runs");
        const int64_t n1 = (int64_t)n_pass + 1;
        int64_t *d_offs = S.get<int64_t>(5 * n1, "the pass offsets");
        const std::vector<int64_t> *offs[5] = {&r_off, &f_off, &o_off, &s_off, &p_off};
        for (int i = 0; i < 5; i++)
            check(cudaMemcpy(d_offs + i * n1, offs[i]->data(), (size_t)n1 * 8, cudaMemcpyHostToDevice), "cudaMemcpy");
        int64_t *d_e = S.get<int64_t>(n_sums, "the error prefix sums");
        int64_t *d_q = want_qual ? S.get<int64_t>(n_sums, "the quality prefix sums") : nullptr;
        double *d_id = S.get<double>(n_pts, "the identity series");
        double *d_mq = want_qual ? S.get<double>(n_pts, "the qscore series") : nullptr;
        ws_k_series<<<(unsigned)n_pass, WS_THREADS>>>(d_read, d_qual, d_ref, d_offs, d_offs + n1, d_ops, d_p0, d_r0, d_offs + 2 * n1,
                                                      window, WS_ITEMS, d_offs + 3 * n1, d_offs + 4 * n1, d_e, d_q, d_id, d_mq);
        check(cudaGetLastError(), "ws_k_series");
        d2h(out_identity, d_id, n_pts);
        if (want_qual) d2h(out_qual, d_mq, n_pts);
        check(cudaDeviceSynchronize(), "ws_k_series");
        return BB_OK;
    });
}
