// bb_tu_inflate.cu — compiles the BGZF inflater (bb_inflate.cuh) and its C ABI entry point, bb_bgzf_decompress.
// Like the model builders' calls it takes a device instead of a context and reports errors through bb_model_error().
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_call.h"
#include "bb_inflate.cuh"

// The host walk of in[0..n): its members and their inflated size; BB_ERR_ARG naming the first member that is not BGZF.
static int64_t walk(const uint8_t *in, int64_t n, std::vector<InflMember> &members) {
    char msg[256];
    int64_t total = 0;
    if (!infl_walk(in, n, members, &total, msg, sizeof(msg))) throw Fail{BB_ERR_ARG, msg};
    return total;
}

// The device step after the walk: uploads the input and its members, inflates them on `st` and checks every member's
// status.  Returns a device buffer of `total` bytes (16 when total is 0); a corrupt member throws BB_ERR_ARG naming it
// by index and offset.
static DevBuf infl_device(cudaStream_t st, const uint8_t *in, int64_t n, const std::vector<InflMember> &members, int64_t total) {
    const char *what = "bb_bgzf_decompress";
    Scratch S;
    DevBuf out = S.result((size_t)(total ? total : 16), what);
    if (!members.empty()) {
        const int64_t n_members = (int64_t)members.size();
        const uint8_t *d_in = S.upload(in, n, what, st);
        const InflMember *d_members = S.upload(members.data(), n_members, what, st);
        int32_t *d_status = S.get<int32_t>(n_members, what);
        (void)cudaGetLastError();   // (report this call's launch only)
        const int64_t grid = (n_members + INFL_WARPS - 1) / INFL_WARPS;
        infl_k_members<<<(unsigned)grid, INFL_THREADS, 0, st>>>(d_in, d_members, n_members, out.as<uint8_t>(), d_status);
        check(cudaGetLastError(), "bb_bgzf_decompress: infl_k_members");
        std::vector<int32_t> status(members.size());
        d2h(status.data(), d_status, n_members, st);
        char msg[256];
        if (infl_first_failure(members, status.data(), msg, sizeof(msg))) throw Fail{BB_ERR_ARG, msg};
    }
    return out;
}

extern "C" int bb_bgzf_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out) {
    if (n < 0 || (n > 0 && !in) || !n_out || out_cap < 0 || (out_cap > 0 && !out)) return bad_argument("bb_bgzf_decompress");
    return model_call([&] {
        std::vector<InflMember> members;
        const int64_t total = walk(in, n, members);
        *n_out = total;
        if (total > out_cap)   // (answered from the host walk: the caller asks again with the room)
            throw Fail{BB_ERR_CAPACITY, "bb_bgzf_decompress: " + std::to_string(total) + " bytes of output, capacity " +
                                            std::to_string(out_cap)};
        if (members.empty()) return BB_OK;
        use_device(device);
        const DevBuf d_out = infl_device(0, in, n, members, total);
        check(cudaMemcpy(out, d_out.p, (size_t)total, cudaMemcpyDeviceToHost), "bb_bgzf_decompress: cudaMemcpy");
        return BB_OK;
    });
}

// Any gzip stream: every member BGZF (the host walk succeeds) through infl_device, one warp per member; anything else
// through the chunked inflater of bb_tu_gunzip.cu.  The choice is made from the input.
DevBuf bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, int64_t *total,
                               bb_gzip_stats *stats) {
    *total = 0;
    *stats = bb_gzip_stats{};
    std::vector<InflMember> members;
    char msg[256];
    if (n > 0 && infl_walk(in, n, members, total, msg, sizeof(msg))) {
        stats->bgzf = 1;
        stats->members = (int64_t)members.size();
        return infl_device(st, in, n, members, *total);
    }
    *total = 0;
    return bbl_gzip_chunked(st, in, n, chunk_bytes, total, stats);
}
