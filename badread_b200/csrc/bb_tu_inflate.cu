// bb_tu_inflate.cu — compiles the BGZF inflater (bb_inflate.cuh) and its C ABI entry point, bb_bgzf_decompress.
// Like the model builders' calls it takes a device instead of a context and reports errors through bb_model_error().
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_inflate.cuh"

void bbm_set_error(const char *msg);   // bb_tu_models.cu
int bbl_bgzf_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, uint8_t **out, int64_t *total, char *msg,
                            size_t msg_len);   // (bb_launch.h)
int bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out,
                            int64_t *total, bb_gzip_stats *stats, char *msg, size_t msg_len);   // (bb_launch.h)
int bbl_gzip_chunked(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out, int64_t *total,
                     bb_gzip_stats *stats, char *msg, size_t msg_len);   // bb_tu_gunzip.cu

namespace {

struct DevBuf {   // released on every exit path
    void *p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
};

int cuda_fail(const char *what, cudaError_t e, char *msg, size_t msg_len) {
    std::snprintf(msg, msg_len, "bb_bgzf_decompress: %s: %s", what, cudaGetErrorString(e));
    return BB_ERR_CUDA;
}

}  // namespace

#define BBI_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(#call, e_, msg, msg_len); } while (0)

// The device step after infl_walk: uploads the input and its members, inflates them on `st` and checks every member's
// status.  On success *out is a device buffer of `total` bytes (16 when total is 0) that the caller frees; otherwise
// msg says why (a corrupt member by index and offset).
static int infl_device(cudaStream_t st, const uint8_t *in, int64_t n, const std::vector<InflMember> &members, int64_t total,
                       uint8_t **out, char *msg, size_t msg_len) {
    DevBuf d_in, d_out, d_members, d_status;
    BBI_TRY(cudaMalloc(&d_out.p, (size_t)(total ? total : 16)));
    if (!members.empty()) {
        const int64_t n_members = (int64_t)members.size();
        BBI_TRY(cudaMalloc(&d_in.p, (size_t)n));
        BBI_TRY(cudaMalloc(&d_members.p, members.size() * sizeof(InflMember)));
        BBI_TRY(cudaMalloc(&d_status.p, members.size() * sizeof(int32_t)));
        BBI_TRY(cudaMemcpyAsync(d_in.p, in, (size_t)n, cudaMemcpyHostToDevice, st));
        BBI_TRY(cudaMemcpyAsync(d_members.p, members.data(), members.size() * sizeof(InflMember), cudaMemcpyHostToDevice, st));
        (void)cudaGetLastError();   // (report this call's launch only)
        const int64_t grid = (n_members + INFL_WARPS - 1) / INFL_WARPS;
        infl_k_members<<<(unsigned)grid, INFL_THREADS, 0, st>>>((const uint8_t *)d_in.p, (const InflMember *)d_members.p,
                                                                 n_members, (uint8_t *)d_out.p, (int32_t *)d_status.p);
        BBI_TRY(cudaGetLastError());
        std::vector<int32_t> status(members.size());
        BBI_TRY(cudaMemcpyAsync(status.data(), d_status.p, members.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        BBI_TRY(cudaStreamSynchronize(st));
        if (infl_first_failure(members, status.data(), msg, msg_len)) return BB_ERR_ARG;
    }
    *out = (uint8_t *)d_out.p;
    d_out.p = nullptr;
    return BB_OK;
}

extern "C" int bb_bgzf_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out) {
    bbm_set_error("");
    char msg[256];
    if (n < 0 || (n > 0 && !in) || !n_out || out_cap < 0 || (out_cap > 0 && !out)) {
        bbm_set_error("bb_bgzf_decompress: invalid argument");
        return BB_ERR_ARG;
    }
    std::vector<InflMember> members;
    int64_t total = 0;
    if (!infl_walk(in, n, members, &total, msg, sizeof(msg))) {
        bbm_set_error(msg);
        return BB_ERR_ARG;
    }
    *n_out = total;
    if (total > out_cap) {   // (answered from the host walk: the caller asks again with the room)
        std::snprintf(msg, sizeof(msg), "bb_bgzf_decompress: %lld bytes of output, capacity %lld", (long long)total,
                      (long long)out_cap);
        bbm_set_error(msg);
        return BB_ERR_CAPACITY;
    }
    if (members.empty()) return BB_OK;
    uint8_t *d_out = nullptr;
    cudaError_t e = cudaSetDevice(device);
    int rc = e == cudaSuccess ? infl_device(0, in, n, members, total, &d_out, msg, sizeof(msg))
                              : cuda_fail("cudaSetDevice", e, msg, sizeof(msg));
    if (rc == BB_OK && (e = cudaMemcpy(out, d_out, (size_t)total, cudaMemcpyDeviceToHost)) != cudaSuccess)
        rc = cuda_fail("cudaMemcpy", e, msg, sizeof(msg));
    cudaFree(d_out);
    if (rc) bbm_set_error(msg);
    return rc;
}

int bbl_bgzf_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, uint8_t **out, int64_t *total, char *msg,
                            size_t msg_len) {
    *out = nullptr;
    *total = 0;
    std::vector<InflMember> members;
    if (!infl_walk(in, n, members, total, msg, msg_len)) return BB_ERR_ARG;
    return infl_device(st, in, n, members, *total, out, msg, msg_len);
}

// Any gzip stream: every member BGZF (the host walk succeeds) through infl_device, one warp per member; anything else
// through the chunked inflater of bb_tu_gunzip.cu.  The choice is made from the input.
int bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out,
                            int64_t *total, bb_gzip_stats *stats, char *msg, size_t msg_len) {
    *out = nullptr;
    *total = 0;
    *stats = bb_gzip_stats{};
    std::vector<InflMember> members;
    if (n > 0 && infl_walk(in, n, members, total, msg, msg_len)) {
        stats->bgzf = 1;
        stats->members = (int64_t)members.size();
        return infl_device(st, in, n, members, *total, out, msg, msg_len);
    }
    *total = 0;
    return bbl_gzip_chunked(st, in, n, chunk_bytes, out, total, stats, msg, msg_len);
}
