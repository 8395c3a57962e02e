// bb_tu_gunzip.cu — compiles the gzip inflater (bb_gunzip.cuh) with its CUDA backend, and its C ABI entry point,
// bb_gzip_decompress.  Like bb_bgzf_decompress it takes a device instead of a context and reports errors through
// bb_model_error().
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_crc32.cuh"
#define INFL_NO_MEMBER_KERNEL
namespace {   // (bb_inflate.cuh's decoder and tables are also bb_tu_inflate.cu's: this unit's copies stay private)
#include "bb_gunzip.cuh"
}

void bbm_set_error(const char *msg);   // bb_tu_models.cu
int bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out,
                            int64_t *total, bb_gzip_stats *stats, char *msg, size_t msg_len);   // (bb_launch.h)
int bbl_gzip_chunked(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out, int64_t *total,
                     bb_gzip_stats *stats, char *msg, size_t msg_len);   // (bb_tu_inflate.cu)

namespace {

int cuda_fail(const char *what, cudaError_t e, char *msg, size_t msg_len) {
    std::snprintf(msg, msg_len, "bb_gzip_decompress: %s: %s", what, cudaGetErrorString(e));
    return BB_ERR_CUDA;
}

struct CudaDev {   // gz_inflate's backend: every copy and launch on one stream
    cudaStream_t st;
    int alloc(void **p, size_t bytes) { return cudaMalloc(p, bytes); }
    void release(void *p) { cudaFree(p); }
    int h2d(void *d, const void *h, size_t bytes) { return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st); }
    int d2h(void *h, const void *d, size_t bytes) { return cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st); }
    int fill(void *d, int v, size_t bytes) { return cudaMemsetAsync(d, v, bytes, st); }
    int sync() {   // (a launch error surfaces here)
        const cudaError_t e = cudaGetLastError();
        return e != cudaSuccess ? e : cudaStreamSynchronize(st);
    }
    int fail(const char *what, int e, char *msg, size_t msg_len) { return cuda_fail(what, (cudaError_t)e, msg, msg_len); }
    template <class... A> void find(unsigned grid, A... a) { gz_k_find<<<grid, GZ_FIND_THREADS, 0, st>>>(a...); }
    template <class... A> void decode(unsigned grid, A... a) { gz_k_decode<<<grid, INFL_THREADS, 0, st>>>(a...); }
    template <class... A> void chain(A... a) { gz_k_chain<<<1, 32, 0, st>>>(a...); }
    template <class... A> void windows(A... a) { gz_k_windows<<<1, GZ_WINDOW_THREADS, 0, st>>>(a...); }
    template <class... A> void resolve(unsigned grid, A... a) { gz_k_resolve<<<grid, GZ_RESOLVE_THREADS, 0, st>>>(a...); }
    template <class... A> void crc(unsigned grid, A... a) { gz_k_crc<<<grid, INFL_THREADS, 0, st>>>(a...); }
};

}  // namespace

// The chunked inflater (gz_inflate) on `st`, for a stream that is not all BGZF; bbl_gzip_inflate_device decides.
int bbl_gzip_chunked(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, uint8_t **out, int64_t *total,
                     bb_gzip_stats *stats, char *msg, size_t msg_len) {
    msg[0] = 0;
    (void)cudaGetLastError();   // (report this call's launches only)
    CudaDev dev{st};
    return gz_inflate(dev, in, n, chunk_bytes, out, total, stats, msg, msg_len);
}

extern "C" int bb_gzip_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out,
                                  int64_t chunk_bytes, bb_gzip_stats *stats) {
    bbm_set_error("");
    char msg[256];
    if (n < 0 || (n > 0 && !in) || !n_out || out_cap < 0 || (out_cap > 0 && !out) || chunk_bytes < 0) {
        bbm_set_error("bb_gzip_decompress: invalid argument");
        return BB_ERR_ARG;
    }
    bb_gzip_stats local;
    if (!stats) stats = &local;
    uint8_t *d_out = nullptr;
    int64_t total = 0;
    cudaError_t e = cudaSetDevice(device);
    int rc = e == cudaSuccess ? bbl_gzip_inflate_device(0, in, n, chunk_bytes, &d_out, &total, stats, msg, sizeof(msg))
                              : cuda_fail("cudaSetDevice", e, msg, sizeof(msg));
    if (rc == BB_OK) {
        *n_out = total;
        if (total > out_cap) {
            std::snprintf(msg, sizeof(msg), "bb_gzip_decompress: %lld bytes of output, capacity %lld", (long long)total,
                          (long long)out_cap);
            rc = BB_ERR_CAPACITY;
        } else if (total && (e = cudaMemcpy(out, d_out, (size_t)total, cudaMemcpyDeviceToHost)) != cudaSuccess) {
            rc = cuda_fail("cudaMemcpy", e, msg, sizeof(msg));
        }
    }
    cudaFree(d_out);
    if (rc) bbm_set_error(msg);
    return rc;
}
