// bb_tu_gunzip.cu — compiles the gzip inflater (bb_gunzip.cuh) with its CUDA backend, and its C ABI entry point,
// bb_gzip_decompress.  Like bb_bgzf_decompress it takes a device instead of a context and reports errors through
// bb_model_error().
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_call.h"
#include "bb_crc32.cuh"
#define INFL_NO_MEMBER_KERNEL
namespace {   // (bb_inflate.cuh's decoder and tables are also bb_tu_inflate.cu's: this unit's copies stay private)
#include "bb_gunzip.cuh"

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
    int fail(const char *what, int e, char *msg, size_t msg_len) {
        std::snprintf(msg, msg_len, "bb_gzip_decompress: %s: %s", what, cudaGetErrorString((cudaError_t)e));
        return BB_ERR_CUDA;
    }
    template <class... A> void find(unsigned grid, A... a) { gz_k_find<<<grid, GZ_FIND_THREADS, 0, st>>>(a...); }
    template <class... A> void decode(unsigned grid, A... a) { gz_k_decode<<<grid, INFL_THREADS, 0, st>>>(a...); }
    template <class... A> void chain(A... a) { gz_k_chain<<<1, 32, 0, st>>>(a...); }
    template <class... A> void windows(A... a) { gz_k_windows<<<1, GZ_WINDOW_THREADS, 0, st>>>(a...); }
    template <class... A> void resolve(unsigned grid, A... a) { gz_k_resolve<<<grid, GZ_RESOLVE_THREADS, 0, st>>>(a...); }
    template <class... A> void crc(unsigned grid, A... a) { gz_k_crc<<<grid, INFL_THREADS, 0, st>>>(a...); }
};

}  // namespace

// The chunked inflater (gz_inflate) on `st`, for a stream that is not all BGZF; bbl_gzip_inflate_device decides.
DevBuf bbl_gzip_chunked(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, int64_t *total, bb_gzip_stats *stats) {
    char msg[256] = "";
    (void)cudaGetLastError();   // (report this call's launches only)
    CudaDev dev{st};
    DevBuf out;
    uint8_t *p = nullptr;
    if (const int rc = gz_inflate(dev, in, n, chunk_bytes, &p, total, stats, msg, sizeof(msg))) throw Fail{rc, msg};
    out.p = p;
    out.cap = (size_t)std::max<int64_t>(*total, 16);
    return out;
}

extern "C" int bb_gzip_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out,
                                  int64_t chunk_bytes, bb_gzip_stats *stats) {
    if (n < 0 || (n > 0 && !in) || !n_out || out_cap < 0 || (out_cap > 0 && !out) || chunk_bytes < 0)
        return bad_argument("bb_gzip_decompress");
    bb_gzip_stats local;
    if (!stats) stats = &local;
    return device_call(device, [&] {
        int64_t total = 0;
        const DevBuf d_out = bbl_gzip_inflate_device(0, in, n, chunk_bytes, &total, stats);
        *n_out = total;
        if (total > out_cap)
            throw Fail{BB_ERR_CAPACITY, "bb_gzip_decompress: " + std::to_string(total) + " bytes of output, capacity " +
                                            std::to_string(out_cap)};
        if (total) check(cudaMemcpy(out, d_out.p, (size_t)total, cudaMemcpyDeviceToHost), "bb_gzip_decompress: cudaMemcpy");
        return BB_OK;
    });
}
