// emu_gunzip.cpp — the gzip inflater (badread_b200/csrc/bb_gunzip.cuh) under the warp emulator: its driver, gz_inflate,
// with a backend that runs every kernel CTA by CTA in host memory (TEST INFRASTRUCTURE).
#include "cuda_emu.h"

inline unsigned atomicXor(unsigned *p, unsigned v) { const unsigned o = *p; *p = o ^ v; return o; }
#define __noinline__ __attribute__((noinline))
#define GZ_WINDOW_THREADS 256   // (the emulator runs at most 512 threads per CTA; the kernel strides over its window)

#include <vector>

#include "../../badread_b200/csrc/bb_gunzip.cuh"

namespace {

template <class F> void run_grid(unsigned grid, int threads, F f) {
    gridDim.x = grid;
    for (unsigned c = 0; c < grid; c++) {
        blockIdx.x = c;
        emu::run_block(threads, f);
    }
    blockIdx.x = 0;
}

struct EmuDev {   // "device" memory is host memory; a launch runs before it returns
    int alloc(void **p, size_t bytes) { *p = std::calloc(1, bytes); return *p ? 0 : 2; }
    void release(void *p) { std::free(p); }
    int h2d(void *d, const void *h, size_t bytes) { std::memcpy(d, h, bytes); return 0; }
    int d2h(void *h, const void *d, size_t bytes) { std::memcpy(h, d, bytes); return 0; }
    int fill(void *d, int v, size_t bytes) { std::memset(d, v, bytes); return 0; }
    int sync() { return 0; }
    int fail(const char *what, int e, char *msg, size_t msg_len) {
        std::snprintf(msg, msg_len, "emu_gunzip: %s: error %d", what, e);
        return BB_ERR_CUDA;
    }
    template <class... A> void find(unsigned grid, A... a) { run_grid(grid, GZ_FIND_THREADS, [&]() { gz_k_find(a...); }); }
    template <class... A> void decode(unsigned grid, A... a) { run_grid(grid, INFL_THREADS, [&]() { gz_k_decode(a...); }); }
    template <class... A> void chain(A... a) { run_grid(1, 32, [&]() { gz_k_chain(a...); }); }
    template <class... A> void windows(A... a) { run_grid(1, GZ_WINDOW_THREADS, [&]() { gz_k_windows(a...); }); }
    template <class... A> void resolve(unsigned grid, A... a) { run_grid(grid, GZ_RESOLVE_THREADS, [&]() { gz_k_resolve(a...); }); }
    template <class... A> void crc(unsigned grid, A... a) { run_grid(grid, INFL_THREADS, [&]() { gz_k_crc(a...); }); }
};

}  // namespace

// bb_gzip_decompress without the device and without the BGZF dispatch: 0, -2 (message in msg) or -4 (*n_out = the size
// needed).  in_copy is an exact-size copy of the input, so that a read past it would leave the input.
extern "C" __attribute__((visibility("default")))
int emu_gzip_decompress(const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out, int64_t chunk_bytes,
                        bb_gzip_stats *stats, char *msg, int msg_len) {
    msg[0] = 0;
    std::vector<uint8_t> in_copy(in, in + n);
    EmuDev dev;
    uint8_t *res = nullptr;
    int64_t total = 0;
    *stats = bb_gzip_stats{};
    const int rc = gz_inflate(dev, in_copy.data(), n, chunk_bytes, &res, &total, stats, msg, (size_t)msg_len);
    if (rc) return rc;
    *n_out = total;
    if (total > out_cap) {
        std::free(res);
        return -4;
    }
    std::memcpy(out, res, (size_t)total);
    std::free(res);
    return 0;
}
