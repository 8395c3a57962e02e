// bb_call.h — how the entry points own device memory and report failures, and the host helpers of the input paths that
// more than one unit calls.  A helper that fails throws Fail, and one wrapper per entry point turns it into the return
// code and the message: bb_last_error() of the context for the context entry points (context_call), bb_model_error(), a
// message per host thread, for the loaders and model builders, which take a device instead (model_call).  The first
// half is plain C++, for the units g++ compiles without the CUDA headers (bb_bam.cpp); the rest needs cuda_runtime.h.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/badread_b200.h"

struct Fail {   // thrown with the return code and the message the entry point reports
    int rc;
    std::string msg;
};

// The message of bb_model_error() for the calling thread
void bbm_set_error(const std::string &msg);

// An entry point's refusal of its arguments, before it touches a device
inline int bad_argument(const char *name) {
    bbm_set_error(std::string(name) + ": invalid argument");
    return BB_ERR_ARG;
}

// Runs an entry point's body() (which returns its code) with the message cleared; a Fail becomes the code and the message.
template <class F>
int model_call(F &&body) {
    bbm_set_error("");
    try {
        return body();
    } catch (const Fail &f) {
        bbm_set_error(f.msg);
        return f.rc;
    }
}

#ifdef __CUDACC__
#include <cuda_runtime.h>

inline void check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) throw Fail{BB_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e)};
}

// Makes `device` current and discards the error an earlier call of this thread left (for instance an out-of-memory of
// another context's scratch, already reported there), so that cudaGetLastError() reports this call's launches only.
inline void use_device(int device) {
    check(cudaSetDevice(device), "cudaSetDevice");
    (void)cudaGetLastError();
}

// model_call for an entry point that takes a device: body() runs with `device` current (use_device)
template <class F>
int device_call(int device, F &&body) {
    return model_call([&] {
        use_device(device);
        return body();
    });
}

// Runs a context entry point's body(), which returns its code or nothing (BB_OK).  A null context is refused with
// BB_ERR_ARG and no message; a Fail becomes the code and the context's message (bb_last_error), which a success leaves
// as it was.
template <class Ctx, class F>
int context_call(Ctx *ctx, F &&body) {
    if (!ctx) return BB_ERR_ARG;
    try {
        if constexpr (std::is_void_v<decltype(body())>) {
            body();
            return BB_OK;
        } else {
            return body();
        }
    } catch (const Fail &f) {
        ctx->err = f.msg;
        return f.rc;
    }
}

// context_call for an entry point that works on the context's device: body() runs with it current (use_device)
template <class Ctx, class F>
int context_device_call(Ctx *ctx, F &&body) {
    return context_call(ctx, [&] {
        use_device(ctx->device);
        return body();
    });
}

struct DevBuf {   // a device allocation, freed with its owner
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;   // (so a Worker or a context cannot be copied either)
    DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) {
            release();
            p = std::exchange(o.p, nullptr);
            cap = std::exchange(o.cap, 0);
        }
        return *this;
    }
    ~DevBuf() { release(); }
    // grow-only: at least `bytes`, with slack for the next call; a failure throws BB_ERR_CUDA "<what>: <error>"
    void ensure(size_t bytes, const char *what) {
        if (bytes <= cap) return;
        release();
        const size_t want = bytes + bytes / 8 + 256;
        const cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) (void)cudaGetLastError();   // (an out-of-memory, say, is not for a later launch to report)
        check(e, what);
        cap = want;
    }
    // exactly `bytes` (at least 1), for buffers the size of their contents
    cudaError_t alloc(size_t bytes) {
        release();
        bytes = bytes ? bytes : 1;
        const cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// The device memory of one call, freed on every exit path.  A failed allocation throws: out of memory with oom_rc =
// BB_ERR_CAPACITY as "Error: not enough device memory for <what> (<n> bytes asked for)", anything else as BB_ERR_CUDA
// "<what>: <error>".  Copies are on the legacy default stream unless a stream is given.
class Scratch {
  public:
    explicit Scratch(int oom_rc = BB_ERR_CUDA) : oom_rc_(oom_rc) {}
    // `count` elements, at least 16 bytes, not initialized
    template <class T> T *get(int64_t count, const char *what) {
        held_.push_back(result((size_t)count * sizeof(T), what));
        return held_.back().as<T>();
    }
    // a copy of src[0..count)
    template <class T> T *upload(const T *src, int64_t count, const char *what, cudaStream_t st = 0) {
        T *d = get<T>(count, what);
        if (count > 0) check(cudaMemcpyAsync(d, src, (size_t)count * sizeof(T), cudaMemcpyHostToDevice, st), "cudaMemcpy");
        return d;
    }
    // src[0..count) in place when it is device memory of `device`, else a copy
    template <class T> const T *input(const T *src, int64_t count, int device, const char *what) {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device == device) return src;
        (void)cudaGetLastError();
        return upload(src, count, what);
    }
    // `bytes` (at least 16) that the call hands out with its results: not freed with the scratch
    DevBuf result(size_t bytes, const char *what) const;

  private:
    int oom_rc_;
    std::vector<DevBuf> held_;
};

// dst[0..count) from device memory, copied on `st` and waited for
template <class T>
void d2h(T *dst, const void *src, int64_t count, cudaStream_t st = 0) {
    if (count > 0) {
        check(cudaMemcpyAsync(dst, src, (size_t)count * sizeof(T), cudaMemcpyDeviceToHost, st), "cudaMemcpy");
        check(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    }
}

// ---- the input paths' helpers (bb_call.cu unless noted)
// An input file data[0..n) in device memory, *len bytes: inflated on `st` when `gzip` (BGZF or not, *stats as
// bb_gzip_decompress reports them; an inflate failure is thrown as it is), else copied as it is into an allocation of
// S's (what: its name).
DevBuf text_to_device(Scratch &S, cudaStream_t st, const uint8_t *data, int64_t n, bool gzip, int64_t *len,
                      bb_gzip_stats *stats, const char *what);
// The n spans [lo[i], hi[i]) of device text gathered on `st` into *bytes: span i is bytes[off[i] .. off[i + 1]), and
// off (n + 1 entries) is returned.  Scratch from S (what: the spans' name).
std::vector<int64_t> gather_spans(Scratch &S, cudaStream_t st, const uint8_t *text, const std::vector<int64_t> &lo,
                                  const std::vector<int64_t> &hi, std::string *bytes, const char *what);

// bb_c_comp's table (misc._COMP_TABLE) into table[256], for every unit that complements on the device (bb_api.cu)
void bbl_comp_table(uint8_t *table);
// dst[dst_off[r] .. dst_off[r + 1]) = src[src_lo[r] ..] for r < n_ranges; total = dst_off[n_ranges] (device arrays;
// bb_tu_fasta.cu)
void bbl_fasta_gather(cudaStream_t st, const uint8_t *src, const int64_t *src_lo, const int64_t *dst_off, int32_t n_ranges,
                      int64_t total, uint8_t *dst);
// A gzip stream in host memory in[0..n) inflated on `st` into a new device allocation of *total bytes (at least 16
// allocated); the input goes through a device buffer of its own, released before the call returns.  Every member BGZF:
// one warp per member, else bbl_gzip_chunked in chunks of chunk_bytes (0: the default; bb_tu_gunzip.cu).  *stats as
// bb_gzip_decompress reports them.  Throws BB_ERR_ARG naming the member (index and offset) for a corrupt stream, as
// bb_gzip_decompress; BB_ERR_CUDA otherwise.  (bb_tu_inflate.cu)
DevBuf bbl_gzip_inflate_device(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, int64_t *total,
                               bb_gzip_stats *stats);
DevBuf bbl_gzip_chunked(cudaStream_t st, const uint8_t *in, int64_t n, int64_t chunk_bytes, int64_t *total, bb_gzip_stats *stats);
// An error model file's text[0..n) in device memory to its tables (bb_em_load.cuh; bb_tu_em_load.cu), in allocations of
// their own.  kmer_to_row[4^k] only when `dense` and k <= 12.  info->fallback set: nothing to install.  Throws
// BB_ERR_CAPACITY when the slot pool outgrows its limit, BB_ERR_CUDA for a CUDA failure.
struct BBEmLoadOut {
    DevBuf kmer_to_row, codes, row_off, cum, probs, flags, slots, pool, rowinfo;
};
void bbl_em_load(cudaStream_t st, const uint8_t *text, int64_t n, bool dense, bb_em_load_info *info, BBEmLoadOut *out);
#endif
