// bb_call.cu — the message of bb_model_error(), the scratch allocations of the entry points and the input paths' shared
// steps (bb_call.h).  Host code only.
#include "bb_call.h"

namespace {
thread_local std::string g_model_error;
}  // namespace

void bbm_set_error(const std::string &msg) { g_model_error = msg; }

extern "C" const char *bb_model_error(void) { return g_model_error.c_str(); }

DevBuf Scratch::result(size_t bytes, const char *what) const {
    DevBuf b;
    bytes = std::max<size_t>(bytes, 16);
    const cudaError_t e = b.alloc(bytes);
    if (e == cudaSuccess) return b;
    (void)cudaGetLastError();
    if (e == cudaErrorMemoryAllocation && oom_rc_ == BB_ERR_CAPACITY)
        throw Fail{BB_ERR_CAPACITY, std::string("Error: not enough device memory for ") + what + " (" + std::to_string(bytes) +
                                        " bytes asked for)"};
    check(e, what);
    return b;
}

DevBuf text_to_device(Scratch &S, cudaStream_t st, const uint8_t *data, int64_t n, bool gzip, int64_t *len,
                      bb_gzip_stats *stats, const char *what) {
    if (gzip) return bbl_gzip_inflate_device(st, data, n, 0, len, stats);
    DevBuf text = S.result((size_t)n, what);
    if (n) check(cudaMemcpyAsync(text.p, data, (size_t)n, cudaMemcpyHostToDevice, st), "cudaMemcpy");
    *len = n;
    return text;
}

std::vector<int64_t> gather_spans(Scratch &S, cudaStream_t st, const uint8_t *text, const std::vector<int64_t> &lo,
                                  const std::vector<int64_t> &hi, std::string *bytes, const char *what) {
    const int64_t n = (int64_t)lo.size();
    std::vector<int64_t> lo_off((size_t)(2 * n + 1));   // bbl_fasta_gather's src_lo, then dst_off
    for (int64_t i = 0; i < n; i++) {
        lo_off[(size_t)i] = lo[(size_t)i];
        lo_off[(size_t)(n + i + 1)] = lo_off[(size_t)(n + i)] + hi[(size_t)i] - lo[(size_t)i];
    }
    const int64_t total = lo_off[(size_t)(2 * n)];
    bytes->resize((size_t)total);
    if (total) {
        const int64_t *idx = S.upload(lo_off.data(), (int64_t)lo_off.size(), what, st);
        uint8_t *d = S.get<uint8_t>(total, what);
        bbl_fasta_gather(st, text, idx, idx + n, (int32_t)n, total, d);
        check(cudaGetLastError(), "bbl_fasta_gather");
        d2h(&(*bytes)[0], d, total, st);
    }
    return std::vector<int64_t>(lo_off.begin() + n, lo_off.end());
}
