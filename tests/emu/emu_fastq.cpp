// emu_fastq.cpp — the FASTQ parser and the slice gather (badread_b200/csrc/bb_fastq.cuh) under the warp emulator, CTA by
// CTA, with the byte tile and the lines per thread as arguments so that tests can put tile edges anywhere (TEST
// INFRASTRUCTURE).  Built with fewer threads per CTA than the device (FQ_THREADS, FQ_SCAN_THREADS in emu_fastq.py) to
// keep the emulator fast and to have each thread of the scan CTAs take several tiles; the code paths are the same.
#include "cuda_emu.h"

#include <vector>

#include "../../badread_b200/csrc/bb_fastq.cuh"

namespace {
template <class F>
void grid(int64_t blocks, int threads, F &&f) {
    gridDim.x = (unsigned)blocks;
    for (int64_t b = 0; b < blocks; b++) {
        blockIdx.x = (unsigned)b;
        emu::run_block(threads, f);
    }
    gridDim.x = 1;
    blockIdx.x = 0;
}
}  // namespace

// The passes of bb_fastq_parse over text[0..n): recs[6 * r ..] the spans of record r (rec_cap records at most),
// *n_rec the records, *err the least (record << 1 | kind) of a failing record or -1.  -4 when rec_cap is too small.
extern "C" __attribute__((visibility("default")))
int emu_fastq_parse(const uint8_t *text, int64_t n, int32_t tile, int32_t lpt, int64_t *recs, int64_t rec_cap, int64_t *n_rec,
                    int64_t *err) {
    if (tile < 1 || lpt < 1 || n < 1) return -2;
    std::vector<uint8_t> in(text, text + n);   // exact size: a read past the end would leave it
    const int64_t n_tiles = (n + tile - 1) / tile;
    std::vector<int64_t> counts((size_t)n_tiles + 1);
    grid(n_tiles, FQ_THREADS, [&]() { fq_k_count_nl(in.data(), n, tile, counts.data()); });
    grid(1, FQ_SCAN_THREADS, [&]() { fq_k_scan64(counts.data(), n_tiles, counts.data() + n_tiles); });
    const int64_t n_nl = counts[(size_t)n_tiles];
    std::vector<int64_t> nl((size_t)n_nl);
    grid(n_tiles, FQ_THREADS, [&]() { fq_k_emit_nl(in.data(), n, tile, counts.data(), nl.data()); });
    const int64_t n_lines = n_nl + (in[(size_t)n - 1] != '\n'), lt = (int64_t)FQ_THREADS * lpt, n_lt = (n_lines + lt - 1) / lt;
    std::vector<FqMap> maps((size_t)n_lt);
    std::vector<int32_t> state((size_t)n_lt);
    std::vector<int64_t> base((size_t)n_lt + 1);
    grid(n_lt, FQ_THREADS, [&]() { fq_k_line_maps(in.data(), nl.data(), n_nl, n, n_lines, lpt, maps.data()); });
    grid(1, FQ_SCAN_THREADS, [&]() { fq_k_scan_maps(maps.data(), n_lt, state.data(), base.data(), base.data() + n_lt); });
    *n_rec = base[(size_t)n_lt];
    if (*n_rec > rec_cap) return -4;
    std::vector<int64_t> rec_line((size_t)*n_rec);
    grid(n_lt, FQ_THREADS, [&]() { fq_k_records(in.data(), nl.data(), n_nl, n, n_lines, lpt, state.data(), base.data(), rec_line.data()); });
    std::vector<FastqRec> R((size_t)*n_rec);
    unsigned long long e = ~0ull;
    grid((*n_rec + FQ_THREADS - 1) / FQ_THREADS, FQ_THREADS,
         [&]() { fq_k_fields(in.data(), nl.data(), n_nl, n, n_lines, rec_line.data(), *n_rec, R.data(), &e); });
    for (int64_t r = 0; r < *n_rec; r++) {
        const FastqRec &x = R[(size_t)r];
        const int64_t v[6] = {x.name_lo, x.name_hi, x.seq_lo, x.seq_hi, x.qual_lo, x.qual_hi};
        std::copy(v, v + 6, recs + 6 * r);
    }
    *err = e == ~0ull ? -1 : (int64_t)e;
    return 0;
}

// bb_flat_build on the emulator: fq_plan, then fq_k_gather.  First call with read == nullptr: sizes[0..3) = read, ref and
// op counts (or the plan's failure in failed[]).  Second call: the arrays, and failed[] = (alignment, 3) for a read with a
// byte >= 0x80.  names / name_off: the records' names as bb_fastq_parse gathers them.
extern "C" __attribute__((visibility("default")))
int emu_fastq_flat(const uint8_t *text, int64_t n, const int64_t *recs, int64_t n_rec, const char *names, const int64_t *name_off,
                   const bb_aln_view *v, int32_t n_aln, const int64_t *records, const int64_t *contig_at, const int64_t *contig_len,
                   const uint8_t *contigs, int64_t contigs_len, const uint8_t *comp, int64_t *sizes, uint8_t *read, uint8_t *qual,
                   uint8_t *ref, uint32_t *ops, int32_t *p0, int32_t *r0, int64_t *read_off, int64_t *ref_off, int64_t *ops_off,
                   int64_t *failed) {
    FqPlan P;
    if (fq_plan(names, name_off, n_rec, v, n_aln, records, contig_at, contig_len, P, failed)) return -2;
    sizes[0] = P.read_off.back();
    sizes[1] = P.ref_off.back();
    sizes[2] = (int64_t)P.ops.size();
    if (!read) return 0;
    std::vector<uint8_t> in(text, text + n), ctg(contigs, contigs + contigs_len);
    std::vector<FastqRec> R((size_t)n_rec);
    for (int64_t r = 0; r < n_rec; r++) {
        const int64_t *x = recs + 6 * r;
        R[(size_t)r] = FastqRec{x[0], x[1], x[2], x[3], x[4], x[5]};
    }
    // exact sizes (a write past the end would leave them), filled with 0xa5 so that a byte the kernel skips shows
    std::vector<uint8_t> rd((size_t)sizes[0], 0xa5), ql((size_t)sizes[0], 0xa5), rf((size_t)sizes[1], 0xa5);
    unsigned long long bad = ~0ull;
    grid(n_aln, FQ_THREADS, [&]() {
        fq_k_gather(in.data(), R.data(), P.alns.data(), P.read_off.data(), P.ref_off.data(), ctg.data(), comp, rd.data(), ql.data(),
                    rf.data(), &bad);
    });
    if (bad != ~0ull) {
        failed[0] = (int64_t)bad;
        failed[1] = 3;
        return -2;
    }
    std::copy(rd.begin(), rd.end(), read);
    std::copy(ql.begin(), ql.end(), qual);
    std::copy(rf.begin(), rf.end(), ref);
    std::copy(P.ops.begin(), P.ops.end(), ops);
    std::copy(P.p0.begin(), P.p0.end(), p0);
    std::copy(P.r0.begin(), P.r0.end(), r0);
    std::copy(P.read_off.begin(), P.read_off.end(), read_off);
    std::copy(P.ref_off.begin(), P.ref_off.end(), ref_off);
    std::copy(P.ops_off.begin(), P.ops_off.end(), ops_off);
    return 0;
}
