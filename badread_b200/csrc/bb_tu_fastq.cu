// bb_tu_fastq.cu — compiles the FASTQ parser and the slice gather (bb_fastq.cuh) and their C ABI for the model builders'
// device route (include/badread_b200.h): bb_fastq_parse, bb_flat_build, bb_flat_view_get, bb_flat_fetch, bb_flat_free,
// bb_fastq_free, bb_device_count.  Like the other builder inputs they take a device instead of a context and report
// failures through bb_model_error(); every launch and copy is on the legacy default stream.
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../include/badread_b200.h"

#include "bb_call.h"
#include "bb_fastq.cuh"

struct bb_fastq_set {
    int device = 0;
    DevBuf text;                  // the (inflated) file, until bb_flat_build has gathered from it
    DevBuf recs;                  // FastqRec[n_rec]
    int64_t n_text = 0, n_rec = 0;
    std::string names;            // record r's name: names[name_off[r] .. name_off[r + 1])
    std::vector<int64_t> name_off;
};

struct bb_flat_set {
    int32_t n = 0;
    DevBuf read, qual, ref, ops, op_read0, op_ref0;
    std::vector<int64_t> read_off{0}, ref_off{0}, ops_off{0};
};

namespace {

unsigned grid(int64_t items, int64_t per) { return (unsigned)((items + per - 1) / per); }

void parse(bb_fastq_set &F) {
    Scratch S(BB_ERR_CAPACITY);
    const uint8_t *text = F.text.as<uint8_t>();
    const int64_t n = F.n_text, n_tiles = (n + FQ_TILE - 1) / FQ_TILE;
    // 1. the newlines
    int64_t *counts = S.get<int64_t>(n_tiles + 1, "the newline scan");
    if (n_tiles) fq_k_count_nl<<<(unsigned)n_tiles, FQ_THREADS>>>(text, n, FQ_TILE, counts);
    fq_k_scan64<<<1, FQ_SCAN_THREADS>>>(counts, n_tiles, counts + n_tiles);
    check(cudaGetLastError(), "fq_k_scan64");
    int64_t n_nl = 0;
    uint8_t last = '\n';
    d2h(&n_nl, counts + n_tiles, 1);
    d2h(&last, text + n - 1, 1);
    int64_t *nl = S.get<int64_t>(n_nl, "the newline positions");
    if (n_tiles) fq_k_emit_nl<<<(unsigned)n_tiles, FQ_THREADS>>>(text, n, FQ_TILE, counts, nl);
    // 2. the records' header lines
    const int64_t n_lines = n_nl + (last != '\n'), n_lt = (n_lines + FQ_THREADS * FQ_LINES_PER_THREAD - 1) / (FQ_THREADS * FQ_LINES_PER_THREAD);
    FqMap *maps = S.get<FqMap>(n_lt, "the line scan");
    int32_t *state = S.get<int32_t>(n_lt, "the line scan");
    int64_t *base = S.get<int64_t>(n_lt + 1, "the line scan");
    if (n_lt) fq_k_line_maps<<<(unsigned)n_lt, FQ_THREADS>>>(text, nl, n_nl, n, n_lines, FQ_LINES_PER_THREAD, maps);
    fq_k_scan_maps<<<1, FQ_SCAN_THREADS>>>(maps, n_lt, state, base, base + n_lt);
    check(cudaGetLastError(), "fq_k_scan_maps");
    int64_t n_rec = 0;
    d2h(&n_rec, base + n_lt, 1);
    if (n_rec > INT32_MAX) throw Fail{BB_ERR_ARG, "Error: the FASTQ holds more than 2^31 - 1 records"};
    int64_t *rec_line = S.get<int64_t>(n_rec, "the record table");
    if (n_lt) fq_k_records<<<(unsigned)n_lt, FQ_THREADS>>>(text, nl, n_nl, n, n_lines, FQ_LINES_PER_THREAD, state, base, rec_line);
    // 3. the spans
    F.recs = S.result((size_t)n_rec * sizeof(FastqRec), "the record table");
    F.n_rec = n_rec;
    FastqRec *recs = F.recs.as<FastqRec>();
    unsigned long long *err = S.get<unsigned long long>(1, "the record table");
    check(cudaMemset(err, 0xff, 8), "cudaMemset");
    if (n_rec) fq_k_fields<<<grid(n_rec, FQ_THREADS), FQ_THREADS>>>(text, nl, n_nl, n, n_lines, rec_line, n_rec, recs, err);
    check(cudaGetLastError(), "fq_k_fields");
    // the names
    std::vector<int64_t> spans((size_t)(2 * n_rec)), lo((size_t)n_rec), hi((size_t)n_rec);
    if (n_rec) check(cudaMemcpy2D(spans.data(), 16, recs, sizeof(FastqRec), 16, (size_t)n_rec, cudaMemcpyDeviceToHost), "cudaMemcpy2D");
    for (int64_t r = 0; r < n_rec; r++) {
        lo[(size_t)r] = spans[(size_t)(2 * r)];
        hi[(size_t)r] = spans[(size_t)(2 * r + 1)];
    }
    F.name_off = gather_spans(S, 0, text, lo, hi, &F.names, "the read names");
    unsigned long long e = 0;
    d2h(&e, err, 1);
    if (e != ~0ull) {
        const int64_t r = (int64_t)(e >> 1);
        const std::string name = F.names.substr((size_t)F.name_off[(size_t)r], (size_t)(F.name_off[(size_t)r + 1] - F.name_off[(size_t)r]));
        throw Fail{BB_ERR_ARG, (e & 1) ? "Error: FASTQ record " + std::to_string(r + 1) + " (" + name +
                                             ") is truncated: the file ends before its quality line"
                                       : "Error: FASTQ record " + std::to_string(r + 1) + " has no read name (its header is a lone '@')"};
    }
}

}  // namespace

extern "C" int bb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int bb_fastq_parse(int device, const uint8_t *data, int64_t n, int is_gzip, bb_fastq_set **out, int64_t *n_records,
                              int32_t *first_byte) {
    if (n < 0 || (n > 0 && !data) || !out || !n_records || !first_byte) return bad_argument("bb_fastq_parse");
    *out = nullptr;
    *n_records = 0;
    *first_byte = -1;
    return device_call(device, [&] {
        std::unique_ptr<bb_fastq_set> F(new bb_fastq_set());
        F->device = device;
        Scratch S(BB_ERR_CAPACITY);
        bb_gzip_stats stats{};
        try {
            F->text = text_to_device(S, 0, data, n, is_gzip, &F->n_text, &stats, "the FASTQ text");
        } catch (const Fail &f) {
            if (!is_gzip) throw;
            throw Fail{f.rc, "Error: the FASTQ could not be inflated (" + f.msg + ")"};
        }
        if (F->n_text) {
            uint8_t c = 0;
            d2h(&c, F->text.p, 1);
            *first_byte = c;
        }
        if (*first_byte == '@') parse(*F);
        *n_records = F->n_rec;
        *out = F.release();
        return BB_OK;
    });
}

extern "C" int bb_fastq_free(bb_fastq_set *F) {
    delete F;
    return BB_OK;
}

extern "C" int bb_flat_build(bb_fastq_set *F, const bb_aln_view *v, int32_t n_aln, const int64_t *records, const int64_t *contig_at,
                             const int64_t *contig_len, const uint8_t *contigs, int64_t contigs_len, bb_flat_set **out,
                             int64_t *failed, int64_t *slice_len) {
    if (!F || !v || n_aln < 0 || (n_aln && (!records || !contig_at || !contig_len)) || contigs_len < 0 ||
        (contigs_len && !contigs) || !out || !failed || (n_aln && !F->text.p))
        return bad_argument("bb_flat_build");
    *out = nullptr;
    return model_call([&] {
        FqPlan P;
        const int kind = fq_plan(F->names.data(), F->name_off.data(), F->n_rec, v, n_aln, records, contig_at, contig_len, P, failed);
        if (kind == 4) {
            const int32_t id = v->read_id[records[failed[0]]];
            failed[0] = -1;
            failed[1] = 0;
            throw Fail{BB_ERR_ARG, "Error: the CIGAR of read " +
                                       std::string(v->read_names + v->read_name_off[id], (size_t)(v->read_name_off[id + 1] - v->read_name_off[id])) +
                                       " spans more than 2^31 - 1 bases"};
        }
        if (kind) return BB_ERR_ARG;
        const std::vector<FastqAln> &alns = P.alns;
        std::unique_ptr<bb_flat_set> flat(new bb_flat_set());
        flat->read_off = P.read_off;
        flat->ref_off = P.ref_off;
        flat->ops_off = P.ops_off;
        flat->n = n_aln;
        const int64_t n_read = flat->read_off.back(), n_ref = flat->ref_off.back(), n_ops = (int64_t)P.ops.size();
        use_device(F->device);
        Scratch S(BB_ERR_CAPACITY);
        flat->read = S.result((size_t)n_read, "the aligned read slices");
        flat->qual = S.result((size_t)n_read, "the aligned quality slices");
        flat->ref = S.result((size_t)n_ref, "the aligned reference slices");
        flat->ops = S.result((size_t)n_ops * 4, "the CIGAR runs");
        flat->op_read0 = S.result((size_t)n_ops * 4, "the CIGAR runs");
        flat->op_ref0 = S.result((size_t)n_ops * 4, "the CIGAR runs");
        if (n_ops) {
            check(cudaMemcpy(flat->ops.p, P.ops.data(), (size_t)n_ops * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
            check(cudaMemcpy(flat->op_read0.p, P.p0.data(), (size_t)n_ops * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
            check(cudaMemcpy(flat->op_ref0.p, P.r0.data(), (size_t)n_ops * 4, cudaMemcpyHostToDevice), "cudaMemcpy");
        }
        if (slice_len && n_aln) {   // (the records' spans: the slices' lengths before fq_k_gather pads or truncates them)
            std::vector<FastqRec> recs((size_t)F->n_rec);
            d2h(recs.data(), F->recs.p, F->n_rec);
            for (int32_t i = 0; i < n_aln; i++) {
                const FastqAln &A = alns[(size_t)i];
                const FastqRec &R = recs[(size_t)A.rec];
                int64_t lo;
                slice_len[3 * (int64_t)i] = fq_slice(R.seq_hi - R.seq_lo, A.read_start, A.read_end, &lo);
                slice_len[3 * (int64_t)i + 1] = fq_slice(R.qual_hi - R.qual_lo, A.read_start, A.read_end, &lo);
                slice_len[3 * (int64_t)i + 2] = fq_slice(A.contig_len, A.ref_start, A.ref_end, &lo);
            }
        }
        const FastqAln *d_alns = S.upload(alns.data(), n_aln, "the alignment descriptors");
        const int64_t *d_read_off = S.upload(flat->read_off.data(), n_aln + 1, "the alignment descriptors");
        const int64_t *d_ref_off = S.upload(flat->ref_off.data(), n_aln + 1, "the alignment descriptors");
        const uint8_t *d_contigs = S.upload(contigs, contigs_len, "the reference contigs");
        uint8_t comp[256];
        bbl_comp_table(comp);
        const uint8_t *d_comp = S.upload(comp, 256, "the reference contigs");
        unsigned long long *bad = S.get<unsigned long long>(1, "the alignment descriptors");
        check(cudaMemset(bad, 0xff, 8), "cudaMemset");
        if (n_aln)
            fq_k_gather<<<(unsigned)n_aln, FQ_THREADS>>>(F->text.as<uint8_t>(), F->recs.as<FastqRec>(), d_alns, d_read_off, d_ref_off,
                                                        d_contigs, d_comp, flat->read.as<uint8_t>(), flat->qual.as<uint8_t>(),
                                                        flat->ref.as<uint8_t>(), bad);
        check(cudaGetLastError(), "fq_k_gather");
        unsigned long long b = 0;
        d2h(&b, bad, 1);
        if (b != ~0ull) {
            failed[0] = (int64_t)b;
            failed[1] = 3;
            return BB_ERR_ARG;
        }
        F->text.release();   // (the text and the record table are no longer needed)
        F->recs.release();
        *out = flat.release();
        return BB_OK;
    });
}

extern "C" int bb_flat_view_get(const bb_flat_set *S, bb_flat_view *v) {
    if (!S || !v) return BB_ERR_ARG;
    v->n = S->n;
    v->read = S->read.as<uint8_t>();
    v->qual = S->qual.as<uint8_t>();
    v->ref = S->ref.as<uint8_t>();
    v->ops = S->ops.as<uint32_t>();
    v->op_read0 = S->op_read0.as<int32_t>();
    v->op_ref0 = S->op_ref0.as<int32_t>();
    v->read_off = S->read_off.data();
    v->ref_off = S->ref_off.data();
    v->ops_off = S->ops_off.data();
    return BB_OK;
}

extern "C" int bb_flat_fetch(const bb_flat_set *S, int which, int64_t lo, int64_t count, void *dst) {
    if (!S || which < 0 || which > 5 || lo < 0 || count < 0 || (count && !dst)) return bad_argument("bb_flat_fetch");
    return model_call([&] {
        const DevBuf *src[6] = {&S->read, &S->qual, &S->ref, &S->ops, &S->op_read0, &S->op_ref0};
        const int64_t size = which < 3 ? 1 : 4;
        const int64_t total = which < 2 ? S->read_off.back() : which == 2 ? S->ref_off.back() : S->ops_off.back();
        if (lo + count > total) throw Fail{BB_ERR_ARG, "bb_flat_fetch: range out of bounds"};
        if (count) check(cudaMemcpy(dst, src[which]->as<uint8_t>() + lo * size, (size_t)(count * size), cudaMemcpyDeviceToHost), "bb_flat_fetch");
        return BB_OK;
    });
}

extern "C" int bb_flat_free(bb_flat_set *S) {
    delete S;
    return BB_OK;
}
