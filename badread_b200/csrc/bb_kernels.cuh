// bb_kernels.cuh — the per-read hot path as sm_90a kernels.
//
//   K1 bb_k_build_fragments   gather fragments from the HBM-resident reference / literal pool, draw the 2k pad
//                             bases (simulate.py:260), reset slot states
//   K2 bb_k_error_loop        simulate.sequence_fragment's while-loop (simulate.py:272-346): one warp per read,
//                             32 loop iterations evaluated speculatively per step (one Philox stream per
//                             iteration), changes committed in order, identity re-measured every 25 changes by
//                             the warp aligner (bb_align.cuh)
//   K3 bb_k_join              ''.join(new_fragment_bases) (simulate.py:351)
//   K4 bb_k_final_align       edlib.align(seq, fragment) of get_qscores (qscore_model.py:37) -> per-base ops
//   K5 bb_k_qscores           per-base CIGAR window -> QScoreModel.get_qscore (qscore_model.py:54-68,273-287)
//   K6 bb_k_compact           seq[start_trim:-end_trim], qual likewise (simulate.py:355-356)
#pragma once
#include <cstdint>
#include <type_traits>

#include "../../include/badread_b200.h"
#include "bb_align.cuh"
#include "bb_em_tables.h"
#include "bb_lane.cuh"
#include "bb_qscore_tables.h"
#include "bb_rng.cuh"

#define BB_SLOT_NONE 0xFFFFFFFFu
#define BB_ALIGNMENT_INTERVAL 25  // settings.py:24
#define BB_ALIGNMENT_SIZE 1000    // settings.py:25
#define BB_WARPS_PER_CTA 4
enum { BB_READ_PENDING = 0, BB_READ_DONE = 1 };  // BBReadDev::status: the error loop of the read has finished

// Everything the common outcome of a model draw needs, in one 32-byte record per table row: random.choices picks
// entry 0 - the unchanged k-mer, p ~ 0.92 (nanopore) ... 0.99 (pacbio) - iff random() * cum_last < cum0.
struct __align__(32) BBRowInfo {
    double cum_last;   // cum[e0 + ne - 1]
    double cum0;       // cum[e0]
    int32_t e0, ne;    // entry range of the row
    int32_t first_is_identity;  // flags[e0] == 1: ''.join(alt) == kmer and not the remainder entry
    int32_t pad;
};

struct BBErrorModelDev {
    int k, type;
    const int32_t *kmer_to_row;
    const int32_t *row_off;
    const double *cum;
    const uint8_t *flags;
    const uint32_t *slots;
    const uint8_t *pool;
    const BBRowInfo *rowinfo;
};

struct BBQScoreModelDev {  // layout: bb_qscore_tables.h
    int kmer_size;
    const uint64_t *hkeys;  // open addressing, 0 = empty
    const int32_t *hvals;
    uint32_t hbits;
    const int32_t *row_off;
    const uint8_t *scores;
    const double *cum;
    // keys longer than 31 symbols
    int long_max_len;             // symbols of the longest one, 0 = none
    uint32_t lbits;
    const BBQLongKey *lkeys;      // open addressing, len 0 = empty
    const uint64_t *lpool;        // their symbols, 32 per word
};

struct BBReadDev {
    long long frag_off;  // into frag / state
    long long seq_off;   // into seq / ops / dcnt / qual
    long long out_off;   // into out_seq / out_qual
    long long fpeq_off;  // into fpeq (match bitmap of the padded fragment), uint4 units
    long long speq_off;  // into speq (match bitmap of the untrimmed read)
    int frag_len;        // padded (2k pad bases included)
    int seq_len;         // untrimmed
    int start_trim, end_trim;
    int upper;           // upper bound on the edit distance seq <-> fragment (injected edits)
    int loop_count, change_count, n_align;
    int matches, dels, lead_del;
    int out_len;
    int flags;
    int kc_loop, kc_align;  // kilo-cycles this read spent in the error loop / final alignment (diagnostics)
    // speculative error loop (bb_loop.cuh)
    long long log_off;   // into chlog (change log), entries
    long long wres_off;  // into wres (window alignment results), entries
    int horizon;         // changes the mutate kernel may log before pausing
    int n_logged;        // changes logged so far
    int n_resume;        // next loop iteration to evaluate
    int stop_reason;     // why the mutate kernel stopped (BB_STOP_*)
    int a_done;          // window alignments already computed
    int status;          // BB_READ_*
};

struct BBBatchDev {
    int n_reads;
    const unsigned long long *read_index;
    const int *seg_off;
    const bb_segment *segs;
    const uint8_t *lit;
    const double *target;
    const int *order;  // reads sorted by decreasing fragment length (work queue order)
    BBReadDev *reads;
    uint8_t *frag;
    uint32_t *state;
    uint8_t *seq;
    uint8_t *ops;
    unsigned int *dcnt;
    uint8_t *qual;
    uint8_t *out_seq, *out_qual;
    uint4 *fpeq, *speq;
    int *kidx;             // per fragment position: table row of the k-mer that starts there (-1: not in the model)
    unsigned int *ctime;   // per slot: ordinal of the change that rewrote it (0 = pristine)
    uint2 *chlog;          // per read: (iteration, position) of every applied change, in order
    int2 *wres;            // per read: (matches, columns) of every window alignment
};

struct BBScratchPool {
    uint2 *hist; long long hist_stride; int hist_cap;
    int8_t *hbuf; long long hbuf_stride; int hbuf_cap;
    int *lr; long long lr_stride; int lr_cap;  // L at [0, lr_cap), R at [lr_cap, 2*lr_cap)
    int *stack; int stack_cap;
    uint8_t *tbuf; long long tbuf_stride;
    uint4 *peq; long long peq_stride; int peq_cap;
    __device__ BBScratch for_warp(int w) const {
        BBScratch s;
        s.hist = hist + (long long)w * hist_stride; s.hist_cap = hist_cap;
        s.hbuf = hbuf + (long long)w * hbuf_stride; s.hbuf_cap = hbuf_cap;
        s.L = lr + (long long)w * lr_stride; s.R = s.L + lr_cap; s.lr_cap = lr_cap;
        s.stack = stack + (long long)w * stack_cap * 5; s.stack_cap = stack_cap;
        s.peq = peq + (long long)w * peq_stride; s.peq_cap = peq_cap;
        return s;
    }
};

__constant__ uint8_t bb_c_comp[256];  // misc.REV_COMP_DICT, unknown -> 'N' (misc.py:56-67)

// ------------------------------------------------------------------------------------------------ K1
// The k-mer index is the dense kmer_to_row[4^k] (k <= 12), or with HASH the open-addressing table `hash` of
// bb_em_tables.h (any k up to 16); either one null: no index (the random model).
template <int BB_TU_ = 0, bool HASH = false>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_build_fragments(BBBatchDev B, const uint8_t *__restrict__ ref, int k,
                                                            unsigned long long seed, const int32_t *__restrict__ kmer_to_row,
                                                            BBEmHashDev hash = BBEmHashDev{nullptr, 0}) {
    const int r = blockIdx.x;
    if (r >= B.n_reads) return;
    const BBReadDev rd = B.reads[r];
    uint8_t *f = B.frag + rd.frag_off;
    uint32_t *st = B.state + rd.frag_off;
    const int flen = rd.frag_len;
    if (threadIdx.x == 0) {
        BBRng rng;
        rng.init(seed, B.read_index[r]);
        rng.stream(BB_PURPOSE_PAD, 0);
        for (int j = 0; j < k; j++) f[j] = rng.random_base();
        for (int j = 0; j < k; j++) f[flen - k + j] = rng.random_base();
    }
    int pos = k;
    for (int s = B.seg_off[r]; s < B.seg_off[r + 1]; s++) {
        const bb_segment sg = B.segs[s];
        if (sg.kind == BB_SEG_REF_FWD) {
            const uint8_t *src = ref + sg.src;
            for (int x = threadIdx.x; x < sg.len; x += blockDim.x) f[pos + x] = __ldg(src + x);
        } else if (sg.kind == BB_SEG_REF_REV) {
            const uint8_t *src = ref + sg.src + sg.len - 1;
            for (int x = threadIdx.x; x < sg.len; x += blockDim.x) f[pos + x] = bb_c_comp[__ldg(src - x)];
        } else {
            const uint8_t *src = B.lit + sg.src;
            for (int x = threadIdx.x; x < sg.len; x += blockDim.x) f[pos + x] = __ldg(src + x);
        }
        pos += sg.len;
    }
    unsigned int *ct = B.ctime + rd.frag_off;
    for (int x = threadIdx.x; x < flen; x += blockDim.x) { st[x] = BB_SLOT_NONE; ct[x] = 0u; }
    // match bitmap of the padded fragment (bb_build_peq layout), one ballot group per 32 bases
    __syncthreads();
    if (HASH ? hash.entries != nullptr : kmer_to_row != nullptr) {  // table row of every k-mer of the fragment: the
        int *kx = B.kidx + rd.frag_off;                               // loop looks a position up with one load
        for (int x = threadIdx.x; x + k <= flen; x += blockDim.x) {
            typename std::conditional<HASH, uint32_t, int>::type idx = 0;   // (a 16-mer's code needs all 32 bits)
            bool ok = true;
            for (int j = 0; j < k; j++) {
                const uint8_t c = f[x + j];
                const int code = c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
                if (code < 0) ok = false;
                idx = idx * 4 + (code & 3);
            }
            if (HASH) kx[x] = ok ? bb_em_find(hash.entries, hash.bits, (uint32_t)idx) : -1;
            else kx[x] = ok ? kmer_to_row[idx] : -1;
        }
    }
    uint4 *pq = B.fpeq + rd.fpeq_off;
    const int lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int fw = (flen + 31) >> 5;
    for (int w = threadIdx.x; w < BB_PEQ_PAD; w += blockDim.x) {
        pq[w] = make_uint4(0u, 0u, 0u, 0u);
        pq[BB_PEQ_PAD + fw + w] = make_uint4(0u, 0u, 0u, 0u);
    }
    for (int w = threadIdx.x >> 5; w < fw; w += nwarps) {
        const int row = 32 * w + lane;
        const uint8_t c = row < flen ? f[row] : 0;
        const uint32_t mA = __ballot_sync(BB_FULL, c == 'A'), mC = __ballot_sync(BB_FULL, c == 'C');
        const uint32_t mG = __ballot_sync(BB_FULL, c == 'G'), mT = __ballot_sync(BB_FULL, c == 'T');
        if (lane == 0) pq[BB_PEQ_PAD + w] = make_uint4(mA, mC, mG, mT);
    }
}

// ------------------------------------------------------------------------------------------------ K2
__device__ __forceinline__ int bb_base_code(uint8_t c) {
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}
__device__ __forceinline__ uint32_t bb_slot_inline(int len, uint8_t c0, uint8_t c1) {
    return (uint32_t)len | ((uint32_t)c0 << 8) | ((uint32_t)c1 << 16);
}
__device__ __forceinline__ uint8_t bb_slot_char(const BBErrorModelDev &em, uint32_t enc, int idx) {
    const int len = enc & 0xff;
    if (len <= 3) return (uint8_t)(enc >> (8 * (idx + 1)));
    return em.pool[(enc >> 8) + idx];
}

// ''.join(new_fragment_bases[lo:lo+count]) into out (warp-cooperative). Returns the joined length; *upper gets
// the number of edits that turn the original slice into the joined one (an upper bound on their edit distance).
static __device__ int bb_join_slots(const BBErrorModelDev &em, const uint8_t *frag, const uint32_t *state, int lo, int count,
                             uint8_t *out, int *upper) {
    const int lane = threadIdx.x & 31;
    int total = 0, up = 0;
    for (int base = 0; base < count; base += 32) {
        const int x = base + lane;
        uint32_t st = BB_SLOT_NONE;
        int len = 0;
        if (x < count) { st = state[lo + x]; len = st == BB_SLOT_NONE ? 1 : (int)(st & 0xff); }
        int incl = len;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(BB_FULL, incl, d);
            if (lane >= d) incl += v;
        }
        const int off = total + incl - len;
        if (x < count) {
            if (st == BB_SLOT_NONE) out[off] = frag[lo + x];
            else {
                for (int c = 0; c < len; c++) out[off + c] = bb_slot_char(em, st, c);
                up += len < 1 ? 1 : len;
            }
        }
        total += __shfl_sync(BB_FULL, incl, 31);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) up += __shfl_xor_sync(BB_FULL, up, d);
    *upper = up;
    __syncwarp();
    return total;
}

// One speculative evaluation of simulate.py:294-296 for loop iteration n: position, k-mer, model draw.
// kind 0: ''.join(new_kmer) == kmer (nothing to do); 1: table entry `payload`; 2: one random change where
// slot `rpos` becomes the inline-encoded string `payload` (error_model.py:163-176).
__device__ __forceinline__ void bb_eval_iteration(const BBErrorModelDev &em, const uint8_t *frag, const int *kidx,
                                                  int max_kmer_index, unsigned long long seed, unsigned long long read,
                                                  unsigned int n, int &kind, int &pos_i, uint32_t &payload,
                                                  int &rpos) {
    BBRng rng;
    rng.init(seed, read);
    rng.stream(BB_PURPOSE_LOOP, n);
    const int k = em.k;
    const int i = (int)rng.randbelow((uint32_t)(max_kmer_index + 1));  // random.randint(0, max_kmer_index)
    pos_i = i;
    bool random_change = (em.type == 0);
    if (!random_change) {
        const int row = kidx[i];  // kmer -> row, -1: not in self.alternatives (error_model.py:143-144) or non-ACGT
        if (row < 0) random_change = true;
        else {
            const BBRowInfo ri = em.rowinfo[row];
            // random.choices: bisect_right(cum, random() * cum[-1]); entry 0 answers whenever the product is below cum[0]
            const double x = __dmul_rn(rng.random(), ri.cum_last);
            int e = ri.e0;
            uint8_t fl;
            if (x < ri.cum0) fl = ri.first_is_identity ? 1 : em.flags[e];
            else {
                const double *cum = em.cum + ri.e0;
                int lo = 1, hi = ri.ne - 1;
                if (lo > hi) lo = hi;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (x < cum[mid]) hi = mid; else lo = mid + 1;
                }
                e += lo;
                fl = em.flags[e];
            }
            if (fl & 2) random_change = true;  // alt is None (error_model.py:157-158)
            else { kind = (fl & 1) ? 0 : 1; payload = (uint32_t)e; rpos = 0; return; }
        }
    }
    // add_one_random_change
    const uint32_t type = rng.randbelow(3);          // random.choice(['s','i','d'])
    const int p = (int)rng.randbelow((uint32_t)k);   // random.randint(0, len(kmer)-1)
    const uint8_t old = frag[i + p];
    if (type == 0) payload = bb_slot_inline(1, rng.random_different_base(old), 0);
    else if (type == 1) {
        if (rng.random() < 0.5) { const uint8_t nb = rng.random_base(); payload = bb_slot_inline(2, old, nb); }
        else { const uint8_t nb = rng.random_base(); payload = bb_slot_inline(2, nb, old); }
    } else payload = bb_slot_inline(0, 0, 0);
    kind = 2; rpos = p;
}

// ------------------------------------------------------------------------------------------------ scan
// Offsets of the per-read regions in seq / ops / dcnt / qual (16-byte aligned), the match bitmaps of the joined reads
// and the packed outputs: three exclusive prefix sums over the reads in batch order, by one CTA (a few ten thousand
// reads).  A read whose regions do not fit the buffers (sized from the fragment lengths before the run) is flagged
// BB_FLAG_NOSPACE and left empty; the host grows the buffers and runs the batch again.
#define BB_FLAG_NOSPACE 0x40000000
struct BBScanOut {
    long long seq_total, out_total, speq_total;
    int n_nospace, max_seq_len, max_upper, n_pending;
};

template <int BB_TU_ = 0>
__global__ void __launch_bounds__(1024)
bb_k_scan(BBBatchDev B, int n, long long seq_cap, long long out_cap, long long speq_cap, BBScanOut *out) {
    __shared__ long long s_w[3][32];
    __shared__ long long s_run[3];
    __shared__ int s_bad, s_maxlen, s_maxup, s_pend;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_run[0] = s_run[1] = s_run[2] = 0; s_bad = 0; s_maxlen = 0; s_maxup = 0; s_pend = 0; }
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int r = base + threadIdx.x;
        long long v[3] = {0, 0, 0};
        int out_len = 0, seq_len = 0;
        bool pending = false;  // the error loop of this read has not finished (too few rounds enqueued): skipped like a
                               // read without room, the host runs the batch again with more rounds
        if (r < n && B.reads[r].status != BB_READ_DONE) pending = true;
        if (r < n && !pending) {
            const BBReadDev &rd = B.reads[r];
            seq_len = rd.seq_len;
            out_len = seq_len - rd.start_trim - rd.end_trim;  // seq[start_trim:-end_trim]
            if (out_len < 0) out_len = 0;
            v[0] = (seq_len + 15) & ~15; v[1] = out_len; v[2] = bb_peq_words(seq_len);
        }
        long long incl[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            long long x = v[c];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const long long y = __shfl_up_sync(BB_FULL, x, d);
                if (lane >= d) x += y;
            }
            incl[c] = x;
            if (lane == 31) s_w[c][wid] = x;
        }
        __syncthreads();
        if (wid == 0) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                long long x = s_w[c][lane];
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const long long y = __shfl_up_sync(BB_FULL, x, d);
                    if (lane >= d) x += y;
                }
                s_w[c][lane] = x;  // inclusive over warps
            }
        }
        __syncthreads();
        long long off[3];
#pragma unroll
        for (int c = 0; c < 3; c++) off[c] = s_run[c] + (wid ? s_w[c][wid - 1] : 0) + incl[c] - v[c];
        if (r < n) {
            BBReadDev &rd = B.reads[r];
            const bool fits = !pending && off[0] + v[0] <= seq_cap && off[1] + v[1] <= out_cap && off[2] + v[2] <= speq_cap;
            rd.seq_off = fits ? off[0] : 0; rd.out_off = fits ? off[1] : 0; rd.speq_off = fits ? off[2] : 0;
            rd.out_len = fits ? out_len : 0;
            rd.lead_del = 0; rd.matches = 0; rd.dels = 0;
            if (!fits) { rd.flags |= BB_FLAG_NOSPACE; atomicAdd(pending ? &s_pend : &s_bad, 1); }
            if (pending) { rd.seq_len = 0; rd.start_trim = 0; rd.end_trim = 0; }
            atomicMax(&s_maxlen, seq_len);
            atomicMax(&s_maxup, rd.upper);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll
            for (int c = 0; c < 3; c++) s_run[c] += s_w[c][31];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out->seq_total = s_run[0]; out->out_total = s_run[1]; out->speq_total = s_run[2];
        out->n_nospace = s_bad; out->max_seq_len = s_maxlen; out->max_upper = s_maxup; out->n_pending = s_pend;
    }
}

// ------------------------------------------------------------------------------------------------ K3
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_join(BBBatchDev B, BBErrorModelDev em) {
    const int r = blockIdx.x;
    if (r >= B.n_reads) return;
    const BBReadDev rd = B.reads[r];
    if (rd.flags & BB_FLAG_NOSPACE) return;
    const uint8_t *frag = B.frag + rd.frag_off;
    const uint32_t *state = B.state + rd.frag_off;
    uint8_t *seq = B.seq + rd.seq_off;
    __shared__ int warp_sum[8];
    __shared__ int running;
    if (threadIdx.x == 0) running = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int cost = 0;  // sum of the exact edit distances base -> slot string: a tighter bound than the loop's count
    for (int base = 0; base < rd.frag_len; base += 256) {
        const int x = base + threadIdx.x;
        uint32_t st = BB_SLOT_NONE;
        int len = 0;
        if (x < rd.frag_len) { st = state[x]; len = st == BB_SLOT_NONE ? 1 : (int)(st & 0xff); }
        int incl = len;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(BB_FULL, incl, d);
            if (lane >= d) incl += v;
        }
        if (lane == 31) warp_sum[wid] = incl;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < wid; w++) woff += warp_sum[w];
        const int off = running + woff + incl - len;
        if (x < rd.frag_len) {
            if (st == BB_SLOT_NONE) seq[off] = frag[x];
            else {
                const uint8_t orig = frag[x];
                int kept = 0;  // the original base survives inside the slot string: the rest are insertions
                for (int c = 0; c < len; c++) {
                    const uint8_t ch = bb_slot_char(em, st, c);
                    seq[off + c] = ch;
                    kept |= (ch == orig) ? 1 : 0;
                }
                cost += len == 0 ? 1 : len - kept;
            }
        }
        __syncthreads();
        if (threadIdx.x == 255) running = off + len;
        __syncthreads();
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cost += __shfl_xor_sync(BB_FULL, cost, d);
    if (lane == 0) warp_sum[wid] = cost;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tight = 0;
        for (int w = 0; w < 8; w++) tight += warp_sum[w];
        if (tight < rd.upper) B.reads[r].upper = tight;
    }
    uint4 *pq = B.speq + rd.speq_off;
    const int nwarps = blockDim.x >> 5;
    const int sw = (rd.seq_len + 31) >> 5;
    for (int w = threadIdx.x; w < BB_PEQ_PAD; w += blockDim.x) {
        pq[w] = make_uint4(0u, 0u, 0u, 0u);
        pq[BB_PEQ_PAD + sw + w] = make_uint4(0u, 0u, 0u, 0u);
    }
    for (int w = wid; w < sw; w += nwarps) {
        const int row = 32 * w + lane;
        const uint8_t c = row < rd.seq_len ? seq[row] : 0;
        const uint32_t mA = __ballot_sync(BB_FULL, c == 'A'), mC = __ballot_sync(BB_FULL, c == 'C');
        const uint32_t mG = __ballot_sync(BB_FULL, c == 'G'), mT = __ballot_sync(BB_FULL, c == 'T');
        if (lane == 0) pq[BB_PEQ_PAD + w] = make_uint4(mA, mC, mG, mT);
    }
}

// ------------------------------------------------------------------------------------------------ K5
__device__ __forceinline__ int bb_qm_find(const BBQScoreModelDev &qm, unsigned long long key) {
    const uint32_t mask = (1u << qm.hbits) - 1u;
    uint32_t h = bb_qm_slot(key, qm.hbits);
    for (;;) {
        const unsigned long long kk = qm.hkeys[h];
        if (kk == key) return qm.hvals[h];
        if (kk == 0ull) return -1;
        h = (h + 1) & mask;
    }
}

// Row of the window [s, e] (ops[s] D^dcnt[s] ops[s+1] ... ops[e]) among the keys of more than 31 symbols, -1 if it
// is none of them.  The walk hashes the symbols as it emits them and stops as soon as the window outgrows the longest
// such key, so a huge dcnt costs one comparison.  A hash hit is confirmed by walking the window again against the
// pooled symbols.
__device__ inline int bb_qm_find_long(const BBQScoreModelDev &qm, const uint8_t *ops, const unsigned int *dcnt, int s, int e) {
    const int bound = qm.long_max_len;
    unsigned long long h = BB_QM_LONG_HASH_INIT;
    int len = 0;
    for (int x = s; x <= e; x++) {
        if (len >= bound) return -1;
        h = bb_qm_long_hash(h, ops[x]);
        len++;
        if (x < e) {
            const unsigned int d = dcnt[x];
            if (d > (unsigned int)(bound - len)) return -1;
            for (unsigned int c = 0; c < d; c++) h = bb_qm_long_hash(h, 3u);
            len += (int)d;
        }
    }
    const uint32_t mask = (1u << qm.lbits) - 1u;
    for (uint32_t slot = bb_qm_slot(h, qm.lbits);; slot = (slot + 1) & mask) {
        const BBQLongKey k = qm.lkeys[slot];
        if (k.len == 0) return -1;
        if (k.len != len || k.hash != h) continue;
        const uint64_t *w = qm.lpool + k.off;
        bool same = true;
        int j = 0;
        for (int x = s; x <= e && same; x++) {
            same = ((w[j >> 5] >> (2 * (j & 31))) & 3u) == ops[x];
            j++;
            if (x < e)
                for (unsigned int c = 0; c < dcnt[x] && same; c++, j++) same = ((w[j >> 5] >> (2 * (j & 31))) & 3u) == 3u;
        }
        if (same) return k.row;
    }
}

// qscore for base i of a read of n bases given per-base ops and deletion counts (qscore_model.py:54-68 and
// QScoreModel.get_qscore :273-287).  partial_cigar = ops[s] D^dcnt[s] ops[s+1] ... ops[e]; a CIGAR that is
// not in the model loses its first and last symbol and then its outer D's, which is exactly the window
// [s+1, e-1] of the same form.  A window of up to 31 symbols is packed into one key of the uint64 table; a longer one
// goes to the side table (bb_qm_find_long) when the model has long keys.
__device__ __forceinline__ uint8_t bb_qscore_base(const BBQScoreModelDev &qm, const uint8_t *ops, const unsigned int *dcnt,
                                                  int n, int i, unsigned long long seed, unsigned long long read) {
    int mm = (qm.kmer_size - 1) / 2;
    if (mm > i) mm = i;
    if (mm > n - 1 - i) mm = n - 1 - i;
    int row = -1;
    for (; mm >= 0 && row < 0; mm--) {
        const int s = i - mm, e = i + mm;
        unsigned long long key = 1ull;
        int len = 0;
        bool ok = true;
        for (int x = s; x <= e && ok; x++) {
            key = (key << 2) | ops[x];
            len++;
            if (x < e) {
                const unsigned int d = dcnt[x];
                if (d > 31u || len + (int)d > 31) ok = false;
                else { for (unsigned int c = 0; c < d; c++) key = (key << 2) | 3ull; len += (int)d; }
            }
        }
        if (ok && len <= 31) row = bb_qm_find(qm, key);
        else if (qm.long_max_len > 0) row = bb_qm_find_long(qm, ops, dcnt, s, e);
    }
    if (row < 0) return 0;  // cannot happen: '=', 'X', 'I' are asserted at model load (qscore_model.py:205-207)
    const int e0 = qm.row_off[row], ne = qm.row_off[row + 1] - e0;
    BBRng rng;
    rng.init(seed, read);
    rng.stream(BB_PURPOSE_QSCORE, (uint32_t)i);
    const int pick = bb_choices(rng, qm.cum + e0, ne);
    return (uint8_t)(qm.scores[e0 + pick] + 33);
}

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_qscores(BBBatchDev B, BBQScoreModelDev qm, unsigned long long seed) {
    const int r = blockIdx.x;
    const BBReadDev rd = B.reads[r];
    if (rd.flags & BB_FLAG_NOSPACE) return;
    const int n = rd.seq_len;
    const uint8_t *ops = B.ops + rd.seq_off;
    const unsigned int *dcnt = B.dcnt + rd.seq_off;
    uint8_t *qual = B.qual + rd.seq_off;
    const unsigned long long read = B.read_index[r];
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        qual[i] = bb_qscore_base(qm, ops, dcnt, n, i, seed, read);
}

// ------------------------------------------------------------------------------------------------ K6
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_compact(BBBatchDev B) {
    const int r = blockIdx.x;
    const BBReadDev rd = B.reads[r];
    const uint8_t *seq = B.seq + rd.seq_off + rd.start_trim;
    const uint8_t *qual = B.qual + rd.seq_off + rd.start_trim;
    uint8_t *os = B.out_seq + rd.out_off, *oq = B.out_qual + rd.out_off;
    for (int i = threadIdx.x; i < rd.out_len; i += blockDim.x) {
        os[i] = seq[i];
        oq[i] = qual[i];
    }
}

// ------------------------------------------------------------------------------------------------ single-pair entry points
// edlib.align(query, target, task='path') for one pair (diagnostics / tests): ops + dcnt + lead_del + counts.
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(32) bb_k_align_pair(const uint8_t *q, int n, const uint8_t *t, int m, int k_upper,
                                                      BBScratchPool pool, uint8_t *ops, unsigned int *dcnt, int *out4) {
    const BBScratch sc = pool.for_warp(0);
    BBEmit em = {ops, dcnt, &out4[3]};
    BBAlnCounts cnt = {0, 0, 0, 0};
    if (bb_peq_words(n) > sc.peq_cap) cnt.err |= 256;
    else {
        bb_build_peq(q, n, sc.peq);
        bb_align<true, 16>(q, n, t, m, k_upper, sc, em, 0, cnt);
    }
    __syncwarp();
    if ((threadIdx.x & 31) == 0) { out4[0] = cnt.matches; out4[1] = cnt.dels; out4[2] = cnt.dist; out4[4] = cnt.err; }
}

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_qscores_pair(const uint8_t *ops, const unsigned int *dcnt, int n,
                                                         BBQScoreModelDev qm, unsigned long long seed,
                                                         unsigned long long read, uint8_t *qual) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        qual[i] = bb_qscore_base(qm, ops, dcnt, n, i, seed, read);
}

#include "bb_tasks.cuh"
#include "bb_loop.cuh"
