// emu_large_k.cpp — the device code of error models with k up to 16 under the warp emulator (TEST INFRASTRUCTURE):
//   emu_count_kmers_wide   bbm_k_kmer_alternatives + bbm_k_compact with 128-bit keys (the interface of
//                          bb_count_kmer_alternatives_wide)
//   emu_build_kidx_hash    K1 bb_k_build_fragments<0, true> for one read, with the hash table of the shared builder
//                          (badread_b200/csrc/bb_em_tables.h)
//   emu_error_loop_kmers   K1 with that table, then the error loop of one read round after round, as emu_align.cpp's
//                          emu_error_loop runs it, and bb_k_join
// Front end: emu_large_k.py.
#include "cuda_emu.h"

#include <string>
#include <type_traits>
#include <vector>

// sm_90's 16-byte atomicCAS (crt/sm_90_rt.h) for the 128-bit keys of bbm_k_kmer_alternatives: any trivially copyable
// 16-byte type, compared bitwise.  Declared before the device code so that its calls resolve to it.
template <typename T, typename = typename std::enable_if<sizeof(T) == 16>::type>
inline T atomicCAS(T *p, T cmp, T v) {
    T o;
    std::memcpy(&o, p, 16);
    if (std::memcmp(&o, &cmp, 16) == 0) std::memcpy(p, &v, 16);
    return o;
}

#include "../../badread_b200/csrc/bb_kernels.cuh"
#include "../../badread_b200/csrc/bb_models.cuh"

static void copy_err(const std::string &err, char *out, int cap) {
    if (cap > 0) { std::strncpy(out, err.c_str(), (size_t)cap - 1); out[cap - 1] = 0; }
}

extern "C" __attribute__((visibility("default")))
int emu_count_kmers_wide(int k, int32_t n_aln, const uint8_t *read, const int64_t *read_off, const uint8_t *ref,
                         const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0, const int32_t *op_ref0,
                         const int64_t *ops_off, int64_t table_cap, uint64_t *keys_out, uint64_t *first_out,
                         uint32_t *counts_out, int64_t *n_entries, int64_t ovf_cap, int32_t *ovf_aln, int32_t *ovf_pos,
                         int32_t *ovf_k, int64_t *n_ovf) {
    BBMAln A;
    A.read = read; A.qual = nullptr; A.ref = ref; A.read_off = read_off; A.ref_off = ref_off; A.ops_off = ops_off; A.ops = ops;
    A.op_read0 = op_read0; A.op_ref0 = op_ref0;
    std::vector<BBMKey128> keys((size_t)table_cap, BBMKey128{BBM_EMPTY, BBM_EMPTY});
    std::vector<unsigned long long> first((size_t)table_cap, BBM_EMPTY);
    std::vector<unsigned int> counts((size_t)table_cap, 0u);
    int status[4] = {0, 0, 0, 0};
    unsigned long long novf = 0, n = 0;
    BBMTableWide T;
    T.keys = keys.data(); T.first = first.data(); T.counts = counts.data(); T.cap = table_cap; T.status = status;
    T.ovf_aln = ovf_aln; T.ovf_pos = ovf_pos; T.ovf_k = ovf_k; T.n_ovf = &novf; T.ovf_cap = ovf_cap;
    std::vector<int> rp((size_t)ref_off[n_aln] + 8);
    std::vector<uint8_t> ism((size_t)ref_off[n_aln] + 8);
    for (int a = 0; a < n_aln; a++) {
        blockIdx.x = (unsigned)a;
        emu::run_block(256, [&]() { bbm_k_kmer_alternatives(A, n_aln, k, rp.data(), ism.data(), T); });
    }
    blockIdx.x = 0;
    *n_ovf = (int64_t)novf;
    if (status[0] || status[1]) { *n_entries = 0; return -4; }
    for (long long b = 0; b < (table_cap + 255) / 256; b++) {
        blockIdx.x = (unsigned)b;
        emu::run_block(256, [&]() { bbm_k_compact(T, 1, (BBMKey128 *)keys_out, (unsigned long long *)first_out, counts_out, &n, table_cap); });
    }
    blockIdx.x = 0;
    *n_entries = (int64_t)n;
    return 0;
}

// K1 for one read described like in bb_batch_upload (n_segs segments (kind, src, len) over `ref` and the literal pool
// `lit`), its k-mer index the hash table of rows r = 0 .. n_rows-1 with k-mer code kmer_codes[r].  Outputs the padded
// fragment and the row per position.  Returns 2 if the builder rejects the codes (message in err_out).
extern "C" __attribute__((visibility("default")))
int emu_build_kidx_hash(const uint8_t *ref, const uint8_t *lit, const int32_t *seg_kind, const int64_t *seg_src,
                        const int32_t *seg_len, int n_segs, int k, int32_t n_rows, const int64_t *kmer_codes,
                        unsigned long long seed, unsigned long long read_index, uint8_t *frag_out, int32_t *kidx_out,
                        char *err_out, int err_cap) {
    BBEmHashTable t;
    std::string err;
    if (!bb_build_em_hash(k, n_rows, kmer_codes, t, err)) { copy_err(err, err_out, err_cap); return 2; }
    uint8_t comp[256];
    std::memset(comp, 'N', sizeof(comp));
    const char *from = "ATGCatgcRYSWKMBVDHNryswkmbvdhn.-?";
    const char *to = "TACGtacgYRSWMKVBHDNyrswmkvbhdn.-?";
    for (int i = 0; from[i]; i++) comp[(uint8_t)from[i]] = (uint8_t)to[i];
    std::memcpy(bb_c_comp, comp, 256);
    std::vector<bb_segment> segs((size_t)n_segs);
    int len = 0;
    for (int s = 0; s < n_segs; s++) { segs[(size_t)s] = bb_segment{seg_src[s], seg_len[s], seg_kind[s]}; len += seg_len[s]; }
    const int frag_len = len + 2 * k;
    int seg_off[2] = {0, n_segs};
    BBReadDev rd;
    std::memset(&rd, 0, sizeof(rd));
    rd.frag_len = frag_len;
    std::vector<uint8_t> fr((size_t)frag_len + 64, 0);
    std::vector<uint32_t> state((size_t)frag_len + 64, 7u);
    std::vector<unsigned int> ctime((size_t)frag_len + 64, 7u);
    std::vector<int> kidx((size_t)frag_len + 64, -7);
    std::vector<uint4> fpeq((size_t)bb_peq_words(frag_len) + 8);
    BBBatchDev B;
    std::memset(&B, 0, sizeof(B));
    B.n_reads = 1; B.read_index = &read_index; B.seg_off = seg_off; B.segs = segs.data(); B.lit = lit; B.reads = &rd;
    B.frag = fr.data(); B.state = state.data(); B.ctime = ctime.data(); B.kidx = kidx.data(); B.fpeq = fpeq.data();
    const BBEmHashDev hash{t.entries.data(), t.bits};
    blockIdx.x = 0;
    emu::run_block(256, [&]() { bb_k_build_fragments<0, true>(B, ref, k, seed, nullptr, hash); });
    std::memcpy(frag_out, fr.data(), (size_t)frag_len);
    for (int x = 0; x + k <= frag_len; x++) kidx_out[x] = kidx[(size_t)x];
    return 0;
}

// The error loop of ONE read with a hash-indexed model: K1 builds the padded fragment (one literal segment) and its
// k-mer rows, then bb_k_mutate -> bb_k_window_tasks -> bb_k_window_lane_hist<4> -> <8> -> bb_k_window_warp ->
// bb_k_replay round after round, then bb_k_join.  out8 / joined_out / the return value as emu_error_loop; -6: the
// builder rejected the codes.
extern "C" __attribute__((visibility("default")))
int emu_error_loop_kmers(const uint8_t *fragment, int n, double target, unsigned long long seed, unsigned long long read_index,
                         int k, int32_t n_rows, const int64_t *kmer_codes, const int32_t *row_off, const double *cum,
                         const uint8_t *flags, const uint32_t *slots, const uint8_t *pool_bytes, int *out8,
                         uint8_t *joined_out, int joined_cap) {
    const int frag_len = n + 2 * k;
    std::vector<uint8_t> fr((size_t)frag_len + 64, 0);
    std::vector<int> kidx((size_t)frag_len + 64, -1);
    {
        const int32_t kind = BB_SEG_LITERAL, len = n;
        const int64_t src = 0;
        char err[256];
        if (emu_build_kidx_hash(nullptr, fragment, &kind, &src, &len, 1, k, n_rows, kmer_codes, seed, read_index, fr.data(),
                                kidx.data(), err, sizeof(err)))
            return -6;
    }
    std::vector<BBRowInfo> info((size_t)n_rows);
    for (int32_t r = 0; r < n_rows; r++) {
        const int32_t e0 = row_off[r], ne = row_off[r + 1] - e0;
        BBRowInfo &ri = info[(size_t)r];
        ri.cum_last = cum[e0 + ne - 1]; ri.cum0 = cum[e0]; ri.e0 = e0; ri.ne = ne;
        ri.first_is_identity = flags[e0] == 1 ? 1 : 0; ri.pad = 0;
    }
    BBErrorModelDev em;
    std::memset(&em, 0, sizeof(em));
    em.k = k; em.type = 1; em.kmer_to_row = nullptr; em.row_off = row_off; em.cum = cum; em.flags = flags; em.slots = slots;
    em.pool = pool_bytes; em.rowinfo = info.data();
    std::vector<uint32_t> state((size_t)frag_len + 64, BB_SLOT_NONE);
    std::vector<unsigned int> ctime((size_t)frag_len + 64, 0u);
    std::vector<uint4> fpeq((size_t)bb_peq_words(frag_len) + 8);
    const int cap = (int)(0.9 * (double)frag_len) + k + 2;
    std::vector<uint2> chlog((size_t)cap + 8);
    std::vector<int2> wres((size_t)cap / BB_ALIGNMENT_INTERVAL + 8, make_int2(-1, -1));
    BBReadDev rd;
    std::memset(&rd, 0, sizeof(rd));
    rd.frag_len = frag_len;
    const double need = (double)frag_len * (1.0 - target);
    rd.horizon = (int)std::min<double>((double)cap, std::max(0.0, 1.25 * need) + 48.0);
    rd.status = BB_READ_PENDING;
    BBBatchDev B;
    std::memset(&B, 0, sizeof(B));
    int order0 = 0;
    B.n_reads = 1; B.read_index = &read_index; B.target = &target; B.order = &order0; B.reads = &rd; B.frag = fr.data();
    B.state = state.data(); B.ctime = ctime.data(); B.kidx = kidx.data(); B.fpeq = fpeq.data(); B.chlog = chlog.data();
    B.wres = wres.data();
    emu::run_warp([&]() { bb_build_peq(fr.data(), frag_len, fpeq.data()); });
    const int big = 2 * BB_WIN_MAX_COLS + frag_len + 64;
    const int NW = BB_WARPS_PER_CTA;
    std::vector<uint2> hist((size_t)NW * 106496), whist((size_t)32 * BB_WIN_MAX_COLS * BB_WIN_LW);
    std::vector<int8_t> hbuf((size_t)NW * big);
    std::vector<int> LR((size_t)NW * 2 * big), stack((size_t)NW * 5 * 64);
    std::vector<uint8_t> wtbuf((size_t)NW * big), ltbuf((size_t)64 * BB_WIN_MAX_COLS);
    std::vector<uint4> wpeq((size_t)NW * (bb_peq_words(big) + 8));
    BBScratchPool pool;
    std::memset(&pool, 0, sizeof(pool));
    pool.hist = hist.data(); pool.hist_stride = 106496; pool.hist_cap = 106496;
    pool.hbuf = hbuf.data(); pool.hbuf_stride = big; pool.hbuf_cap = big;
    pool.lr = LR.data(); pool.lr_stride = 2 * (long long)big; pool.lr_cap = big;
    pool.stack = stack.data(); pool.stack_cap = 64;
    pool.tbuf = wtbuf.data(); pool.tbuf_stride = big;
    pool.peq = wpeq.data(); pool.peq_stride = bb_peq_words(big) + 8; pool.peq_cap = bb_peq_words(big) + 8;
    std::vector<BBWinTask> tasks((size_t)cap / BB_ALIGNMENT_INTERVAL + 8), fb1(tasks.size()), fb2(tasks.size());
    int rounds = 0;
    for (; rounds < 12 && rd.status != BB_READ_DONE; rounds++) {
        int c_mut = 0, n_tasks = 0, c4 = 0, n_fb1 = 0, c8 = 0, n_fb2 = 0, cw = 0, pending = 0;
        emu::run_block(BB_MUTP_THREADS, [&]() { bb_k_mutate(B, em, seed, &c_mut, &order0, 1); });
        emu::run_warp([&]() { bb_k_window_tasks(B, &order0, 1, tasks.data(), &n_tasks); });
        emu::run_warp([&]() {
            bb_k_window_lane_hist<4, 4>(B, em, tasks.data(), &n_tasks, seed, whist.data(), ltbuf.data(), &c4, fb1.data(), &n_fb1);
        });
        emu::run_warp([&]() {
            bb_k_window_lane_hist<BB_WIN_LW, 4>(B, em, fb1.data(), &n_fb1, seed, whist.data(), ltbuf.data(), &c8, fb2.data(), &n_fb2);
        });
        emu::run_block(BB_WARPS_PER_CTA * 32, [&]() { bb_k_window_warp(B, em, pool, fb2.data(), &n_fb2, seed, &cw); });
        emu::run_warp([&]() { bb_k_replay(B, &order0, 1, k, &pending); });
    }
    if (rd.status != BB_READ_DONE) return -1;
    std::vector<uint8_t> seq((size_t)rd.seq_len + 64, 0);
    std::vector<uint4> speq((size_t)bb_peq_words(rd.seq_len) + 8);
    B.seq = seq.data(); B.speq = speq.data();
    emu::run_block(256, [&]() { bb_k_join(B, em); });
    out8[0] = rd.loop_count; out8[1] = rd.change_count; out8[2] = rd.n_align; out8[3] = rd.seq_len;
    out8[4] = rd.start_trim; out8[5] = rd.end_trim; out8[6] = rd.upper; out8[7] = rd.flags;
    std::memcpy(joined_out, seq.data(), (size_t)std::min(rd.seq_len, joined_cap));
    return rounds;
}
