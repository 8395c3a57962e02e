// bb_tasks.cuh — the final alignment (edlib.align(seq, fragment), qscore_model.py:37) as level-synchronous tasks.
//
// edlib's recursion (Hirschberg split on the target until its traceback estimate drops below 1 MiB, then a leaf
// traceback) is a tree whose nodes are independent once their parent has chosen the split row.  Instead of one
// warp walking the tree of one read depth-first, every level of all reads' trees is processed by a few kernel
// launches:
//   node kernels   forward pass over the left half + reverse pass over the right half of the node, split row by
//                  edlib's rule, children appended to the next level's queues (or to the leaf queues)
//   leaf kernels   forward pass with history + traceback, emitting the per-base ops / deletion counts
// Tasks are routed by band width: narrow bands go to LANE kernels (one task per thread, persistent lanes that all
// execute the same column step; 32 tasks per warp), wide bands to WARP kernels (the wavefront of bb_align.cuh).
// The root needs no separate distance pass: with the band derived from the injected-edit bound, the minimum of
// forward + reverse scores over the split column IS the edit distance.
#pragma once
#include <cstdint>

#include "bb_align.cuh"
#include "bb_lane.cuh"

#define BB_NODE_LW_SMALL 8   // window words of the lane node kernel (bands up to 32*6 rows)
#define BB_LEAF_LW 8         // window words of the lane leaf kernel
#define BB_LEAF_LANE_COLS 2048

// Node classes, one queue (per level parity) and one kernel each: lane mode for narrow short nodes; single warps with
// the forward and the reverse pass in its two 16-lane halves, 1 / 2 / 4 words per lane (one build per width: the
// narrow ones need a third of the registers of the wide one and run at three times the occupancy); warp pairs beyond.
enum { BBQ_NODE_LANE8 = 0, BBQ_NODE_LEAN1 = 1, BBQ_NODE_LEAN2 = 2, BBQ_NODE_LEAN4 = 3, BBQ_NODE_WIDE = 4, BBQ_NODE_CLASSES = 5 };
#define BBQ_COUNT(cls, parity) ((parity) * BBQ_NODE_CLASSES + (cls))  // Q.count index of a node queue's length
#define BBQ_LEAF_COUNT 10  // Q.count index of the leaf counters (lane, warp)
#define BBQ_OVERFLOW 12
// Node kernels take `parity | BBQ_BACKWARDS` to walk their queue from its end.  Below the roots a level's queue fills in
// the order the parents finish - the longest nodes are queued last, and taken in that order they start when everything
// else is done; from the end, the longest go first.
#define BBQ_BACKWARDS 2

struct BBNode { int r, q0, nn, t0, mm, best; };  // best < 0: root (band from the read's edit bound)

struct BBQueues {
    BBNode *node[BBQ_NODE_CLASSES][2];  // [class][level parity]
    BBNode *leaf[2];     // lane, warp
    int *count;          // node counts: [BBQ_COUNT(class, parity)]; leaf counts: [BBQ_LEAF_COUNT + which]
    int *overflow;
    int cap_node, cap_leaf;
    int lane8_cols;      // longest target a lane node task may have (longer ones go to the warp kernels)
};

struct BBAlignOut {      // where a read's alignment goes
    uint8_t *ops;
    unsigned int *dcnt;
    BBReadDev *rd;
};

__device__ __forceinline__ void bb_add_dels(const BBAlignOut &o, int qidx_after, int count) {
    // `count` deletion columns that follow query base qidx_after (-1: before the first base)
    if (count <= 0) return;
    if (qidx_after >= 0) atomicAdd(&o.dcnt[qidx_after], (unsigned int)count);
    else atomicAdd(&o.rd->lead_del, count);
}

// Band a task will be processed with (the root uses the injected-edit bound of its read).
__device__ __forceinline__ void bb_task_band(const BBNode &nd, int upper, int &a, int &b) {
    int k = nd.best >= 0 ? nd.best : upper;
    const int diff = nd.nn > nd.mm ? nd.nn - nd.mm : nd.mm - nd.nn;
    if (k < diff) k = diff;
    const int mx = nd.nn > nd.mm ? nd.nn : nd.mm;
    if (k > mx) k = mx;
    bb_band(nd.nn, nd.mm, k, a, b);
    // an even band (a wider band is always valid): the chunks of the two-column wavefront then begin and end on whole
    // column pairs (bb_band_pass_bp)
    a += a & 1; b += b & 1;
}

// Queue a child (or finish it on the spot when one side is empty, edlib.cpp obtainAlignment).
static __device__ void bb_push_task(const BBQueues &Q, int next_parity, const BBAlignOut &o, const BBNode &nd, int upper) {
    if (nd.nn == 0) {
        atomicAdd(&o.rd->dels, nd.mm);
        bb_add_dels(o, nd.q0 - 1, nd.mm);
        return;
    }
    if (nd.mm == 0) {
        for (int x = 0; x < nd.nn; x++) o.ops[nd.q0 + x] = BB_OP_I;
        return;
    }
    int a, b;
    bb_task_band(nd, upper, a, b);
    const int lw = bb_lane_words(a, b);
    if (bb_uses_traceback(nd.nn, nd.mm)) {
        const int which = (lw <= BB_LEAF_LW && nd.mm <= BB_LEAF_LANE_COLS) ? 0 : 1;
        const int idx = atomicAdd(&Q.count[BBQ_LEAF_COUNT + which], 1);
        if (idx >= Q.cap_leaf) { atomicExch(Q.overflow, 1); return; }
        Q.leaf[which][idx] = nd;
    } else {
        // a lane walks its node alone, one column after the other: only short nodes go there (they are the many
        // ones); a long narrow node would hold a whole launch up and runs ~15x sooner as a warp wavefront
        const int L2 = bb_pick_L<4>(a, b, 16);  // words per lane that let two 16-lane groups share a warp (0: too wide)
        const int cls = (lw <= BB_NODE_LW_SMALL && nd.mm <= Q.lane8_cols) ? BBQ_NODE_LANE8
                        : L2 == 1 ? BBQ_NODE_LEAN1 : L2 == 2 ? BBQ_NODE_LEAN2 : L2 == 4 ? BBQ_NODE_LEAN4 : BBQ_NODE_WIDE;
        const int idx = atomicAdd(&Q.count[BBQ_COUNT(cls, next_parity)], 1);
        if (idx >= Q.cap_node) { atomicExch(Q.overflow, 1); return; }
        Q.node[cls][next_parity][idx] = nd;
    }
}

// edlib.cpp obtainAlignmentHirschberg's choice of the split row from the two column-score arrays
// (L[r - loL] = D(q[0..r], t[0..left_w)), R[x - loR] = D(rq[0..x], rt[0..right_w))), sequential version.
// best < 0 (root): the minimum over all splits is the edit distance.  Returns false if no split matches.
static __device__ bool bb_choose_split_seq(const int *L, int loL, int hiL, const int *R, int loR, int hiR, int nn, int left_w,
                                    int right_w, int &best, int &split, int &ls, int &rs) {
    int rlo = max(loL, nn - 2 - hiR); if (rlo < 0) rlo = 0;
    int rhi = min(hiL, nn - 2 - loR); if (rhi > nn - 2) rhi = nn - 2;
    const bool have_top = nn - 1 >= loR && nn - 1 <= hiR;  // empty query prefix on the left
    const bool have_bot = nn - 1 >= loL && nn - 1 <= hiL;  // empty query suffix on the right
    if (best < 0) {
        int mn = BB_INF;
        for (int r = rlo; r <= rhi; r++) mn = min(mn, L[r - loL] + R[(nn - 2 - r) - loR]);
        if (have_top) mn = min(mn, left_w + R[(nn - 1) - loR]);
        if (have_bot) mn = min(mn, L[(nn - 1) - loL] + right_w);
        best = mn;
    }
    for (int r = rlo; r <= rhi; r++) {
        const int lv = L[r - loL], rv = R[(nn - 2 - r) - loR];
        if (lv + rv == best) { split = r; ls = lv; rs = rv; return true; }
    }
    if (have_top) {
        const int v = R[(nn - 1) - loR];
        if (left_w + v == best) { split = -1; ls = left_w; rs = v; return true; }
    }
    if (have_bot) {
        const int v = L[(nn - 1) - loL];
        if (v + right_w == best) { split = nn - 1; ls = v; rs = right_w; return true; }
    }
    return false;
}

// Roots of all reads of the batch (same routing rule as every other task).
// Reads whose root has a wide band form their own pipeline (QW): its levels are not held up by, and do not hold
// up, the levels of all other reads (QN).
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(256) bb_k_push_roots(BBBatchDev B, BBQueues QN, BBQueues QW, const int *order) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n_reads) return;
    const int r = order[i];  // longest fragments first, so the biggest nodes start early
    BBReadDev *rd = &B.reads[r];
    if (rd->flags & BB_FLAG_NOSPACE) return;  // no room for this read (bb_k_scan): the host runs the batch again
    BBAlignOut o;
    o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
    const BBNode nd = {r, 0, rd->seq_len, 0, rd->frag_len, -1};
    int a, b;
    bb_task_band(nd, rd->upper, a, b);
    const bool wide = !bb_uses_traceback(nd.nn, nd.mm) && bb_pick_L<4>(a, b, 16) == 0;
    bb_push_task(wide ? QW : QN, 0, o, nd, rd->upper);
}

// ---------------------------------------------------------------------------------------------- lane column step
// State of one banded pass owned by one thread (window of LW words following the band).
template <int LW>
struct BBLanePass {
    uint32_t Pv[LW], Mv[LW], eA[LW], eC[LW], eG[LW], eT[LW];
    int wt, score, c;
};

template <int LW>
__device__ __forceinline__ void bb_lane_begin(BBLanePass<LW> &S, const BBProb &P) {
#pragma unroll
    for (int x = 0; x < LW; x++) {
        S.Pv[x] = ~0u; S.Mv[x] = 0u;
        bb_fetch_peq(P, 32 * x, S.eA[x], S.eC[x], S.eG[x], S.eT[x]);
    }
    S.wt = 0; S.score = 32 * LW; S.c = 0;
}

// One column of the pass. hist (optional): with HSTRIDE == 1, this column's band slice, the bb_band_words(a, b) words
// from row max(0, c - a) on (the traceback never leaves the band); otherwise all LW window words, HSTRIDE apart.
template <int LW, bool HIST, int HSTRIDE = 1>
__device__ __forceinline__ void bb_lane_step(BBLanePass<LW> &S, const BBProb &P, uint2 *hist) {
    const int c = S.c;
    if (c - P.a >= 32 * (S.wt + 1)) {  // slide the window down one word
#pragma unroll
        for (int x = 0; x + 1 < LW; x++) {
            S.Pv[x] = S.Pv[x + 1]; S.Mv[x] = S.Mv[x + 1];
            S.eA[x] = S.eA[x + 1]; S.eC[x] = S.eC[x + 1]; S.eG[x] = S.eG[x + 1]; S.eT[x] = S.eT[x + 1];
        }
        S.wt++;
        S.Pv[LW - 1] = ~0u; S.Mv[LW - 1] = 0u;
        bb_fetch_peq(P, 32 * (S.wt + LW - 1), S.eA[LW - 1], S.eC[LW - 1], S.eG[LW - 1], S.eT[LW - 1]);
        S.score += 32;
    }
    const uint32_t tc = P.t[(long long)c * P.ts];
    const uint32_t code = (tc >> 1) & 3u;  // A->0, C->1, T->2, G->3
    const bool acgt = ((0x47544341u >> (8 * code)) & 0xffu) == tc;
    uint32_t Eq[LW], Xv[LW], A[LW], Sm[LW], Ph[LW], Mh[LW];
#pragma unroll
    for (int x = 0; x < LW; x++)
        Eq[x] = (code & 2u) ? ((code & 1u) ? S.eG[x] : S.eT[x]) : ((code & 1u) ? S.eC[x] : S.eA[x]);
    if (!acgt) {
#pragma unroll
        for (int x = 0; x < LW; x++) {
            Eq[x] = 0u;
            const int row0 = (S.wt + x) * 32;
            for (int r = 0; r < 32; r++)
                if (row0 + r < P.n && P.q[(long long)(row0 + r) * P.qs] == tc) Eq[x] |= 1u << r;
        }
    }
#pragma unroll
    for (int x = 0; x < LW; x++) { Xv[x] = Eq[x] | S.Mv[x]; A[x] = Eq[x] & S.Pv[x]; }
    bb_add_words<LW>(A, S.Pv, Sm);
#pragma unroll
    for (int x = 0; x < LW; x++) {
        const uint32_t Xh = (Sm[x] ^ S.Pv[x]) | Eq[x];
        Ph[x] = S.Mv[x] | ~(Xh | S.Pv[x]);
        Mh[x] = S.Pv[x] & Xh;
    }
    S.score += (int)(Ph[LW - 1] >> 31) - (int)(Mh[LW - 1] >> 31);
#pragma unroll
    for (int x = LW - 1; x >= 0; x--) {
        const uint32_t phs = __funnelshift_l(x > 0 ? Ph[x - 1] : 0x80000000u, Ph[x], 1);
        const uint32_t mhs = __funnelshift_l(x > 0 ? Mh[x - 1] : 0u, Mh[x], 1);
        const uint32_t raw = Ph[x];
        S.Pv[x] = mhs | ~(Xv[x] | phs);
        S.Mv[x] = phs & Xv[x];
        if (HIST && HSTRIDE != 1) hist[x * HSTRIDE] = make_uint2(S.Pv[x], raw);
    }
    if (HIST && HSTRIDE == 1) {
        // the band's top row is bit off of window word 0 (wt = max(0, (c - a) >> 5)); Ph still holds the raw words
        const int bw = bb_band_words(P.a, P.b);
        const int off = c >= P.a ? (c - P.a) & 31 : 0;
#pragma unroll
        for (int y = 0; y + 1 < LW; y++)
            if (y < bw) hist[y] = make_uint2(__funnelshift_r(S.Pv[y], S.Pv[y + 1], off), __funnelshift_r(Ph[y], Ph[y + 1], off));
    }
    S.c = c + 1;
}

// D[row][last column] of the window rows in [lo, hi] -> out[row - lo]; returns D[n-1][last] if inside the window.
template <int LW>
__device__ int bb_lane_column_scores(const BBLanePass<LW> &S, int n, int lo, int hi, int *out) {
    int result = BB_INF;
    int run = S.score;
#pragma unroll
    for (int x = LW - 1; x >= 0; x--) {
        const int row0 = (S.wt + x) * 32;
        int rr = run;
        for (int r = 31; r >= 0; r--) {
            const int row = row0 + r;
            if (row < n) {
                if (out && row >= lo && row <= hi) out[row - lo] = rr;
                if (row == n - 1) result = rr;
            }
            rr -= (int)((S.Pv[x] >> r) & 1u) - (int)((S.Mv[x] >> r) & 1u);
        }
        run -= __popc(S.Pv[x]) - __popc(S.Mv[x]);
    }
    return result;
}

// D[n-1][last column] of a finished pass (BB_INF if row n-1 is outside the window).
template <int LW>
__device__ __forceinline__ int bb_lane_corner(const BBLanePass<LW> &S, int n) {
    int result = BB_INF;
    int run = S.score;
#pragma unroll
    for (int x = LW - 1; x >= 0; x--) {
        const int row0 = (S.wt + x) * 32;
        if (row0 <= n - 1 && n - 1 < row0 + 32) {
            const int bit = (n - 1) - row0;
            const uint32_t up = bit == 31 ? 0u : (S.Pv[x] >> (bit + 1));
            const uint32_t um = bit == 31 ? 0u : (S.Mv[x] >> (bit + 1));
            result = run - __popc(up) + __popc(um);
        }
        run -= __popc(S.Pv[x]) - __popc(S.Mv[x]);
    }
    return result;
}

// ---------------------------------------------------------------------------------------------- lane node kernel
template <int LW>
__global__ void __launch_bounds__(64, 6)
bb_k_node_lane(BBBatchDev B, BBQueues Q, int parity_order, int *cursor) {
    constexpr int CLS = BBQ_NODE_LANE8;
    const int parity = parity_order & 1;
    const bool backwards = (parity_order & BBQ_BACKWARDS) != 0;
    const BBNode *list = Q.node[CLS][parity];
    const int count = min(Q.count[BBQ_COUNT(CLS, parity)], Q.cap_node);
    BBLanePass<LW> S;
    BBProb P;
    BBNode nd;
    int Lc[32 * LW], Rc[32 * LW];
    int loL = 0, hiL = 0, loR = 0, hiR = 0, left_w = 0, right_w = 0, ncols = 0, upper = 0;
    int phase = 0;  // 0: fetch, 1: forward pass, 2: reverse pass, 3: done
    BBAlignOut o;
    for (;;) {
        if (phase == 0) {
            const int w = atomicAdd(cursor, 1);
            if (w >= count) phase = 3;
            else {
                nd = list[backwards ? count - 1 - w : w];
                BBReadDev *rd = &B.reads[nd.r];
                o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
                upper = rd->upper;
                bb_task_band(nd, upper, P.a, P.b);
                left_w = nd.mm / 2; right_w = nd.mm - left_w;
                loL = max(0, left_w - 1 - P.a); hiL = min(nd.nn - 1, left_w - 1 + P.b);
                loR = max(0, right_w - 1 - P.a); hiR = min(nd.nn - 1, right_w - 1 + P.b);
                P.n = nd.nn; P.peq = B.speq + rd->speq_off;
                P.q = B.seq + rd->seq_off + nd.q0; P.qs = 1; P.peq_bit0 = nd.q0 + BB_PEQ_BIT0;
                P.t = B.frag + rd->frag_off + nd.t0; P.ts = 1;
                ncols = left_w;
                bb_lane_begin<LW>(S, P);
                phase = 1;
            }
        }
        if (__all_sync(BB_FULL, phase == 3)) break;
        // the hot loop: every lane advances its current pass by one column per iteration
        for (int it = 0; it < 128; it++) {
            if (phase == 1 || phase == 2) {
                bb_lane_step<LW, false>(S, P, nullptr);
                if (S.c >= ncols) {
                    if (phase == 1) {
                        bb_lane_column_scores<LW>(S, nd.nn, loL, hiL, Lc);
                        const BBReadDev *rd = o.rd;
                        P.q = B.seq + rd->seq_off + nd.q0 + nd.nn - 1; P.qs = -1; P.peq_bit0 = nd.q0 + nd.nn - 1 + BB_PEQ_BIT0;
                        P.t = B.frag + rd->frag_off + nd.t0 + nd.mm - 1; P.ts = -1;
                        ncols = right_w;
                        bb_lane_begin<LW>(S, P);
                        phase = 2;
                    } else {
                        bb_lane_column_scores<LW>(S, nd.nn, loR, hiR, Rc);
                        int best = nd.best, split = 0, ls = 0, rs = 0;
                        if (!bb_choose_split_seq(Lc, loL, hiL, Rc, loR, hiR, nd.nn, left_w, right_w, best, split, ls, rs)) {
                            atomicOr(&o.rd->flags, 32 << 8);
                        } else {
                            BBNode c0 = {nd.r, nd.q0, split + 1, nd.t0, left_w, ls};
                            BBNode c1 = {nd.r, nd.q0 + split + 1, nd.nn - split - 1, nd.t0 + left_w, right_w, rs};
                            bb_push_task(Q, parity ^ 1, o, c0, upper);
                            bb_push_task(Q, parity ^ 1, o, c1, upper);
                        }
                        phase = 0;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- lane leaf kernel
// One leaf per thread, 32 at a time per warp in lock step: forward pass with a checkpoint of the vertical deltas every
// BB_LEAF_TILE columns, then the traceback tile by tile out of shared memory (the scheme of bb_k_window_lane; round 1
// kept 64 bytes of history per column per leaf in global memory).
#define BB_LEAF_TILE 16
#define BB_LEAF_CKPT_WORDS (2 * BB_LEAF_LW + 2)
#define BB_LEAF_MAX_TILES (BB_LEAF_LANE_COLS / BB_LEAF_TILE)
#define BB_LEAF_SMEM_BYTES (BB_LEAF_TILE * BB_LEAF_LW * 64 * 8)

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(64, 3)
bb_k_leaf_lane(BBBatchDev B, BBQueues Q, uint32_t *ckpt_pool, int *cursor) {
    constexpr int LW = BB_LEAF_LW, CKW = BB_LEAF_CKPT_WORDS;
#ifdef BB_EMULATOR
    static uint2 s_hist[BB_LEAF_TILE * LW * 64];
#else
    extern __shared__ __align__(16) uint2 s_hist[];  // [column in tile][word][thread]
#endif
    const BBNode *list = Q.leaf[0];
    const int count = min(Q.count[BBQ_LEAF_COUNT], Q.cap_leaf);
    uint32_t *const ckpt = ckpt_pool + ((long long)blockIdx.x * blockDim.x + threadIdx.x) * (long long)(BB_LEAF_MAX_TILES * CKW);
    uint2 *const hs = s_hist + threadIdx.x;
    for (;;) {
        const int w = atomicAdd(cursor, 1);
        const bool active = w < count;
        if (!__any_sync(BB_FULL, active)) break;
        BBNode nd = {0, 0, 0, 0, 0, 0};
        BBAlignOut o = {nullptr, nullptr, nullptr};
        BBProb P;
        P.a = 0; P.b = 1;
        BBLanePass<LW> S;
        const uint8_t *qp = nullptr, *tp = nullptr;
        int mm = 0;
        if (active) {
            nd = list[w];
            BBReadDev *rd = &B.reads[nd.r];
            o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
            bb_task_band(nd, rd->upper, P.a, P.b);
            P.n = nd.nn; P.peq = B.speq + rd->speq_off;
            qp = B.seq + rd->seq_off + nd.q0; tp = B.frag + rd->frag_off + nd.t0;
            P.q = qp; P.qs = 1; P.peq_bit0 = nd.q0 + BB_PEQ_BIT0; P.t = tp; P.ts = 1;
            bb_lane_begin<LW>(S, P);
            mm = nd.mm;
        }
        // ---- forward pass, a checkpoint every BB_LEAF_TILE columns
        const int mm_max = __reduce_max_sync(BB_FULL, mm);
        for (int c = 0; c < mm_max; c++) {
            if (c < mm) {
                if ((c & (BB_LEAF_TILE - 1)) == 0) {
                    uint32_t *ck = ckpt + (c / BB_LEAF_TILE) * CKW;
#pragma unroll
                    for (int x = 0; x < LW; x++) { ck[x] = S.Pv[x]; ck[LW + x] = S.Mv[x]; }
                    ck[2 * LW] = (uint32_t)S.wt; ck[2 * LW + 1] = (uint32_t)S.score;
                }
                bb_lane_step<LW, false>(S, P, nullptr);
            }
        }
        if (active) {
            const int d = bb_lane_column_scores<LW>(S, nd.nn, 0, -1, nullptr);
            if (nd.best >= 0 && d != nd.best) atomicOr(&o.rd->flags, 8 << 8);
        }
        // ---- traceback (edlib's rule: 'I' > 'D' > diagonal), tile by tile
        int ti = nd.nn - 1, tj = mm - 1, matches = 0, dels = 0;
        bool walking = active && ti >= 0 && tj >= 0;
        bool need_tile = walking;
        int tile_lo = 0;
        // (every round moves every walking lane at least once: nn + mm rounds bound the loop whatever the data)
        for (int round = 0; round < (1 << 16) && __any_sync(BB_FULL, walking); round++) {
            if (walking && need_tile) {  // all walking lanes get here together (see the inner loop's exit)
                const int tile = tj / BB_LEAF_TILE;
                tile_lo = tile * BB_LEAF_TILE;
                const uint32_t *ck = ckpt + tile * CKW;
#pragma unroll
                for (int x = 0; x < LW; x++) { S.Pv[x] = ck[x]; S.Mv[x] = ck[LW + x]; }
                S.wt = (int)ck[2 * LW]; S.score = (int)ck[2 * LW + 1]; S.c = tile_lo;
#pragma unroll
                for (int x = 0; x < LW; x++) bb_fetch_peq(P, 32 * (S.wt + x), S.eA[x], S.eC[x], S.eG[x], S.eT[x]);
                const int hi = min(tile_lo + BB_LEAF_TILE, mm);
                for (int c = tile_lo; c < hi; c++) bb_lane_step<LW, true, 64>(S, P, hs + ((c - tile_lo) * LW) * 64);
                need_tile = false;
            }
            for (int mv = 0; mv < 64; mv++) {
                const bool can = walking && !need_tile;
                if (!__any_sync(BB_FULL, can)) break;
                if (can) {
                    int wt = (tj - P.a) >> 5; if (wt < 0) wt = 0;
                    const int x = (ti >> 5) - wt;
                    if (x < 0 || x >= LW) { atomicOr(&o.rd->flags, 1 << 8); ti = -1; tj = -1; }
                    else {
                        const uint2 e = hs[((tj - tile_lo) * LW + x) * 64];
                        const int bit = ti & 31;
                        if ((e.x >> bit) & 1u) { o.ops[nd.q0 + ti] = BB_OP_I; ti--; }
                        else if ((e.y >> bit) & 1u) { bb_add_dels(o, nd.q0 + ti, 1); dels++; tj--; }
                        else {
                            const bool eq = qp[ti] == tp[tj];
                            o.ops[nd.q0 + ti] = eq ? BB_OP_EQ : BB_OP_X;
                            matches += eq ? 1 : 0;
                            ti--; tj--;
                        }
                    }
                    if (ti < 0 || tj < 0) walking = false;
                    else if (tj < tile_lo) need_tile = true;
                }
            }
        }
        if (active) {
            if (walking) atomicOr(&o.rd->flags, 1 << 8);  // cannot happen: the round bound above was hit
            for (int x = 0; x <= ti; x++) o.ops[nd.q0 + x] = BB_OP_I;  // column boundary: insertions remain
            if (tj >= 0) { bb_add_dels(o, nd.q0 - 1, tj + 1); dels += tj + 1; }  // row boundary: deletions
            atomicAdd(&o.rd->matches, matches);
            atomicAdd(&o.rd->dels, dels);
        }
    }
}

// ---------------------------------------------------------------------------------------------- lane leaf kernel (default)
// Persistent lanes with per-column history in global memory, walked back through the shared-memory staging ring
// (see bb_k_window_lane_hist and bb_ring_tick).
#ifndef BB_LEAF_RING_T
#define BB_LEAF_RING_T 4
#endif
#define BB_LEAF_RING_BYTES BB_RING_BYTES(BB_LEAF_LW, BB_LEAF_RING_T)

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(64)
bb_k_leaf_lane_hist(BBBatchDev B, BBQueues Q, uint2 *hist_pool, int *cursor) {
    constexpr int LW = BB_LEAF_LW, T = BB_LEAF_RING_T;
#ifdef BB_EMULATOR
    static uint2 s_ring[BB_LEAF_RING_BYTES / 8];
#else
    extern __shared__ __align__(16) uint2 s_ring[];  // BB_LEAF_RING_BYTES: [column mod 2T][word][thread]
#endif
    const BBNode *list = Q.leaf[0];
    const int count = min(Q.count[BBQ_LEAF_COUNT], Q.cap_leaf);
    uint2 *const hist = hist_pool + ((long long)blockIdx.x * blockDim.x + threadIdx.x) * (long long)(BB_LEAF_LANE_COLS * (LW - 1));
    uint2 *const ring = s_ring + threadIdx.x;
    BBLanePass<LW> S;
    BBProb P;
    BBNode nd;
    BBAlignOut o;
    const uint8_t *qp = nullptr, *tp = nullptr;
    int phase = 0;  // 0: fetch, 1: forward pass, 2: traceback, 3: done
    int ti = 0, tj = 0, matches = 0, dels = 0, staged_lo = 0;
    for (;;) {
        if (phase == 0) {
            const int w = atomicAdd(cursor, 1);
            if (w >= count) phase = 3;
            else {
                nd = list[w];
                BBReadDev *rd = &B.reads[nd.r];
                o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
                bb_task_band(nd, rd->upper, P.a, P.b);
                P.n = nd.nn; P.peq = B.speq + rd->speq_off;
                qp = B.seq + rd->seq_off + nd.q0; tp = B.frag + rd->frag_off + nd.t0;
                P.q = qp; P.qs = 1; P.peq_bit0 = nd.q0 + BB_PEQ_BIT0; P.t = tp; P.ts = 1;
                bb_lane_begin<LW>(S, P);
                phase = 1;
            }
        }
        if (__all_sync(BB_FULL, phase == 3)) break;
        for (int it = 0; it < 128; it++) {  // forward columns with history
            if (phase == 1) {
                bb_lane_step<LW, true>(S, P, hist + (long long)S.c * bb_band_words(P.a, P.b));
                if (S.c >= nd.mm) {
                    const int d = bb_lane_corner<LW>(S, nd.nn);
                    if (nd.best >= 0 && d != nd.best) atomicOr(&o.rd->flags, 8 << 8);
                    ti = nd.nn - 1; tj = nd.mm - 1; matches = 0; dels = 0; staged_lo = nd.mm;
                    phase = 2;
                }
            }
        }
        for (int it = 0; it < 256; it++) {  // traceback moves (edlib's rule: 'I' > 'D' > diagonal)
            if (phase == 2) {
                if (ti >= 0 && tj >= 0) {
                    // (it is the same for all lanes: the walking lanes of the warp tick together)
                    const int bw = bb_band_words(P.a, P.b);  // (recomputed, not kept: a live register more spills)
                    if ((it & (T - 1)) == 0) bb_ring_tick<LW - 1, T>(ring, hist, bw, tj, staged_lo);
                    const int k = ti - max(0, tj - P.a);  // row in the band slice of column tj
                    if (k < 0 || k >= 32 * bw) { atomicOr(&o.rd->flags, 1 << 8); ti = -1; tj = -1; }
                    else {
                        const uint2 e = bb_ring_entry<LW - 1, T>(ring, tj, k >> 5);
                        const int bit = k & 31;
                        if ((e.x >> bit) & 1u) { o.ops[nd.q0 + ti] = BB_OP_I; ti--; }
                        else if ((e.y >> bit) & 1u) { bb_add_dels(o, nd.q0 + ti, 1); dels++; tj--; }
                        else {
                            const bool eq = qp[ti] == tp[tj];
                            o.ops[nd.q0 + ti] = eq ? BB_OP_EQ : BB_OP_X;
                            matches += eq ? 1 : 0;
                            ti--; tj--;
                        }
                    }
                } else {
                    bb_cp_async_wait<0>();  // nothing of this walk may land in the ring after the next walk's copies
                    for (int x = 0; x <= ti; x++) o.ops[nd.q0 + x] = BB_OP_I;  // column boundary: insertions remain
                    if (tj >= 0) { bb_add_dels(o, nd.q0 - 1, tj + 1); dels += tj + 1; }  // row boundary: deletions
                    atomicAdd(&o.rd->matches, matches);
                    atomicAdd(&o.rd->dels, dels);
                    phase = 0;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- warp kernels
// One Hirschberg node per warp: the forward pass over the left half of the target and the reverse pass over the right
// half run side by side in the warp's two 16-lane groups with exactly L words per lane (class BBQ_NODE_LEAN<L>), several
// columns per wavefront step on bit planes (bb_band_pass_bp); then the split row by edlib's rule.
template <int L>
__global__ void __launch_bounds__(BB_WARPS_PER_CTA * 32, (L == 1 ? 6 : L == 2 ? 5 : 3))
bb_k_node_warp(BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity_order, int *cursor, int warp_base) {
    constexpr int CLS = L == 1 ? BBQ_NODE_LEAN1 : L == 2 ? BBQ_NODE_LEAN2 : BBQ_NODE_LEAN4;
    const int parity = parity_order & 1;
    const bool backwards = (parity_order & BBQ_BACKWARDS) != 0;
    const int lane = threadIdx.x & 31;
    const int warp = warp_base + blockIdx.x * BB_WARPS_PER_CTA + (threadIdx.x >> 5);
    BBScratch sc = pool.for_warp(warp);
    const BBNode *list = Q.node[CLS][parity];
    const int count = min(Q.count[BBQ_COUNT(CLS, parity)], Q.cap_node);
    for (;;) {
        int w = 0;
        if (lane == 0) w = atomicAdd(cursor, 1);
        w = __shfl_sync(BB_FULL, w, 0);
        if (w >= count) break;
        const BBNode nd = list[backwards ? count - 1 - w : w];
        BBReadDev *rd = &B.reads[nd.r];
        BBAlignOut o;
        o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
        sc.peq = B.speq + rd->speq_off;
        const uint8_t *q = B.seq + rd->seq_off, *t = B.frag + rd->frag_off;
        int a, b;
        bb_task_band(nd, rd->upper, a, b);
        const int left_w = nd.mm / 2, right_w = nd.mm - left_w;
        const int loL = max(0, left_w - 1 - a), hiL = min(nd.nn - 1, left_w - 1 + b);
        const int loR = max(0, right_w - 1 - a), hiR = min(nd.nn - 1, right_w - 1 + b);
        int best = nd.best, split = 0, ls = 0, rs = 0, err = 0;
        if (hiL - loL + 1 > sc.lr_cap || hiR - loR + 1 > sc.lr_cap) err = 16;
        else {
            BBProb P;
            P.n = nd.nn; P.a = a; P.b = b; P.peq = sc.peq; P.hist = nullptr; P.nb_alloc = 0;
            P.tpeq = B.fpeq + rd->fpeq_off;
            if (lane < 16) {
                P.q = q + nd.q0; P.qs = 1; P.t = t + nd.t0; P.ts = 1; P.ncols = left_w;
                P.peq_bit0 = nd.q0 + BB_PEQ_BIT0; P.cols_out = sc.L; P.cols_lo = loL;
                P.tpeq_bit0 = nd.t0 + BB_PEQ_BIT0;
            } else {
                P.q = q + nd.q0 + nd.nn - 1; P.qs = -1; P.t = t + nd.t0 + nd.mm - 1; P.ts = -1; P.ncols = right_w;
                P.peq_bit0 = nd.q0 + nd.nn - 1 + BB_PEQ_BIT0; P.cols_out = sc.R; P.cols_lo = loR;
                P.tpeq_bit0 = nd.t0 + nd.mm - 1 + BB_PEQ_BIT0;
            }
            bb_band_pass_bp<L>(P, 16);
            __syncwarp();
            err = bb_split_warp(sc, loL, hiL, loR, hiR, nd.nn, left_w, right_w, best, split, ls, rs);
        }
        __syncwarp();
        if (lane == 0) {
            if (err) atomicOr(&rd->flags, err << 8);
            else {
                BBNode c0 = {nd.r, nd.q0, split + 1, nd.t0, left_w, ls};
                BBNode c1 = {nd.r, nd.q0 + split + 1, nd.nn - split - 1, nd.t0 + left_w, right_w, rs};
                bb_push_task(Q, parity ^ 1, o, c0, rd->upper);
                bb_push_task(Q, parity ^ 1, o, c1, rd->upper);
            }
        }
        __syncwarp();
    }
}

#define BB_PAIR_SMEM_BYTES (BB_WARPS_PER_CTA * bb_esm_words(32) * 4)

// Rendezvous of the two warps of a pair (named barrier `id`, 64 threads).
__device__ __forceinline__ void bb_pair_sync(int id) {
#ifdef BB_EMULATOR
    emu::named_barrier(id, 64);
#else
    asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory");
#endif
}

// Wide-band nodes: a PAIR of warps per node.  The even warp runs the forward pass over the left half of the target,
// the odd warp the reverse pass over the right half, each as a full 32-lane wavefront (half the words per lane of
// the paired single-warp variant, so the steps are half as long); the even warp then picks the split.
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_WARPS_PER_CTA * 32, 2)
bb_k_node_pair(BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity_order, int *cursor, int warp_base) {
    const int parity = parity_order & 1;
    const bool backwards = (parity_order & BBQ_BACKWARDS) != 0;
    __shared__ int s_task[BB_WARPS_PER_CTA / 2];
#ifdef BB_EMULATOR
    static uint32_t s_eq[BB_PAIR_SMEM_BYTES / 4];
#else
    extern __shared__ __align__(16) uint32_t s_eq[];  // BB_PAIR_SMEM_BYTES: one match-word cache per warp
#endif
    const int lane = threadIdx.x & 31;
    const int wi = threadIdx.x >> 5;
    const int pair = wi >> 1;
    const bool rev = (wi & 1) != 0;
    // both warps of a pair use the even warp's scratch (L and R live there)
    BBScratch sc = pool.for_warp(warp_base + blockIdx.x * BB_WARPS_PER_CTA + (wi & ~1));
    const BBNode *list = Q.node[BBQ_NODE_WIDE][parity];
    const int count = min(Q.count[BBQ_COUNT(BBQ_NODE_WIDE, parity)], Q.cap_node);
    for (;;) {
        if (!rev && lane == 0) s_task[pair] = atomicAdd(cursor, 1);
        bb_pair_sync(pair + 1);
        const int w = s_task[pair];
        bb_pair_sync(pair + 1);
        if (w >= count) break;
        const BBNode nd = list[backwards ? count - 1 - w : w];
        BBReadDev *rd = &B.reads[nd.r];
        sc.peq = B.speq + rd->speq_off;
        const uint8_t *q = B.seq + rd->seq_off, *t = B.frag + rd->frag_off;
        int a, b;
        bb_task_band(nd, rd->upper, a, b);
        const int left_w = nd.mm / 2, right_w = nd.mm - left_w;
        const int loL = max(0, left_w - 1 - a), hiL = min(nd.nn - 1, left_w - 1 + b);
        const int loR = max(0, right_w - 1 - a), hiR = min(nd.nn - 1, right_w - 1 + b);
        const int L = bb_pick_L<32>(a, b, 32);
        int err = 0;
        if (hiL - loL + 1 > sc.lr_cap || hiR - loR + 1 > sc.lr_cap) err = 16;
        else if (L > 0) {
            BBProb P;
            P.n = nd.nn; P.a = a; P.b = b; P.peq = sc.peq; P.hist = nullptr; P.nb_alloc = 0;
            if (!rev) {
                P.q = q + nd.q0; P.qs = 1; P.t = t + nd.t0; P.ts = 1; P.ncols = left_w;
                P.peq_bit0 = nd.q0 + BB_PEQ_BIT0; P.cols_out = sc.L; P.cols_lo = loL;
            } else {
                P.q = q + nd.q0 + nd.nn - 1; P.qs = -1; P.t = t + nd.t0 + nd.mm - 1; P.ts = -1; P.ncols = right_w;
                P.peq_bit0 = nd.q0 + nd.nn - 1 + BB_PEQ_BIT0; P.cols_out = sc.R; P.cols_lo = loR;
            }
            P.esm = s_eq + wi * bb_esm_words(32);
            bb_band_dispatch<false, true, 32, true>(P, 32, L);
        }
        __threadfence_block();
        bb_pair_sync(pair + 1);
        if (!rev) {
            int best = nd.best, split = 0, ls = 0, rs = 0;
            if (!err) {
                if (L > 0) err = bb_split_warp(sc, loL, hiL, loR, hiR, nd.nn, left_w, right_w, best, split, ls, rs);
                else err = bb_node_warp<1>(q, t, nd.q0, nd.nn, nd.t0, nd.mm, a, b, sc, best, split, ls, rs);  // strips
            }
            if (lane == 0) {
                BBAlignOut o;
                o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
                if (err) atomicOr(&rd->flags, err << 8);
                else {
                    BBNode c0 = {nd.r, nd.q0, split + 1, nd.t0, left_w, ls};
                    BBNode c1 = {nd.r, nd.q0 + split + 1, nd.nn - split - 1, nd.t0 + left_w, right_w, rs};
                    bb_push_task(Q, parity ^ 1, o, c0, rd->upper);
                    bb_push_task(Q, parity ^ 1, o, c1, rd->upper);
                }
            }
            __syncwarp();
        }
    }
}

// Wide-band nodes by a whole CTA of 8 warps: warps 0-3 run the forward pass over the left half of the target as one
// 128-lane wavefront (bb_band_pass_mw), warps 4-7 the reverse pass over the right half; warp 0 then picks the split.
// A quarter of the words per lane of the single-warp wavefront and four schedulers per pass: the dependent chain of
// columns of the longest reads - what bounds a whole step from below - runs about three times faster.
#define BB_QUAD_WARPS 4
#define BB_QUAD_THREADS (2 * BB_QUAD_WARPS * 32)
#define BB_QUAD_SMEM_BYTES (2 * BB_QUAD_WARPS * bb_esm_words(32) * 4)

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_QUAD_THREADS, 1)
bb_k_node_quad(BBBatchDev B, BBQueues Q, BBScratchPool pool, int parity_order, int *cursor, int warp_base) {
    const int parity = parity_order & 1;
    const bool backwards = (parity_order & BBQ_BACKWARDS) != 0;
    __shared__ int s_task;
    __shared__ uint32_t s_mbox[2][BB_QUAD_WARPS * 8];
    __shared__ int s_progress[2][BB_QUAD_WARPS];
    __shared__ int s_err;
#ifdef BB_EMULATOR
    static uint32_t s_eq[BB_QUAD_SMEM_BYTES / 4];
#else
    extern __shared__ __align__(16) uint32_t s_eq[];  // BB_QUAD_SMEM_BYTES: one match-word cache per warp
#endif
    const int lane = threadIdx.x & 31;
    const int wi = threadIdx.x >> 5;
    const bool rev = wi >= BB_QUAD_WARPS;
    const int wg = wi % BB_QUAD_WARPS;
    BBScratch sc = pool.for_warp(warp_base + blockIdx.x);  // L and R of the CTA's current node
    const BBNode *list = Q.node[BBQ_NODE_WIDE][parity];
    const int count = min(Q.count[BBQ_COUNT(BBQ_NODE_WIDE, parity)], Q.cap_node);
    for (;;) {
        if (threadIdx.x == 0) { s_task = atomicAdd(cursor, 1); s_err = 0; }
        if (threadIdx.x < 2 * BB_QUAD_WARPS) s_progress[threadIdx.x / BB_QUAD_WARPS][threadIdx.x % BB_QUAD_WARPS] = 0;
        __syncthreads();
        const int w = s_task;
        __syncthreads();
        if (w >= count) break;
        const BBNode nd = list[backwards ? count - 1 - w : w];
        BBReadDev *rd = &B.reads[nd.r];
        sc.peq = B.speq + rd->speq_off;
        const uint8_t *q = B.seq + rd->seq_off, *t = B.frag + rd->frag_off;
        int a, b;
        bb_task_band(nd, rd->upper, a, b);
        const int left_w = nd.mm / 2, right_w = nd.mm - left_w;
        const int loL = max(0, left_w - 1 - a), hiL = min(nd.nn - 1, left_w - 1 + b);
        const int loR = max(0, right_w - 1 - a), hiR = min(nd.nn - 1, right_w - 1 + b);
        const int L = bb_pick_L<32>(a, b, 32 * BB_QUAD_WARPS);
        int err = 0;
        if (hiL - loL + 1 > sc.lr_cap || hiR - loR + 1 > sc.lr_cap) err = 16;
        else if (L > 0) {
            BBProb P;
            P.n = nd.nn; P.a = a; P.b = b; P.peq = sc.peq; P.hist = nullptr; P.nb_alloc = 0;
            if (!rev) {
                P.q = q + nd.q0; P.qs = 1; P.t = t + nd.t0; P.ts = 1; P.ncols = left_w;
                P.peq_bit0 = nd.q0 + BB_PEQ_BIT0; P.cols_out = sc.L; P.cols_lo = loL;
            } else {
                P.q = q + nd.q0 + nd.nn - 1; P.qs = -1; P.t = t + nd.t0 + nd.mm - 1; P.ts = -1; P.ncols = right_w;
                P.peq_bit0 = nd.q0 + nd.nn - 1 + BB_PEQ_BIT0; P.cols_out = sc.R; P.cols_lo = loR;
            }
            P.esm = s_eq + wi * bb_esm_words(32);
            volatile uint32_t *mb = s_mbox[rev ? 1 : 0];
            volatile int *pg = s_progress[rev ? 1 : 0];
            int e;
            if (L == 1) e = bb_band_pass_mw<1, BB_QUAD_WARPS>(P, wg, mb, pg);
            else if (L == 2) e = bb_band_pass_mw<2, BB_QUAD_WARPS>(P, wg, mb, pg);
            else if (L == 4) e = bb_band_pass_mw<4, BB_QUAD_WARPS>(P, wg, mb, pg);
            else if (L == 8) e = bb_band_pass_mw<8, BB_QUAD_WARPS>(P, wg, mb, pg);
            else if (L == 16) e = bb_band_pass_mw<16, BB_QUAD_WARPS>(P, wg, mb, pg);
            else e = bb_band_pass_mw<32, BB_QUAD_WARPS>(P, wg, mb, pg);
            if (e && lane == 0) atomicOr(&s_err, e);
        }
        __threadfence_block();
        __syncthreads();
        if (wi == 0) {
            err |= s_err;
            int best = nd.best, split = 0, ls = 0, rs = 0;
            if (!err) {
                if (L > 0) err = bb_split_warp(sc, loL, hiL, loR, hiR, nd.nn, left_w, right_w, best, split, ls, rs);
                else err = bb_node_warp<1>(q, t, nd.q0, nd.nn, nd.t0, nd.mm, a, b, sc, best, split, ls, rs);  // strips
            }
            if (lane == 0) {
                BBAlignOut o;
                o.ops = B.ops + rd->seq_off; o.dcnt = B.dcnt + rd->seq_off; o.rd = rd;
                if (err) atomicOr(&rd->flags, err << 8);
                else {
                    BBNode c0 = {nd.r, nd.q0, split + 1, nd.t0, left_w, ls};
                    BBNode c1 = {nd.r, nd.q0 + split + 1, nd.nn - split - 1, nd.t0 + left_w, right_w, rs};
                    bb_push_task(Q, parity ^ 1, o, c0, rd->upper);
                    bb_push_task(Q, parity ^ 1, o, c1, rd->upper);
                }
            }
            __syncwarp();
        }
    }
}

// One leaf per warp (bands or lengths beyond the lane kernel's limits).
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_WARPS_PER_CTA * 32, 2)
bb_k_leaf_warp(BBBatchDev B, BBQueues Q, BBScratchPool pool, int *cursor, int warp_base) {
    const int lane = threadIdx.x & 31;
    const int warp = warp_base + blockIdx.x * BB_WARPS_PER_CTA + (threadIdx.x >> 5);
    BBScratch sc = pool.for_warp(warp);
    const BBNode *list = Q.leaf[1];
    const int count = min(Q.count[BBQ_LEAF_COUNT + 1], Q.cap_leaf);
    for (;;) {
        int w = 0;
        if (lane == 0) w = atomicAdd(cursor, 1);
        w = __shfl_sync(BB_FULL, w, 0);
        if (w >= count) break;
        const BBNode nd = list[w];
        BBReadDev *rd = &B.reads[nd.r];
        sc.peq = B.speq + rd->speq_off;
        BBEmit em;
        em.ops = B.ops + rd->seq_off; em.dcnt = B.dcnt + rd->seq_off; em.lead_del = &rd->lead_del;
        BBAlnCounts cnt = {0, 0, 0, 0};
        int k = nd.best >= 0 ? nd.best : rd->upper;
        {
            const int diff = nd.nn > nd.mm ? nd.nn - nd.mm : nd.mm - nd.nn;
            if (k < diff) k = diff;
            const int mx = nd.nn > nd.mm ? nd.nn : nd.mm;
            if (k > mx) k = mx;
        }
        const int d = bb_leaf<true, 16>(B.seq + rd->seq_off + nd.q0, nd.nn, B.frag + rd->frag_off + nd.t0, nd.mm, k, sc, em,
                                        nd.q0, nd.q0, cnt);
        if (nd.best >= 0 && d != nd.best) cnt.err |= 8;
        __syncwarp();
        if (lane == 0) {
            atomicAdd(&rd->matches, cnt.matches);
            atomicAdd(&rd->dels, cnt.dels);
            if (cnt.err) atomicOr(&rd->flags, cnt.err << 8);
        }
        __syncwarp();
    }
}
