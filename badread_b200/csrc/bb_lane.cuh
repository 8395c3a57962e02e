// bb_lane.cuh — lane-level banded alignment for narrow bands (one problem per THREAD).
//
// The identity re-measurements of the error loop (simulate.py:325-346) align a 1000-base window against its
// mutated copy: the Ukkonen band is only a few dozen rows wide, so a warp-wide wavefront would keep two or three
// lanes busy.  Here every lane owns a complete problem: it keeps a window of LW 32-row words that follows the
// band down the diagonal (shifted by one word every 32 columns) and advances one column per iteration with a
// single 32*LW-bit Myers step (one add carry chain, no shuffles).  Thirty-two reads progress per warp.
// Same path semantics as bb_align.cuh (edlib's traceback rule); the history layout is per lane:
// hist[c * LW + x] = (Pv, PhRaw) of window word x at column c.
#pragma once
#include <cstdint>

#include "bb_align.cuh"

struct BBLaneProb {
    const uint4 *peq;   // match bitmap of the read that holds the query (bb_build_peq layout)
    int peq_bit0;       // bit index of query row 0 in that bitmap (index of q[0] in the read + 32)
    const uint8_t *q;   // query characters (for non-ACGT targets and the traceback)
    int n;
    const uint8_t *t;   // target characters
    int m;
    int a, b;           // band
    uint2 *hist;        // m * LW entries
};

// Window words needed for a band: the window top is word max(0, (c - a) >> 5); rows up to c + b must fit.
__device__ __forceinline__ int bb_lane_words(int a, int b) { return ((a + b) >> 5) + 2; }
// Words of a band slice, the a + b + 1 rows c - a ... c + b of column c from row max(0, c - a) on: at most
// bb_lane_words(a, b) - 1, so a window of LW words never needs more than LW - 1.
__device__ __forceinline__ int bb_band_words(int a, int b) { return ((a + b) >> 5) + 1; }

__device__ __forceinline__ void bb_lane_fetch(const BBLaneProb &P, int word, uint32_t &mA, uint32_t &mC, uint32_t &mG,
                                              uint32_t &mT) {
    mA = mC = mG = mT = 0u;
    const int R = word * 32;
    const int valid = P.n - R;
    if (valid <= 0) return;
    const int s = P.peq_bit0 + R;
    const int idx = s >> 5, sh = s & 31;
    const uint4 lo = P.peq[idx], hi = P.peq[idx + 1];
    mA = __funnelshift_r(lo.x, hi.x, sh); mC = __funnelshift_r(lo.y, hi.y, sh);
    mG = __funnelshift_r(lo.z, hi.z, sh); mT = __funnelshift_r(lo.w, hi.w, sh);
    if (valid < 32) {
        const uint32_t keep = (1u << valid) - 1u;
        mA &= keep; mC &= keep; mG &= keep; mT &= keep;
    }
}

// Forward pass with history. Returns D[n-1][m-1]. Requires bb_lane_words(a, b) <= LW and a + b >= 1.
template <int LW>
__device__ int bb_lane_pass(const BBLaneProb &P) {
    const int n = P.n, m = P.m, a = P.a;
    uint32_t Pv[LW], Mv[LW], eA[LW], eC[LW], eG[LW], eT[LW];
#pragma unroll
    for (int x = 0; x < LW; x++) {
        Pv[x] = ~0u; Mv[x] = 0u;
        bb_lane_fetch(P, x, eA[x], eC[x], eG[x], eT[x]);
    }
    int wt = 0;               // window top word
    int score = 32 * LW;      // D at the window's bottom row, previous column
    uint2 *h = P.hist;
    for (int c = 0; c < m; c++) {
        if (c - a >= 32 * (wt + 1)) {  // the band has left the top word: slide the window down one word
#pragma unroll
            for (int x = 0; x + 1 < LW; x++) {
                Pv[x] = Pv[x + 1]; Mv[x] = Mv[x + 1];
                eA[x] = eA[x + 1]; eC[x] = eC[x + 1]; eG[x] = eG[x + 1]; eT[x] = eT[x + 1];
            }
            wt++;
            Pv[LW - 1] = ~0u; Mv[LW - 1] = 0u;  // all-(+1) upper bound below the old bottom row
            bb_lane_fetch(P, wt + LW - 1, eA[LW - 1], eC[LW - 1], eG[LW - 1], eT[LW - 1]);
            score += 32;
        }
        const uint32_t tc = P.t[c];
        const uint32_t code = (tc >> 1) & 3u;  // A->0, C->1, T->2, G->3
        const bool acgt = ((0x47544341u >> (8 * code)) & 0xffu) == tc;
        uint32_t Eq[LW], Xv[LW], A[LW], S[LW], Ph[LW], Mh[LW];
#pragma unroll
        for (int x = 0; x < LW; x++)
            Eq[x] = (code & 2u) ? ((code & 1u) ? eG[x] : eT[x]) : ((code & 1u) ? eC[x] : eA[x]);
        if (!acgt) {
#pragma unroll
            for (int x = 0; x < LW; x++) {
                Eq[x] = 0u;
                const int row0 = (wt + x) * 32;
                for (int r = 0; r < 32; r++)
                    if (row0 + r < n && P.q[row0 + r] == tc) Eq[x] |= 1u << r;
            }
        }
        // horizontal delta entering the window top is +1: exact on row 0, an upper bound below it
#pragma unroll
        for (int x = 0; x < LW; x++) { Xv[x] = Eq[x] | Mv[x]; A[x] = Eq[x] & Pv[x]; }
        bb_add_words<LW>(A, Pv, S);
#pragma unroll
        for (int x = 0; x < LW; x++) {
            const uint32_t Xh = (S[x] ^ Pv[x]) | Eq[x];
            Ph[x] = Mv[x] | ~(Xh | Pv[x]);
            Mh[x] = Pv[x] & Xh;
        }
        score += (int)(Ph[LW - 1] >> 31) - (int)(Mh[LW - 1] >> 31);
#pragma unroll
        for (int x = LW - 1; x >= 0; x--) {
            const uint32_t phs = __funnelshift_l(x > 0 ? Ph[x - 1] : 0x80000000u, Ph[x], 1);
            const uint32_t mhs = __funnelshift_l(x > 0 ? Mh[x - 1] : 0u, Mh[x], 1);
            const uint32_t raw = Ph[x];
            Pv[x] = mhs | ~(Xv[x] | phs);
            Mv[x] = phs & Xv[x];
            h[x] = make_uint2(Pv[x], raw);
        }
        h += LW;
    }
    // D[n-1][m-1] from the window's bottom-row score and the vertical deltas below row n-1
    int result = BB_INF;
    int run = score;
#pragma unroll
    for (int x = LW - 1; x >= 0; x--) {
        const int row0 = (wt + x) * 32;
        if (row0 <= n - 1 && n - 1 < row0 + 32) {
            const int bit = (n - 1) - row0;
            const uint32_t up = bit == 31 ? 0u : (Pv[x] >> (bit + 1));
            const uint32_t um = bit == 31 ? 0u : (Mv[x] >> (bit + 1));
            result = run - __popc(up) + __popc(um);
        }
        run -= __popc(Pv[x]) - __popc(Mv[x]);
    }
    return result;
}

// edlib's traceback rule on the lane history: counts '=' columns and 'D' columns.
template <int LW>
__device__ void bb_lane_traceback(const BBLaneProb &P, int &matches, int &dels, int &err) {
    const int a = P.a;
    int i = P.n - 1, j = P.m - 1;
    int mt = 0, dl = 0;
    while (i >= 0 && j >= 0) {
        int wt = (j - a) >> 5; if (wt < 0) wt = 0;
        const int x = (i >> 5) - wt;
        if (x < 0 || x >= LW) { err |= 1; break; }
        const uint2 e = P.hist[j * LW + x];
        const int bit = i & 31;
        if ((e.x >> bit) & 1u) { i--; }                       // 'I'
        else if ((e.y >> bit) & 1u) { dl++; j--; }            // 'D'
        else { mt += (P.q[i] == P.t[j]) ? 1 : 0; i--; j--; }  // '=' / 'X'
    }
    if (j >= 0) dl += j + 1;
    matches = mt; dels = dl;
}

// Traceback reads one history entry per step, each depending on the previous one, out of a per-lane history that no
// longer sits in any cache: ask L2 for the line three lines down the path (the path moves at most one column a step).
template <int LW>
__device__ __forceinline__ void bb_prefetch_history(const uint2 *hist, int tj) {
#if defined(__CUDA_ARCH__)
    const long long e = (long long)tj * LW;
    if ((e & 15) == 0 && e >= 48) asm volatile("prefetch.global.L2 [%0];" ::"l"(hist + (e - 48)));
#endif
}

// ---------------------------------------------------------------------------------------------- traceback staging ring
// A lane's traceback is a chain of dependent history loads, one per move, out of a per-lane history far too large for
// any cache: with 3-4 warps per scheduler the kernels sat on that latency (ncu, round 1: 78 % of the stall cycles on the
// L1TEX scoreboard, issue slots 18 % busy).  The ring stages the history the path is about to walk through in SHARED
// memory with cp.async: all walking lanes of a warp "tick" at the same loop iteration, every T moves; a tick asks for the
// columns down to tj - 2T + 1 that are not staged yet and waits only for the copies of the PREVIOUS tick.  A move goes at
// most one column to the left, so the T columns a lane can reach before the next tick were requested one tick (T moves)
// earlier and have arrived; the moves themselves read shared memory.  Slot of column c: c mod 2T (the columns a tick
// overwrites are the ones the path has left behind).  The history holds the band slice of every column (bw words at
// hist[c * bw], bb_lane_step), at most LW - 1 words for a window of LW words.  Layout: ring[(slot * (LW - 1) + word) * 64
// + thread] (64 threads per CTA: consecutive threads, consecutive 8-byte entries, no bank conflicts).
#define BB_RING_BYTES(LW, T) (2 * (T) * ((LW) - 1) * 64 * 8)

__device__ __forceinline__ void bb_cp_async8(uint2 *smem, const uint2 *gmem) {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
#else
    *smem = *gmem;
#endif
}
__device__ __forceinline__ void bb_cp_async_commit() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N>
__device__ __forceinline__ void bb_cp_async_wait() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}

// One tick of a walking lane at column tj (>= 0) of a history of bw words per column; RW = LW - 1 words per ring slot.
// staged_lo: lowest column requested so far; > tj marks a walk that has not staged anything yet (it then issues two
// groups, so that the uniform wait below covers its first T columns).
template <int RW, int T>
__device__ __forceinline__ void bb_ring_tick(uint2 *ring, const uint2 *hist, int bw, int tj, int &staged_lo) {
    const bool fresh = staged_lo > tj;
    if (fresh) {
        const int lo1 = max(0, tj - T + 1);
        for (int col = tj; col >= lo1; col--) {
#pragma unroll
            for (int x = 0; x < RW; x++)
                if (x < bw) bb_cp_async8(ring + ((col & (2 * T - 1)) * RW + x) * 64, hist + (long long)col * bw + x);
        }
        bb_cp_async_commit();
        staged_lo = lo1;
    }
    const int want_lo = max(0, tj - 2 * T + 1);
    for (int col = staged_lo - 1; col >= want_lo; col--) {
#pragma unroll
        for (int x = 0; x < RW; x++)
            if (x < bw) bb_cp_async8(ring + ((col & (2 * T - 1)) * RW + x) * 64, hist + (long long)col * bw + x);
    }
    bb_cp_async_commit();
    if (want_lo < staged_lo) staged_lo = want_lo;
#if defined(__CUDA_ARCH__)
    // what the tick after the next one will ask for: into L2 now (HBM latency is more than one tick long)
    {
        constexpr int MAX_LINES = (T * RW * 8 + 127) / 128 + 1;
        const int lines = (T * bw * 8 + 127) / 128 + 1;
        const long long e = ((long long)tj - 4 * T) * bw;
#pragma unroll
        for (int x = 0; x < 2 * MAX_LINES; x++)
            if (e + 16 * x >= 0 && x < (fresh ? 2 : 1) * lines) asm volatile("prefetch.global.L2 [%0];" ::"l"(hist + e + 16 * x));
    }
#endif
    bb_cp_async_wait<1>();
}

template <int RW, int T>
__device__ __forceinline__ uint2 bb_ring_entry(const uint2 *ring, int col, int x) {
    return ring[((col & (2 * T - 1)) * RW + x) * 64];
}
