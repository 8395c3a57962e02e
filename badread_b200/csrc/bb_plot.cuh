// bb_plot.cuh — `badread plot`'s window series on the device (plot_window_identity.get_window_means of the reference).
//
// Input: the model builders' flat arrays (model_builders.FlatAlignments / DeviceFlat).  For an alignment of read slice
// length L the errors per read position e[0..L) are: 1 where an M base differs from the reference base, 1 for an I base,
// plus n at the read offset where a D run of n starts (adjacent runs add up).  The host has refused every alignment whose
// CIGAR does not cover the read slice exactly or has a D run at offset L, so every read position lies in exactly one M or
// I run of non-zero length, and every D run starts where the next such run starts.  For i in [0, L - w) the series is
//   identity[i] = 100 * (1 - (E[i + w] - E[i]) / w)      mean qscore[i] = (Q[i + w] - Q[i]) / w
// with E, Q the inclusive prefix sums (E[0] = 0) of e and of (quality byte - 33): integers, so each difference equals the
// reference's running sum, and the three double operations are the reference's, rounded the same way (no contraction).
//
// One CTA per alignment walks its read slice in tiles of blockDim.x * items positions, items consecutive positions per
// thread: it finds each position's run (a binary search per thread and tile, then a walk), scans the tile, stores the
// prefix sums (64-bit) in scratch and, once the tile's sums are stored, writes the windows that end in the tile.  A
// window reaches back at most w positions, into this tile or an earlier one of the same CTA.
#pragma once
#ifndef BB_EMULATOR
#include <cuda_runtime.h>
#endif
#include <cstdint>

#ifndef WS_THREADS
#define WS_THREADS 256               // threads per CTA
#endif
#define WS_ITEMS 8                   // the most positions per thread and tile (items <= WS_ITEMS is a kernel argument)

// Exclusive block scan of two values per thread (WS_THREADS threads): *ta, *tb the block's sums.  Every thread calls it.
__device__ __forceinline__ void ws_block_scan2(int64_t a, int64_t b, int64_t *ea, int64_t *eb, int64_t *ta, int64_t *tb) {
    __shared__ int64_t s_a[WS_THREADS / 32], s_b[WS_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t ia = a, ib = b;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t oa = __shfl_up_sync(0xffffffffu, ia, d), ob = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= d) {
            ia += oa;
            ib += ob;
        }
    }
    if (lane == 31) {
        s_a[w] = ia;
        s_b[w] = ib;
    }
    __syncthreads();
    int64_t ba = 0, bb = 0, sa = 0, sb = 0;
    for (int k = 0; k < WS_THREADS / 32; k++) {
        if (k == w) {
            ba = sa;
            bb = sb;
        }
        sa += s_a[k];
        sb += s_b[k];
    }
    __syncthreads();   // (the next call may overwrite s_a / s_b)
    *ea = ba + ia - a;
    *eb = bb + ib - b;
    *ta = sa;
    *tb = sb;
}

// Alignment a = blockIdx.x of a pass: its read slice read[read_off[a] ..] (quality slice alike), reference slice
// ref[ref_off[a] ..], runs ops[ops_off[a] .. ops_off[a + 1]) ((length << 2) | 0 M, 1 I, 2 D, at read / reference offsets
// op_read0 / op_ref0).  E / Q: scratch of L + 1 int64 each at scratch_off[a] (Q unused without qual); the window series
// go to identity[point_off[a] ..] and mean_qual[point_off[a] ..] (max(0, L - window) each).  qual == nullptr: no qscores.
__global__ void __launch_bounds__(WS_THREADS)
ws_k_series(const uint8_t *__restrict__ read, const uint8_t *__restrict__ qual, const uint8_t *__restrict__ ref,
            const int64_t *__restrict__ read_off, const int64_t *__restrict__ ref_off, const uint32_t *__restrict__ ops,
            const int32_t *__restrict__ op_read0, const int32_t *__restrict__ op_ref0, const int64_t *__restrict__ ops_off,
            int64_t window, int items, const int64_t *__restrict__ scratch_off, const int64_t *__restrict__ point_off,
            int64_t *__restrict__ E, int64_t *__restrict__ Q, double *__restrict__ identity, double *__restrict__ mean_qual) {
    const int64_t a = blockIdx.x;
    const int64_t r0 = read_off[a], L = read_off[a + 1] - r0, f0 = ref_off[a], o_lo = ops_off[a], o_hi = ops_off[a + 1];
    const bool want_qual = qual != nullptr;
    int64_t *const e_sum = E + scratch_off[a];
    int64_t *const q_sum = want_qual ? Q + scratch_off[a] : nullptr;
    double *const out_id = identity + point_off[a];
    double *const out_q = want_qual ? mean_qual + point_off[a] : nullptr;
    const double w = (double)window;
    if (threadIdx.x == 0) {
        e_sum[0] = 0;
        if (want_qual) q_sum[0] = 0;
    }
    const int64_t tile = (int64_t)WS_THREADS * items;
    int64_t carry_e = 0, carry_q = 0;
    for (int64_t t0 = 0; t0 < L; t0 += tile) {
        const int64_t p_first = t0 + (int64_t)threadIdx.x * items;
        int64_t ev[WS_ITEMS], qv[WS_ITEMS], sum_e = 0, sum_q = 0;
        int64_t o = o_lo;
        if (p_first < L) {   // the last run starting at or before p_first (an M or I run: see the top of the file)
            int64_t lo = o_lo, hi = o_hi - 1;
            while (lo < hi) {
                const int64_t mid = (lo + hi + 1) >> 1;
                if (op_read0[mid] <= p_first) lo = mid;
                else hi = mid - 1;
            }
            o = lo;
        }
#pragma unroll
        for (int k = 0; k < WS_ITEMS; k++) {
            ev[k] = qv[k] = 0;
            const int64_t p = p_first + k;
            if (k >= items || p >= L) continue;
            while (o + 1 < o_hi && op_read0[o + 1] <= p) o++;
            const uint32_t run = ops[o];
            const int32_t p0 = op_read0[o];
            int64_t e = 1;
            if ((run & 3u) == 0u) e = read[r0 + p] != ref[f0 + op_ref0[o] + (p - p0)];
            // the runs just before this one that start at p too: D runs, whose lengths add here, and empty M / I runs
            for (int64_t d = o - 1; p == p0 && d >= o_lo && op_read0[d] == p0; d--)
                if ((ops[d] & 3u) == 2u) e += ops[d] >> 2;
            ev[k] = e;
            if (want_qual) qv[k] = (int64_t)qual[r0 + p] - 33;
            sum_e += ev[k];
            sum_q += qv[k];
        }
        int64_t ex_e, ex_q, tot_e, tot_q;
        ws_block_scan2(sum_e, sum_q, &ex_e, &ex_q, &tot_e, &tot_q);
        int64_t run_e = carry_e + ex_e, run_q = carry_q + ex_q;
#pragma unroll
        for (int k = 0; k < WS_ITEMS; k++) {
            const int64_t p = p_first + k;
            if (k >= items || p >= L) continue;
            run_e += ev[k];
            run_q += qv[k];
            e_sum[p + 1] = run_e;
            if (want_qual) q_sum[p + 1] = run_q;
        }
        carry_e += tot_e;
        carry_q += tot_q;
        __syncthreads();   // the tile's prefix sums are stored
        // windows i = j - window whose last prefix index j = p + 1 lies in this tile; j = L is the reference's dropped window
#pragma unroll
        for (int k = 0; k < WS_ITEMS; k++) {
            const int64_t j = p_first + k + 1, i = j - window;
            if (k >= items || j >= L || i < 0) continue;
            const double s = (double)(e_sum[j] - e_sum[i]);
            out_id[i] = __dmul_rn(100.0, __dsub_rn(1.0, __ddiv_rn(s, w)));
            if (want_qual) out_q[i] = __ddiv_rn((double)(q_sum[j] - q_sum[i]), w);
        }
    }
}
