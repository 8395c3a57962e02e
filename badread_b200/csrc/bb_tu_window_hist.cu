// bb_tu_window_hist.cu — compiles the default lane-mode window aligners bb_k_window_lane_hist<4>, <8> (bb_loop.cuh).
#include "bb_launch.h"

// ring_t: columns staged per traceback tick (bb_ring_tick); 8 halves the ticks of the 4-word build (24 KB of shared
// memory per CTA)
void bbl_window_lane_hist(int words, int ring_t, int grid, cudaStream_t st, BBBatchDev B, BBErrorModelDev em,
                          const BBWinTask *tasks, const int *n_tasks, unsigned long long seed, uint2 *hist_pool,
                          uint8_t *tbuf_pool, int *cursor, BBWinTask *fallback, int *fallback_count) {
    if (words == 4 && ring_t == 8)
        bb_k_window_lane_hist<4, 8><<<grid, 64, BB_RING_BYTES(4, 8), st>>>(B, em, tasks, n_tasks, seed, hist_pool, tbuf_pool, cursor,
                                                                             fallback, fallback_count);
    else if (words == 4 && ring_t == 2)
        bb_k_window_lane_hist<4, 2><<<grid, 64, BB_RING_BYTES(4, 2), st>>>(B, em, tasks, n_tasks, seed, hist_pool, tbuf_pool, cursor,
                                                                             fallback, fallback_count);
    else if (words == 4)
        bb_k_window_lane_hist<4, 4><<<grid, 64, BB_RING_BYTES(4, 4), st>>>(B, em, tasks, n_tasks, seed, hist_pool, tbuf_pool, cursor,
                                                                             fallback, fallback_count);
    else
        bb_k_window_lane_hist<BB_WIN_LW, 4><<<grid, 64, BB_RING_BYTES(BB_WIN_LW, 4), st>>>(B, em, tasks, n_tasks, seed, hist_pool,
                                                                                             tbuf_pool, cursor, fallback, fallback_count);
}
