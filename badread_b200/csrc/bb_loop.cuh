// bb_loop.cuh — simulate.sequence_fragment's error loop (simulate.py:272-346) decoupled from its identity
// re-measurements.
//
// Which slot mutates, and into what, never depends on the running error estimate `errors`: the position and the
// alternative come from the iteration's own random stream, and whether a slot takes the change depends only on
// the slots changed before.  `errors` (and with it every window alignment) decides one thing only: at the top of
// which iteration the loop stops.  So the loop is split into three kernels that can each use the whole GPU:
//   bb_k_mutate        one CTA per read runs the k-mer loop AHEAD without any alignment, logging every applied
//                      change (iteration, position) and stamping the slot with the change's ordinal; it stops at
//                      the loop's own guards (simulate.py:278-286) or when a generous horizon of changes is reached.
//   bb_k_window_lane   every identity re-measurement of every read is an independent task: "the window as it was
//                      after 25*a changes" is rebuilt from the ordinals; one task per THREAD (bb_lane.cuh), so
//                      several hundred thousand alignments are in flight at once.  Windows beyond the lane limits
//                      go to bb_k_window_warp.
//   bb_k_replay        one thread per read replays the scalar recurrence of `errors` over the change log with the
//                      alignment results, finds the iteration at whose top the reference loop breaks, and rolls
//                      back the changes logged past it.  A read whose horizon was too short is resumed.
// The result is identical to running the loop sequentially (the oracle does exactly that).
#pragma once
#include <cstdint>

#include "bb_lane.cuh"

enum { BB_STOP_HORIZON = 0, BB_STOP_LIMIT = 1, BB_STOP_COUNT = 2, BB_STOP_NOLOOP = 3 };

#define BB_WIN_LW 8          // window words of the lane window aligner (bands up to 32*6 rows)
#define BB_WIN_MAX_COLS 2048 // joined window length a lane can keep

struct BBWinTask { int r, a; };  // read, alignment ordinal (1-based: after 25*a changes)

// ------------------------------------------------------------------------------------------------ mutate
// One CTA (5 warps) per read.  A step covers 128 consecutive loop iterations: warps 1-4 evaluate them (position, k-mer,
// model draw: chains of dependent loads, independent across iterations), warp 0 commits the iterations that change
// something, in order.  The evaluation runs ONE STEP AHEAD of the commit: what an iteration would change depends on its
// own random stream and on the fragment only, never on earlier commits, and the next step starts at n0 + 128 unless the
// loop stops - so while warp 0 commits the candidates of step i, warps 1-4 already evaluate step i + 1 into the other
// half of a double buffer.  A step costs max(evaluate, commit) instead of their sum (the evaluate-then-commit build
// spent most of its warp stall cycles at the CTA barrier between the two).  If
// the loop stops, the speculative step is simply dropped - the resume point is the commit's.
#define BB_MUTP_THREADS (BB_WARPS_PER_CTA * 32 + 32)

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_MUTP_THREADS)
bb_k_mutate(BBBatchDev B, BBErrorModelDev em, unsigned long long seed, int *work_counter, const int *order,
                 int n_items) {
    constexpr int NE = BB_WARPS_PER_CTA * 32;  // evaluator threads = iterations per step
    __shared__ int s_kind[2][NE], s_pos[2][NE], s_rpos[2][NE];
    __shared__ uint32_t s_pay[2][NE];
    __shared__ int s_w, s_stop, s_cc;
    __shared__ long long s_n0;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int ev = threadIdx.x - 32;  // evaluator index (warps 1 ... 4)
    const int k = em.k;
    for (;;) {
        if (threadIdx.x == 0) s_w = atomicAdd(work_counter, 1);
        __syncthreads();
        const int w = s_w;
        __syncthreads();
        if (w >= n_items) break;
        const int r = order[w];
        BBReadDev *rd = &B.reads[r];
        if (rd->status == BB_READ_DONE) continue;  // later rounds: only reads whose horizon was too short go on
        const long long clk0 = clock64();
        const uint8_t *frag = B.frag + rd->frag_off;
        uint32_t *state = B.state + rd->frag_off;
        unsigned int *ctime = B.ctime + rd->frag_off;
        const int *kidx = B.kidx + rd->frag_off;
        uint2 *chlog = B.chlog + rd->log_off;
        const int frag_len = rd->frag_len;
        const unsigned long long read = B.read_index[r];
        const double target = B.target[r];
        const double fl = (double)frag_len;
        const int max_kmer_index = frag_len - 1 - k;
        const long long limit = 100ll * frag_len;  // loop_count > 100 * frag_len stops the loop (simulate.py:279)
        const double cc_limit = __dmul_rn(0.9, fl);
        const int horizon = rd->horizon;
        if (threadIdx.x == 0) {
            int stop = -1;
            if (__dmul_rn(fl, __dsub_rn(1.0, target)) < 0.5) stop = BB_STOP_NOLOOP;  // simulate.py:274
            else if ((double)rd->n_logged > cc_limit) stop = BB_STOP_COUNT;
            s_stop = stop; s_cc = rd->n_logged; s_n0 = rd->n_resume;
        }
        __syncthreads();
        // every thread follows n0 in a register: it advances by NE per step for as long as the loop goes on (warp 0
        // rewrites s_n0 while the evaluators are at work)
        long long n0 = s_n0;
        auto evaluate = [&](long long first, int buf) {
            const long long n = first + ev;
            int kind = 0, pos_i = 0, rpos = 0;
            uint32_t payload = 0;
            if (n < limit) bb_eval_iteration(em, frag, kidx, max_kmer_index, seed, read, (unsigned int)n, kind, pos_i, payload, rpos);
            s_kind[buf][ev] = kind; s_pos[buf][ev] = pos_i; s_rpos[buf][ev] = rpos; s_pay[buf][ev] = payload;
        };
        int cur = 0;
        if (s_stop < 0 && warp > 0) evaluate(n0, 0);
        __syncthreads();
        while (s_stop < 0) {
            if (warp > 0) evaluate(n0 + NE, cur ^ 1);   // one step ahead
            else if (n0 >= limit) {
                if (lane == 0) s_stop = BB_STOP_LIMIT;
            } else {
                int change_count = s_cc, stop = -1;
                long long next_n0 = n0 + NE;
                for (int g = 0; g < BB_WARPS_PER_CTA && stop < 0; g++) {
                    uint32_t cmask = __ballot_sync(BB_FULL, s_kind[cur][32 * g + lane] != 0);
                    while (cmask) {
                        const int L = 32 * g + __ffs(cmask) - 1;
                        cmask &= cmask - 1;
                        const long long nL = n0 + L;
                        if (change_count >= horizon) { stop = BB_STOP_HORIZON; next_n0 = nL; break; }  // pause at an iteration top
                        const int bi = s_pos[cur][L], bkind = s_kind[cur][L], brpos = s_rpos[cur][L];
                        const uint32_t bpay = s_pay[cur][L];
                        uint32_t enc = 0;
                        bool app = false;
                        if (lane < k) {
                            const uint8_t fb = frag[bi + lane];
                            enc = bkind == 1 ? em.slots[(long long)bpay * k + lane]
                                             : (lane == brpos ? bpay : bb_slot_inline(1, fb, 0));
                            const bool differs = !((enc & 0xff) == 1 && ((enc >> 8) & 0xff) == fb);
                            app = differs && state[bi + lane] == BB_SLOT_NONE;  // simulate.py:309
                        }
                        const uint32_t amask = __ballot_sync(BB_FULL, app);
                        if (app) {  // slots of one k-mer are distinct positions: applied together, ordinals in slot order
                            const int ord = change_count + __popc(amask & ((1u << lane) - 1u)) + 1;
                            state[bi + lane] = enc;
                            ctime[bi + lane] = (unsigned int)ord;
                            chlog[ord - 1] = make_uint2((unsigned int)nL, (unsigned int)(bi + lane) | ((enc & 0xffu) << 24));
                        }
                        change_count += __popc(amask);
                        __syncwarp();
                        // the guard at the top of the next iteration (simulate.py:285) can only change after a commit
                        if ((double)change_count > cc_limit) { stop = BB_STOP_COUNT; next_n0 = nL + 1; break; }
                    }
                }
                __syncwarp();
                if (lane == 0) { s_cc = change_count; s_stop = stop; s_n0 = next_n0; }
            }
            __syncthreads();
            cur ^= 1;
            n0 += NE;
        }
        if (threadIdx.x == 0) {
            rd->n_logged = s_cc;
            rd->n_resume = (int)(s_n0 > 0x7fffffff ? 0x7fffffff : s_n0);
            rd->stop_reason = s_stop;
            rd->kc_loop += (int)((clock64() - clk0) >> 10);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ mutate (latency build)
// The same loop as bb_k_mutate for the reads whose dependent chain of stages bounds the step: the HEAD batch of the
// longest reads (bb_batch_upload).  bb_k_mutate commits a change with a global round trip (~1 us each, thousands of
// them in a row for a 150 kb read) but has the higher throughput when tens of CTAs share an SM; this build takes the
// round trips out of the serial part:
// One CTA (4 warps) per read.  A step covers BB_MUT_ITERS consecutive loop iterations:
//   1. every thread evaluates its iterations (position, k-mer row, model draw: chains of dependent loads, independent
//      across iterations);
//   2. the iterations that change something are compacted, in order, into a candidate list;
//   3. all threads prefetch what committing a candidate needs - the k encoded slot strings, whether each differs from
//      the original base, whether the slot is still pristine - into shared memory, k lanes per candidate;
//   4. warp 0 commits the candidates in iteration order out of shared memory.  A slot rewritten earlier in the same
//      step is recognised through a small position bitmap and re-read from global memory (the only serial loads left).
// The commit is the reference's `if new_fragment_bases[i+j] is None` (simulate.py:309) in iteration order: identical
// results, but the serial part costs tens of nanoseconds per change instead of a global round trip.
#define BB_MUT_IPT 2                                        // iterations per thread and step
#define BB_MUT_ITERS (BB_WARPS_PER_CTA * 32 * BB_MUT_IPT)   // iterations per step
#define BB_MUT_KMAX 16                                      // slots per candidate in shared memory (k <= 16)
#define BB_MUT_DIRTY_WORDS 128                              // bitmap over positions mod 4096

template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_WARPS_PER_CTA * 32)
bb_k_mutate_chain(BBBatchDev B, BBErrorModelDev em, unsigned long long seed, int *work_counter, const int *order,
            int n_items) {
    constexpr int NT = BB_WARPS_PER_CTA * 32, NI = BB_MUT_ITERS, NG = NI / 32;
    __shared__ int s_pos[NI];
    __shared__ uint32_t s_pay[NI];
    __shared__ uint8_t s_kind[NI], s_rpos[NI];
    __shared__ unsigned short s_cidx[NI];
    __shared__ uint32_t s_enc[NI][BB_MUT_KMAX];
    __shared__ uint8_t s_flag[NI][BB_MUT_KMAX];   // 0: same as the original base, 1: differs but the slot is taken, 2: differs, pristine
    __shared__ uint32_t s_dirty[BB_MUT_DIRTY_WORDS];
    __shared__ int s_gcount[NG];
    __shared__ int s_w, s_stop, s_cc, s_ncand;
    __shared__ long long s_n0;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int k = em.k;
    for (;;) {
        if (threadIdx.x == 0) s_w = atomicAdd(work_counter, 1);
        __syncthreads();
        const int w = s_w;
        __syncthreads();
        if (w >= n_items) break;
        const int r = order[w];
        BBReadDev *rd = &B.reads[r];
        if (rd->status == BB_READ_DONE) continue;  // later rounds: only reads whose horizon was too short go on
        const long long clk0 = clock64();
        const uint8_t *frag = B.frag + rd->frag_off;
        uint32_t *state = B.state + rd->frag_off;
        unsigned int *ctime = B.ctime + rd->frag_off;
        const int *kidx = B.kidx + rd->frag_off;
        uint2 *chlog = B.chlog + rd->log_off;
        const int frag_len = rd->frag_len;
        const unsigned long long read = B.read_index[r];
        const double target = B.target[r];
        const double fl = (double)frag_len;
        const int max_kmer_index = frag_len - 1 - k;
        const long long limit = 100ll * frag_len;  // loop_count > 100 * frag_len stops the loop (simulate.py:279)
        const double cc_limit = __dmul_rn(0.9, fl);
        const int horizon = rd->horizon;
        if (threadIdx.x == 0) {
            int stop = -1;
            if (__dmul_rn(fl, __dsub_rn(1.0, target)) < 0.5) stop = BB_STOP_NOLOOP;  // simulate.py:274
            else if ((double)rd->n_logged > cc_limit) stop = BB_STOP_COUNT;
            s_stop = stop; s_cc = rd->n_logged; s_n0 = rd->n_resume;
        }
        __syncthreads();
        while (s_stop < 0) {
            const long long n0 = s_n0;
            if (n0 >= limit) {
                __syncthreads();
                if (threadIdx.x == 0) s_stop = BB_STOP_LIMIT;
                __syncthreads();
                break;
            }
            // 1. evaluate: slot i of the step is iteration n0 + i; thread t owns slots t, t + NT, ...
#pragma unroll
            for (int j = 0; j < BB_MUT_IPT; j++) {
                const int i = j * NT + threadIdx.x;
                const long long n = n0 + i;
                int kind = 0, pos_i = 0, rpos = 0;
                uint32_t payload = 0;
                if (n < limit) bb_eval_iteration(em, frag, kidx, max_kmer_index, seed, read, (unsigned int)n, kind, pos_i, payload, rpos);
                s_kind[i] = (uint8_t)kind; s_pos[i] = pos_i; s_rpos[i] = (uint8_t)rpos; s_pay[i] = payload;
            }
            if (threadIdx.x < BB_MUT_DIRTY_WORDS) s_dirty[threadIdx.x] = 0u;
            __syncthreads();
            // 2. candidate list in iteration order
            for (int g = warp; g < NG; g += BB_WARPS_PER_CTA) {
                const uint32_t m = __ballot_sync(BB_FULL, s_kind[32 * g + lane] != 0);
                if (lane == 0) s_gcount[g] = __popc(m);
            }
            __syncthreads();
            for (int g = warp; g < NG; g += BB_WARPS_PER_CTA) {
                int off = 0;
                for (int h = 0; h < g; h++) off += s_gcount[h];
                const bool c = s_kind[32 * g + lane] != 0;
                const uint32_t m = __ballot_sync(BB_FULL, c);
                if (c) s_cidx[off + __popc(m & ((1u << lane) - 1u))] = (unsigned short)(32 * g + lane);
                if (g == NG - 1 && lane == 0) s_ncand = off + __popc(m);
            }
            __syncthreads();
            const int ncand = s_ncand;
            // 3. prefetch, BB_MUT_KMAX lanes per candidate
            for (int c = threadIdx.x / BB_MUT_KMAX; c < ncand; c += NT / BB_MUT_KMAX) {
                const int l = threadIdx.x % BB_MUT_KMAX;
                if (l < k) {
                    const int i = s_cidx[c];
                    const int bi = s_pos[i];
                    const uint8_t fb = frag[bi + l];
                    const uint32_t enc = s_kind[i] == 1 ? em.slots[(long long)s_pay[i] * k + l]
                                                        : (l == s_rpos[i] ? s_pay[i] : bb_slot_inline(1, fb, 0));
                    const bool differs = !((enc & 0xff) == 1 && ((enc >> 8) & 0xff) == fb);
                    s_enc[c][l] = enc;
                    s_flag[c][l] = differs ? (state[bi + l] == BB_SLOT_NONE ? 2 : 1) : 0;
                }
            }
            __syncthreads();
            // 4. ordered commit by warp 0
            if (warp == 0) {
                int change_count = s_cc, stop = -1;
                long long next_n0 = n0 + NI;
                for (int c = 0; c < ncand; c++) {
                    const int i = s_cidx[c];
                    const long long nL = n0 + i;
                    if (change_count >= horizon) { stop = BB_STOP_HORIZON; next_n0 = nL; break; }  // pause at an iteration top
                    const int bi = s_pos[i];
                    uint32_t enc = 0;
                    bool app = false;
                    if (lane < k) {
                        const int pos = bi + lane;
                        enc = s_enc[c][lane];
                        const int fg = s_flag[c][lane];
                        if (fg) {
                            const bool dirty = (s_dirty[(pos >> 5) & (BB_MUT_DIRTY_WORDS - 1)] >> (pos & 31)) & 1u;
                            app = dirty ? (state[pos] == BB_SLOT_NONE) : (fg == 2);  // simulate.py:309
                        }
                    }
                    const uint32_t amask = __ballot_sync(BB_FULL, app);
                    if (app) {  // slots of one k-mer are distinct positions: applied together, ordinals in slot order
                        const int pos = bi + lane;
                        const int ord = change_count + __popc(amask & ((1u << lane) - 1u)) + 1;
                        state[pos] = enc;
                        ctime[pos] = (unsigned int)ord;
                        chlog[ord - 1] = make_uint2((unsigned int)nL, (unsigned int)pos | ((enc & 0xffu) << 24));
                        atomicOr(&s_dirty[(pos >> 5) & (BB_MUT_DIRTY_WORDS - 1)], 1u << (pos & 31));
                    }
                    change_count += __popc(amask);
                    __syncwarp();
                    // the guard at the top of the next iteration (simulate.py:285) can only change after a commit
                    if ((double)change_count > cc_limit) { stop = BB_STOP_COUNT; next_n0 = nL + 1; break; }
                }
                __syncwarp();  // every lane has read s_cc / s_n0 before lane 0 replaces them
                if (lane == 0) { s_cc = change_count; s_stop = stop; s_n0 = next_n0; }
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            rd->n_logged = s_cc;
            rd->n_resume = (int)(s_n0 > 0x7fffffff ? 0x7fffffff : s_n0);
            rd->stop_reason = s_stop;
            rd->kc_loop += (int)((clock64() - clk0) >> 10);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ window task list
// One thread per read: the identity re-measurements its newly logged changes call for ("after 25 a changes", a from
// a_done + 1 to n_logged / 25) become tasks.  Built on the device so that a round of the loop needs no host round trip.
template <int BB_TU_ = 0>
__global__ void __launch_bounds__(256)
bb_k_window_tasks(BBBatchDev B, const int *order, int n_items, BBWinTask *tasks, int *n_tasks) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_items) return;
    const int r = order[w];
    const BBReadDev *rd = &B.reads[r];
    if (rd->status == BB_READ_DONE) return;
    const int a0 = rd->a_done + 1, a1 = rd->n_logged / BB_ALIGNMENT_INTERVAL;
    if (a1 < a0) return;
    const int base = atomicAdd(n_tasks, a1 - a0 + 1);
    for (int a = a0; a <= a1; a++) tasks[base + a - a0] = BBWinTask{r, a};
}

// ------------------------------------------------------------------------------------------------ window alignments
// The window of identity re-measurement `a` of a read (simulate.py:325-346): position and length.
__device__ __forceinline__ void bb_window_of(int frag_len, unsigned long long seed, unsigned long long read, int a,
                                             int &qpos, int &qn) {
    qpos = 0; qn = frag_len;
    if (frag_len > BB_ALIGNMENT_SIZE) {
        BBRng wr;
        wr.init(seed, read);
        wr.stream(BB_PURPOSE_WINDOW, (uint32_t)(a - 1));
        qpos = (int)wr.randbelow((uint32_t)(frag_len - BB_ALIGNMENT_SIZE + 1));
        qn = BB_ALIGNMENT_SIZE;
    }
}

// One window alignment per thread, 32 at a time per warp in lock step: join -> forward pass -> traceback.
// The forward pass keeps no per-column history.  It saves the lane's vertical deltas every BB_WIN_TILE columns (a
// checkpoint: 2 LW + 2 words); the traceback walks the tiles from the last to the first, re-running each tile's columns
// from its checkpoint into SHARED memory (per-column vertical / horizontal delta words, the two bits per cell edlib's
// traceback rule needs) and following the path through it.  Round 1 wrote 8 LW bytes per column per window to global
// memory and read them back along the path, with the traceback stalled on those loads most of the time; now a window
// moves ~9 KB.
#define BB_WIN_TILE 16
#define BB_WIN_CKPT_WORDS(LW) (2 * (LW) + 2)
#define BB_WIN_MAX_TILES (BB_WIN_MAX_COLS / BB_WIN_TILE)
#define BB_WIN_SMEM_BYTES(LW) (BB_WIN_TILE * (LW) * 64 * 8)

template <int LW>
__global__ void __launch_bounds__(64, (LW <= 4 ? 6 : 3))
bb_k_window_lane(BBBatchDev B, BBErrorModelDev em, const BBWinTask *tasks, const int *n_tasks_ptr, unsigned long long seed,
                 uint32_t *ckpt_pool, uint8_t *tbuf_pool, int *cursor, BBWinTask *fallback, int *fallback_count) {
#ifdef BB_EMULATOR
    static uint2 s_hist[BB_WIN_TILE * LW * 64];
#else
    extern __shared__ __align__(16) uint2 s_hist[];  // [column in tile][word][thread]
#endif
    constexpr int CKW = BB_WIN_CKPT_WORDS(LW);
    const int n_tasks = *n_tasks_ptr;
    const long long gl = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *const ckpt = ckpt_pool + gl * (long long)(BB_WIN_MAX_TILES * CKW);
    uint8_t *const tbuf = tbuf_pool + gl * (long long)BB_WIN_MAX_COLS;
    uint2 *const hs = s_hist + threadIdx.x;
    for (;;) {
        const int w = atomicAdd(cursor, 1);
        bool active = w < n_tasks;
        if (!__any_sync(BB_FULL, active)) break;
        BBWinTask tk = {0, 0};
        const BBReadDev *rd = nullptr;
        const uint8_t *frag = nullptr;
        const uint32_t *state = nullptr;
        const unsigned int *ctime = nullptr;
        int qpos = 0, qn = 0;
        unsigned int tmax = 0;
        if (active) {
            tk = tasks[w];
            rd = &B.reads[tk.r];
            frag = B.frag + rd->frag_off; state = B.state + rd->frag_off; ctime = B.ctime + rd->frag_off;
            bb_window_of(rd->frag_len, seed, B.read_index[tk.r], tk.a, qpos, qn);
            tmax = (unsigned int)(BB_ALIGNMENT_INTERVAL * tk.a);
        }
        // ---- join: ''.join(new_fragment_bases[pos:pos2]) as it was after 25*a changes
        int tm = 0, uw = 0;
        const int qn_max = __reduce_max_sync(BB_FULL, qn);
        for (int j0 = 0; j0 < qn_max; j0 += 4) {
            if (active && j0 < qn) {
                unsigned int ct4[4];
                uint8_t fb4[4];
#pragma unroll
                for (int h = 0; h < 4; h++) {  // four slots per iteration: their loads are issued together
                    const int j = min(j0 + h, qn - 1);
                    ct4[h] = ctime[qpos + j];
                    fb4[h] = frag[qpos + j];
                }
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    if (j0 + h < qn) {
                        if (ct4[h] == 0u || ct4[h] > tmax) { if (tm < BB_WIN_MAX_COLS) tbuf[tm] = fb4[h]; tm++; }
                        else {
                            const uint32_t st = state[qpos + j0 + h];
                            const int sl = (int)(st & 0xff);
                            for (int c = 0; c < sl; c++) { if (tm < BB_WIN_MAX_COLS) tbuf[tm] = bb_slot_char(em, st, c); tm++; }
                            uw += sl < 1 ? 1 : sl;
                        }
                    }
                }
            }
        }
        BBProb P;
        P.a = 0; P.b = 1;
        if (active) {
            const int diff = qn > tm ? qn - tm : tm - qn;
            if (uw < diff) uw = diff;
            const int mx = qn > tm ? qn : tm;
            if (uw > mx) uw = mx;
            bb_band(qn, tm, uw, P.a, P.b);
            if (tm > BB_WIN_MAX_COLS || bb_lane_words(P.a, P.b) > LW || !bb_uses_traceback(qn, tm)) {
                fallback[atomicAdd(fallback_count, 1)] = tk;  // the next kernel handles this window
                active = false;
            }
        }
        if (!active) tm = 0;
        // ---- forward pass, a checkpoint every BB_WIN_TILE columns
        BBLanePass<LW> S;
        if (active) {
            P.n = qn; P.peq = B.fpeq + rd->fpeq_off; P.q = frag + qpos; P.qs = 1;
            P.peq_bit0 = qpos + BB_PEQ_BIT0; P.t = tbuf; P.ts = 1;
            bb_lane_begin<LW>(S, P);
        }
        const int tm_max = __reduce_max_sync(BB_FULL, tm);
        for (int c = 0; c < tm_max; c++) {
            if (c < tm) {
                if ((c & (BB_WIN_TILE - 1)) == 0) {
                    uint32_t *ck = ckpt + (c / BB_WIN_TILE) * CKW;
#pragma unroll
                    for (int x = 0; x < LW; x++) { ck[x] = S.Pv[x]; ck[LW + x] = S.Mv[x]; }
                    ck[2 * LW] = (uint32_t)S.wt; ck[2 * LW + 1] = (uint32_t)S.score;
                }
                bb_lane_step<LW, false>(S, P, nullptr);
            }
        }
        // ---- traceback (edlib's rule: 'I' > 'D' > diagonal), tile by tile, counting '=' and 'D' columns
        int ti = qn - 1, tj = tm - 1, matches = 0, dels = 0;
        bool walking = active && ti >= 0 && tj >= 0;
        bool need_tile = walking;
        int tile_lo = 0;
        // (every round moves every walking lane at least once: qn + tm rounds bound the loop whatever the data)
        for (int round = 0; round < 2 * BB_WIN_MAX_COLS + 64 && __any_sync(BB_FULL, walking); round++) {
            if (walking && need_tile) {  // all walking lanes get here together (see the inner loop's exit)
                const int tile = tj / BB_WIN_TILE;
                tile_lo = tile * BB_WIN_TILE;
                const uint32_t *ck = ckpt + tile * CKW;
#pragma unroll
                for (int x = 0; x < LW; x++) { S.Pv[x] = ck[x]; S.Mv[x] = ck[LW + x]; }
                S.wt = (int)ck[2 * LW]; S.score = (int)ck[2 * LW + 1]; S.c = tile_lo;
#pragma unroll
                for (int x = 0; x < LW; x++) bb_fetch_peq(P, 32 * (S.wt + x), S.eA[x], S.eC[x], S.eG[x], S.eT[x]);
                const int hi = min(tile_lo + BB_WIN_TILE, tm);
                for (int c = tile_lo; c < hi; c++) bb_lane_step<LW, true, 64>(S, P, hs + ((c - tile_lo) * LW) * 64);
                need_tile = false;
            }
            for (int mv = 0; mv < 64; mv++) {
                const bool can = walking && !need_tile;
                if (!__any_sync(BB_FULL, can)) break;
                if (can) {
                    int wt = (tj - P.a) >> 5; if (wt < 0) wt = 0;
                    const int x = (ti >> 5) - wt;
                    if (x < 0 || x >= LW) { atomicOr(&B.reads[tk.r].flags, 1); ti = -1; tj = -1; }
                    else {
                        const uint2 e = hs[((tj - tile_lo) * LW + x) * 64];
                        const int bit = ti & 31;
                        if ((e.x >> bit) & 1u) ti--;
                        else if ((e.y >> bit) & 1u) { dels++; tj--; }
                        else { matches += (frag[qpos + ti] == tbuf[tj]) ? 1 : 0; ti--; tj--; }
                    }
                    if (ti < 0 || tj < 0) walking = false;
                    else if (tj < tile_lo) need_tile = true;
                }
            }
        }
        if (active) {
            if (walking) atomicOr(&B.reads[tk.r].flags, 1);  // cannot happen: the round bound above was hit
            if (tj >= 0) dels += tj + 1;
            B.wres[rd->wres_off + tk.a - 1] = make_int2(matches, qn + dels);
        }
    }
}

// The DEFAULT window aligner: one window alignment per thread; persistent lanes, all on the same step of the same phase;
// per-column history (Pv, PhRaw of the band slice, bb_lane_step) in global memory.  The traceback does not chase it
// there: the columns ahead of the path are staged in shared memory by cp.async, T columns per tick (bb_ring_tick), so a
// move costs a shared-memory load instead of an L2 / HBM round trip.  The checkpoint build above (BADREAD_B200_LOWMEM=1)
// moves ~9 KB per window instead of up to ~48 KB and is slower per step: recomputing tiles costs more than the traffic
// it saves.
#ifndef BB_WIN_RING_T
#define BB_WIN_RING_T 4
#endif
template <int LW, int T = BB_WIN_RING_T>
__global__ void __launch_bounds__(64, (LW <= 4 ? 8 : 4))
bb_k_window_lane_hist(BBBatchDev B, BBErrorModelDev em, const BBWinTask *tasks, const int *n_tasks_ptr, unsigned long long seed,
                 uint2 *hist_pool, uint8_t *tbuf_pool, int *cursor, BBWinTask *fallback, int *fallback_count) {
#ifdef BB_EMULATOR
    static uint2 s_ring[BB_RING_BYTES(LW, T) / 8];
#else
    extern __shared__ __align__(16) uint2 s_ring[];  // BB_RING_BYTES(LW, T): [column mod 2T][word][thread]
#endif
    const int n_tasks = *n_tasks_ptr;
    const long long gl = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    uint2 *const hist = hist_pool + gl * (long long)(BB_WIN_MAX_COLS * (LW - 1));
    uint8_t *const tbuf = tbuf_pool + gl * (long long)BB_WIN_MAX_COLS;
    uint2 *const ring = s_ring + threadIdx.x;
    BBLanePass<LW> S;
    BBProb P;
    BBWinTask tk = {0, 0};
    const uint8_t *frag = nullptr;
    const uint32_t *state = nullptr;
    const unsigned int *ctime = nullptr;
    int phase = 0;  // 0: fetch, 1: join, 2: forward pass, 3: traceback, 4: done
    int qpos = 0, qn = 0, jx = 0, tm = 0, uw = 0, ti = 0, tj = 0, diags = 0, dels = 0, dist = 0, staged_lo = 0, bw = 1;
    unsigned int tmax = 0;
    for (;;) {
        if (phase == 0) {
            const int w = atomicAdd(cursor, 1);
            if (w >= n_tasks) phase = 4;
            else {
                tk = tasks[w];
                const BBReadDev *rd = &B.reads[tk.r];
                frag = B.frag + rd->frag_off; state = B.state + rd->frag_off; ctime = B.ctime + rd->frag_off;
                bb_window_of(rd->frag_len, seed, B.read_index[tk.r], tk.a, qpos, qn);
                tmax = (unsigned int)(BB_ALIGNMENT_INTERVAL * tk.a);
                jx = 0; tm = 0; uw = 0;
                phase = 1;
            }
        }
        if (__all_sync(BB_FULL, phase == 4)) break;
        for (int it = 0; it < 64; it++) {  // ''.join(new_fragment_bases[pos:pos2]) as it was after 25*a changes
            if (phase == 1) {
                // four slots per iteration: their loads are issued together, the (serial) appends follow
                unsigned int ct4[4];
                uint8_t fb4[4];
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    const int j = min(jx + h, qn - 1);
                    ct4[h] = ctime[qpos + j];
                    fb4[h] = frag[qpos + j];
                }
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    if (jx < qn) {
                        if (ct4[h] == 0u || ct4[h] > tmax) { if (tm < BB_WIN_MAX_COLS) tbuf[tm] = fb4[h]; tm++; }
                        else {
                            const uint32_t st = state[qpos + jx];
                            const int sl = (int)(st & 0xff);
                            for (int c = 0; c < sl; c++) { if (tm < BB_WIN_MAX_COLS) tbuf[tm] = bb_slot_char(em, st, c); tm++; }
                            uw += sl < 1 ? 1 : sl;
                        }
                        jx++;
                    }
                }
                if (jx >= qn) {
                    const int diff = qn > tm ? qn - tm : tm - qn;
                    if (uw < diff) uw = diff;
                    const int mx = qn > tm ? qn : tm;
                    if (uw > mx) uw = mx;
                    bb_band(qn, tm, uw, P.a, P.b);
                    if (tm > BB_WIN_MAX_COLS || bb_lane_words(P.a, P.b) > LW || !bb_uses_traceback(qn, tm)) {
                        fallback[atomicAdd(fallback_count, 1)] = tk;  // the warp kernel handles this window
                        phase = 0;
                    } else {
                        const BBReadDev *rd = &B.reads[tk.r];
                        P.n = qn; P.peq = B.fpeq + rd->fpeq_off; P.q = frag + qpos; P.qs = 1;
                        P.peq_bit0 = qpos + BB_PEQ_BIT0; P.t = tbuf; P.ts = 1;
                        bb_lane_begin<LW>(S, P);
                        bw = bb_band_words(P.a, P.b);
                        phase = 2;
                    }
                }
            }
        }
        for (int it = 0; it < 128; it++) {  // forward columns with history
            if (phase == 2) {
                bb_lane_step<LW, true>(S, P, hist + (long long)S.c * bw);
                if (S.c >= tm) {
                    // '=' columns without looking at the characters again: the path's 'X' columns are the edit distance
                    // minus its 'I' and 'D' columns, and the diagonal moves are '=' or 'X'
                    dist = bb_lane_corner<LW>(S, qn);
                    ti = qn - 1; tj = tm - 1; diags = 0; dels = 0; staged_lo = tm; phase = 3;
                }
            }
        }
        for (int it = 0; it < 256; it++) {  // traceback (edlib's rule), counting '=' and 'D' columns
            if (phase == 3) {
                if (ti >= 0 && tj >= 0) {
                    // (it is the same for all lanes: the walking lanes of the warp tick together)
                    if ((it & (T - 1)) == 0) bb_ring_tick<LW - 1, T>(ring, hist, bw, tj, staged_lo);
                    const int k = ti - max(0, tj - P.a);  // row in the band slice of column tj
                    if (k < 0 || k >= 32 * bw) { atomicOr(&B.reads[tk.r].flags, 1); ti = -1; tj = -1; }
                    else {
                        const uint2 e = bb_ring_entry<LW - 1, T>(ring, tj, k >> 5);
                        const int bit = k & 31;
                        if ((e.x >> bit) & 1u) ti--;
                        else if ((e.y >> bit) & 1u) { dels++; tj--; }
                        else { diags++; ti--; tj--; }
                    }
                } else {
                    bb_cp_async_wait<0>();  // nothing of this walk may land in the ring after the next walk's copies
                    if (tj >= 0) dels += tj + 1;
                    // rows = diagonal + 'I' moves, so 'I' = qn - diags; 'X' = dist - 'I' - 'D'
                    const int matches = diags - (dist - (qn - diags) - dels);
                    if (dist >= BB_INF) atomicOr(&B.reads[tk.r].flags, 1);
                    B.wres[B.reads[tk.r].wres_off + tk.a - 1] = make_int2(matches, qn + dels);
                    phase = 0;
                }
            }
        }
    }
}

// Windows beyond the lane limits: one warp each, with the general aligner.
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(BB_WARPS_PER_CTA * 32, 4)
bb_k_window_warp(BBBatchDev B, BBErrorModelDev em, BBScratchPool pool, const BBWinTask *tasks, const int *n_tasks_ptr,
                 unsigned long long seed, int *cursor) {
    const int lane = threadIdx.x & 31;
    const int warp = blockIdx.x * BB_WARPS_PER_CTA + (threadIdx.x >> 5);
    BBScratch sc = pool.for_warp(warp);
    uint8_t *tbuf = pool.tbuf + (long long)warp * pool.tbuf_stride;
    const int n_tasks = *n_tasks_ptr;
    BBEmit no_emit = {nullptr, nullptr, nullptr};
    for (;;) {
        int w = 0;
        if (lane == 0) w = atomicAdd(cursor, 1);
        w = __shfl_sync(BB_FULL, w, 0);
        if (w >= n_tasks) break;
        const BBWinTask tk = tasks[w];
        BBReadDev *rd = &B.reads[tk.r];
        const uint8_t *frag = B.frag + rd->frag_off;
        const uint32_t *state = B.state + rd->frag_off;
        const unsigned int *ctime = B.ctime + rd->frag_off;
        int qpos, qn;
        bb_window_of(rd->frag_len, seed, B.read_index[tk.r], tk.a, qpos, qn);
        const unsigned int tmax = (unsigned int)(BB_ALIGNMENT_INTERVAL * tk.a);
        // warp-cooperative join of the snapshot
        int total = 0, up = 0;
        for (int base = 0; base < qn; base += 32) {
            const int x = base + lane;
            uint32_t st = BB_SLOT_NONE;
            int len = 0;
            if (x < qn) {
                const unsigned int ct = ctime[qpos + x];
                if (ct != 0u && ct <= tmax) st = state[qpos + x];
                len = st == BB_SLOT_NONE ? 1 : (int)(st & 0xff);
            }
            int incl = len;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(BB_FULL, incl, d);
                if (lane >= d) incl += v;
            }
            const int off = total + incl - len;
            if (x < qn) {
                if (st == BB_SLOT_NONE) tbuf[off] = frag[qpos + x];
                else {
                    for (int c = 0; c < len; c++) tbuf[off + c] = bb_slot_char(em, st, c);
                    up += len < 1 ? 1 : len;
                }
            }
            total += __shfl_sync(BB_FULL, incl, 31);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) up += __shfl_xor_sync(BB_FULL, up, d);
        __syncwarp();
        sc.peq = B.fpeq + rd->fpeq_off;
        BBAlnCounts cnt = {0, 0, 0, 0};
        bb_align<false, 1>(frag + qpos, qn, tbuf, total, up, sc, no_emit, qpos, cnt);
        __syncwarp();
        if (lane == 0) {
            if (cnt.err) atomicOr(&rd->flags, cnt.err);
            B.wres[rd->wres_off + tk.a - 1] = make_int2(cnt.matches, qn + cnt.dels);
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------ replay
// One warp per read: the scalar recurrence of simulate.py:290-346 over the change log.  The recurrence itself is serial
// (every lane computes it redundantly); the log is read 32 entries at a time, coalesced, and handed round by shuffles,
// so the dependent chain of a long read is arithmetic only.
template <int BB_TU_ = 0>  // a template: only the translation unit that launches it compiles it
__global__ void __launch_bounds__(128)
bb_k_replay(BBBatchDev B, const int *order, int n_items, int k, int *n_pending) {
    const int lane = threadIdx.x & 31;
    const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= n_items) return;
    const int r = order[w];
    BBReadDev *rd = &B.reads[r];
    if (rd->status == BB_READ_DONE) return;
    uint32_t *state = B.state + rd->frag_off;
    const uint2 *chlog = B.chlog + rd->log_off;
    const int2 *wres = B.wres + rd->wres_off;
    const int frag_len = rd->frag_len;
    const double target = B.target[r];
    const double fl = (double)frag_len;
    const double cc_limit = __dmul_rn(0.9, fl);
    const long long limit = 100ll * frag_len;
    const int n_logged = rd->n_logged;
    const int stop_reason = rd->stop_reason, n_resume = rd->n_resume;
    double errors = 0.0, est_id = 1.0, scale = 1.0;
    int total = frag_len, st_trim = k, en_trim = k, upper = 0;
    long long loop_count = -1;
    int kstop = n_logged;  // changes that survive
    bool stopped = false;
    if (stop_reason == BB_STOP_NOLOOP) { stopped = true; loop_count = 0; kstop = 0; }
    else if (1.0 <= target) { stopped = true; loop_count = 1; kstop = 0; }  // first check of the first iteration
    long long cur_n = -1;  // iteration whose changes are being applied (-1: none yet)
    // the checks at the top of iteration cur_n + 1 (simulate.py:278-292), after `c` changes
    auto close_group = [&](int c) {
        est_id = __dsub_rn(1.0, __ddiv_rn(errors, fl));
        if (cur_n + 1 >= limit) { stopped = true; loop_count = limit + 1; kstop = c; }
        else if ((double)c > cc_limit || est_id <= target) { stopped = true; loop_count = cur_n + 2; kstop = c; }
    };
    for (int c0 = 0; c0 < n_logged && !stopped; c0 += 32) {
        uint2 mine = make_uint2(0u, 0u);
        if (c0 + lane < n_logged) mine = chlog[c0 + lane];
        const int m = min(32, n_logged - c0);
        for (int j = 0; j < m && !stopped; j++) {
            const unsigned int n = __shfl_sync(BB_FULL, mine.x, j);
            const unsigned int py = __shfl_sync(BB_FULL, mine.y, j);
            int c = c0 + j;  // changes applied before this one
            if ((long long)n != cur_n) {
                if (cur_n >= 0) { close_group(c); if (stopped) break; }
                cur_n = n;
                // all changes of one iteration use est_id from the top of that iteration (simulate.py:290,321)
                scale = __dmul_rn(est_id, __dsqrt_rn(est_id));
            }
            const int pos = (int)(py & 0xffffffu), len = (int)(py >> 24);
            c++;
            upper += len < 1 ? 1 : len;
            total += len - 1;
            if (pos < k) st_trim += len - 1;
            if (pos >= frag_len - k) en_trim += len - 1;
            errors = __dadd_rn(errors, __dmul_rn((double)(len < 2 ? 1 : len - 1), scale));
            if (c % BB_ALIGNMENT_INTERVAL == 0) {  // simulate.py:325-346
                const int2 res = wres[c / BB_ALIGNMENT_INTERVAL - 1];
                const double actual = res.y ? __ddiv_rn((double)res.x, (double)res.y) : 0.0;
                if (frag_len <= BB_ALIGNMENT_SIZE) {
                    errors = __dmul_rn(__dsub_rn(1.0, actual), fl);
                } else {
                    const double est_err = __dmul_rn(__dsub_rn(1.0, actual), fl);
                    const double weight = __ddiv_rn((double)BB_ALIGNMENT_SIZE, fl);
                    errors = __dadd_rn(__dmul_rn(est_err, weight), __dmul_rn(errors, __dsub_rn(1.0, weight)));
                }
            }
        }
    }
    if (!stopped && cur_n >= 0) close_group(n_logged);
    if (!stopped) {
        if (stop_reason == BB_STOP_LIMIT) { stopped = true; loop_count = limit + 1; kstop = n_logged; }
        else if (stop_reason == BB_STOP_COUNT) { stopped = true; loop_count = (long long)n_resume + 1; kstop = n_logged; }
    }
    if (!stopped) {  // the horizon was too short: log more changes and come back
        if (lane == 0) {
            rd->horizon = n_logged + max(64, n_logged / 2);
            rd->a_done = n_logged / BB_ALIGNMENT_INTERVAL;
            atomicAdd(n_pending, 1);
        }
        return;
    }
    for (int x = kstop + lane; x < n_logged; x += 32) {  // changes logged past the stop never happened
        state[chlog[x].y & 0xffffffu] = BB_SLOT_NONE;
    }
    if (lane == 0) {
        rd->seq_len = total; rd->start_trim = st_trim; rd->end_trim = en_trim; rd->upper = upper;
        rd->loop_count = (int)(loop_count > 0x7fffffff ? 0x7fffffff : loop_count);
        rd->change_count = kstop; rd->n_align = kstop / BB_ALIGNMENT_INTERVAL;
        rd->status = BB_READ_DONE;
    }
}
