// bb_api.cu — C ABI of libbadread_b200.so (see include/badread_b200.h): context, one-time uploads, batch
// orchestration. All hot-path work is done by the kernels in bb_kernels.cuh; there is no CPU path here.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "bb_kernels.cuh"
#include "bb_launch.h"

namespace {

struct DevBuf {  // grow-only device allocation, freed with its owner
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;  // (so a Worker or a context cannot be copied either)
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ~DevBuf() { release(); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

constexpr int BB_MAX_ROUNDS = 15;  // error-loop rounds a run can enqueue (16 counters each, see BB_ROUND_BASE)
// per-level snapshot of the queue counters (bb_last_run_work): [pipeline][level < BB_MAX_LEVELS][the BBQ_NODE_CLASSES
// node counts; at level 0 also the two leaf counters right after bb_k_push_roots]
constexpr int BB_SNAP_WORDS = 8, BB_SNAP_LEAF = BBQ_NODE_CLASSES;
static_assert(BB_SNAP_LEAF + 2 <= BB_SNAP_WORDS, "snapshot row too short");
static_assert(int(BB_NODE_CLASSES) == int(BBQ_NODE_CLASSES) && int(BB_NODE_LANE8) == int(BBQ_NODE_LANE8) &&
              int(BB_NODE_LEAN1) == int(BBQ_NODE_LEAN1) && int(BB_NODE_LEAN2) == int(BBQ_NODE_LEAN2) &&
              int(BB_NODE_LEAN4) == int(BBQ_NODE_LEAN4) && int(BB_NODE_WIDE) == int(BBQ_NODE_WIDE),
              "bb_node_class must follow the node queues");

// Queue counters of an alignment pipeline: one block of kQueueCounts ints, the BBQ_* counts first, then from
// kCursorBase one work cursor per node / leaf launch (5 per level at most, 2 for the leaves).
constexpr int kQueueCounts = 512, kCursorBase = 16;
static_assert(BBQ_OVERFLOW < kCursorBase && kCursorBase + 5 * BB_MAX_LEVELS + 2 <= kQueueCounts, "queue counter block");

// The single-warp node kernels (4, 2 and 1 words per lane) of both pipelines are resident at once: each launch owns
// a fixed range of warp slots in pool_lean, sized for its grid cap of kLeanCtasPerSm CTAs per SM.
enum { LEAN4, LEAN2, LEAN1 };
constexpr int kLeanCtasPerSm[3] = {4, 6, 6};
constexpr int kLeanCtasPerSmBoth = 2 * (kLeanCtasPerSm[LEAN4] + kLeanCtasPerSm[LEAN2] + kLeanCtasPerSm[LEAN1]);

const char *kStageNames[BB_N_STAGES] = {"build_fragments", "error_loop", "scan", "join", "final_align", "qscores",
                                        "compact", "total"};

enum GridKnob { G_MUTATE, G_WIN4, G_WIN8, G_WARP1, G_WARP2, G_WARP4, G_LANE8, G_LEAF, kGridKnobs };
const char *const kGridNames[kGridKnobs] = {"MUTATE", "WIN4", "WIN8", "WARP1", "WARP2", "WARP4", "LANE8", "LEAF"};

// The BADREAD_B200_* environment variables, read once by bb_create (see README).
struct Knobs {
    bool trace = false;        // TRACE: an event after every launch / host step of a run (bb_trace_dump)
    int n_workers = 2;         // SUBBATCHES
    bool head_priority = true; // HEAD_PRIORITY: worker 0 on high-priority streams
    bool head_worker = true;   // HEAD_WORKER: worker 0 = the longest reads only (see bb_batch_upload)
    int grid_div = 0;          // GRID_DIV: > 0 replaces the share of the SMs the workers of a split batch ask for
    int grid[kGridKnobs] = {}; // GRID_<name>: > 0 replaces the kernel's CTAs per SM
    int lane8_cols = 4096;     // routing limit of the lane node kernel
    int pair_ctas = 1;         // CTAs per SM of the warp-pair node kernel
    bool lpt_order = true;     // node queues below the roots walked from the end (longest nodes first)
    int ring_t = 4;            // columns per traceback tick of the 4-word window aligner (2, 4 or 8)
    bool lowmem = false;       // window / leaf aligners with checkpoints + shared-memory tiles instead of global history
    bool use_quad = false;     // wide nodes by 8-warp CTAs (bb_k_node_quad) instead of warp pairs
    // starting values of the limits w_finish grows when a batch outgrows them (the results do not depend on them);
    // lr_cap > 0: the split-score scratch of a batch starts at this many rows
    int n_rounds = 3, extra_levels = 0, lr_cap = 0;
    double slack = 1.25;
};

Knobs read_knobs() {
    Knobs k;
    auto env = [](const std::string &name) { return std::getenv(("BADREAD_B200_" + name).c_str()); };
    if (const char *e = env("TRACE")) k.trace = (e[0] == '1');
    if (const char *e = env("SUBBATCHES")) k.n_workers = std::max(1, std::min(8, std::atoi(e)));
    if (const char *e = env("HEAD_PRIORITY")) k.head_priority = (e[0] != '0');
    if (const char *e = env("HEAD_WORKER")) k.head_worker = (e[0] != '0');
    if (const char *e = env("GRID_DIV")) k.grid_div = std::atoi(e);
    for (int g = 0; g < kGridKnobs; g++) if (const char *e = env(std::string("GRID_") + kGridNames[g])) k.grid[g] = std::atoi(e);
    if (const char *e = env("LANE8_COLS")) k.lane8_cols = std::atoi(e);
    if (const char *e = env("PAIR_CTAS")) k.pair_ctas = (e[0] == '2') ? 2 : 1;
    if (const char *e = env("LPT")) k.lpt_order = (e[0] != '0');
    if (const char *e = env("RING_T")) k.ring_t = (e[0] == '8') ? 8 : (e[0] == '2') ? 2 : 4;
    if (const char *e = env("LOWMEM")) k.lowmem = (e[0] != '0');
    if (const char *e = env("QUAD")) k.use_quad = (e[0] != '0');
    if (const char *e = env("ROUNDS")) k.n_rounds = std::max(1, std::min(BB_MAX_ROUNDS, std::atoi(e)));
    if (const char *e = env("SLACK")) { const double v = std::atof(e); if (v > 0.0) k.slack = v; }
    if (const char *e = env("EXTRA_LEVELS")) k.extra_levels = std::atoi(e);
    if (const char *e = env("LR_CAP")) k.lr_cap = std::max(0, std::atoi(e));
    return k;
}

// One kernel chain of a context: its streams, the part of the batch it was dealt, and the buffers, scratch and queues
// its kernels run on.  The reference, the models and the knobs are the context's.
struct Worker {
    bb_ctx *ctx;
    cudaStream_t stream = nullptr, stream2 = nullptr;
    cudaStream_t side[2][3] = {};   // per alignment pipeline: the streams of the node classes that run next to the main one
    cudaEvent_t ev_side[2][3] = {}, ev_level[2] = {};
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_scan = nullptr;
    cudaEvent_t ev[BB_N_STAGES + 1] = {};
    std::string err;  // batch uploads run on one host thread per worker
    int64_t launches = 0;

    // batch
    int n_reads = 0;
    bool uploaded = false, ran = false, finished = false;
    bool is_head = false;      // this worker holds the head batch of the current upload
    std::vector<BBReadDev> h_reads;
    std::vector<int32_t> h_inlen;
    std::vector<double> h_target;
    int64_t frag_total = 0;
    int64_t seq_cap = 0, out_cap = 0, speq_cap = 0;  // capacities of the per-batch buffers (from the fragment lengths)
    int64_t log_total = 0, wres_total = 0, fpeq_total = 0;
    int max_len = 0;
    // sizing knobs a retry raises (bb_k_scan / the node kernels flag what did not fit; see w_finish)
    double slack;              // joined reads may be this much longer than their fragments in total
    int n_rounds;              // mutate -> windows -> replay rounds enqueued without asking the device in between
    int n_levels = 0;          // Hirschberg levels enqueued (from the longest fragment)
    int extra_levels;
    bool lr_worst = false;     // size the split-score scratch for the worst case instead of the expected edit count
    struct RunInfo {
        BBScanOut scan; int counters[256]; int qcount[2][32];
        int levels[2][BB_MAX_LEVELS][BB_SNAP_WORDS];  // queue counters at the start of every level (d_levels)
    } *h_info = nullptr;  // pinned
    std::vector<BBReadDev> h_res;  // per-read records of the finished run
    bool reran = false;        // w_finish had to run the batch again (copies enqueued before that are stale)
    int n_reruns = 0;          // runs of the current batch after the first (bb_last_run_retries)
    uint32_t rerun_reasons = 0;  // BB_RERUN_* bits of what did not fit
    DevBuf d_read_index, d_seg_off, d_segs, d_lit, d_target, d_order, d_reads;
    DevBuf d_kidx, d_frag, d_state, d_seq, d_ops, d_dcnt, d_qual, d_out_seq, d_out_qual, d_counter, d_fpeq, d_speq, d_scan;
    DevBuf d_levels;  // int[2][BB_MAX_LEVELS][BB_SNAP_WORDS]: what RunInfo::levels is copied from
    DevBuf d_ctime, d_chlog, d_wres, d_wtasks, d_wfallback;

    // Where the kernels of a run find their share of the queues and scratch (set by w_prepare)
    struct Layout {
        int cap_node = 0;          // entries of every node and leaf queue
        int lane_ctas = 0;         // 64-thread CTAs of the lane leaf kernel of one pipeline (its grid cap)
        size_t hist_per_pipe = 0;  // elements of s_lanehist (s_leafhist with lowmem) that one pipeline's leaf kernel owns
        int64_t fb_len = 0;        // entries of each of the two window fall-back lists in d_wfallback
        int lean_base[2][3] = {};  // first pool_lean slot of each pipeline's LEAN4 / LEAN2 / LEAN1 node kernel
    } L;

    // scratch
    BBScratchPool pool{}, pool_lean{};  // pool_lean: split-score arrays of the single-warp node kernels (bands < 2048 rows)
    DevBuf s_hist, s_hbuf, s_lr, s_stack, s_tbuf, s_peq, s_ltbuf, s_leafhist, s_lr_lean, s_wckpt, s_lanehist;
    DevBuf p_q, p_t, p_ops, p_dcnt, p_out, p_qual;  // single-pair entry points (bb_align_path / bb_get_qscores): kept between calls
    struct QueueBufs { DevBuf node[BBQ_NODE_CLASSES][2], leaf[2], count; } qbuf[2];  // [0] normal, [1] wide-root reads

    // launch trace (BADREAD_B200_TRACE=1): an event after every launch / host step of a run, dumped by bb_trace_dump
    struct Mark { const char *name; int stream; cudaEvent_t ev; };
    std::vector<Mark> marks;
    std::vector<cudaEvent_t> mark_pool;
    size_t mark_used = 0;

    Worker(bb_ctx *c, const Knobs &k) : ctx(c), slack(k.slack), n_rounds(k.n_rounds), extra_levels(k.extra_levels) {}
    ~Worker() {
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : {ev_fork, ev_join, ev_scan, ev_level[0], ev_level[1]}) if (e) cudaEventDestroy(e);
        for (auto &row : ev_side) for (cudaEvent_t e : row) if (e) cudaEventDestroy(e);
        for (cudaStream_t s : {stream, stream2}) if (s) cudaStreamDestroy(s);
        for (auto &row : side) for (cudaStream_t s : row) if (s) cudaStreamDestroy(s);
        for (cudaEvent_t e : mark_pool) cudaEventDestroy(e);
        if (h_info) cudaFreeHost(h_info);
    }
};

// The BGZF compressor of a context (bb_bgzf_compress, bb_bam_compress*): a stream and scratch of its own, so that a call
// leaves the workers alone.
struct Bgzf {
    cudaStream_t stream = nullptr;
    int64_t *h = nullptr;   // pinned: line_pref[n_chunks] and offsets[n_chunks] of the last pass
    DevBuf in, slots, lines, sizes, pref, off, out;
    cudaError_t open() {   // the stream and the pinned words, made by the first call that needs them
        cudaError_t e = stream ? cudaSuccess : cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        if (e == cudaSuccess && !h) e = cudaHostAlloc((void **)&h, 2 * sizeof(int64_t), cudaHostAllocPortable);
        return e;
    }
    ~Bgzf() {
        if (stream) cudaStreamDestroy(stream);
        if (h) cudaFreeHost(h);
    }
};

}  // namespace

struct bb_ctx {
    int device = 0;
    int sm_count = 0;
    int n_warps = 0;  // warp slots of a worker's pool (4 CTAs of BB_WARPS_PER_CTA warps per SM)
    uint64_t seed = 0;
    std::string err;
    Knobs knobs;

    // reference + models, shared by the workers
    DevBuf ref; int64_t ref_len = 0;
    // a FASTA parsed by bb_fasta_parse (fa_n_kept >= 0): its kept bytes, header texts and each header's kept offset,
    // until bb_fasta_reference forms the reference from them
    DevBuf fa_kept; int64_t fa_n_kept = -1;
    bb_gzip_stats gz_stats{};   // how the last bb_fasta_parse inflated its input
    std::string fa_text; std::vector<int64_t> fa_text_off, fa_kept_off;
    bool have_em = false, have_qm = false;
    BBErrorModelDev em{}; DevBuf em_k2r, em_rowoff, em_cum, em_flags, em_slots, em_pool, em_rowinfo;
    BBEmHashDev em_hash{}; DevBuf em_hentries;  // k-mer index as a hash table (bb_upload_error_model_kmers)
    // the model installed by bb_load_error_model_file (em_loaded): what bb_download_error_model copies besides the tables
    bool em_loaded = false; DevBuf em_probs, em_codes; bb_em_load_info em_info{};
    BBQScoreModelDev qm{}; DevBuf qm_hkeys, qm_hvals, qm_lkeys, qm_lpool, qm_rowoff, qm_scores, qm_cum;

    // Sub-batches: a batch is dealt out over the workers and their kernel chains run side by side on their own
    // streams, so that one worker's tails and host round trips are covered by the others' kernels.  Worker 0 also
    // runs the uploads and the single-pair entry points.
    std::vector<std::unique_ptr<Worker>> workers;
    int n_split = 1;                          // workers the uploaded batch is spread over
    std::vector<std::vector<int32_t>> part;   // part[w][i] = batch position of worker w's i-th read
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;

    void *nccl_comm = nullptr;   // ncclComm_t of this context's device (bb_comm_init_rank / bb_comm_init_all)
    DevBuf d_red;                // two int64: send, receive of bb_allreduce_bases

    Bgzf bgzf;

    // BAM output (bb_bam_*), on bgzf.stream.  The last fetched batch: its workers' blocks start at out_base[w] of the
    // concatenated output (out_base[n_split] = its size).
    bool fetched = false;
    std::vector<int64_t> out_base;
    // The record stream bytes [bam_base, bam_base + bam_len) in bam_buf[bam_cur], and the (offset, length) pairs of the
    // seq and qual fields that start in it in bam_fields[bam_fcur], their offsets also on the host (bam_field_off).  The
    // other buffer of each pair takes the carried rest when the stream is compressed.
    DevBuf bam_buf[2], bam_fields[2], bam_recs, bam_pos, bam_text, bam_hfields;
    int bam_cur = 0, bam_fcur = 0;
    int64_t bam_base = 0, bam_len = 0;
    std::vector<int64_t> bam_field_off;
    // the records of the last bb_bam_build: stream offset and size of each (bam_last_at < 0: taken off the stream)
    int64_t bam_last_at = -1;
    std::vector<int64_t> bam_last_pos, bam_last_size;
    uint8_t *h_bam = nullptr;   // pinned staging of bb_bam_fetch_records
    int64_t h_bam_cap = 0;

    Worker &w0() { return *workers[0]; }
    ~bb_ctx() {
        for (cudaEvent_t e : {ev_t0, ev_t1}) if (e) cudaEventDestroy(e);
        if (h_bam) cudaFreeHost(h_bam);
    }
};

// Records "the work enqueued on `st` up to here is done" under `name` (tracing only).
static void mark(Worker &w, cudaStream_t st, const char *name) {
    if (!w.ctx->knobs.trace) return;
    if (w.mark_used == w.mark_pool.size()) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        w.mark_pool.push_back(e);
    }
    cudaEvent_t e = w.mark_pool[w.mark_used++];
    cudaEventRecord(e, st);
    int id = st == w.stream ? 0 : st == w.stream2 ? 1 : -1;
    for (int p = 0; p < 2 && id < 0; p++)
        for (int x = 0; x < 3; x++)
            if (st == w.side[p][x]) id = 2 + 4 * p + x;
    w.marks.push_back(Worker::Mark{name, id < 0 ? 0 : id, e});
}

static thread_local std::string g_create_error;

// A context drives up to 7 streams per worker (2 workers by default).  CUDA multiplexes streams onto
// CUDA_DEVICE_MAX_CONNECTIONS hardware queues (default 8); streams that share a queue serialize behind each other's
// pending waits.  Ask for the maximum unless the user chose a value; it only takes effect if CUDA is not initialized yet
// in this process (badread_b200/_lib.py and bench.py set it before anything touches CUDA).
namespace {
struct ConnectionsDefault {
    ConnectionsDefault() { setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0); }
} g_connections_default;
}  // namespace

// (ctx) is a bb_ctx or a Worker: whichever reports the error
#define BB_CUDA(ctx, call)                                                                                   \
    do {                                                                                                     \
        cudaError_t e_ = (call);                                                                             \
        if (e_ != cudaSuccess) {                                                                             \
            (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                                 \
            return BB_ERR_CUDA;                                                                              \
        }                                                                                                    \
    } while (0)

template <typename O>
static int set_err(O *o, int code, const std::string &msg) {
    if (o) o->err = msg;
    return code;
}

// Calls f(worker, w) for the workers of the current split in order; the first failure's code and message become the context's.
template <typename F>
static int each_worker(bb_ctx *ctx, F &&f) {
    for (int w = 0; w < ctx->n_split; w++) {
        Worker &wk = *ctx->workers[(size_t)w];
        if (const int rc = f(wk, w)) return set_err(ctx, rc, wk.err);
    }
    return BB_OK;
}

// misc.REV_COMP_DICT (misc.py:56-61); anything else complements to 'N' (misc.py:64-68)
void bbl_comp_table(uint8_t *table) {
    std::memset(table, 'N', 256);
    const char *from = "ATGCatgcRYSWKMBVDHNryswkmbvdhn.-?";
    const char *to = "TACGtacgYRSWMKVBHDNyrswmkvbhdn.-?";
    for (int i = 0; from[i]; i++) table[(uint8_t)from[i]] = (uint8_t)to[i];
}

extern "C" const char *bb_version(void) { return "badread_b200 0.1.0 (sm_90a)"; }

extern "C" const char *bb_last_error(const bb_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

extern "C" const char *bb_stage_name(int stage) {
    return (stage >= 0 && stage < BB_N_STAGES) ? kStageNames[stage] : "";
}

extern "C" int64_t bb_launch_count(const bb_ctx *ctx) {
    if (!ctx) return 0;
    int64_t total = 0;
    for (const auto &w : ctx->workers) total += w->launches;
    return total;
}

static int add_worker(bb_ctx *ctx, bool high_priority) {
    ctx->workers.push_back(std::make_unique<Worker>(ctx, ctx->knobs));
    Worker &w = *ctx->workers.back();
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    const int prio = high_priority ? prio_hi : prio_lo;
    cudaError_t e = cudaStreamCreateWithPriority(&w.stream, cudaStreamNonBlocking, prio);
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return BB_ERR_CUDA; }
    cudaStreamCreateWithPriority(&w.stream2, cudaStreamNonBlocking, prio);
    for (auto &row : w.side) for (cudaStream_t &s : row) cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, prio);
    for (cudaEvent_t &e : w.ev) cudaEventCreate(&e);
    for (cudaEvent_t *e : {&w.ev_fork, &w.ev_join, &w.ev_scan, &w.ev_level[0], &w.ev_level[1]}) cudaEventCreateWithFlags(e, cudaEventDisableTiming);
    for (auto &row : w.ev_side) for (cudaEvent_t &e : row) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    if (cudaHostAlloc((void **)&w.h_info, sizeof(Worker::RunInfo), cudaHostAllocPortable) == cudaSuccess) return BB_OK;
    w.h_info = nullptr;
    g_create_error = "cudaHostAlloc failed";
    return BB_ERR_CUDA;
}

static void (*nccl_destroy)(void *) = nullptr;  // set once NCCL is loaded (bb_comm_init_*)

extern "C" int bb_create(bb_ctx **out, int device, uint64_t seed) {
    if (!out) return BB_ERR_ARG;
    *out = nullptr;
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev <= 0) {
        g_create_error = std::string("no CUDA device available: ") + cudaGetErrorString(e) +
                         " (badread_b200 has no CPU path)";
        return BB_ERR_CUDA;
    }
    if (device < 0 || device >= n_dev) { g_create_error = "invalid device ordinal"; return BB_ERR_ARG; }
    e = cudaSetDevice(device);
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return BB_ERR_CUDA; }
    std::unique_ptr<bb_ctx> ctx(new bb_ctx());
    ctx->device = device;
    ctx->seed = seed;
    ctx->knobs = read_knobs();
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return BB_ERR_CUDA; }
    ctx->sm_count = prop.multiProcessorCount;
    // persistent warps: 4 CTAs of 4 warps per SM for the warp-per-read kernels
    ctx->n_warps = ctx->sm_count * 4 * BB_WARPS_PER_CTA;
    uint8_t comp[256];
    bbl_comp_table(comp);
    e = cudaMemcpyToSymbol(bb_c_comp, comp, 256);
    if (e == cudaSuccess) e = bbl_node_pair_init();
    if (e == cudaSuccess) e = bbl_node_quad_init();
    if (e == cudaSuccess) e = bbl_window_lane_init();
    if (e == cudaSuccess) e = bbl_leaf_lane_init();
    if (e == cudaSuccess) e = bbl_bgzf_init();
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return BB_ERR_CUDA; }
    // 2 workers on H100 (132 SMs, 80 GB): as fast as 3 and 12 % faster than 4 on config 1, and their scratch (lane
    // histories sized by the SM count) leaves room for a second context on the same GPU (~39 GB peak against 66 with 4).
    // Worker 0 carries the longest reads of a split batch (bb_batch_upload): their dependent chain of stages bounds the
    // step from below, so its kernels go first whenever the block scheduler has a choice.
    for (int w = 0; w < ctx->knobs.n_workers; w++)
        if (const int rc = add_worker(ctx.get(), w == 0 && ctx->knobs.head_priority)) return rc;
    cudaEventCreate(&ctx->ev_t0);
    cudaEventCreate(&ctx->ev_t1);
    *out = ctx.release();
    return BB_OK;
}

extern "C" int bb_destroy(bb_ctx *ctx) {
    if (!ctx) return BB_OK;
    cudaSetDevice(ctx->device);  // the frees below act on the current device
    for (const auto &w : ctx->workers) cudaStreamSynchronize(w->stream);
    if (ctx->bgzf.stream) cudaStreamSynchronize(ctx->bgzf.stream);
    if (ctx->nccl_comm && nccl_destroy) nccl_destroy(ctx->nccl_comm);
    delete ctx;
    return BB_OK;
}

template <typename O, typename T>
static int upload(O *o, cudaStream_t st, DevBuf &buf, const T *src, size_t count) {
    BB_CUDA(o, buf.ensure(std::max<size_t>(count, 1) * sizeof(T)));
    if (count) BB_CUDA(o, cudaMemcpyAsync(buf.p, src, count * sizeof(T), cudaMemcpyHostToDevice, st));
    return BB_OK;
}

extern "C" int bb_upload_reference(bb_ctx *ctx, const uint8_t *bases, int64_t n_bases) {
    if (!ctx || n_bases < 0 || (n_bases && !bases)) return set_err(ctx, BB_ERR_ARG, "bb_upload_reference: bad arguments");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->w0().stream;
    int rc = upload(ctx, st, ctx->ref, bases, (size_t)n_bases);
    if (rc) return rc;
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->ref_len = n_bases;
    return BB_OK;
}

extern "C" int bb_download_reference(bb_ctx *ctx, int64_t offset, int64_t n, uint8_t *out) {
    if (!ctx || offset < 0 || n < 0 || (n && !out)) return set_err(ctx, BB_ERR_ARG, "bb_download_reference: bad arguments");
    if (offset + n > ctx->ref_len) return set_err(ctx, BB_ERR_ARG, "bb_download_reference: range beyond the reference");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n) BB_CUDA(ctx, cudaMemcpy(out, ctx->ref.as<uint8_t>() + offset, (size_t)n, cudaMemcpyDeviceToHost));
    return BB_OK;
}

// ---- the reference from a FASTA file parsed on the device (bb_fasta.cuh)
// Exactly `bytes` (at least 1) in buf: the loader's buffers are the size of the reference, so no slack.
static cudaError_t alloc_exact(DevBuf &buf, size_t bytes) {
    buf.release();
    bytes = std::max<size_t>(bytes, 1);
    cudaError_t e = cudaMalloc(&buf.p, bytes);
    if (e == cudaSuccess) buf.cap = bytes;
    return e;
}

static void fasta_reset(bb_ctx *ctx) {
    ctx->fa_kept.release();
    ctx->fa_n_kept = -1;
    ctx->fa_text.clear();
    ctx->fa_text_off.clear();
    ctx->fa_kept_off.clear();
}

extern "C" int bb_fasta_parse(bb_ctx *ctx, const uint8_t *data, int64_t n, int is_bgzf, int32_t *n_headers, int64_t *text_bytes,
                              int64_t *n_kept) {
    if (!ctx || n < 0 || (n && !data) || !n_headers || !text_bytes || !n_kept)
        return set_err(ctx, BB_ERR_ARG, "bb_fasta_parse: bad arguments");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    for (const auto &w : ctx->workers) BB_CUDA(ctx, cudaStreamSynchronize(w->stream));
    fasta_reset(ctx);
    ctx->gz_stats = bb_gzip_stats{};
    ctx->ref.release();   // (replaced by bb_fasta_reference; freed first, so that the parse has its memory)
    ctx->ref_len = 0;
    const cudaStream_t st = ctx->w0().stream;
    DevBuf text, scratch, hdr, idx, htext;
    int64_t len = n;
    if (is_bgzf) {
        uint8_t *p = nullptr;
        char msg[256];
        if (const int rc = bbl_gzip_inflate_device(st, data, n, 0, &p, &len, &ctx->gz_stats, msg, sizeof(msg)))
            return set_err(ctx, rc, msg);
        text.p = p;
        text.cap = (size_t)std::max<int64_t>(len, 16);
    } else {
        BB_CUDA(ctx, alloc_exact(text, (size_t)n));
        if (n) BB_CUDA(ctx, cudaMemcpyAsync(text.p, data, (size_t)n, cudaMemcpyHostToDevice, st));
    }
    BB_CUDA(ctx, alloc_exact(scratch, bbl_fasta_scratch_bytes(len)));
    bbl_fasta_scan(st, text.as<uint8_t>(), len, scratch.p);
    int64_t totals[2] = {0, 0};
    BB_CUDA(ctx, cudaMemcpyAsync(totals, bbl_fasta_totals(scratch.p, len), sizeof(totals), cudaMemcpyDeviceToHost, st));
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    const int64_t kept = totals[0], nh = totals[1];
    if (nh > INT32_MAX) return set_err(ctx, BB_ERR_ARG, "bb_fasta_parse: more than 2^31 - 1 header lines");
    BB_CUDA(ctx, alloc_exact(ctx->fa_kept, (size_t)kept));
    BB_CUDA(ctx, alloc_exact(hdr, 3 * sizeof(int64_t) * (size_t)nh));
    int64_t *d_start = hdr.as<int64_t>(), *d_end = d_start + nh, *d_kept = d_end + nh;
    bbl_fasta_emit(st, text.as<uint8_t>(), len, scratch.p, ctx->fa_kept.as<uint8_t>(), d_start, d_end, d_kept);
    BB_CUDA(ctx, cudaGetLastError());
    std::vector<int64_t> h((size_t)(3 * nh));
    if (nh) BB_CUDA(ctx, cudaMemcpyAsync(h.data(), hdr.p, h.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    // the header texts (after the '>', up to the newline) gathered into one buffer
    std::vector<int64_t> lo_off((size_t)(2 * nh + 1));
    lo_off[(size_t)nh] = 0;
    for (int64_t k = 0; k < nh; k++) {
        lo_off[(size_t)k] = h[(size_t)k] + 1;
        lo_off[(size_t)(nh + k + 1)] = lo_off[(size_t)(nh + k)] + (h[(size_t)(nh + k)] - h[(size_t)k] - 1);
    }
    const int64_t tlen = lo_off[(size_t)(2 * nh)];
    ctx->fa_text.resize((size_t)tlen);
    if (tlen) {
        if (const int rc = upload(ctx, st, idx, lo_off.data(), lo_off.size())) return rc;
        BB_CUDA(ctx, alloc_exact(htext, (size_t)tlen));
        bbl_fasta_gather(st, text.as<uint8_t>(), idx.as<int64_t>(), idx.as<int64_t>() + nh, (int32_t)nh, tlen, htext.as<uint8_t>());
        BB_CUDA(ctx, cudaGetLastError());
        BB_CUDA(ctx, cudaMemcpyAsync(&ctx->fa_text[0], htext.p, (size_t)tlen, cudaMemcpyDeviceToHost, st));
        BB_CUDA(ctx, cudaStreamSynchronize(st));
    }
    ctx->fa_text_off.assign(lo_off.begin() + nh, lo_off.end());
    ctx->fa_kept_off.assign(h.begin() + 2 * nh, h.end());
    ctx->fa_n_kept = kept;
    *n_headers = (int32_t)nh;
    *text_bytes = tlen;
    *n_kept = kept;
    return BB_OK;
}

extern "C" int bb_last_gzip_stats(const bb_ctx *ctx, bb_gzip_stats *stats) {
    if (!ctx || !stats) return BB_ERR_ARG;
    *stats = ctx->gz_stats;
    return BB_OK;
}

extern "C" int bb_fasta_headers(bb_ctx *ctx, char *text, int64_t text_cap, int64_t *text_off, int64_t *kept_off, int32_t n_cap) {
    if (!ctx || text_cap < 0 || n_cap < 0) return set_err(ctx, BB_ERR_ARG, "bb_fasta_headers: bad arguments");
    if (ctx->fa_n_kept < 0) return set_err(ctx, BB_ERR_STATE, "bb_fasta_headers: no FASTA parsed (bb_fasta_parse)");
    const size_t nh = ctx->fa_kept_off.size();
    if ((size_t)n_cap < nh || (size_t)text_cap < ctx->fa_text.size())
        return set_err(ctx, BB_ERR_CAPACITY, "bb_fasta_headers: " + std::to_string(nh) + " headers of " +
                                                 std::to_string(ctx->fa_text.size()) + " bytes, capacity " + std::to_string(n_cap) +
                                                 " of " + std::to_string(text_cap));
    if (!text_off || !kept_off || (!ctx->fa_text.empty() && !text)) return set_err(ctx, BB_ERR_ARG, "bb_fasta_headers: bad arguments");
    if (!ctx->fa_text.empty()) std::memcpy(text, ctx->fa_text.data(), ctx->fa_text.size());
    std::copy(ctx->fa_text_off.begin(), ctx->fa_text_off.end(), text_off);
    std::copy(ctx->fa_kept_off.begin(), ctx->fa_kept_off.end(), kept_off);
    kept_off[nh] = ctx->fa_n_kept;
    return BB_OK;
}

extern "C" int bb_fasta_reference(bb_ctx *ctx, int32_t n_contigs, const int64_t *lo, const int64_t *hi) {
    if (!ctx || n_contigs < 0 || (n_contigs && (!lo || !hi))) return set_err(ctx, BB_ERR_ARG, "bb_fasta_reference: bad arguments");
    if (ctx->fa_n_kept < 0) return set_err(ctx, BB_ERR_STATE, "bb_fasta_reference: no FASTA parsed (bb_fasta_parse)");
    std::vector<int64_t> lo_off((size_t)(2 * n_contigs + 1));
    bool in_place = true;   // the contigs are the kept bytes as they lie
    for (int32_t c = 0; c < n_contigs; c++) {
        if (lo[c] < 0 || lo[c] > hi[c] || hi[c] > ctx->fa_n_kept) return set_err(ctx, BB_ERR_ARG, "bb_fasta_reference: contig out of range");
        lo_off[(size_t)c] = lo[c];
        lo_off[(size_t)(n_contigs + c + 1)] = lo_off[(size_t)(n_contigs + c)] + (hi[c] - lo[c]);
        in_place = in_place && lo[c] == (c ? hi[c - 1] : 0);
    }
    const int64_t total = lo_off[(size_t)(2 * n_contigs)];
    in_place = in_place && total == ctx->fa_n_kept;
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->w0().stream;
    if (in_place) {
        ctx->ref.release();
        std::swap(ctx->ref.p, ctx->fa_kept.p);
        std::swap(ctx->ref.cap, ctx->fa_kept.cap);
    } else {
        DevBuf idx;
        BB_CUDA(ctx, alloc_exact(ctx->ref, (size_t)total));
        if (const int rc = upload(ctx, st, idx, lo_off.data(), lo_off.size())) return rc;
        bbl_fasta_gather(st, ctx->fa_kept.as<uint8_t>(), idx.as<int64_t>(), idx.as<int64_t>() + n_contigs, n_contigs, total,
                         ctx->ref.as<uint8_t>());
        BB_CUDA(ctx, cudaGetLastError());
        BB_CUDA(ctx, cudaStreamSynchronize(st));
    }
    ctx->ref_len = total;
    fasta_reset(ctx);
    return BB_OK;
}

// The per-entry tables of a model (everything but the k-mer index) and the per-row summaries derived from them.
static int upload_em_rows(bb_ctx *ctx, int k, int32_t n_rows, const int32_t *row_off, const double *cum,
                          const uint8_t *flags, const uint32_t *slots, const uint8_t *pool, int64_t pool_len) {
    const cudaStream_t st = ctx->w0().stream;
    const int64_t ne = row_off[n_rows];
    int rc;
    if ((rc = upload(ctx, st, ctx->em_rowoff, row_off, (size_t)n_rows + 1))) return rc;
    if ((rc = upload(ctx, st, ctx->em_cum, cum, (size_t)ne))) return rc;
    if ((rc = upload(ctx, st, ctx->em_flags, flags, (size_t)ne))) return rc;
    if ((rc = upload(ctx, st, ctx->em_slots, slots, (size_t)ne * k))) return rc;
    if ((rc = upload(ctx, st, ctx->em_pool, pool, (size_t)pool_len))) return rc;
    std::vector<BBRowInfo> info((size_t)n_rows);
    for (int32_t r = 0; r < n_rows; r++) {
        const int32_t e0 = row_off[r], ne = row_off[r + 1] - e0;
        if (ne <= 0) return set_err(ctx, BB_ERR_ARG, "error model: empty table row");
        BBRowInfo &ri = info[(size_t)r];
        ri.cum_last = cum[e0 + ne - 1]; ri.cum0 = cum[e0]; ri.e0 = e0; ri.ne = ne;
        ri.first_is_identity = flags[e0] == 1 ? 1 : 0; ri.pad = 0;
    }
    if ((rc = upload(ctx, st, ctx->em_rowinfo, info.data(), info.size()))) return rc;
    BB_CUDA(ctx, cudaStreamSynchronize(st));  // `info` is about to go out of scope
    ctx->em.row_off = ctx->em_rowoff.as<int32_t>();
    ctx->em.cum = ctx->em_cum.as<double>(); ctx->em.flags = ctx->em_flags.as<uint8_t>();
    ctx->em.slots = ctx->em_slots.as<uint32_t>(); ctx->em.pool = ctx->em_pool.as<uint8_t>();
    ctx->em.rowinfo = ctx->em_rowinfo.as<BBRowInfo>();
    return BB_OK;
}

extern "C" int bb_upload_error_model(bb_ctx *ctx, int k, int type, const int32_t *kmer_to_row, int64_t n_index,
                                     int32_t n_rows, const int32_t *row_off, const double *cum, const uint8_t *flags,
                                     const uint32_t *slots, const uint8_t *pool, int64_t pool_len) {
    if (!ctx) return BB_ERR_ARG;
    if (k < 1 || k > 12 || (type != 0 && type != 1)) return set_err(ctx, BB_ERR_ARG, "error model: k must be 1..12");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    ctx->em = BBErrorModelDev{};
    ctx->em_loaded = false;
    ctx->em_hash = BBEmHashDev{};
    ctx->em.k = k; ctx->em.type = type;
    if (type == 1) {
        if (!kmer_to_row || !row_off || !cum || !flags || !slots || n_rows <= 0 || n_index != (1ll << (2 * k)))
            return set_err(ctx, BB_ERR_ARG, "error model: missing tables");
        int rc;
        if ((rc = upload(ctx, ctx->w0().stream, ctx->em_k2r, kmer_to_row, (size_t)n_index))) return rc;
        if ((rc = upload_em_rows(ctx, k, n_rows, row_off, cum, flags, slots, pool, pool_len))) return rc;
        ctx->em.kmer_to_row = ctx->em_k2r.as<int32_t>();
    }
    BB_CUDA(ctx, cudaStreamSynchronize(ctx->w0().stream));
    ctx->have_em = true;
    for (const auto &w : ctx->workers) w->uploaded = false;  // the fragment layout of a batch depends on k
    return BB_OK;
}

extern "C" int bb_upload_error_model_kmers(bb_ctx *ctx, int k, int32_t n_rows, const int64_t *kmer_codes,
                                           const int32_t *row_off, const double *cum, const uint8_t *flags,
                                           const uint32_t *slots, const uint8_t *pool, int64_t pool_len) {
    if (!ctx) return BB_ERR_ARG;
    if (!kmer_codes || !row_off || !cum || !flags || !slots || n_rows <= 0 || pool_len < 0 || (pool_len && !pool))
        return set_err(ctx, BB_ERR_ARG, "error model: missing tables");
    BBEmHashTable t;
    std::string err;
    if (!bb_build_em_hash(k, n_rows, kmer_codes, t, err)) return set_err(ctx, BB_ERR_ARG, err);
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    ctx->em = BBErrorModelDev{};
    ctx->em_loaded = false;
    ctx->em_hash = BBEmHashDev{};
    ctx->have_em = false;
    int rc;
    if ((rc = upload(ctx, ctx->w0().stream, ctx->em_hentries, t.entries.data(), t.entries.size()))) return rc;
    if ((rc = upload_em_rows(ctx, k, n_rows, row_off, cum, flags, slots, pool, pool_len))) return rc;  // (synchronizes)
    ctx->em.k = k; ctx->em.type = 1;
    ctx->em_hash.entries = ctx->em_hentries.as<unsigned long long>(); ctx->em_hash.bits = t.bits;
    ctx->have_em = true;
    for (const auto &w : ctx->workers) w->uploaded = false;  // the fragment layout of a batch depends on k
    return BB_OK;
}

// Takes ownership of a device allocation
static void adopt(DevBuf &buf, void *p, size_t bytes) {
    buf.release();
    buf.p = p;
    buf.cap = bytes;
}

extern "C" int bb_load_error_model_file(bb_ctx *ctx, const uint8_t *bytes, int64_t n, bb_em_load_info *info) {
    if (!ctx || n < 0 || (n && !bytes) || !info) return set_err(ctx, BB_ERR_ARG, "bb_load_error_model_file: bad arguments");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    for (const auto &w : ctx->workers) BB_CUDA(ctx, cudaStreamSynchronize(w->stream));
    *info = bb_em_load_info{};
    const auto t0 = std::chrono::steady_clock::now();
    const cudaStream_t st = ctx->w0().stream;
    // misc.get_compression_type's magic numbers: gzip (BGZF or not) is inflated here, bzip2 and zip are the host's to refuse
    const bool gz = n >= 3 && bytes[0] == 0x1f && bytes[1] == 0x8b && bytes[2] == 0x08;
    if ((n >= 3 && bytes[0] == 'B' && bytes[1] == 'Z' && bytes[2] == 'h') ||
        (n >= 4 && bytes[0] == 'P' && bytes[1] == 'K' && bytes[2] == 3 && bytes[3] == 4)) {
        info->fallback = BB_EM_FALLBACK_INPUT;
        return BB_OK;
    }
    DevBuf text;
    int64_t len = n;
    if (gz) {
        uint8_t *p = nullptr;
        char msg[256];
        bb_gzip_stats stats{};
        const int rc = bbl_gzip_inflate_device(st, bytes, n, 0, &p, &len, &stats, msg, sizeof(msg));
        if (rc == BB_ERR_ARG) {   // not a stream gzip.open reads either: the host loader reports it
            info->fallback = BB_EM_FALLBACK_INPUT;
            return BB_OK;
        }
        if (rc) return set_err(ctx, rc, msg);
        text.p = p;
        text.cap = (size_t)std::max<int64_t>(len, 16);
    } else {
        BB_CUDA(ctx, alloc_exact(text, (size_t)n));
        if (n) BB_CUDA(ctx, cudaMemcpyAsync(text.p, bytes, (size_t)n, cudaMemcpyHostToDevice, st));
        BB_CUDA(ctx, cudaStreamSynchronize(st));
    }
    auto t = std::chrono::steady_clock::now();
    info->ms_inflate = std::chrono::duration<double, std::milli>(t - t0).count();
    info->text_bytes = len;
    BBEmLoadOut out;
    char msg[256];
    int rc = bbl_em_load(st, text.as<uint8_t>(), len, true, info, &out, msg, sizeof(msg));
    text.release();
    // the hash index for k > 12: BBEmHashTable's builder over the row codes made on the device
    BBEmHashTable hash;
    if (rc == BB_OK && !info->fallback && !out.kmer_to_row) {
        std::vector<int64_t> codes((size_t)info->n_rows);
        BB_CUDA(ctx, cudaMemcpy(codes.data(), out.codes, codes.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
        std::string err;
        if (!bb_build_em_hash(info->k, (int32_t)info->n_rows, codes.data(), hash, err)) info->fallback |= BB_EM_FALLBACK_DUPLICATE;
    }
    if (rc != BB_OK || info->fallback) {
        bbl_em_load_free(&out);
        return rc == BB_OK ? BB_OK : set_err(ctx, rc, msg);
    }
    ctx->have_em = false;
    ctx->em = BBErrorModelDev{};
    ctx->em_hash = BBEmHashDev{};
    const size_t ne = (size_t)info->n_entries, nr = (size_t)info->n_rows;
    if (out.kmer_to_row) {
        adopt(ctx->em_k2r, out.kmer_to_row, ((size_t)1 << (2 * info->k)) * sizeof(int32_t));
        info->index = 1;
    } else {
        if (const int urc = upload(ctx, st, ctx->em_hentries, hash.entries.data(), hash.entries.size())) {
            bbl_em_load_free(&out);
            return urc;
        }
        info->index = 2;
    }
    adopt(ctx->em_codes, out.codes, nr * sizeof(int64_t));
    adopt(ctx->em_rowoff, out.row_off, (nr + 1) * sizeof(int32_t));
    adopt(ctx->em_cum, out.cum, ne * sizeof(double));
    adopt(ctx->em_probs, out.probs, ne * sizeof(double));
    adopt(ctx->em_flags, out.flags, std::max<size_t>(ne, 1));
    adopt(ctx->em_slots, out.slots, std::max<size_t>(ne * info->k, 1) * sizeof(uint32_t));
    adopt(ctx->em_pool, out.pool, (size_t)std::max<int64_t>(info->pool_bytes, 1));
    adopt(ctx->em_rowinfo, out.rowinfo, nr * sizeof(BBRowInfo));
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    const auto t1 = std::chrono::steady_clock::now();
    info->ms_index = std::chrono::duration<double, std::milli>(t1 - t).count() - info->ms_parse - info->ms_align - info->ms_tables;
    info->ms_total = std::chrono::duration<double, std::milli>(t1 - t0).count();
    ctx->em.k = info->k; ctx->em.type = 1;
    ctx->em.kmer_to_row = info->index == 1 ? ctx->em_k2r.as<int32_t>() : nullptr;
    ctx->em.row_off = ctx->em_rowoff.as<int32_t>();
    ctx->em.cum = ctx->em_cum.as<double>(); ctx->em.flags = ctx->em_flags.as<uint8_t>();
    ctx->em.slots = ctx->em_slots.as<uint32_t>(); ctx->em.pool = ctx->em_pool.as<uint8_t>();
    ctx->em.rowinfo = ctx->em_rowinfo.as<BBRowInfo>();
    if (info->index == 2) { ctx->em_hash.entries = ctx->em_hentries.as<unsigned long long>(); ctx->em_hash.bits = hash.bits; }
    ctx->em_info = *info;
    ctx->em_loaded = true;
    ctx->have_em = true;
    for (const auto &w : ctx->workers) w->uploaded = false;  // the fragment layout of a batch depends on k
    return BB_OK;
}

extern "C" int bb_download_error_model(bb_ctx *ctx, int32_t *kmer_to_row, int64_t *kmer_codes, int32_t *row_off, double *cum,
                                       double *probs, uint8_t *flags, uint32_t *slots, uint8_t *pool) {
    if (!ctx) return BB_ERR_ARG;
    if (!ctx->em_loaded) return set_err(ctx, BB_ERR_STATE, "bb_download_error_model: no model installed by bb_load_error_model_file");
    const bb_em_load_info &I = ctx->em_info;
    if (kmer_to_row && I.index != 1) return set_err(ctx, BB_ERR_ARG, "bb_download_error_model: the model has no dense index");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t ne = (size_t)I.n_entries, nr = (size_t)I.n_rows;
    const struct { void *dst; const DevBuf &src; size_t bytes; } parts[] = {
        {kmer_to_row, ctx->em_k2r, ((size_t)1 << (2 * I.k)) * sizeof(int32_t)}, {kmer_codes, ctx->em_codes, nr * sizeof(int64_t)},
        {row_off, ctx->em_rowoff, (nr + 1) * sizeof(int32_t)}, {cum, ctx->em_cum, ne * sizeof(double)},
        {probs, ctx->em_probs, ne * sizeof(double)}, {flags, ctx->em_flags, ne}, {slots, ctx->em_slots, ne * I.k * sizeof(uint32_t)},
        {pool, ctx->em_pool, (size_t)std::max<int64_t>(I.pool_bytes, 1)}};
    for (const auto &p : parts)
        if (p.dst && p.bytes) BB_CUDA(ctx, cudaMemcpy(p.dst, p.src.p, p.bytes, cudaMemcpyDeviceToHost));
    return BB_OK;
}

extern "C" int bb_upload_qscore_model_cigars(bb_ctx *ctx, int kmer_size, int32_t n_keys, const uint8_t *key_chars,
                                             const int32_t *key_off, const int32_t *row_off, const uint8_t *scores,
                                             const double *cum) {
    if (!ctx) return BB_ERR_ARG;
    if (kmer_size < 1 || (kmer_size & 1) == 0 || n_keys <= 0 || !key_chars || !key_off || !row_off || !scores || !cum)
        return set_err(ctx, BB_ERR_ARG, "qscore model: bad arguments");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    BBQScoreTables t;
    std::string err;
    if (!bb_build_qscore_tables(n_keys, key_chars, key_off, t, err)) return set_err(ctx, BB_ERR_ARG, err);
    const cudaStream_t st = ctx->w0().stream;
    const int64_t ne = row_off[n_keys];
    int rc;
    if ((rc = upload(ctx, st, ctx->qm_hkeys, t.hkeys.data(), t.hkeys.size()))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_hvals, t.hvals.data(), t.hvals.size()))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_lkeys, t.lkeys.data(), t.lkeys.size()))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_lpool, t.lpool.data(), t.lpool.size()))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_rowoff, row_off, (size_t)n_keys + 1))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_scores, scores, (size_t)ne))) return rc;
    if ((rc = upload(ctx, st, ctx->qm_cum, cum, (size_t)ne))) return rc;
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->qm.kmer_size = kmer_size; ctx->qm.hbits = t.hbits;
    ctx->qm.hkeys = ctx->qm_hkeys.as<uint64_t>(); ctx->qm.hvals = ctx->qm_hvals.as<int32_t>();
    ctx->qm.row_off = ctx->qm_rowoff.as<int32_t>(); ctx->qm.scores = ctx->qm_scores.as<uint8_t>();
    ctx->qm.cum = ctx->qm_cum.as<double>();
    ctx->qm.long_max_len = t.long_max_len; ctx->qm.lbits = t.lbits;
    ctx->qm.lkeys = ctx->qm_lkeys.as<BBQLongKey>(); ctx->qm.lpool = ctx->qm_lpool.as<uint64_t>();
    ctx->have_qm = true;
    return BB_OK;
}

extern "C" int bb_upload_qscore_model(bb_ctx *ctx, int kmer_size, int32_t n_keys, const uint64_t *keys,
                                      const int32_t *row_off, const uint8_t *scores, const double *cum) {
    if (!ctx) return BB_ERR_ARG;
    if (n_keys <= 0 || !keys) return set_err(ctx, BB_ERR_ARG, "qscore model: bad arguments");
    std::vector<uint8_t> chars;
    std::vector<int32_t> off;
    if (!bb_unpack_qscore_keys(n_keys, keys, chars, off)) return set_err(ctx, BB_ERR_ARG, "qscore model: invalid packed key");
    return bb_upload_qscore_model_cigars(ctx, kmer_size, n_keys, chars.data(), off.data(), row_off, scores, cum);
}

// Scratch shared by the warp-per-read kernels. hist is sized for the largest traceback edlib's 1 MiB rule
// admits (ceil(n/64)*m < 52429 -> < 104858 32-row blocks); tbuf holds a joined 1000-slot window.
static int ensure_scratch(Worker &w, int hbuf_need, int lr_need, int len_need, int lr_floor = 4096) {
    const int n_warps = w.ctx->n_warps;
    const int hist_cap = 106496;
    const int tbuf_stride = 1000 * 255 + 1024;
    const int stack_cap = 64;
    int hbuf_cap = std::max(hbuf_need + 64, tbuf_stride);
    hbuf_cap = (hbuf_cap + 255) & ~255;
    int lr_cap = std::max(lr_need + 64, lr_floor);
    lr_cap = (lr_cap + 255) & ~255;
    int peq_cap = bb_peq_words(len_need) + 8;
    peq_cap = (peq_cap + 63) & ~63;
    if (w.pool.peq_cap >= peq_cap) peq_cap = w.pool.peq_cap;
    if (w.pool.hbuf_cap >= hbuf_cap) hbuf_cap = w.pool.hbuf_cap;
    if (w.pool.lr_cap >= lr_cap) lr_cap = w.pool.lr_cap;
    BB_CUDA(&w, w.s_hist.ensure((size_t)n_warps * hist_cap * sizeof(uint2)));
    BB_CUDA(&w, w.s_tbuf.ensure((size_t)n_warps * tbuf_stride));
    BB_CUDA(&w, w.s_stack.ensure((size_t)n_warps * stack_cap * 5 * sizeof(int)));
    BB_CUDA(&w, w.s_hbuf.ensure((size_t)n_warps * hbuf_cap));
    BB_CUDA(&w, w.s_lr.ensure((size_t)n_warps * lr_cap * 2 * sizeof(int)));
    BB_CUDA(&w, w.s_peq.ensure((size_t)n_warps * peq_cap * sizeof(uint4)));
    BBScratchPool &p = w.pool;
    p.hist = w.s_hist.as<uint2>(); p.hist_stride = hist_cap; p.hist_cap = hist_cap;
    p.hbuf = w.s_hbuf.as<int8_t>(); p.hbuf_stride = hbuf_cap; p.hbuf_cap = hbuf_cap;
    p.lr = w.s_lr.as<int>(); p.lr_stride = 2ll * lr_cap; p.lr_cap = lr_cap;
    p.stack = w.s_stack.as<int>(); p.stack_cap = stack_cap;
    p.tbuf = w.s_tbuf.as<uint8_t>(); p.tbuf_stride = tbuf_stride;
    p.peq = w.s_peq.as<uint4>(); p.peq_stride = peq_cap; p.peq_cap = peq_cap;
    // the single-warp node kernels only touch the split-score arrays
    constexpr int lean_cap = 2048;  // > a + b + 1 of the widest lean class (bb_pick_L<4>(a, b, 16) > 0: a + b < 1920)
    const size_t lean_warps = (size_t)w.ctx->sm_count * kLeanCtasPerSmBoth * BB_WARPS_PER_CTA;
    BB_CUDA(&w, w.s_lr_lean.ensure(lean_warps * lean_cap * 2 * sizeof(int)));
    w.pool_lean = p;
    w.pool_lean.lr = w.s_lr_lean.as<int>(); w.pool_lean.lr_stride = 2ll * lean_cap; w.pool_lean.lr_cap = lean_cap;
    return BB_OK;
}

static BBBatchDev batch_dev(const Worker &w) {
    BBBatchDev B{};
    B.n_reads = w.n_reads;
    B.read_index = w.d_read_index.as<unsigned long long>();
    B.seg_off = w.d_seg_off.as<int>();
    B.segs = w.d_segs.as<bb_segment>();
    B.lit = w.d_lit.as<uint8_t>();
    B.target = w.d_target.as<double>();
    B.order = w.d_order.as<int>();
    B.reads = w.d_reads.as<BBReadDev>();
    B.frag = w.d_frag.as<uint8_t>();
    B.state = w.d_state.as<uint32_t>();
    B.kidx = w.d_kidx.as<int>();
    B.seq = w.d_seq.as<uint8_t>();
    B.ops = w.d_ops.as<uint8_t>();
    B.dcnt = w.d_dcnt.as<unsigned int>();
    B.qual = w.d_qual.as<uint8_t>();
    B.out_seq = w.d_out_seq.as<uint8_t>();
    B.out_qual = w.d_out_qual.as<uint8_t>();
    B.fpeq = w.d_fpeq.as<uint4>();
    B.speq = w.d_speq.as<uint4>();
    B.ctime = w.d_ctime.as<unsigned int>();
    B.chlog = w.d_chlog.as<uint2>();
    B.wres = w.d_wres.as<int2>();
    return B;
}

// Counters of a run live in d_counter (256 ints, cleared once per run): [0, 16) spare; round r of the error loop owns
// the 16 ints from BB_ROUND_BASE(r).
#define BB_N_COUNTERS 256
#define BB_ROUND_BASE(r) (16 + 16 * (r))
enum { BBC_MUTATE = 0, BBC_NTASKS = 1, BBC_LANE4 = 2, BBC_FB1 = 3, BBC_LANE8 = 4, BBC_FB2 = 5, BBC_WARP = 6, BBC_PENDING = 7 };

// Hirschberg levels a fragment of max_len bases can need: a node is split while edlib's traceback estimate
// 20 ceil(nn/64) mm + 8 mm reaches 1 MiB; mm halves per level and nn <= 2 mm + 64 bounds the query side generously.
static int level_bound(int max_len, double slack) {
    long long mm = (long long)(max_len * slack) + 64;
    int d = 0;
    while (20ll * ((2 * mm + 64 + 63) / 64) * mm + 8ll * mm >= 1048576ll) { mm = (mm + 1) / 2; d++; }
    return d + 1;
}

// Every allocation a run needs, sized from the fragment lengths: a run is pure enqueueing, nothing on the host
// depends on a value the device computes.  What turns out too small is flagged by the kernels and w_finish grows
// the knobs (slack, n_rounds, levels, lr_worst) and runs the batch again.
static int w_prepare(Worker &w) {
    const bb_ctx &c = *w.ctx;
    BB_CUDA(&w, cudaSetDevice(c.device));
    Worker::Layout &L = w.L;
    const int n = w.n_reads;
    const int64_t off = w.frag_total;
    w.seq_cap = (int64_t)((double)off * w.slack) + 16ll * n + 65536;
    w.out_cap = w.seq_cap;
    w.speq_cap = w.seq_cap / 32 + (2ll * BB_PEQ_PAD + 2) * n + 64;
    L.fb_len = w.wres_total + 8;
    BB_CUDA(&w, w.d_frag.ensure((size_t)off + 16));
    BB_CUDA(&w, w.d_state.ensure(((size_t)off + 16) * sizeof(uint32_t)));
    BB_CUDA(&w, w.d_kidx.ensure(((size_t)off + 16) * sizeof(int)));
    BB_CUDA(&w, w.d_counter.ensure(BB_N_COUNTERS * sizeof(int)));
    BB_CUDA(&w, w.d_scan.ensure(sizeof(BBScanOut)));
    BB_CUDA(&w, w.d_levels.ensure(sizeof(Worker::RunInfo::levels)));
    BB_CUDA(&w, w.d_fpeq.ensure(((size_t)w.fpeq_total + 4) * sizeof(uint4)));
    BB_CUDA(&w, w.d_ctime.ensure(((size_t)off + 16) * sizeof(unsigned int)));
    BB_CUDA(&w, w.d_chlog.ensure(((size_t)w.log_total + 16) * sizeof(uint2)));
    BB_CUDA(&w, w.d_wres.ensure(((size_t)w.wres_total + 16) * sizeof(int2)));
    BB_CUDA(&w, w.d_wtasks.ensure(((size_t)w.wres_total + 16) * sizeof(BBWinTask)));
    BB_CUDA(&w, w.d_wfallback.ensure(2 * (size_t)L.fb_len * sizeof(BBWinTask)));
    BB_CUDA(&w, w.d_seq.ensure((size_t)w.seq_cap + 16));
    BB_CUDA(&w, w.d_ops.ensure((size_t)w.seq_cap + 16));
    BB_CUDA(&w, w.d_dcnt.ensure(((size_t)w.seq_cap + 16) * sizeof(unsigned int)));
    BB_CUDA(&w, w.d_qual.ensure((size_t)w.seq_cap + 16));
    BB_CUDA(&w, w.d_speq.ensure(((size_t)w.speq_cap + 4) * sizeof(uint4)));
    BB_CUDA(&w, w.d_out_seq.ensure((size_t)w.out_cap + 16));
    BB_CUDA(&w, w.d_out_qual.ensure((size_t)w.out_cap + 16));
    // Lane pools of the window aligners and the leaf aligner.  Each alignment pipeline's leaf kernel owns half of the
    // history (checkpoints with lowmem), one lane per thread of its lane_ctas CTAs.  The window kernels run before the
    // alignment and use the whole pool: the 4-word build up to 2 * lane_ctas CTAs (band slices of up to 3 words per
    // column), the 8-word build half as many (up to 7), with lowmem both up to 2 * lane_ctas.
    L.lane_ctas = c.sm_count * 4;
    const size_t lanes = (size_t)L.lane_ctas * 64;
    if (c.knobs.lowmem) {
        L.hist_per_pipe = lanes * BB_LEAF_MAX_TILES * BB_LEAF_CKPT_WORDS;
        BB_CUDA(&w, w.s_leafhist.ensure(2 * L.hist_per_pipe * sizeof(uint32_t)));
    } else {
        L.hist_per_pipe = lanes * BB_LEAF_LANE_COLS * (BB_LEAF_LW - 1);  // per-column band slices
        BB_CUDA(&w, w.s_lanehist.ensure(2 * L.hist_per_pipe * sizeof(uint2)));
    }
    BB_CUDA(&w, w.s_ltbuf.ensure(2 * lanes * BB_WIN_MAX_COLS));
    // window aligners: a checkpoint (2 LW + 2 words) per 16 columns per lane instead of a per-column history
    if (c.knobs.lowmem) BB_CUDA(&w, w.s_wckpt.ensure(2 * lanes * BB_WIN_MAX_TILES * BB_WIN_CKPT_WORDS(BB_WIN_LW) * sizeof(uint32_t)));
    // per-warp scratch: strip carries / bitmaps for the longest joined read; split-score arrays for the widest band
    // (expected: a few times the injected edits; worst case: the whole read; BADREAD_B200_LR_CAP replaces the expected
    // size and its floor)
    const int len_b = (int)std::min<double>((double)w.max_len * w.slack + 64.0, (double)(1 << 24));
    const int lr_floor = c.knobs.lr_cap > 0 ? c.knobs.lr_cap : 4096;
    int lr_need = lr_floor;
    for (int r = 0; r < n; r++) {
        const double len = (double)w.h_reads[(size_t)r].frag_len;
        const double worst = len * w.slack + 64.0;
        const double expect = c.knobs.lr_cap > 0 ? 0.0 : 3.0 * (1.0 - w.h_target[(size_t)r]) * len + 0.02 * len + 512.0;
        lr_need = std::max(lr_need, (int)std::min(worst, w.lr_worst ? worst : expect));
    }
    int rc = ensure_scratch(w, len_b, lr_need, len_b, lr_floor);
    if (rc) return rc;
    int slot = 0;
    for (int s = 0; s < 2; s++)
        for (int k = 0; k < 3; k++) {
            L.lean_base[s][k] = slot;
            slot += c.sm_count * kLeanCtasPerSm[k] * BB_WARPS_PER_CTA;
        }
    L.cap_node = (int)std::min<int64_t>(w.seq_cap / 256 + 4ll * n + 1024, 0x7ffffff0);
    for (int s = 0; s < 2; s++) {
        auto &qb = w.qbuf[s];
        for (int k = 0; k < BBQ_NODE_CLASSES; k++)
            for (int p = 0; p < 2; p++) BB_CUDA(&w, qb.node[k][p].ensure((size_t)L.cap_node * sizeof(BBNode)));
        for (int x = 0; x < 2; x++) BB_CUDA(&w, qb.leaf[x].ensure((size_t)L.cap_node * sizeof(BBNode)));
        BB_CUDA(&w, qb.count.ensure(kQueueCounts * sizeof(int)));
    }
    w.n_levels = std::max(1, std::min(BB_MAX_LEVELS, level_bound(w.max_len, w.slack) + w.extra_levels));
    return BB_OK;
}

// Checks the descriptors of a whole batch and sums each read's segment lengths into len.
static int check_batch(bb_ctx *ctx, int32_t n_reads, const int32_t *seg_off, const bb_segment *segs, int64_t literal_len,
                       std::vector<int64_t> &len) {
    const int k = ctx->em.k;
    len.assign((size_t)n_reads, 0);
    for (int32_t r = 0; r < n_reads; r++) {
        if (seg_off[r + 1] < seg_off[r]) return set_err(ctx, BB_ERR_ARG, "seg_off must be non-decreasing");
        for (int32_t s = seg_off[r]; s < seg_off[r + 1]; s++) {
            const bb_segment &sg = segs[s];
            if (sg.len < 0 || sg.src < 0) return set_err(ctx, BB_ERR_ARG, "negative segment");
            if (sg.kind == BB_SEG_LITERAL) { if (sg.src + sg.len > literal_len) return set_err(ctx, BB_ERR_ARG, "literal segment out of range"); }
            else if (sg.kind == BB_SEG_REF_FWD || sg.kind == BB_SEG_REF_REV) { if (sg.src + sg.len > ctx->ref_len) return set_err(ctx, BB_ERR_ARG, "reference segment out of range"); }
            else return set_err(ctx, BB_ERR_ARG, "unknown segment kind");
            len[(size_t)r] += sg.len;
        }
        if (len[(size_t)r] + 2 * k >= (1 << 24)) return set_err(ctx, BB_ERR_ARG, "fragment too long (16 Mb limit)");
    }
    return BB_OK;
}

// Uploads a worker's reads, whose descriptors check_batch has accepted.
static int w_batch_upload(Worker &w, int32_t n_reads, const uint64_t *read_index, const int32_t *seg_off,
                          const bb_segment *segs, const uint8_t *literal_pool, int64_t literal_len,
                          const double *target_identity) {
    BB_CUDA(&w, cudaSetDevice(w.ctx->device));
    const int k = w.ctx->em.k;
    w.h_reads.assign((size_t)n_reads, BBReadDev{});
    w.h_inlen.assign((size_t)n_reads, 0);
    w.h_target.assign(target_identity, target_identity + n_reads);
    int64_t off = 0, peq_off = 0, log_off = 0, wres_off = 0;
    int max_len = 0;
    for (int32_t r = 0; r < n_reads; r++) {
        int64_t len = 0;
        for (int32_t s = seg_off[r]; s < seg_off[r + 1]; s++) len += segs[s].len;
        w.h_inlen[(size_t)r] = (int32_t)len;
        BBReadDev &rd = w.h_reads[(size_t)r];
        rd.frag_off = off;
        rd.frag_len = (int)(len + 2 * k);
        rd.fpeq_off = peq_off;
        peq_off += bb_peq_words(rd.frag_len);
        {   // speculative loop bookkeeping: the loop cannot apply more than 0.9*len + k changes (simulate.py:285)
            const int cap = (int)(0.9 * (double)rd.frag_len) + k + 2;
            rd.log_off = log_off; rd.wres_off = wres_off;
            log_off += cap; wres_off += cap / BB_ALIGNMENT_INTERVAL + 1;
            const double need = (double)rd.frag_len * (1.0 - target_identity[r]);
            rd.horizon = (int)std::min<double>((double)cap, std::max(0.0, 1.25 * need) + 48.0);
            rd.n_logged = 0; rd.n_resume = 0; rd.a_done = 0; rd.status = BB_READ_PENDING; rd.stop_reason = 0;
        }
        off += (rd.frag_len + 15) & ~15;
        max_len = std::max(max_len, rd.frag_len);
    }
    w.frag_total = off; w.fpeq_total = peq_off; w.log_total = log_off; w.wres_total = wres_off;
    w.max_len = max_len;
    std::vector<int> order((size_t)n_reads);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(),
                     [&](int x, int y) { return w.h_reads[(size_t)x].frag_len > w.h_reads[(size_t)y].frag_len; });
    w.n_reads = n_reads;
    const cudaStream_t st = w.stream;
    int rc;
    if ((rc = upload(&w, st, w.d_read_index, read_index, (size_t)n_reads))) return rc;
    if ((rc = upload(&w, st, w.d_seg_off, seg_off, (size_t)n_reads + 1))) return rc;
    if ((rc = upload(&w, st, w.d_segs, segs, (size_t)seg_off[n_reads]))) return rc;
    if ((rc = upload(&w, st, w.d_lit, literal_pool, (size_t)literal_len))) return rc;
    if ((rc = upload(&w, st, w.d_target, target_identity, (size_t)n_reads))) return rc;
    if ((rc = upload(&w, st, w.d_order, order.data(), (size_t)n_reads))) return rc;
    if ((rc = upload(&w, st, w.d_reads, w.h_reads.data(), (size_t)n_reads))) return rc;
    if ((rc = w_prepare(w))) return rc;
    BB_CUDA(&w, cudaStreamSynchronize(st));
    w.uploaded = true;
    w.ran = false;
    w.finished = false;
    return BB_OK;
}

// Persistent grids (CTAs that pull work from a queue until it is empty) of `per_sm` CTAs per SM at full size, or of
// the GRID_<knob> setting.  The workers of a split batch run side by side: each launches its share (GRID_DIV; all of
// the SMs by default), so that their kernels are resident together instead of queueing behind each other's CTAs.
static int pgrid(const Worker &w, int per_sm, int knob = kGridKnobs) {
    const bb_ctx &c = *w.ctx;
    if (knob < kGridKnobs && c.knobs.grid[knob] > 0) per_sm = c.knobs.grid[knob];
    const int div = c.n_split > 1 && c.knobs.grid_div > 0 ? c.knobs.grid_div : 1;
    return std::max(c.sm_count / 2, (c.sm_count * per_sm + div - 1) / div);
}

// The error loop decoupled from its identity re-measurements (bb_loop.cuh): mutate ahead -> task list -> all window
// alignments as independent lane tasks -> scalar replay, n_rounds times back to back.  A round after the last read
// has finished costs six launches that find nothing to do; a read that is still pending after the last round is
// reported by the replay kernel's counter and w_finish runs the batch again with more rounds.
static int enqueue_error_loop(Worker &w, const BBBatchDev &B) {
    const bb_ctx &c = *w.ctx;
    const Worker::Layout &L = w.L;
    const BBErrorModelDev &em = c.em;
    cudaStream_t st = w.stream;
    const int n = w.n_reads;
    const int win_grid = 2 * L.lane_ctas;  // what the lane pools hold (see w_prepare)
    int *cnt = w.d_counter.as<int>();
    const int *order = w.d_order.as<int>();
    BBWinTask *tasks = w.d_wtasks.as<BBWinTask>();
    BBWinTask *fb1 = w.d_wfallback.as<BBWinTask>(), *fb2 = fb1 + L.fb_len;
    for (int round = 0; round < w.n_rounds; round++) {
        int *cr = cnt + BB_ROUND_BASE(round);
        bbl_mutate(std::min(pgrid(w, 8, G_MUTATE), n), st, B, em, c.seed, cr + BBC_MUTATE, order, n, w.is_head);
        mark(w, st, "mutate");
        bb_k_window_tasks<<<(n + 255) / 256, 256, 0, st>>>(B, order, n, tasks, cr + BBC_NTASKS);
        mark(w, st, "window_tasks");
        // 4-word windows first (bands up to 64 rows: almost every window); what does not fit falls through to the
        // 8-word build and from there to the warp kernel
        if (c.knobs.lowmem)
            bbl_window_lane4(std::min(pgrid(w, 6, G_WIN4), win_grid), st, B, em, tasks, cr + BBC_NTASKS, c.seed,
                             w.s_wckpt.as<uint32_t>(), w.s_ltbuf.as<uint8_t>(), cr + BBC_LANE4, fb1, cr + BBC_FB1);
        else
            bbl_window_lane_hist(4, c.knobs.ring_t, std::min(pgrid(w, 8, G_WIN4), win_grid), st, B, em, tasks, cr + BBC_NTASKS,
                                 c.seed, w.s_lanehist.as<uint2>(), w.s_ltbuf.as<uint8_t>(), cr + BBC_LANE4, fb1, cr + BBC_FB1);
        mark(w, st, "window_lane4");
        if (c.knobs.lowmem)
            bbl_window_lane8(std::min(pgrid(w, 3, G_WIN8), win_grid), st, B, em, fb1, cr + BBC_FB1, c.seed,
                             w.s_wckpt.as<uint32_t>(), w.s_ltbuf.as<uint8_t>(), cr + BBC_LANE8, fb2, cr + BBC_FB2);
        else
            bbl_window_lane_hist(8, 4, std::min(pgrid(w, 4, G_WIN8), win_grid / 2), st, B, em, fb1, cr + BBC_FB1, c.seed,
                                 w.s_lanehist.as<uint2>(), w.s_ltbuf.as<uint8_t>(), cr + BBC_LANE8, fb2, cr + BBC_FB2);
        mark(w, st, "window_lane8");
        bbl_window_warp(pgrid(w, 2), st, B, em, w.pool, fb2, cr + BBC_FB2, c.seed, cr + BBC_WARP);
        mark(w, st, "window_warp");
        bb_k_replay<<<(n + 3) / 4, 128, 0, st>>>(B, order, n, em.k, cr + BBC_PENDING);
        mark(w, st, "replay");
        w.launches += 6;
    }
    return BB_OK;
}

// Final alignment as level-synchronous tasks (bb_tasks.cuh): every level of all reads' Hirschberg trees is a few
// launches (warp-pair, lean-warp and lane nodes), leaves run at the end.  The number of levels comes from the longest
// fragment; nodes left over after the last level are reported by the queue counters (w_finish adds levels).
static int enqueue_align_tasks(Worker &w, const BBBatchDev &B) {
    const bb_ctx &c = *w.ctx;
    const Knobs &kn = c.knobs;
    const Worker::Layout &L = w.L;
    cudaStream_t stream[2] = {w.stream, w.stream2};
    const int n = w.n_reads;
    BBQueues Q[2];
    int *cnt[2];
    for (int s = 0; s < 2; s++) {
        auto &qb = w.qbuf[s];
        for (int k = 0; k < BBQ_NODE_CLASSES; k++)
            for (int p = 0; p < 2; p++) Q[s].node[k][p] = qb.node[k][p].as<BBNode>();
        for (int x = 0; x < 2; x++) Q[s].leaf[x] = qb.leaf[x].as<BBNode>();
        cnt[s] = qb.count.as<int>();
        Q[s].count = cnt[s]; Q[s].overflow = cnt[s] + BBQ_OVERFLOW; Q[s].cap_node = L.cap_node; Q[s].cap_leaf = L.cap_node;
        Q[s].lane8_cols = kn.lane8_cols;
        BB_CUDA(&w, cudaMemsetAsync(cnt[s], 0, kQueueCounts * sizeof(int), stream[0]));
    }
    int *snap = w.d_levels.as<int>();
    BB_CUDA(&w, cudaMemsetAsync(snap, 0, sizeof(Worker::RunInfo::levels), stream[0]));
    bb_k_push_roots<<<(n + 255) / 256, 256, 0, stream[0]>>>(B, Q[0], Q[1], w.d_order.as<int>());
    w.launches++;
    // pipeline 0 (stream 0): every read whose root band fits the lean / lane kernels; pipeline 1 (stream 1): reads
    // with a wide root (long or noisy reads).  The two never wait for each other's levels.
    BB_CUDA(&w, cudaEventRecord(w.ev_fork, stream[0]));
    BB_CUDA(&w, cudaStreamWaitEvent(stream[1], w.ev_fork, 0));
    int *cursor[2] = {cnt[0] + kCursorBase, cnt[1] + kCursorBase};
    const int warp_base[2] = {0, c.n_warps / 2};
    // The node classes of a level read the same queues and push into the next level's: they are independent and run
    // side by side on their own streams; the level ends when all of them have finished.
    for (int level = 0; level < w.n_levels; level++) {
        // (the roots are queued longest read first; every later queue fills in the order the parents finish, longest
        // last, and is walked from its end)
        const int p = (level & 1) | (level > 0 && kn.lpt_order ? BBQ_BACKWARDS : 0);
        for (int s = 0; s < 2; s++) {
            cudaStream_t st = stream[s];
            // this level's node counts are final here and cleared when the next level starts: keep them
            // (bb_last_run_work); the leaf counters at level 0 are the roots' leaves
            int *row = snap + (s * BB_MAX_LEVELS + level) * BB_SNAP_WORDS;
            BB_CUDA(&w, cudaMemcpyAsync(row, cnt[s] + BBQ_COUNT(0, p & 1), BBQ_NODE_CLASSES * sizeof(int), cudaMemcpyDeviceToDevice, st));
            if (level == 0)
                BB_CUDA(&w, cudaMemcpyAsync(row + BB_SNAP_LEAF, cnt[s] + BBQ_LEAF_COUNT, 2 * sizeof(int), cudaMemcpyDeviceToDevice, st));
            BB_CUDA(&w, cudaMemsetAsync(cnt[s] + BBQ_COUNT(0, (p & 1) ^ 1), 0, BBQ_NODE_CLASSES * sizeof(int), st));
            BB_CUDA(&w, cudaEventRecord(w.ev_level[s], st));
            int n_side = 0;
            auto on_side = [&]() -> cudaStream_t {
                cudaStream_t x = w.side[s][n_side++];
                cudaStreamWaitEvent(x, w.ev_level[s], 0);
                mark(w, x, "fork");
                return x;
            };
            if (s == 1) {
                cudaStream_t x = on_side();
                if (kn.use_quad) bbl_node_quad(c.sm_count, x, B, Q[s], w.pool, p, cursor[s]++, warp_base[s]);
                else bbl_node_pair(c.sm_count * kn.pair_ctas, x, B, Q[s], w.pool, p, cursor[s]++, warp_base[s]);
                w.launches++;
                mark(w, x, kn.use_quad ? "node_quad" : "node_pair");
            }
            {
                cudaStream_t x = on_side();   // the two narrow single-warp classes share a stream
                bbl_node_warp(2, std::min(pgrid(w, 3, G_WARP2), c.sm_count * kLeanCtasPerSm[LEAN2]), x, B, Q[s], w.pool_lean, p, cursor[s]++,
                              L.lean_base[s][LEAN2]);
                mark(w, x, "node_warp2");
                bbl_node_warp(1, std::min(pgrid(w, 3, G_WARP1), c.sm_count * kLeanCtasPerSm[LEAN1]), x, B, Q[s], w.pool_lean, p, cursor[s]++,
                              L.lean_base[s][LEAN1]);
                mark(w, x, "node_warp1");
                x = on_side();
                bbl_node_lane8(pgrid(w, 6, G_LANE8), x, B, Q[s], p, cursor[s]++);
                mark(w, x, "node_lane8");
            }
            bbl_node_warp(4, std::min(pgrid(w, 2, G_WARP4), c.sm_count * kLeanCtasPerSm[LEAN4]), st, B, Q[s], w.pool_lean, p, cursor[s]++,
                          L.lean_base[s][LEAN4]);
            mark(w, st, "node_warp4");
            w.launches += 4;
            for (int x = 0; x < n_side; x++) {
                BB_CUDA(&w, cudaEventRecord(w.ev_side[s][x], w.side[s][x]));
                BB_CUDA(&w, cudaStreamWaitEvent(st, w.ev_side[s][x], 0));
            }
        }
    }
    for (int s = 0; s < 2; s++) {
        cudaStream_t st = stream[s];
        bbl_leaf_warp(c.sm_count, st, B, Q[s], w.pool, cursor[s]++, warp_base[s]);
        mark(w, st, "leaf_warp");
        if (kn.lowmem)
            bbl_leaf_lane(std::min(pgrid(w, 3, G_LEAF), L.lane_ctas), st, B, Q[s], w.s_leafhist.as<uint32_t>() + s * L.hist_per_pipe, cursor[s]++);
        else
            bbl_leaf_lane_hist(std::min(pgrid(w, 4, G_LEAF), L.lane_ctas), st, B, Q[s], w.s_lanehist.as<uint2>() + s * L.hist_per_pipe, cursor[s]++);
        mark(w, st, "leaf_lane");
        w.launches += 2;
    }
    BB_CUDA(&w, cudaEventRecord(w.ev_join, stream[1]));
    BB_CUDA(&w, cudaStreamWaitEvent(stream[0], w.ev_join, 0));
    for (int s = 0; s < 2; s++)
        BB_CUDA(&w, cudaMemcpyAsync(w.h_info->qcount[s], cnt[s], 32 * sizeof(int), cudaMemcpyDeviceToHost, stream[0]));
    BB_CUDA(&w, cudaMemcpyAsync(w.h_info->levels, snap, sizeof(Worker::RunInfo::levels), cudaMemcpyDeviceToHost, stream[0]));
    return BB_OK;
}

// Enqueues the whole hot path of the uploaded batch on the worker's streams and returns: no host round trip inside.
static int w_enqueue(Worker &w) {
    if (!w.uploaded) return set_err(&w, BB_ERR_STATE, "bb_batch_run: no batch uploaded");
    const bb_ctx &c = *w.ctx;
    BB_CUDA(&w, cudaSetDevice(c.device));
    cudaStream_t st = w.stream;
    const int n = w.n_reads;
    BBBatchDev B = batch_dev(w);
    w.finished = false;
    // the per-read records start from the uploaded state on every run (bb_batch_run may be repeated)
    BB_CUDA(&w, cudaMemcpyAsync(w.d_reads.p, w.h_reads.data(), (size_t)n * sizeof(BBReadDev), cudaMemcpyHostToDevice, st));
    BB_CUDA(&w, cudaMemsetAsync(w.d_counter.p, 0, BB_N_COUNTERS * sizeof(int), st));
    w.marks.clear(); w.mark_used = 0;
    mark(w, st, "begin");
    BB_CUDA(&w, cudaEventRecord(w.ev[0], st));
    if (c.em.type == 1 && c.em_hash.entries)
        bb_k_build_fragments<0, true><<<n, 256, 0, st>>>(B, c.ref.as<uint8_t>(), c.em.k, c.seed, nullptr, c.em_hash);
    else
        bb_k_build_fragments<<<n, 256, 0, st>>>(B, c.ref.as<uint8_t>(), c.em.k, c.seed,
                                                 c.em.type == 1 ? c.em.kmer_to_row : nullptr);
    w.launches++;
    mark(w, st, "build_fragments");
    BB_CUDA(&w, cudaEventRecord(w.ev[1], st));
    int rc = enqueue_error_loop(w, B);
    if (rc) return rc;
    BB_CUDA(&w, cudaEventRecord(w.ev[2], st));
    // offsets of the per-read regions of the joined reads, on the device
    bb_k_scan<<<1, 1024, 0, st>>>(B, n, w.seq_cap, w.out_cap, w.speq_cap, w.d_scan.as<BBScanOut>());
    w.launches++;
    BB_CUDA(&w, cudaMemcpyAsync(&w.h_info->scan, w.d_scan.p, sizeof(BBScanOut), cudaMemcpyDeviceToHost, st));
    BB_CUDA(&w, cudaEventRecord(w.ev_scan, st));  // from here on the host can learn the size of this worker's output
    BB_CUDA(&w, cudaMemsetAsync(w.d_dcnt.p, 0, ((size_t)w.seq_cap + 16) * sizeof(unsigned int), st));
    mark(w, st, "scan");
    BB_CUDA(&w, cudaEventRecord(w.ev[3], st));
    bb_k_join<<<n, 256, 0, st>>>(B, c.em);
    w.launches++;
    mark(w, st, "join");
    BB_CUDA(&w, cudaEventRecord(w.ev[4], st));
    if ((rc = enqueue_align_tasks(w, B))) return rc;
    mark(w, st, "align_tail");
    BB_CUDA(&w, cudaEventRecord(w.ev[5], st));
    bb_k_qscores<<<n, 256, 0, st>>>(B, c.qm, c.seed);
    w.launches++;
    mark(w, st, "qscores");
    BB_CUDA(&w, cudaEventRecord(w.ev[6], st));
    bb_k_compact<<<n, 256, 0, st>>>(B);
    w.launches++;
    mark(w, st, "compact");
    BB_CUDA(&w, cudaEventRecord(w.ev[7], st));
    BB_CUDA(&w, cudaMemcpyAsync(w.h_info->counters, w.d_counter.p, BB_N_COUNTERS * sizeof(int), cudaMemcpyDeviceToHost, st));
    BB_CUDA(&w, cudaGetLastError());
    w.ran = true;
    return BB_OK;
}

// Waits for the worker's run and checks what the device reported.  Returns BB_OK when the results are final; when
// something did not fit (buffers sized from the fragment lengths, rounds, levels, split-score scratch) the knob is
// raised and the batch runs again - the results do not depend on any of them.
static int w_finish(Worker &w) {
    if (!w.ran) return set_err(&w, BB_ERR_STATE, "no run to finish");
    if (w.finished) return BB_OK;
    BB_CUDA(&w, cudaSetDevice(w.ctx->device));
    const int n = w.n_reads;
    for (int attempt = 0;; attempt++) {
        w.h_res.resize((size_t)n);
        BB_CUDA(&w, cudaMemcpyAsync(w.h_res.data(), w.d_reads.p, (size_t)n * sizeof(BBReadDev), cudaMemcpyDeviceToHost, w.stream));
        BB_CUDA(&w, cudaStreamSynchronize(w.stream));
        const Worker::RunInfo &info = *w.h_info;
        uint32_t again = 0;
        std::string why;
        if (info.counters[BB_ROUND_BASE(w.n_rounds - 1) + BBC_PENDING] > 0 || info.scan.n_pending > 0) {
            w.n_rounds = std::min(BB_MAX_ROUNDS, w.n_rounds + 3); again |= BB_RERUN_ROUNDS; why += " error-loop rounds";
        }
        if (info.scan.n_nospace > 0) {  // (reads still pending after the last round are counted separately)
            const double need = (double)std::max(info.scan.seq_total, info.scan.out_total) / (double)std::max<int64_t>(1, w.frag_total);
            w.slack = std::max(w.slack * 1.5, need * 1.1 + 0.05); again |= BB_RERUN_SLACK; why += " buffer slack";
        }
        const int last_parity = w.n_levels & 1;  // the queues the level after the last one would read
        int left = 0, overflow = 0;
        for (int s = 0; s < 2; s++) {
            for (int c = 0; c < BBQ_NODE_CLASSES; c++) left += info.qcount[s][BBQ_COUNT(c, last_parity)];
            overflow += info.qcount[s][BBQ_OVERFLOW];
        }
        if (left > 0) { w.extra_levels += 8; again |= BB_RERUN_LEVELS; why += " levels"; }
        if (overflow) { w.slack *= 1.5; again |= BB_RERUN_QUEUES; why += " task queues"; }
        for (int r = 0; r < n && !w.lr_worst; r++) {
            const int f = (w.h_res[(size_t)r].flags & ~BB_FLAG_NOSPACE) >> 8;
            if (f & (16 | 4 | 2)) { w.lr_worst = true; w.slack *= 1.25; again |= BB_RERUN_SCRATCH; why += " alignment scratch"; }
        }
        if (!again) break;
        w.reran = true;
        w.rerun_reasons |= again;
        if (attempt >= 3) return set_err(&w, BB_ERR_INTERNAL, "batch did not fit after growing:" + why);
        w.n_reruns++;
        int rc = w_prepare(w);
        if (rc) return rc;
        if ((rc = w_enqueue(w))) return rc;
    }
    w.finished = true;
    return BB_OK;
}

extern "C" int bb_host_alloc(void **ptr, int64_t bytes) {
    if (!ptr || bytes <= 0) return BB_ERR_ARG;
    *ptr = nullptr;
    return cudaHostAlloc(ptr, (size_t)bytes, cudaHostAllocPortable) == cudaSuccess ? BB_OK : BB_ERR_CUDA;
}

extern "C" int bb_host_free(void *ptr) {
    if (!ptr) return BB_OK;
    return cudaFreeHost(ptr) == cudaSuccess ? BB_OK : BB_ERR_CUDA;
}

extern "C" int bb_synchronize(bb_ctx *ctx) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    for (const auto &w : ctx->workers) BB_CUDA(ctx, cudaStreamSynchronize(w->stream));
    return BB_OK;
}

// A member holds a chunk and at most 31 bytes more: the gzip header with the BC field (18), a stored block's 5 bytes
// when the chunk does not code smaller, CRC32 and ISIZE (8).
extern "C" int64_t bb_bgzf_bound(int64_t n) {
    return n <= 0 ? 0 : n + (n + BB_BGZF_CHUNK - 1) / BB_BGZF_CHUNK * 31;
}

// Input passes of at most this many chunks (134 MB) bound the scratch the context keeps after a call to about 450 MB
// (input, member slots and packed members, each with DevBuf's 1/8 slack).  Fewer chunks per pass leave the compressor
// few waves to even out its slow chunks: 256 (57 MB of scratch) took 51 ms of kernel time on config 1's FASTQ on an H100
// against 34 ms with 2048.
constexpr int64_t kBgzfPassChunks = 2048;

// The start of every compress call (`who` names it in the messages): *use = the bytes it takes, all n with `final`,
// else its whole chunks; the outputs zeroed (n_consumed may be null); out_cap checked against their bound, which
// becomes *n_out when it is short; then the device and the compressor's stream, unless *use is 0.
static int bgzf_begin(bb_ctx *ctx, const char *who, int64_t n, int final, const uint8_t *out, int64_t out_cap,
                      int64_t *n_out, int64_t *n_consumed, int64_t *use) {
    *use = final ? n : n / BB_BGZF_CHUNK * BB_BGZF_CHUNK;
    *n_out = 0;
    if (n_consumed) *n_consumed = 0;
    if (bb_bgzf_bound(*use) > out_cap || (*use && !out)) {
        *n_out = bb_bgzf_bound(*use);
        return set_err(ctx, BB_ERR_CAPACITY, std::string(who) + ": out_cap is less than bb_bgzf_bound of the input");
    }
    if (!*use) return BB_OK;
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    BB_CUDA(ctx, ctx->bgzf.open());
    return BB_OK;
}

// Compresses `use` bytes in passes of at most kBgzfPassChunks chunks and copies the members to out (checked by
// bgzf_begin).  enqueue(done, len, n_chunks) enqueues on the compressor's stream the kernels of the pass over input
// bytes [done, done + len), which write the members to bgzf.out and their offsets to bgzf.off.
template <typename Enqueue>
static int bgzf_passes(bb_ctx *ctx, const char *who, int64_t use, uint8_t *out, int64_t *n_out, Enqueue &&enqueue) {
    Bgzf &b = ctx->bgzf;
    int64_t done = 0, written = 0;
    while (done < use) {
        const int64_t len = std::min(use - done, kBgzfPassChunks * BB_BGZF_CHUNK);
        const int nc = (int)((len + BB_BGZF_CHUNK - 1) / BB_BGZF_CHUNK);
        BB_CUDA(ctx, b.slots.ensure((size_t)nc * 65536));
        BB_CUDA(ctx, b.sizes.ensure((size_t)nc * sizeof(int32_t)));
        BB_CUDA(ctx, b.off.ensure((size_t)(nc + 1) * sizeof(int64_t)));
        BB_CUDA(ctx, b.out.ensure((size_t)bb_bgzf_bound(len)));
        if (const int rc = enqueue(done, len, nc)) return rc;
        BB_CUDA(ctx, cudaGetLastError());
        BB_CUDA(ctx, cudaMemcpyAsync(b.h + 1, b.off.as<int64_t>() + nc, sizeof(int64_t), cudaMemcpyDeviceToHost, b.stream));
        BB_CUDA(ctx, cudaStreamSynchronize(b.stream));
        const int64_t bytes = b.h[1];
        if (bytes <= 0 || bytes > bb_bgzf_bound(len))
            return set_err(ctx, BB_ERR_INTERNAL, std::string(who) + ": members of " + std::to_string(bytes) + " bytes");
        BB_CUDA(ctx, cudaMemcpyAsync(out + written, b.out.p, (size_t)bytes, cudaMemcpyDeviceToHost, b.stream));
        BB_CUDA(ctx, cudaStreamSynchronize(b.stream));
        written += bytes;
        done += len;
    }
    *n_out = written;
    return BB_OK;
}

extern "C" int bb_bgzf_compress(bb_ctx *ctx, const uint8_t *in, int64_t n, int line_mod4, int final, uint8_t *out,
                                int64_t out_cap, int64_t *n_out, int64_t *n_consumed) {
    if (!ctx || n < 0 || (n && !in) || line_mod4 < 0 || line_mod4 > 3 || out_cap < 0 || !n_out || !n_consumed)
        return set_err(ctx, BB_ERR_ARG, "bb_bgzf_compress: bad arguments");
    int64_t use;
    if (const int rc = bgzf_begin(ctx, "bb_bgzf_compress", n, final, out, out_cap, n_out, n_consumed, &use); rc || !use)
        return rc;
    Bgzf &b = ctx->bgzf;
    int mod4 = line_mod4;
    // each pass also reads back the line index of its end (line_pref[n_chunks]): the next pass starts there
    const int rc = bgzf_passes(ctx, "bb_bgzf_compress", use, out, n_out, [&](int64_t done, int64_t len, int nc) {
        if (done) mod4 = (int)(b.h[0] & 3);
        BB_CUDA(ctx, b.in.ensure((size_t)len));
        BB_CUDA(ctx, b.lines.ensure((size_t)nc * sizeof(int32_t)));
        BB_CUDA(ctx, b.pref.ensure((size_t)(nc + 1) * sizeof(int64_t)));
        BB_CUDA(ctx, cudaMemcpyAsync(b.in.p, in + done, (size_t)len, cudaMemcpyHostToDevice, b.stream));
        bbl_bgzf_pass(b.stream, b.in.as<uint8_t>(), len, nc, mod4, b.lines.as<int32_t>(), b.pref.as<int64_t>(),
                      b.slots.as<uint8_t>(), b.sizes.as<int32_t>(), b.off.as<int64_t>(), b.out.as<uint8_t>());
        BB_CUDA(ctx, cudaMemcpyAsync(b.h, b.pref.as<int64_t>() + nc, sizeof(int64_t), cudaMemcpyDeviceToHost, b.stream));
        return BB_OK;
    });
    if (!rc) *n_consumed = use;
    return rc;
}

// Enqueues the device-to-host copies of a finished (or at least scanned) worker's packed block on its stream.
static int w_copy_out(Worker &w, int64_t base, uint8_t *seq_out, uint8_t *qual_out) {
    BB_CUDA(&w, cudaSetDevice(w.ctx->device));
    const int64_t total = w.h_info->scan.out_total;
    if (total > 0) {
        if (!seq_out || !qual_out) return set_err(&w, BB_ERR_ARG, "null output buffers");
        BB_CUDA(&w, cudaMemcpyAsync(seq_out + base, w.d_out_seq.p, (size_t)total, cudaMemcpyDeviceToHost, w.stream));
        BB_CUDA(&w, cudaMemcpyAsync(qual_out + base, w.d_out_qual.p, (size_t)total, cudaMemcpyDeviceToHost, w.stream));
    }
    return BB_OK;
}

// results[pos[i]] describes the worker's i-th read, its out_off shifted by `base` (from the records w_finish fetched).
static int w_results(Worker &w, bb_read_result *results, const int32_t *pos, int64_t base) {
    const int n = w.n_reads;
    int bad = 0, bad_read = -1;
    for (int r = 0; r < n; r++) {
        const BBReadDev &rd = w.h_res[(size_t)r];
        if (results) {
            bb_read_result &o = results[pos ? pos[r] : r];
            o.out_off = base + rd.out_off; o.out_len = rd.out_len; o.frag_len = w.h_inlen[(size_t)r];
            o.matches = rd.matches; o.columns = rd.seq_len + rd.dels; o.loop_count = rd.loop_count;
            o.change_count = rd.change_count; o.n_alignments = rd.n_align; o.flags = rd.flags;
            o.loop_kcycles = rd.kc_loop; o.align_kcycles = rd.kc_align;
        }
        if (rd.flags && !bad) { bad = rd.flags; bad_read = r; }
    }
    if (bad) {
        char msg[160];
        std::snprintf(msg, sizeof(msg), "device invariant violated: read %d flags 0x%x", pos ? pos[bad_read] : bad_read, bad);
        return set_err(&w, BB_ERR_INTERNAL, msg);
    }
    return BB_OK;
}

// ---- batch entry points: deal the reads out over the workers ---------------------------------------------
extern "C" int bb_batch_upload(bb_ctx *ctx, int32_t n_reads, const uint64_t *read_index, const int32_t *seg_off,
                               const bb_segment *segs, const uint8_t *literal_pool, int64_t literal_len,
                               const double *target_identity) {
    if (!ctx) return BB_ERR_ARG;
    if (n_reads <= 0 || !read_index || !seg_off || !segs || !target_identity || literal_len < 0)
        return set_err(ctx, BB_ERR_ARG, "bb_batch_upload: bad arguments");
    if (!ctx->have_em || !ctx->have_qm) return set_err(ctx, BB_ERR_STATE, "upload the error and qscore models first");
    ctx->fetched = false;   // the workers' output buffers are about to be reused
    std::vector<int64_t> len;
    if (const int rc = check_batch(ctx, n_reads, seg_off, segs, literal_len, len)) return rc;
    const int n_workers = (int)ctx->workers.size();
    const int S = ctx->n_split = (n_workers > 1 && n_reads >= 64 * n_workers) ? n_workers : 1;
    ctx->w0().is_head = false;
    if (S == 1)
        return each_worker(ctx, [&](Worker &w, int) -> int { return w_batch_upload(w, n_reads, read_index, seg_off, segs, literal_pool, literal_len, target_identity); });
    // deal the reads out longest first, so that every worker sees the same length distribution
    std::vector<int32_t> order((size_t)n_reads);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return len[(size_t)x] > len[(size_t)y]; });
    ctx->part.assign((size_t)S, std::vector<int32_t>());
    // The chain of Hirschberg levels of the longest reads is the longest dependent chain of the batch.  Worker 0 is a
    // small HEAD batch of the longest reads: its error loop is short, so their alignment starts early and overlaps the
    // other workers' error loops instead of trailing the step.  The other workers share the rest evenly.
    int32_t n_head = 0;
    if (S >= 3 && ctx->knobs.head_worker) {
        int64_t total = 0, hb = 0;
        for (int32_t r = 0; r < n_reads; r++) total += len[(size_t)r];
        const int64_t longest = len[(size_t)order[0]];
        while (n_head < n_reads / 16 && hb < total / S &&
               (10 * len[(size_t)order[(size_t)n_head]] >= 6 * longest || hb < total / (4 * S))) {
            hb += len[(size_t)order[(size_t)n_head]];
            ctx->part[0].push_back(order[(size_t)n_head++]);
        }
        if (n_head < 16) { ctx->part[0].clear(); n_head = 0; }
    }
    ctx->w0().is_head = n_head > 0;
    if (n_head > 0) for (int32_t i = n_head; i < n_reads; i++) ctx->part[(size_t)(1 + (i - n_head) % (S - 1))].push_back(order[(size_t)i]);
    else for (int32_t i = 0; i < n_reads; i++) ctx->part[(size_t)(i % S)].push_back(order[(size_t)i]);
    std::vector<int> rcs((size_t)S, 0);
    std::vector<std::thread> threads;
    auto upload_part = [&](int w) {
        std::vector<int32_t> &mine = ctx->part[(size_t)w];
        std::sort(mine.begin(), mine.end());
        std::vector<uint64_t> ridx; std::vector<int32_t> soff(1, 0); std::vector<bb_segment> sg; std::vector<uint8_t> lit;
        std::vector<double> ident;
        for (int32_t r : mine) {
            ridx.push_back(read_index[r]);
            ident.push_back(target_identity[r]);
            for (int32_t x = seg_off[r]; x < seg_off[r + 1]; x++) {
                bb_segment g = segs[x];
                if (g.kind == BB_SEG_LITERAL) {
                    const int64_t at = (int64_t)lit.size();
                    lit.insert(lit.end(), literal_pool + g.src, literal_pool + g.src + g.len);
                    g.src = at;
                }
                sg.push_back(g);
            }
            soff.push_back((int32_t)sg.size());
        }
        rcs[(size_t)w] = w_batch_upload(*ctx->workers[(size_t)w], (int32_t)mine.size(), ridx.data(), soff.data(), sg.data(),
                                        lit.data(), (int64_t)lit.size(), ident.data());
    };
    for (int w = 1; w < S; w++) threads.emplace_back(upload_part, w);
    upload_part(0);
    for (auto &t : threads) t.join();
    return each_worker(ctx, [&](Worker &, int w) -> int { return rcs[(size_t)w]; });
}

// Asynchronous: the kernel chains of all workers are enqueued from this thread and overlap on the device.
extern "C" int bb_batch_run(bb_ctx *ctx) {
    if (!ctx) return BB_ERR_ARG;
    ctx->fetched = false;   // the run rewrites the workers' output buffers
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    const cudaStream_t st0 = ctx->w0().stream;
    BB_CUDA(ctx, cudaEventRecord(ctx->ev_t0, st0));
    int rc = each_worker(ctx, [&](Worker &w, int i) -> int {
        w.reran = false; w.n_reruns = 0; w.rerun_reasons = 0;
        if (i > 0) BB_CUDA(&w, cudaStreamWaitEvent(w.stream, ctx->ev_t0, 0));
        return w_enqueue(w);
    });
    if (rc) return rc;
    for (int w = 1; w < ctx->n_split; w++) BB_CUDA(ctx, cudaStreamWaitEvent(st0, ctx->workers[(size_t)w]->ev[BB_N_STAGES - 1], 0));
    BB_CUDA(ctx, cudaEventRecord(ctx->ev_t1, st0));
    return BB_OK;
}

extern "C" int bb_last_run_retries(const bb_ctx *ctx, int32_t *n_reruns, uint32_t *reasons) {
    if (!ctx) return BB_ERR_ARG;
    int32_t total = 0;
    uint32_t bits = 0;
    for (int w = 0; w < ctx->n_split; w++) {
        total += ctx->workers[(size_t)w]->n_reruns;
        bits |= ctx->workers[(size_t)w]->rerun_reasons;
    }
    if (n_reruns) *n_reruns = total;
    if (reasons) *reasons = bits;
    return BB_OK;
}

// Task counts of the last run of every worker (see include/badread_b200.h); read from the counters w_finish fetched.
extern "C" int bb_last_run_work(const bb_ctx *ctx, int64_t *work, int64_t *level_nodes, int32_t level_cap, int32_t *n_levels) {
    if (!ctx) return BB_ERR_ARG;
    bb_ctx *mctx = const_cast<bb_ctx *>(ctx);  // for the error message
    if (level_cap < 0 || (level_cap > 0 && !level_nodes)) return set_err(mctx, BB_ERR_ARG, "bb_last_run_work: bad arguments");
    int64_t w[BB_WORK_SLOTS] = {};
    if (level_nodes) std::fill(level_nodes, level_nodes + (size_t)level_cap * BBQ_NODE_CLASSES, 0);
    int levels = 0;
    const int rc = each_worker(mctx, [&](Worker &wk, int) -> int {
        if (!wk.finished) return set_err(&wk, BB_ERR_STATE, "bb_last_run_work: fetch the batch first");
        const Worker::RunInfo &info = *wk.h_info;
        for (int r = 0; r < wk.n_rounds; r++) {  // each kernel passes what it cannot take on to the next
            const int *c = info.counters + BB_ROUND_BASE(r);
            w[BB_WORK_WINDOW_LANE4] += c[BBC_NTASKS] - c[BBC_FB1];
            w[BB_WORK_WINDOW_LANE8] += c[BBC_FB1] - c[BBC_FB2];
            w[BB_WORK_WINDOW_WARP] += c[BBC_FB2];
        }
        for (int s = 0; s < 2; s++) {
            w[BB_WORK_LEAF_LANE] += info.qcount[s][BBQ_LEAF_COUNT];
            w[BB_WORK_LEAF_WARP] += info.qcount[s][BBQ_LEAF_COUNT + 1];
            w[BB_WORK_ROOT_LEAF_LANE] += info.levels[s][0][BB_SNAP_LEAF];
            w[BB_WORK_ROOT_LEAF_WARP] += info.levels[s][0][BB_SNAP_LEAF + 1];
            for (int l = 0; l < std::min(level_cap, BB_MAX_LEVELS); l++)
                for (int c = 0; c < BBQ_NODE_CLASSES; c++) level_nodes[(size_t)l * BBQ_NODE_CLASSES + c] += info.levels[s][l][c];
        }
        levels = std::max(levels, wk.n_levels);
        return BB_OK;
    });
    if (rc) return rc;
    if (work) std::memcpy(work, w, sizeof(w));
    if (n_levels) *n_levels = levels;
    return BB_OK;
}

// Whole-batch device time from the first worker's first kernel to the last worker's last one.  With several
// workers the stages of different workers overlap in time: each stage is reported as its share of the summed
// per-worker stage times, scaled to the whole-batch time.
extern "C" int bb_last_run_ms(bb_ctx *ctx, float *total_ms, float *stage_ms) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    float sum[BB_N_STAGES] = {};
    const int rc = each_worker(ctx, [&](Worker &w, int) -> int {
        if (!w.ran) return set_err(&w, BB_ERR_STATE, "no run to time");
        BB_CUDA(&w, cudaEventSynchronize(w.ev[BB_N_STAGES - 1]));
        for (int i = 0; i < BB_N_STAGES; i++) {  // between consecutive events; the last stage is the whole chain
            const bool all = i == BB_N_STAGES - 1;
            float t = 0.f;
            BB_CUDA(&w, cudaEventElapsedTime(&t, w.ev[all ? 0 : i], w.ev[all ? i : i + 1]));
            sum[i] += t;
        }
        return BB_OK;
    });
    if (rc) return rc;
    BB_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1));
    float total = 0.f;
    BB_CUDA(ctx, cudaEventElapsedTime(&total, ctx->ev_t0, ctx->ev_t1));
    const float scale = sum[BB_N_STAGES - 1] > 0.f ? total / sum[BB_N_STAGES - 1] : 0.f;
    if (total_ms) *total_ms = total;
    for (int i = 0; stage_ms && i < BB_N_STAGES; i++) stage_ms[i] = i < BB_N_STAGES - 1 ? sum[i] * scale : total;
    return BB_OK;
}

// Launch trace of the last run (BADREAD_B200_TRACE=1) as CSV: worker, stream, name, begin_ms, end_ms relative to the
// first worker's first mark; "begin" is the previous mark on the same worker and stream.
extern "C" int bb_trace_dump(bb_ctx *ctx, const char *path) {
    if (!ctx || !path) return BB_ERR_ARG;
    if (!ctx->knobs.trace || ctx->w0().marks.empty()) return set_err(ctx, BB_ERR_STATE, "no trace (set BADREAD_B200_TRACE=1 before bb_create)");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    BB_CUDA(ctx, cudaDeviceSynchronize());
    FILE *f = std::fopen(path, "w");
    if (!f) return set_err(ctx, BB_ERR_ARG, "cannot open trace file");
    std::fprintf(f, "worker,stream,name,begin_ms,end_ms\n");
    const cudaEvent_t base = ctx->w0().marks[0].ev;
    each_worker(ctx, [&](Worker &wk, int w) -> int {
        float prev[10] = {};
        bool have[10] = {};
        for (const Worker::Mark &m : wk.marks) {
            float t = 0.f;
            if (cudaEventElapsedTime(&t, base, m.ev) != cudaSuccess) continue;
            const float b = have[m.stream] ? prev[m.stream] : (have[0] ? prev[0] : t);
            std::fprintf(f, "%d,%d,%s,%.4f,%.4f\n", w, m.stream, m.name, b, t);
            prev[m.stream] = t; have[m.stream] = true;
        }
        return BB_OK;
    });
    std::fclose(f);
    return BB_OK;
}

// Finishes every worker's run, packs their blocks back to back in the caller's buffers and fills the results.
// eager: the copies of a worker were already enqueued behind its kernels with these bases (bb_sequence_batch).
// Without `copy` the blocks stay on the device (bb_fetch_last_batch_results).
static int fetch_all(bb_ctx *ctx, bb_read_result *results, uint8_t *seq_out, uint8_t *qual_out, int64_t out_cap,
                     int64_t *out_total, const std::vector<int64_t> *eager_bases, bool copy = true) {
    ctx->fetched = false;
    std::vector<int64_t> base((size_t)ctx->n_split, 0);
    int64_t total = 0;
    bool moved = false;  // a worker's output size changed after the eager copies were placed (it had to run again)
    int rc = each_worker(ctx, [&](Worker &w, int i) -> int {
        if (!w.ran) return set_err(&w, BB_ERR_STATE, "bb_fetch_last_batch: nothing to fetch");
        if (const int rc = w_finish(w)) return rc;
        if (w.reran) moved = true;
        base[(size_t)i] = total;
        total += w.h_info->scan.out_total;
        return BB_OK;
    });
    if (rc) return rc;
    if (out_total) *out_total = total;
    if (copy) {
        if (out_cap < total) return set_err(ctx, BB_ERR_CAPACITY, "output buffers too small");
        if (total && (!seq_out || !qual_out)) return set_err(ctx, BB_ERR_ARG, "null output buffers");
        const bool have_eager = eager_bases && !moved && *eager_bases == base;
        if (!have_eager && (rc = each_worker(ctx, [&](Worker &w, int i) -> int { return w_copy_out(w, base[(size_t)i], seq_out, qual_out); })))
            return rc;
    }
    rc = each_worker(ctx, [&](Worker &w, int i) -> int {
        BB_CUDA(&w, cudaSetDevice(ctx->device));
        BB_CUDA(&w, cudaStreamSynchronize(w.stream));
        return w_results(w, results, ctx->n_split == 1 ? nullptr : ctx->part[(size_t)i].data(), base[(size_t)i]);
    });
    if (rc) return rc;
    ctx->out_base = base;
    ctx->out_base.push_back(total);
    ctx->fetched = true;
    return BB_OK;
}

extern "C" int bb_fetch_last_batch_results(bb_ctx *ctx, bb_read_result *results, int64_t *out_total) {
    if (!ctx) return BB_ERR_ARG;
    if (!results) return set_err(ctx, BB_ERR_ARG, "bb_fetch_last_batch_results: bad arguments");
    return fetch_all(ctx, results, nullptr, nullptr, 0, out_total, nullptr, false);
}

extern "C" int bb_fetch_last_batch(bb_ctx *ctx, bb_read_result *results, uint8_t *seq_out, uint8_t *qual_out,
                                   int64_t out_cap, int64_t *out_total) {
    if (!ctx) return BB_ERR_ARG;
    return fetch_all(ctx, results, seq_out, qual_out, out_cap, out_total, nullptr);
}

extern "C" int bb_sequence_batch(bb_ctx *ctx, int32_t n_reads, const uint64_t *read_index, const int32_t *seg_off,
                                 const bb_segment *segs, const uint8_t *literal_pool, int64_t literal_len,
                                 const double *target_identity, bb_read_result *results, uint8_t *seq_out,
                                 uint8_t *qual_out, int64_t out_cap, int64_t *out_total) {
    int rc = bb_batch_upload(ctx, n_reads, read_index, seg_off, segs, literal_pool, literal_len, target_identity);
    if (rc) return rc;
    if ((rc = bb_batch_run(ctx))) return rc;
    // each worker's block is copied out as soon as its own chain is done, while the others still compute: its place
    // in the caller's buffers only needs the output sizes of the workers before it, known since their scans
    const int S = ctx->n_split;
    std::vector<int64_t> base((size_t)S, 0);
    int64_t total = 0;
    bool eager = true;
    for (int w = 0; w < S && eager; w++) {
        Worker &wk = *ctx->workers[(size_t)w];
        BB_CUDA(ctx, cudaSetDevice(ctx->device));
        BB_CUDA(ctx, cudaEventSynchronize(wk.ev_scan));
        base[(size_t)w] = total;
        total += wk.h_info->scan.out_total;
        // (a worker with reads that did not fit or did not finish runs again: its size and everything after it moves)
        if (wk.h_info->scan.n_nospace > 0 || wk.h_info->scan.n_pending > 0 || total > out_cap) { eager = false; break; }
        if ((rc = w_copy_out(wk, base[(size_t)w], seq_out, qual_out))) { eager = false; break; }
    }
    return fetch_all(ctx, results, seq_out, qual_out, out_cap, out_total, eager ? &base : nullptr);
}

// ---- BAM output: records built on the device, compressed by the BGZF compressor --------------------------
// Makes the current buffer of `pair` (index cur) hold at least `bytes`: when it is too small, its first `keep` bytes move
// to the other buffer, which becomes the current one.
static int grow_keep(bb_ctx *ctx, DevBuf (&pair)[2], int &cur, size_t bytes, size_t keep) {
    if (bytes <= pair[cur].cap) return BB_OK;
    BB_CUDA(ctx, pair[1 - cur].ensure(bytes));
    if (keep) BB_CUDA(ctx, cudaMemcpyAsync(pair[1 - cur].p, pair[cur].p, keep, cudaMemcpyDeviceToDevice, ctx->bgzf.stream));
    BB_CUDA(ctx, cudaStreamSynchronize(ctx->bgzf.stream));
    pair[cur].release();
    cur = 1 - cur;
    return BB_OK;
}

extern "C" int bb_bam_build(bb_ctx *ctx, int32_t n, const bb_bam_record *recs, const uint8_t *text, int64_t text_len) {
    if (!ctx) return BB_ERR_ARG;
    if (n < 0 || (n && !recs) || text_len < 0 || (text_len && !text)) return set_err(ctx, BB_ERR_ARG, "bb_bam_build: bad arguments");
    if (!ctx->fetched) return set_err(ctx, BB_ERR_STATE, "bb_bam_build: no fetched batch (bb_fetch_last_batch_results)");
    const std::vector<int64_t> &base = ctx->out_base;
    const int n_src = (int)base.size() - 1;
    std::vector<int64_t> pos((size_t)n), size((size_t)n);
    int64_t at = ctx->bam_len;
    for (int32_t i = 0; i < n; i++) {
        const bb_bam_record &r = recs[i];
        int k = 0;
        while (k + 1 < n_src && r.out_off >= base[(size_t)k + 1]) k++;
        if (r.out_off < 0 || r.out_len < 0 || r.out_off + r.out_len > base[(size_t)k + 1] || r.name_len < 0 || r.name_len > 254 ||
            r.co_len < 0 || r.text_off < 0 || r.text_off + r.name_len + r.co_len > text_len) {
            char msg[160];
            std::snprintf(msg, sizeof(msg), "bb_bam_build: record %d lies outside the batch output or the text", i);
            return set_err(ctx, BB_ERR_ARG, msg);
        }
        pos[(size_t)i] = at;
        size[(size_t)i] = bbl_bam_record_size(r.name_len, r.out_len, r.co_len);
        at += size[(size_t)i];
    }
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    BB_CUDA(ctx, ctx->bgzf.open());
    const cudaStream_t st = ctx->bgzf.stream;
    const size_t nf = ctx->bam_field_off.size();
    if (int rc = grow_keep(ctx, ctx->bam_buf, ctx->bam_cur, (size_t)std::max<int64_t>(at, 1), (size_t)ctx->bam_len)) return rc;
    if (int rc = grow_keep(ctx, ctx->bam_fields, ctx->bam_fcur, (nf + 2 * (size_t)n + 1) * 2 * sizeof(int64_t),
                           nf * 2 * sizeof(int64_t)))
        return rc;
    if (n > 0) {
        int rc;
        if ((rc = upload(ctx, st, ctx->bam_recs, recs, (size_t)n))) return rc;
        if ((rc = upload(ctx, st, ctx->bam_pos, pos.data(), (size_t)n))) return rc;
        if ((rc = upload(ctx, st, ctx->bam_text, text, (size_t)text_len))) return rc;
        std::vector<const uint8_t *> seq((size_t)n_src), qual((size_t)n_src);
        for (int k = 0; k < n_src; k++) {
            seq[(size_t)k] = ctx->workers[(size_t)k]->d_out_seq.as<uint8_t>();
            qual[(size_t)k] = ctx->workers[(size_t)k]->d_out_qual.as<uint8_t>();
        }
        bbl_bam_records(st, n, ctx->bam_recs.as<bb_bam_record>(), ctx->bam_pos.as<int64_t>(), ctx->bam_text.as<uint8_t>(), n_src,
                        seq.data(), qual.data(), base.data(), ctx->bam_buf[ctx->bam_cur].as<uint8_t>(), ctx->bam_base,
                        ctx->bam_fields[ctx->bam_fcur].as<int64_t>() + 2 * nf);
        BB_CUDA(ctx, cudaGetLastError());
    }
    BB_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->bam_last_at = ctx->bam_base + ctx->bam_len;
    ctx->bam_last_pos.assign(pos.begin(), pos.end());
    ctx->bam_last_size.assign(size.begin(), size.end());
    for (int32_t i = 0; i < n; i++) {
        const int64_t o_seq = ctx->bam_base + pos[(size_t)i] + 36 + recs[i].name_len + 1;
        ctx->bam_field_off.push_back(o_seq);
        ctx->bam_field_off.push_back(o_seq + (recs[i].out_len + 1) / 2);
    }
    ctx->bam_len = at;
    return BB_OK;
}

extern "C" int bb_bam_compress_device(bb_ctx *ctx, int final, uint8_t *out, int64_t out_cap, int64_t *n_out) {
    if (!ctx) return BB_ERR_ARG;
    if (out_cap < 0 || !n_out) return set_err(ctx, BB_ERR_ARG, "bb_bam_compress_device: bad arguments");
    int64_t use;
    if (const int rc = bgzf_begin(ctx, "bb_bam_compress_device", ctx->bam_len, final, out, out_cap, n_out, nullptr, &use);
        rc || !use)
        return rc;
    Bgzf &b = ctx->bgzf;
    const int cur = ctx->bam_cur, fcur = ctx->bam_fcur;
    const int64_t nf = (int64_t)ctx->bam_field_off.size();
    if (const int rc = bgzf_passes(ctx, "bb_bam_compress_device", use, out, n_out, [&](int64_t done, int64_t len, int nc) {
            bbl_bgzf_pass_bam(b.stream, ctx->bam_buf[cur].as<uint8_t>() + done, len, nc, ctx->bam_fields[fcur].as<int64_t>(), nf,
                              ctx->bam_base + done, b.slots.as<uint8_t>(), b.sizes.as<int32_t>(), b.off.as<int64_t>(),
                              b.out.as<uint8_t>());
            return BB_OK;
        }))
        return rc;
    // the rest (less than a chunk) and the fields that start in it move to the front of the other buffers
    const int64_t rest = ctx->bam_len - use, new_base = ctx->bam_base + use;
    const int64_t keep_from = std::upper_bound(ctx->bam_field_off.begin(), ctx->bam_field_off.end(), new_base) -
                              ctx->bam_field_off.begin();
    const int64_t nk = nf - keep_from;
    BB_CUDA(ctx, ctx->bam_buf[1 - cur].ensure((size_t)std::max<int64_t>(rest, 1)));
    BB_CUDA(ctx, ctx->bam_fields[1 - fcur].ensure((size_t)std::max<int64_t>(nk, 1) * 2 * sizeof(int64_t)));
    if (rest) BB_CUDA(ctx, cudaMemcpyAsync(ctx->bam_buf[1 - cur].p, ctx->bam_buf[cur].as<uint8_t>() + use, (size_t)rest,
                                           cudaMemcpyDeviceToDevice, b.stream));
    if (nk) BB_CUDA(ctx, cudaMemcpyAsync(ctx->bam_fields[1 - fcur].p, ctx->bam_fields[fcur].as<int64_t>() + 2 * keep_from,
                                         (size_t)nk * 2 * sizeof(int64_t), cudaMemcpyDeviceToDevice, b.stream));
    BB_CUDA(ctx, cudaStreamSynchronize(b.stream));
    ctx->bam_cur = 1 - cur;
    ctx->bam_fcur = 1 - fcur;
    ctx->bam_field_off.erase(ctx->bam_field_off.begin(), ctx->bam_field_off.begin() + keep_from);
    ctx->bam_base = new_base;
    ctx->bam_len = rest;
    ctx->bam_last_at = -1;
    return BB_OK;
}

extern "C" int bb_bam_fetch_records(bb_ctx *ctx, const int64_t *dst_off, uint8_t *out, int64_t out_cap, int64_t *n_bytes) {
    if (!ctx) return BB_ERR_ARG;
    if (!n_bytes || out_cap < 0) return set_err(ctx, BB_ERR_ARG, "bb_bam_fetch_records: bad arguments");
    *n_bytes = 0;
    if (ctx->bam_last_at < 0) return set_err(ctx, BB_ERR_STATE, "bb_bam_fetch_records: no records built since the stream was last compressed or fetched");
    const int64_t from = ctx->bam_last_at - ctx->bam_base, bytes = ctx->bam_len - from;
    const size_t n = ctx->bam_last_pos.size();
    *n_bytes = bytes;
    if (bytes && !out) return set_err(ctx, BB_ERR_ARG, "bb_bam_fetch_records: bad arguments");
    for (size_t i = 0; i < n; i++) {
        const int64_t to = dst_off ? dst_off[i] : ctx->bam_last_pos[i] - from;
        if (to < 0 || to + ctx->bam_last_size[i] > out_cap)
            return set_err(ctx, BB_ERR_CAPACITY, "bb_bam_fetch_records: record " + std::to_string(i) + " does not fit out_cap");
    }
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (bytes > ctx->h_bam_cap) {
        if (ctx->h_bam) cudaFreeHost(ctx->h_bam);
        ctx->h_bam = nullptr;
        ctx->h_bam_cap = 0;
        BB_CUDA(ctx, cudaHostAlloc((void **)&ctx->h_bam, (size_t)(bytes + bytes / 4), cudaHostAllocPortable));
        ctx->h_bam_cap = bytes + bytes / 4;
    }
    if (bytes) {
        BB_CUDA(ctx, cudaMemcpyAsync(ctx->h_bam, ctx->bam_buf[ctx->bam_cur].as<uint8_t>() + from, (size_t)bytes,
                                     cudaMemcpyDeviceToHost, ctx->bgzf.stream));
        BB_CUDA(ctx, cudaStreamSynchronize(ctx->bgzf.stream));
    }
    for (size_t i = 0; i < n; i++) {
        const int64_t at = ctx->bam_last_pos[i] - from;
        std::memcpy(out + (dst_off ? dst_off[i] : at), ctx->h_bam + at, (size_t)ctx->bam_last_size[i]);
    }
    ctx->bam_len = from;
    ctx->bam_field_off.resize(ctx->bam_field_off.size() - 2 * n);
    ctx->bam_last_at = -1;
    return BB_OK;
}

extern "C" int bb_bam_compress(bb_ctx *ctx, const uint8_t *in, int64_t n, int64_t stream_base, const int64_t *fields,
                               int64_t n_fields, int final, uint8_t *out, int64_t out_cap, int64_t *n_out, int64_t *n_consumed) {
    if (!ctx) return BB_ERR_ARG;
    if (n < 0 || (n && !in) || stream_base < 0 || n_fields < 0 || (n_fields && !fields) || out_cap < 0 || !n_out || !n_consumed)
        return set_err(ctx, BB_ERR_ARG, "bb_bam_compress: bad arguments");
    for (int64_t i = 0; i < n_fields; i++)   // block starts must come in order, at least a field apart
        if (fields[2 * i + 1] < 0 || (i && fields[2 * i - 2] + fields[2 * i - 1] > fields[2 * i]))
            return set_err(ctx, BB_ERR_ARG, "bb_bam_compress: fields overlap or are out of order");
    int64_t use;
    if (const int rc = bgzf_begin(ctx, "bb_bam_compress", n, final, out, out_cap, n_out, n_consumed, &use); rc || !use)
        return rc;
    Bgzf &b = ctx->bgzf;
    int64_t f0 = 0, f1 = n_fields;   // the fields that start inside in[0 .. use)
    while (f0 < n_fields && fields[2 * f0] < stream_base) f0++;
    while (f1 > f0 && fields[2 * (f1 - 1)] >= stream_base + use) f1--;
    if (int rc = upload(ctx, b.stream, ctx->bam_hfields, fields + 2 * f0, (size_t)(f1 - f0) * 2)) return rc;
    const int rc = bgzf_passes(ctx, "bb_bam_compress", use, out, n_out, [&](int64_t done, int64_t len, int nc) {
        BB_CUDA(ctx, b.in.ensure((size_t)len));
        BB_CUDA(ctx, cudaMemcpyAsync(b.in.p, in + done, (size_t)len, cudaMemcpyHostToDevice, b.stream));
        bbl_bgzf_pass_bam(b.stream, b.in.as<uint8_t>(), len, nc, ctx->bam_hfields.as<int64_t>(), f1 - f0, stream_base + done,
                          b.slots.as<uint8_t>(), b.sizes.as<int32_t>(), b.off.as<int64_t>(), b.out.as<uint8_t>());
        return BB_OK;
    });
    if (!rc) *n_consumed = use;
    return rc;
}

// ---- single-pair entry points (worker 0's stream and scratch) ----------------------------------------------
static int align_pair_device(bb_ctx *ctx, const uint8_t *q, int n, const uint8_t *t, int m, int out5[5]) {
    Worker &w = ctx->w0();
    int rc;
    if ((rc = upload(ctx, w.stream, w.p_q, q, (size_t)n))) return rc;
    if ((rc = upload(ctx, w.stream, w.p_t, t, (size_t)m))) return rc;
    BB_CUDA(ctx, w.p_ops.ensure((size_t)n + 16));
    BB_CUDA(ctx, w.p_dcnt.ensure(((size_t)n + 16) * sizeof(unsigned int)));
    BB_CUDA(ctx, w.p_out.ensure(8 * sizeof(int)));
    if ((rc = ensure_scratch(w, std::max(n, m), std::max(n, m), std::max(n, m)))) return set_err(ctx, rc, w.err);
    BB_CUDA(ctx, cudaMemsetAsync(w.p_dcnt.p, 0, ((size_t)n + 16) * sizeof(unsigned int), w.stream));
    BB_CUDA(ctx, cudaMemsetAsync(w.p_out.p, 0, 8 * sizeof(int), w.stream));
    bbl_align_pair(w.stream, w.p_q.as<uint8_t>(), n, w.p_t.as<uint8_t>(), m, std::max(n, m), w.pool, w.p_ops.as<uint8_t>(),
                   w.p_dcnt.as<unsigned int>(), w.p_out.as<int>());
    w.launches++;
    BB_CUDA(ctx, cudaMemcpyAsync(out5, w.p_out.p, 5 * sizeof(int), cudaMemcpyDeviceToHost, w.stream));
    BB_CUDA(ctx, cudaStreamSynchronize(w.stream));
    if (out5[4]) {
        char msg[96];
        std::snprintf(msg, sizeof(msg), "aligner invariant violated (code 0x%x)", out5[4]);
        return set_err(ctx, BB_ERR_INTERNAL, msg);
    }
    return BB_OK;
}

extern "C" int bb_align_path(bb_ctx *ctx, const uint8_t *query, int32_t q_len, const uint8_t *target, int32_t t_len,
                             uint8_t *ops_out, int64_t ops_cap, int64_t *n_ops, int32_t *distance) {
    if (!ctx) return BB_ERR_ARG;
    if (!query || !target || q_len <= 0 || t_len <= 0) return set_err(ctx, BB_ERR_ARG, "bb_align_path: empty sequence");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    const Worker &w = ctx->w0();
    int out5[5] = {0, 0, 0, 0, 0};
    int rc = align_pair_device(ctx, query, q_len, target, t_len, out5);
    std::vector<uint8_t> ops((size_t)q_len);
    std::vector<unsigned int> dcnt((size_t)q_len);
    if (rc == BB_OK) {
        cudaMemcpy(ops.data(), w.p_ops.p, (size_t)q_len, cudaMemcpyDeviceToHost);
        cudaMemcpy(dcnt.data(), w.p_dcnt.p, (size_t)q_len * sizeof(unsigned int), cudaMemcpyDeviceToHost);
    }
    if (rc) return rc;
    const int64_t total = (int64_t)q_len + out5[1];
    if (n_ops) *n_ops = total;
    if (distance) *distance = out5[2];
    if (total > ops_cap) return set_err(ctx, BB_ERR_CAPACITY, "ops buffer too small");
    static const char sym[3] = {'=', 'X', 'I'};
    int64_t x = 0;
    for (int i = 0; i < out5[3]; i++) ops_out[x++] = 'D';
    for (int i = 0; i < q_len; i++) {
        ops_out[x++] = (uint8_t)sym[ops[(size_t)i] < 3 ? ops[(size_t)i] : 0];
        for (unsigned int d = 0; d < dcnt[(size_t)i]; d++) ops_out[x++] = 'D';
    }
    if (x != total) return set_err(ctx, BB_ERR_INTERNAL, "column count mismatch");
    return BB_OK;
}

extern "C" int bb_get_qscores(bb_ctx *ctx, uint64_t read_index, const uint8_t *seq, int32_t seq_len,
                              const uint8_t *frag, int32_t frag_len, uint8_t *qual_out, int32_t *matches,
                              int32_t *columns) {
    if (!ctx) return BB_ERR_ARG;
    if (!seq || !frag || seq_len <= 0 || frag_len <= 0 || !qual_out) return set_err(ctx, BB_ERR_ARG, "bb_get_qscores: bad arguments");
    if (!ctx->have_qm) return set_err(ctx, BB_ERR_STATE, "upload the qscore model first");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    Worker &w = ctx->w0();
    int out5[5] = {0, 0, 0, 0, 0};
    int rc = align_pair_device(ctx, seq, seq_len, frag, frag_len, out5);
    if (rc == BB_OK) {
        cudaError_t e = w.p_qual.ensure((size_t)seq_len + 16);
        if (e != cudaSuccess) rc = set_err(ctx, BB_ERR_CUDA, cudaGetErrorString(e));
    }
    if (rc == BB_OK) {
        bb_k_qscores_pair<<<(seq_len + 255) / 256, 256, 0, w.stream>>>(w.p_ops.as<uint8_t>(), w.p_dcnt.as<unsigned int>(), seq_len,
                                                                        ctx->qm, ctx->seed, read_index, w.p_qual.as<uint8_t>());
        w.launches++;
        cudaMemcpyAsync(qual_out, w.p_qual.p, (size_t)seq_len, cudaMemcpyDeviceToHost, w.stream);
        cudaError_t e = cudaStreamSynchronize(w.stream);
        if (e != cudaSuccess) rc = set_err(ctx, BB_ERR_CUDA, cudaGetErrorString(e));
    }
    if (rc) return rc;
    if (matches) *matches = out5[0];
    if (columns) *columns = seq_len + out5[1];
    return BB_OK;
}

// ---- the one collective of the path: SUM of emitted bases over the GPUs (stop condition, simulate.py:63) ----------
// Reads shard over GPUs by read index and never exchange data; the only thing the GPUs have to agree on is the running
// total of emitted bases that ends the simulation.  NCCL is loaded at run time (the process's own libnccl.so.2 if one
// is already mapped - e.g. PyTorch's - else the system library), so the library has no link-time dependency on it.
namespace {
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, bb_nccl_id, int) = nullptr;
    int (*CommInitAll)(void **, int, const int *) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool ok = false;
};

NcclApi &nccl() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    // NCCL writes its banner / warnings to stdout unless told otherwise: stdout is where the FASTQ goes
    setenv("NCCL_DEBUG_FILE", "/dev/stderr", 0);
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
    if (!h) return api;
    api.lib = h;
    api.GetUniqueId = (int (*)(void *))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void **, int, bb_nccl_id, int))dlsym(h, "ncclCommInitRank");
    api.CommInitAll = (int (*)(void **, int, const int *))dlsym(h, "ncclCommInitAll");
    api.AllReduce = (int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclAllReduce");
    api.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
    api.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
    api.CommDestroy = (int (*)(void *))dlsym(h, "ncclCommAbort");  // teardown must not wait for peers that already left
    if (!api.CommDestroy) api.CommDestroy = (int (*)(void *))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
    nccl_destroy = (void (*)(void *))api.CommDestroy;
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommInitAll && api.AllReduce && api.GroupStart && api.GroupEnd;
    return api;
}
constexpr int kNcclInt64 = 4, kNcclSum = 0;  // ncclDataType_t / ncclRedOp_t values (nccl.h)

int nccl_err(bb_ctx *ctx, const char *what, int rc) {
    const char *msg = nccl().GetErrorString ? nccl().GetErrorString(rc) : "?";
    return set_err(ctx, BB_ERR_CUDA, std::string(what) + ": " + msg);
}
}  // namespace

extern "C" int bb_nccl_available(void) { return nccl().ok ? 1 : 0; }

// NCCL prints its version banner with a plain printf to stdout when NCCL_DEBUG=VERSION (init.cc showVersion; the debug
// file setting does not apply to it) - and stdout is where `badread simulate` writes the FASTQ (measured: 29 bytes that
// made the 2-GPU output differ from the 1-GPU one).  While a communicator is created, file descriptor 1 points at stderr.
struct StdoutToStderr {
    int saved = -1;
    StdoutToStderr() {
        fflush(stdout);
        saved = dup(1);
        if (saved >= 0) dup2(2, 1);
    }
    ~StdoutToStderr() {
        fflush(stdout);
        if (saved >= 0) { dup2(saved, 1); close(saved); }
    }
};

extern "C" int bb_comm_unique_id(bb_nccl_id *id) {
    if (!id) return BB_ERR_ARG;
    if (!nccl().ok) return BB_ERR_STATE;
    return nccl().GetUniqueId(id) == 0 ? BB_OK : BB_ERR_CUDA;
}

extern "C" int bb_comm_init_rank(bb_ctx *ctx, const bb_nccl_id *id, int rank, int world) {
    if (!ctx || !id || rank < 0 || rank >= world) return BB_ERR_ARG;
    if (!nccl().ok) return set_err(ctx, BB_ERR_STATE, "libnccl.so.2 could not be loaded");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->nccl_comm && nccl().CommDestroy) { nccl().CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
    int rc;
    {
        StdoutToStderr guard;
        rc = nccl().CommInitRank(&ctx->nccl_comm, world, *id, rank);
    }
    if (rc) return nccl_err(ctx, "ncclCommInitRank", rc);
    BB_CUDA(ctx, ctx->d_red.ensure(2 * sizeof(long long)));
    return BB_OK;
}

extern "C" int bb_comm_init_all(bb_ctx **ctxs, int n) {
    if (!ctxs || n <= 0) return BB_ERR_ARG;
    if (!nccl().ok) return set_err(ctxs[0], BB_ERR_STATE, "libnccl.so.2 could not be loaded");
    std::vector<int> devs((size_t)n);
    std::vector<void *> comms((size_t)n, nullptr);
    for (int i = 0; i < n; i++) { if (!ctxs[i]) return BB_ERR_ARG; devs[(size_t)i] = ctxs[i]->device; }
    int rc;
    {
        StdoutToStderr guard;
        rc = nccl().CommInitAll(comms.data(), n, devs.data());
    }
    if (rc) return nccl_err(ctxs[0], "ncclCommInitAll", rc);
    for (int i = 0; i < n; i++) {
        ctxs[i]->nccl_comm = comms[(size_t)i];
        BB_CUDA(ctxs[i], cudaSetDevice(ctxs[i]->device));
        BB_CUDA(ctxs[i], ctxs[i]->d_red.ensure(2 * sizeof(long long)));
    }
    return BB_OK;
}

// One process per GPU: every rank passes its local count, all get the sum.
extern "C" int bb_allreduce_bases(bb_ctx *ctx, int64_t local, int64_t *total) {
    if (!ctx || !total) return BB_ERR_ARG;
    if (!ctx->nccl_comm) return set_err(ctx, BB_ERR_STATE, "bb_allreduce_bases: no communicator (bb_comm_init_rank)");
    BB_CUDA(ctx, cudaSetDevice(ctx->device));
    long long *d = ctx->d_red.as<long long>();
    const long long v = local;
    BB_CUDA(ctx, cudaMemcpyAsync(d, &v, sizeof(v), cudaMemcpyHostToDevice, ctx->w0().stream));
    const int rc = nccl().AllReduce(d, d + 1, 1, kNcclInt64, kNcclSum, ctx->nccl_comm, ctx->w0().stream);
    if (rc) return nccl_err(ctx, "ncclAllReduce", rc);
    long long out = 0;
    BB_CUDA(ctx, cudaMemcpyAsync(&out, d + 1, sizeof(out), cudaMemcpyDeviceToHost, ctx->w0().stream));
    BB_CUDA(ctx, cudaStreamSynchronize(ctx->w0().stream));
    *total = out;
    return BB_OK;
}

// One process, several GPUs (the CLI's --gpus N): the contexts' counts are summed in one NCCL group call.
extern "C" int bb_allreduce_bases_all(bb_ctx **ctxs, int n, const int64_t *local, int64_t *total) {
    if (!ctxs || n <= 0 || !local || !total) return BB_ERR_ARG;
    for (int i = 0; i < n; i++)
        if (!ctxs[i] || !ctxs[i]->nccl_comm) return set_err(ctxs[0], BB_ERR_STATE, "bb_allreduce_bases_all: no communicator (bb_comm_init_all)");
    for (int i = 0; i < n; i++) {
        BB_CUDA(ctxs[i], cudaSetDevice(ctxs[i]->device));
        const long long v = local[i];
        BB_CUDA(ctxs[i], cudaMemcpyAsync(ctxs[i]->d_red.p, &v, sizeof(v), cudaMemcpyHostToDevice, ctxs[i]->w0().stream));
        BB_CUDA(ctxs[i], cudaStreamSynchronize(ctxs[i]->w0().stream));  // `v` leaves scope
    }
    int rc = nccl().GroupStart();
    for (int i = 0; i < n && !rc; i++) {
        long long *d = ctxs[i]->d_red.as<long long>();
        rc = nccl().AllReduce(d, d + 1, 1, kNcclInt64, kNcclSum, ctxs[i]->nccl_comm, ctxs[i]->w0().stream);
    }
    const int rc2 = nccl().GroupEnd();
    if (rc || rc2) return nccl_err(ctxs[0], "ncclAllReduce (group)", rc ? rc : rc2);
    long long out = 0;
    BB_CUDA(ctxs[0], cudaSetDevice(ctxs[0]->device));
    BB_CUDA(ctxs[0], cudaMemcpyAsync(&out, ctxs[0]->d_red.as<long long>() + 1, sizeof(out), cudaMemcpyDeviceToHost, ctxs[0]->w0().stream));
    for (int i = 0; i < n; i++) {
        BB_CUDA(ctxs[i], cudaSetDevice(ctxs[i]->device));
        BB_CUDA(ctxs[i], cudaStreamSynchronize(ctxs[i]->w0().stream));
    }
    *total = out;
    return BB_OK;
}
