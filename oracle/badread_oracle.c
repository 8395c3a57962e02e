/*
 * badread_oracle.c — CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE)
 *
 * A plain-C restatement of the Badread per-read error-injection hot path.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this library.
 * The product (badread_b200/) never links, imports or calls anything in oracle/.
 *
 * What is restated (all citations relative to /root/reference/):
 *   - CPython `random` module primitives (MT19937, getrandbits, _randbelow, random(), choices):
 *       Lib/random.py of CPython 3.12 as consumed by badread/misc.py:156-182, error_model.py:135-176,
 *       simulate.py:294,338 and qscore_model.py:273-287.
 *   - simulate.sequence_fragment                      badread/simulate.py:256-358
 *   - ErrorModel.add_errors_to_kmer / add_one_random_change   badread/error_model.py:135-176
 *   - get_qscores / QScoreModel.get_qscore            badread/qscore_model.py:32-75, 273-287
 *   - identity_from_edlib_cigar                       badread/misc.py:228-240
 *   - edlib.align(query, target, task='path') (third-party `edlib`, NOT in /root/reference,
 *     un-pinned in requirements.txt:1 / setup.py:95).  Restated from edlib's published algorithm
 *     (Šošić & Šikić 2017; edlib.cpp >= 1.2): Myers bit-vector NW; path = traceback with priority
 *     UP(I) > LEFT(D) > DIAGONAL when the edlib traceback state estimate
 *     (2*8+4)*ceil(|q|/64)*|t| + 2*4*|t| is < 1 MiB, otherwise Hirschberg split on the target at
 *     |t|/2 choosing the smallest interior query row whose left+right scores equal the best score
 *     (then row -1, then row |q|-1), recursing with the same size switch.
 *     PARITY UNPINNED at this boundary: edlib is absent from this image, the reference's tests
 *     declare ties "all acceptable" (test/test_error_model.py:63-80,111-135); see DESIGN.md.
 *
 * Two RNG disciplines:
 *   mode 0 "mt"     one sequential MT19937 stream — byte-for-byte what the reference consumes; used to pin
 *                   this oracle against the unmodified reference (tests/golden/).
 *   mode 1 "philox" counter-based Philox4x32-10 keyed by (seed, read index, purpose, index) — the discipline
 *                   the CUDA path implements; GPU output must equal this mode byte for byte.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define BO_EXPORT __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------
 * RNG
 * ---------------------------------------------------------------------------------------------- */
enum { BO_RNG_MT = 0, BO_RNG_PHILOX = 1 };
enum { BO_PURPOSE_PAD = 2, BO_PURPOSE_LOOP = 3, BO_PURPOSE_WINDOW = 4, BO_PURPOSE_QSCORE = 5 };

typedef struct {
    int mode;
    uint32_t mt[624];
    int mti;
    uint32_t key[2];
    uint32_t ctr[4];
    uint32_t buf[4];
    int bufpos;
} bo_rng;

static void mt_init_genrand(bo_rng *r, uint32_t s) {
    r->mt[0] = s;
    for (int i = 1; i < 624; i++)
        r->mt[i] = 1812433253u * (r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) + (uint32_t)i;
    r->mti = 624;
}

/* random.seed(int) == init_by_array(little-endian 32-bit words of abs(seed)) (CPython _randommodule.c) */
static void mt_init_by_array(bo_rng *r, const uint32_t *key, int klen) {
    mt_init_genrand(r, 19650218u);
    int i = 1, j = 0;
    int k = 624 > klen ? 624 : klen;
    for (; k; k--) {
        r->mt[i] = (r->mt[i] ^ ((r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
        i++; j++;
        if (i >= 624) { r->mt[0] = r->mt[623]; i = 1; }
        if (j >= klen) j = 0;
    }
    for (k = 623; k; k--) {
        r->mt[i] = (r->mt[i] ^ ((r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
        i++;
        if (i >= 624) { r->mt[0] = r->mt[623]; i = 1; }
    }
    r->mt[0] = 0x80000000u;
    r->mti = 624;
}

static uint32_t mt_next(bo_rng *r) {
    if (r->mti >= 624) {
        uint32_t *mt = r->mt;
        int kk;
        for (kk = 0; kk < 624 - 397; kk++) {
            uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
            mt[kk] = mt[kk + 397] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        for (; kk < 623; kk++) {
            uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
            mt[kk] = mt[kk + (397 - 624)] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        uint32_t y = (mt[623] & 0x80000000u) | (mt[0] & 0x7fffffffu);
        mt[623] = mt[396] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        r->mti = 0;
    }
    uint32_t y = r->mt[r->mti++];
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}

static void philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3];
    uint32_t k0 = key[0], k1 = key[1];
    for (int i = 0; i < 10; i++) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* Philox stream layout shared with the CUDA path (badread_b200/csrc/bb_rng.cuh):
 *   key = (seed_lo, seed_hi); ctr = (index, purpose<<24 | block, read_lo, read_hi); words consumed in order. */
static void rng_stream(bo_rng *r, uint32_t purpose, uint32_t index) {
    if (r->mode != BO_RNG_PHILOX) return;
    r->ctr[0] = index;
    r->ctr[1] = purpose << 24;
    r->bufpos = 4;
}

static uint32_t rng_u32(bo_rng *r) {
    if (r->mode == BO_RNG_MT) return mt_next(r);
    if (r->bufpos >= 4) {
        philox4x32_10(r->ctr, r->key, r->buf);
        r->ctr[1]++;
        r->bufpos = 0;
    }
    return r->buf[r->bufpos++];
}

static uint32_t rng_getrandbits(bo_rng *r, int k) { /* 1 <= k <= 32 */
    return rng_u32(r) >> (32 - k);
}

static int bit_length(uint32_t n) {
    int k = 0;
    while (n) { k++; n >>= 1; }
    return k;
}

/* Random._randbelow_with_getrandbits (CPython 3.12 Lib/random.py) */
static uint32_t rng_randbelow(bo_rng *r, uint32_t n) {
    int k = bit_length(n);
    uint32_t v = rng_getrandbits(r, k);
    while (v >= n) v = rng_getrandbits(r, k);
    return v;
}

/* random.random(): 53-bit double from two words (CPython _randommodule.c) */
static double rng_random(bo_rng *r) {
    uint32_t a = rng_u32(r) >> 5, b = rng_u32(r) >> 6;
    return (a * 67108864.0 + b) * (1.0 / 9007199254740992.0);
}

/* random.choices(pop, weights=w)[0] with cum = list(accumulate(w)) precomputed:
 * bisect_right(cum, random()*cum[-1], 0, n-1) */
static int rng_choices(bo_rng *r, const double *cum, int n) {
    double x = rng_random(r) * cum[n - 1];
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        int mid = (lo + hi) / 2;
        if (x < cum[mid]) hi = mid; else lo = mid + 1;
    }
    return lo;
}

static const char BASES[4] = {'A', 'C', 'G', 'T'};

/* misc.get_random_base: RANDOM_SEQ_DICT[random.randint(0, 3)]  (misc.py:159-163) */
static uint8_t rng_random_base(bo_rng *r) { return (uint8_t)BASES[rng_randbelow(r, 4)]; }

/* misc.get_random_different_base (misc.py:166-170) */
static uint8_t rng_random_different_base(bo_rng *r, uint8_t b) {
    uint8_t x = rng_random_base(r);
    while (x == b) x = rng_random_base(r);
    return x;
}

BO_EXPORT bo_rng *bo_rng_create(int mode, uint64_t seed, uint64_t read_index) {
    bo_rng *r = (bo_rng *)calloc(1, sizeof(bo_rng));
    r->mode = mode;
    if (mode == BO_RNG_MT) {
        uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
        mt_init_by_array(r, key, key[1] ? 2 : 1);
    } else {
        r->key[0] = (uint32_t)seed; r->key[1] = (uint32_t)(seed >> 32);
        r->ctr[2] = (uint32_t)read_index; r->ctr[3] = (uint32_t)(read_index >> 32);
        r->bufpos = 4;
    }
    return r;
}
BO_EXPORT void bo_rng_destroy(bo_rng *r) { free(r); }
BO_EXPORT uint32_t bo_rng_u32(bo_rng *r) { return rng_u32(r); }
BO_EXPORT double bo_rng_random(bo_rng *r) { return rng_random(r); }
BO_EXPORT uint32_t bo_rng_randbelow(bo_rng *r, uint32_t n) { return rng_randbelow(r, n); }
BO_EXPORT void bo_rng_stream(bo_rng *r, uint32_t purpose, uint32_t index) { rng_stream(r, purpose, index); }
BO_EXPORT void bo_philox(const uint32_t *ctr, const uint32_t *key, uint32_t *out) { philox4x32_10(ctr, key, out); }

/* ------------------------------------------------------------------------------------------------
 * Aligner: edlib.align(query, target, mode='NW', task='path') restated
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    uint8_t *ops; /* '=', 'X', 'I', 'D', one per alignment column */
    int64_t n, cap;
} opbuf;

static void op_push(opbuf *o, uint8_t c, int64_t count) {
    if (o->n + count > o->cap) {
        while (o->n + count > o->cap) o->cap = o->cap ? o->cap * 2 : 1024;
        o->ops = (uint8_t *)realloc(o->ops, (size_t)o->cap);
    }
    memset(o->ops + o->n, c, (size_t)count);
    o->n += count;
}

/* edlib's switch between traceback and Hirschberg (edlib.cpp obtainAlignment):
 * alignmentDataSize = (2*sizeof(Word)+sizeof(int))*maxNumBlocks*targetLength + 2*sizeof(int)*targetLength */
static int64_t g_traceback_limit = 1024 * 1024;
BO_EXPORT void bo_set_traceback_limit(int64_t v) { g_traceback_limit = v; }
BO_EXPORT int64_t bo_get_traceback_limit(void) { return g_traceback_limit; }

static int uses_traceback(int64_t n, int64_t m) {
    int64_t blocks = (n + 63) / 64;
    return (20 * blocks * m + 8 * m) < g_traceback_limit;
}

typedef struct { int64_t a, b; } band_t; /* a cell (i,j) is inside when j - a <= i <= j + b */

static band_t band_for(int64_t n, int64_t m, int64_t k) {
    /* a path of cost <= k from (0,0) to (n,m) has at most (k-(n-m))/2 deletions and (k+(n-m))/2 insertions */
    band_t bd;
    bd.a = (k - (n - m)) / 2;
    bd.b = (k + (n - m)) / 2;
    if (bd.a < 0) bd.a = 0;
    if (bd.b < 0) bd.b = 0;
    return bd;
}

typedef struct {
    int64_t nblocks;
    int nsym;
    int sym_of[256];
    uint64_t *peq; /* [nsym+1][nblocks]; last row all zero */
} peq_t;

static void peq_build(peq_t *p, const uint8_t *q, int64_t n) {
    p->nblocks = (n + 63) / 64;
    p->nsym = 0;
    for (int i = 0; i < 256; i++) p->sym_of[i] = -1;
    for (int64_t i = 0; i < n; i++)
        if (p->sym_of[q[i]] < 0) p->sym_of[q[i]] = p->nsym++;
    p->peq = (uint64_t *)calloc((size_t)((p->nsym + 1) * p->nblocks), sizeof(uint64_t));
    for (int64_t i = 0; i < n; i++)
        p->peq[p->sym_of[q[i]] * p->nblocks + (i >> 6)] |= 1ull << (i & 63);
}
static const uint64_t *peq_row(const peq_t *p, uint8_t c) {
    int s = p->sym_of[c];
    if (s < 0) s = p->nsym;
    return p->peq + (int64_t)s * p->nblocks;
}
static void peq_free(peq_t *p) { free(p->peq); }

/* One Myers/Hyyrö block step (edlib.cpp calculateBlock). Returns hout; *ph_raw is the horizontal +1 delta
 * vector of this column before the shift (bit r set <=> D[r][j] - D[r][j-1] == +1). */
static inline int block_step(uint64_t *Pv, uint64_t *Mv, uint64_t Eq, int hin, uint64_t *ph_raw) {
    uint64_t hin_neg = (hin < 0) ? 1ull : 0ull;
    uint64_t Xv = Eq | *Mv;
    Eq |= hin_neg;
    uint64_t Xh = (((Eq & *Pv) + *Pv) ^ *Pv) | Eq;
    uint64_t Ph = *Mv | ~(Xh | *Pv);
    uint64_t Mh = *Pv & Xh;
    int hout = (int)(Ph >> 63) - (int)(Mh >> 63);
    if (ph_raw) *ph_raw = Ph;
    Ph <<= 1; Mh <<= 1;
    Mh |= hin_neg;
    if (hin > 0) Ph |= 1ull;
    *Pv = Mh | ~(Xv | Ph);
    *Mv = Ph & Xv;
    return hout;
}

#define SCORE_INF (INT64_C(1) << 40)

/* Banded NW over columns [0, ncols) of t against all of q (n rows).
 * hist (optional): (Pv, PhRaw) pairs per (column, block - first_block(column)), nb_alloc pairs per column.
 * colscore (optional): D[i][ncols-1] for all i (SCORE_INF outside the band).
 * Returns D[n-1][ncols-1] (upper bound if the true value exceeds what the band admits). */
/* Work accounting (bench.py's integer-pipe figure): 64-row block updates of the passes a PATH needs - the two passes
 * of every Hirschberg node and the history pass of every leaf, with bands from exact scores - not those of the
 * distance search in front (edlib's k = 64, 128, ... loop; the GPU path has the bound up front and skips it). */
static __thread int t_count_blocks = 0;
static int64_t g_block_steps = 0;
BO_EXPORT void bo_block_steps_reset(void) { __atomic_store_n(&g_block_steps, 0, __ATOMIC_RELAXED); }
BO_EXPORT int64_t bo_block_steps(void) { return __atomic_load_n(&g_block_steps, __ATOMIC_RELAXED); }

static int64_t banded_nw(const uint8_t *q, int64_t n, const uint8_t *t, int64_t ncols, band_t bd,
                         uint64_t *hist, int64_t nb_alloc, int64_t *colscore) {
    int64_t n_steps = 0;
    peq_t pq;
    peq_build(&pq, q, n);
    int64_t nblocks = pq.nblocks;
    uint64_t *P = (uint64_t *)malloc((size_t)nblocks * 8), *M = (uint64_t *)malloc((size_t)nblocks * 8);
    int64_t *score = (int64_t *)malloc((size_t)nblocks * 8); /* D at the bottom row of each block */
    int64_t first = 0, last = -1;
    for (int64_t j = 0; j < ncols; j++) {
        int64_t lo_row = j - bd.a; if (lo_row < 0) lo_row = 0;
        int64_t hi_row = j + bd.b; if (hi_row > n - 1) hi_row = n - 1;
        int64_t nf = lo_row >> 6, nl = hi_row >> 6;
        if (nf > nblocks - 1) nf = nblocks - 1;
        if (nf > first) first = nf;
        while (last < nl) { /* a block entering the band starts from the all-(+1) upper bound */
            last++;
            P[last] = ~0ull; M[last] = 0;
            /* column j-1 value at the block's bottom row; score[last-1] has not been stepped for column j yet */
            score[last] = (last == 0) ? (j + 64) : score[last - 1] + 64;
        }
        const uint64_t *eq = peq_row(&pq, t[j]);
        int hin = 1;
        n_steps += last - first + 1;
        for (int64_t b = first; b <= last; b++) {
            uint64_t ph;
            hin = block_step(&P[b], &M[b], eq[b], hin, &ph);
            score[b] += hin;
            if (hist) {
                int64_t slot = (j * nb_alloc + (b - nf)) * 2;
                if (b - nf >= 0 && b - nf < nb_alloc) { hist[slot] = P[b]; hist[slot + 1] = ph; }
            }
        }
    }
    int64_t result = SCORE_INF;
    if (ncols > 0) {
        int64_t j = ncols - 1;
        if (colscore) for (int64_t i = 0; i < n; i++) colscore[i] = SCORE_INF;
        int64_t lo_row = j - bd.a; if (lo_row < 0) lo_row = 0;
        int64_t hi_row = j + bd.b; if (hi_row > n - 1) hi_row = n - 1;
        for (int64_t b = first; b <= last; b++) {
            int64_t s = score[b];
            for (int r = 63; r >= 0; r--) {
                int64_t i = b * 64 + r;
                if (i < n) {
                    if (colscore && i >= lo_row && i <= hi_row) colscore[i] = s;
                    if (i == n - 1) result = s;
                }
                s -= (int64_t)((P[b] >> r) & 1) - (int64_t)((M[b] >> r) & 1);
            }
        }
    }
    free(P); free(M); free(score); peq_free(&pq);
    if (t_count_blocks) __atomic_fetch_add(&g_block_steps, n_steps, __ATOMIC_RELAXED);
    return result;
}

/* NW edit distance (edlib phase 1: k = 64, 128, ... until the banded result is <= k) */
static int64_t nw_distance(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m) {
    if (n == 0) return m;
    if (m == 0) return n;
    int64_t k = 64;
    for (;;) {
        int64_t diff = n > m ? n - m : m - n;
        if (k >= diff) {
            int64_t kk = k; int64_t mx = n > m ? n : m; if (kk > mx) kk = mx;
            int64_t d = banded_nw(q, n, t, m, band_for(n, m, kk), NULL, 0, NULL);
            if (d <= kk) return d;
        }
        k *= 2;
    }
}

/* edlib.cpp obtainAlignmentTraceback, expressed on the stored vertical/horizontal +1 deltas:
 * at (i,j): UP (emit I) if D[i][j]-D[i-1][j]==1, else LEFT (emit D) if D[i][j]-D[i][j-1]==1, else diagonal. */
static void leaf_traceback(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int64_t best, opbuf *out) {
    band_t bd = band_for(n, m, best);
    int64_t nb_alloc = ((bd.a + bd.b) >> 6) + 2;
    uint64_t *hist = (uint64_t *)malloc((size_t)(m * nb_alloc * 2) * 8);
    int64_t d = banded_nw(q, n, t, m, bd, hist, nb_alloc, NULL);
    if (d != best) { fprintf(stderr, "oracle: leaf score mismatch %lld != %lld\n", (long long)d, (long long)best); abort(); }
    opbuf rev = {0};
    int64_t i = n - 1, j = m - 1;
    while (i >= 0 && j >= 0) {
        int64_t lo_row = j - bd.a; if (lo_row < 0) lo_row = 0;
        int64_t nf = lo_row >> 6; if (nf > (n + 63) / 64 - 1) nf = (n + 63) / 64 - 1;
        int64_t b = (i >> 6) - nf;
        if (b < 0 || b >= nb_alloc) { fprintf(stderr, "oracle: traceback left the band\n"); abort(); }
        uint64_t pv = hist[(j * nb_alloc + b) * 2], ph = hist[(j * nb_alloc + b) * 2 + 1];
        int r = (int)(i & 63);
        if ((pv >> r) & 1) { op_push(&rev, 'I', 1); i--; }
        else if ((ph >> r) & 1) { op_push(&rev, 'D', 1); j--; }
        else { op_push(&rev, q[i] == t[j] ? '=' : 'X', 1); i--; j--; }
    }
    if (i >= 0) op_push(&rev, 'I', i + 1);
    if (j >= 0) op_push(&rev, 'D', j + 1);
    for (int64_t x = rev.n - 1; x >= 0; x--) op_push(out, rev.ops[x], 1);
    free(rev.ops); free(hist);
}

static uint8_t *reversed(const uint8_t *s, int64_t n) {
    uint8_t *r = (uint8_t *)malloc((size_t)(n ? n : 1));
    for (int64_t i = 0; i < n; i++) r[i] = s[n - 1 - i];
    return r;
}

/* Tree of a final alignment (tests only).  After bo_tree_arm(1), this thread's next final alignment - the one
 * get_qscores makes, or a bo_align_path call - records every obtain_alignment / naive_obtain call with n > 0 and m > 0
 * in call order, BO_TREE_FIELDS values each: depth, q0, nn, t0, mm, best, is_leaf, target_has_non_acgt.  The window
 * alignments of the error loop are never recorded.  Thread-local: bo_sequence_batch's workers record their own reads. */
#define BO_TREE_FIELDS 8
typedef struct { int64_t *v; int64_t n, cap; const uint8_t *q_base, *t_base; } tree_rec;
static __thread int t_tree_armed = 0;
static __thread tree_rec t_tree_buf = {0};   /* the last recorded tree, until bo_tree_take */
static __thread tree_rec *t_tree = NULL;     /* set while a final alignment records */

static void tree_begin(const uint8_t *q, const uint8_t *t) {
    if (!t_tree_armed) return;
    t_tree_armed = 0;
    free(t_tree_buf.v);
    memset(&t_tree_buf, 0, sizeof(t_tree_buf));
    t_tree_buf.q_base = q; t_tree_buf.t_base = t;
    t_tree = &t_tree_buf;
}
static void tree_end(void) { t_tree = NULL; }
static void tree_add(int depth, const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int64_t best, int leaf) {
    tree_rec *r = t_tree;
    if (!r) return;
    if (r->n + BO_TREE_FIELDS > r->cap) {
        r->cap = r->cap ? 2 * r->cap : 64 * BO_TREE_FIELDS;
        r->v = (int64_t *)realloc(r->v, (size_t)r->cap * sizeof(int64_t));
    }
    int non_acgt = 0;
    for (int64_t j = 0; j < m && !non_acgt; j++) non_acgt = t[j] != 'A' && t[j] != 'C' && t[j] != 'G' && t[j] != 'T';
    int64_t *e = r->v + r->n;
    r->n += BO_TREE_FIELDS;
    e[0] = depth; e[1] = q - r->q_base; e[2] = n; e[3] = t - r->t_base; e[4] = m; e[5] = best; e[6] = leaf; e[7] = non_acgt;
}
BO_EXPORT void bo_tree_arm(int on) { t_tree_armed = on; }
/* Hands the last recorded tree over: returns its number of entries, *out (release with bo_free) their values. */
BO_EXPORT int64_t bo_tree_take(int64_t **out) {
    const int64_t n = t_tree_buf.n / BO_TREE_FIELDS;
    *out = t_tree_buf.v;
    memset(&t_tree_buf, 0, sizeof(t_tree_buf));
    return n;
}

/* edlib.cpp obtainAlignment / obtainAlignmentHirschberg (depth: of this call in the recursion, for the tree) */
static void obtain_alignment(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int64_t best, opbuf *out, int depth) {
    if (n == 0) { op_push(out, 'D', m); return; }
    if (m == 0) { op_push(out, 'I', n); return; }
    tree_add(depth, q, n, t, m, best, uses_traceback(n, m));
    if (uses_traceback(n, m)) { leaf_traceback(q, n, t, m, best, out); return; }

    int64_t left_w = m / 2, right_w = m - left_w;
    band_t bd = band_for(n, m, best);
    int64_t *sl = (int64_t *)malloc((size_t)n * 8), *sr = (int64_t *)malloc((size_t)n * 8);
    banded_nw(q, n, t, left_w, bd, NULL, 0, sl); /* sl[r] = D(q[0..r], t[0..left_w)) */
    uint8_t *rq = reversed(q, n), *rt = reversed(t, m);
    band_t rbd = band_for(n, m, best);
    banded_nw(rq, n, rt, right_w, rbd, NULL, 0, sr); /* sr[x] = D(rq[0..x], rt[0..right_w)) */
    free(rq); free(rt);
    /* right[r] (forward coordinates, suffix q[r..]) = sr[n-1-r] */
    int64_t split = -2, left_score = -1, right_score = -1;
    for (int64_t r = 0; r <= n - 2; r++) {
        int64_t ls = sl[r], rs = sr[n - 1 - (r + 1)];
        if (ls + rs == best) { split = r; left_score = ls; right_score = rs; break; }
    }
    if (split == -2) { /* boundary: empty query prefix on the left */
        int64_t rs = sr[n - 1];
        if (left_w + rs == best) { split = -1; left_score = left_w; right_score = rs; }
    }
    if (split == -2) { /* boundary: empty query suffix on the right */
        int64_t ls = sl[n - 1];
        if (ls + right_w == best) { split = n - 1; left_score = ls; right_score = right_w; }
    }
    free(sl); free(sr);
    if (split == -2) { fprintf(stderr, "oracle: Hirschberg found no split\n"); abort(); }
    int64_t ul_h = split + 1;
    obtain_alignment(q, ul_h, t, left_w, left_score, out, depth + 1);
    obtain_alignment(q + ul_h, n - ul_h, t + left_w, right_w, right_score, out, depth + 1);
}

/* Full expanded CIGAR of edlib.align(q, t, task='path'); caller frees out->ops. */
static void align_path(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, opbuf *out, int64_t *dist) {
    int64_t best = nw_distance(q, n, t, m);
    if (dist) *dist = best;
    t_count_blocks = 1;
    obtain_alignment(q, n, t, m, best, out, 0);
    t_count_blocks = 0;
}

/* Definitional checker: full-matrix DP + the same traceback / Hirschberg rules on exact scores.
 * O(n*m) memory; used by tests to cross-check the banded bit-vector implementation above. */
static void naive_matrix(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int32_t *D) {
    int64_t w = m + 1;
    for (int64_t j = 0; j <= m; j++) D[j] = (int32_t)j;
    for (int64_t i = 1; i <= n; i++) {
        D[i * w] = (int32_t)i;
        for (int64_t j = 1; j <= m; j++) {
            int32_t v = D[(i - 1) * w + j - 1] + (q[i - 1] != t[j - 1]);
            int32_t u = D[(i - 1) * w + j] + 1; if (u < v) v = u;
            int32_t l = D[i * w + j - 1] + 1; if (l < v) v = l;
            D[i * w + j] = v;
        }
    }
}
static void naive_obtain(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int64_t best, opbuf *out, int depth) {
    if (n == 0) { op_push(out, 'D', m); return; }
    if (m == 0) { op_push(out, 'I', n); return; }
    tree_add(depth, q, n, t, m, best, uses_traceback(n, m));
    int64_t w = m + 1;
    if (uses_traceback(n, m)) {
        int32_t *D = (int32_t *)malloc((size_t)((n + 1) * w) * 4);
        naive_matrix(q, n, t, m, D);
        opbuf rev = {0};
        int64_t i = n, j = m;
        while (i > 0 && j > 0) {
            int32_t cur = D[i * w + j];
            if (D[(i - 1) * w + j] + 1 == cur) { op_push(&rev, 'I', 1); i--; }
            else if (D[i * w + j - 1] + 1 == cur) { op_push(&rev, 'D', 1); j--; }
            else { op_push(&rev, D[(i - 1) * w + j - 1] == cur ? '=' : 'X', 1); i--; j--; }
        }
        if (i > 0) op_push(&rev, 'I', i);
        if (j > 0) op_push(&rev, 'D', j);
        for (int64_t x = rev.n - 1; x >= 0; x--) op_push(out, rev.ops[x], 1);
        free(rev.ops); free(D);
        return;
    }
    int64_t left_w = m / 2, right_w = m - left_w;
    int32_t *DL = (int32_t *)malloc((size_t)((n + 1) * (left_w + 1)) * 4);
    naive_matrix(q, n, t, left_w, DL);
    uint8_t *rq = reversed(q, n), *rt = reversed(t, m);
    int32_t *DR = (int32_t *)malloc((size_t)((n + 1) * (right_w + 1)) * 4);
    naive_matrix(rq, n, rt, right_w, DR);
    free(rq); free(rt);
    int64_t split = -2, ls = 0, rs = 0;
    for (int64_t r = 0; r <= n - 2; r++) {
        int64_t a = DL[(r + 1) * (left_w + 1) + left_w], b = DR[(n - 1 - r) * (right_w + 1) + right_w];
        if (a + b == best) { split = r; ls = a; rs = b; break; }
    }
    if (split == -2) { int64_t b = DR[n * (right_w + 1) + right_w]; if (left_w + b == best) { split = -1; ls = left_w; rs = b; } }
    if (split == -2) { int64_t a = DL[n * (left_w + 1) + left_w]; if (a + right_w == best) { split = n - 1; ls = a; rs = right_w; } }
    free(DL); free(DR);
    if (split == -2) { fprintf(stderr, "oracle: naive Hirschberg found no split\n"); abort(); }
    naive_obtain(q, split + 1, t, left_w, ls, out, depth + 1);
    naive_obtain(q + split + 1, n - split - 1, t + left_w, right_w, rs, out, depth + 1);
}

/* Python-facing: expanded CIGAR into a malloc'd buffer the caller releases with bo_free. */
BO_EXPORT int64_t bo_align_path(const uint8_t *q, int64_t n, const uint8_t *t, int64_t m, int naive,
                                uint8_t **ops_out, int64_t *dist_out) {
    opbuf out = {0};
    tree_begin(q, t);
    if (n == 0 || m == 0) { /* edlibAlign returns no alignment when either sequence is empty */
        tree_end();
        *ops_out = NULL; if (dist_out) *dist_out = n > m ? n : m; return -1;
    }
    int64_t best;
    if (naive) {
        int32_t *D = (int32_t *)malloc((size_t)((n + 1) * (m + 1)) * 4);
        naive_matrix(q, n, t, m, D);
        best = D[n * (m + 1) + m];
        free(D);
        naive_obtain(q, n, t, m, best, &out, 0);
    } else {
        align_path(q, n, t, m, &out, &best);
    }
    tree_end();
    if (dist_out) *dist_out = best;
    *ops_out = out.ops;
    return out.n;
}
BO_EXPORT void bo_free(void *p) { free(p); }

/* misc.identity_from_edlib_cigar (misc.py:228-240): '=' columns / all columns */
static void identity_counts(const opbuf *o, int64_t *matches, int64_t *cols) {
    int64_t mt = 0;
    for (int64_t i = 0; i < o->n; i++) mt += (o->ops[i] == '=');
    *matches = mt; *cols = o->n;
}

/* ------------------------------------------------------------------------------------------------
 * Model tables (flat arrays built by the host; same layout the CUDA path uploads)
 * ---------------------------------------------------------------------------------------------- */
#define SLOT_NONE 0xFFFFFFFFu /* first slot of the "random change" (None) entry */

typedef struct {
    int k;
    int type; /* 0 = 'random', 1 = 'model' */
    int64_t n_index; /* 4^k */
    int32_t *kmer_to_row;
    int32_t n_rows;
    int32_t *row_off;  /* n_rows + 1, entry index */
    double *cum;       /* per entry: list(accumulate(probs)) */
    uint8_t *flags;    /* per entry: bit0 = ''.join(alt) == kmer, bit1 = None entry */
    uint32_t *slots;   /* per entry: k slot strings; low 8 bits len; len<=3 inline bytes 1..3, else pool offset */
    uint8_t *pool;
    int64_t pool_len;
} bo_em;

static void *dup_mem(const void *p, size_t bytes) {
    void *r = malloc(bytes ? bytes : 1);
    if (bytes) memcpy(r, p, bytes);
    return r;
}

BO_EXPORT bo_em *bo_em_create(int k, int type, const int32_t *kmer_to_row, int64_t n_index, int32_t n_rows,
                              const int32_t *row_off, const double *cum, const uint8_t *flags,
                              const uint32_t *slots, const uint8_t *pool, int64_t pool_len) {
    bo_em *m = (bo_em *)calloc(1, sizeof(bo_em));
    m->k = k; m->type = type; m->n_index = n_index; m->n_rows = n_rows; m->pool_len = pool_len;
    if (type == 1) {
        int64_t ne = row_off[n_rows];
        m->kmer_to_row = (int32_t *)dup_mem(kmer_to_row, (size_t)n_index * 4);
        m->row_off = (int32_t *)dup_mem(row_off, (size_t)(n_rows + 1) * 4);
        m->cum = (double *)dup_mem(cum, (size_t)ne * 8);
        m->flags = (uint8_t *)dup_mem(flags, (size_t)ne);
        m->slots = (uint32_t *)dup_mem(slots, (size_t)ne * k * 4);
        m->pool = (uint8_t *)dup_mem(pool, (size_t)pool_len);
    }
    return m;
}
BO_EXPORT void bo_em_destroy(bo_em *m) {
    if (!m) return;
    free(m->kmer_to_row); free(m->row_off); free(m->cum); free(m->flags); free(m->slots); free(m->pool); free(m);
}

typedef struct {
    int kmer_size;
    int32_t n_keys;
    uint8_t *key_chars; int32_t *key_off; /* key i = key_chars[key_off[i] .. key_off[i+1]) */
    int32_t *row_off; uint8_t *scores; double *cum;
    int32_t *htab; int64_t hsize;
} bo_qm;

static uint64_t str_hash(const uint8_t *s, int64_t n) {
    uint64_t h = 1469598103934665603ull;
    for (int64_t i = 0; i < n; i++) { h ^= s[i]; h *= 1099511628211ull; }
    return h;
}

BO_EXPORT bo_qm *bo_qm_create(int kmer_size, int32_t n_keys, const uint8_t *key_chars, const int32_t *key_off,
                              const int32_t *row_off, const uint8_t *scores, const double *cum) {
    bo_qm *m = (bo_qm *)calloc(1, sizeof(bo_qm));
    m->kmer_size = kmer_size; m->n_keys = n_keys;
    m->key_chars = (uint8_t *)dup_mem(key_chars, (size_t)key_off[n_keys]);
    m->key_off = (int32_t *)dup_mem(key_off, (size_t)(n_keys + 1) * 4);
    m->row_off = (int32_t *)dup_mem(row_off, (size_t)(n_keys + 1) * 4);
    m->scores = (uint8_t *)dup_mem(scores, (size_t)row_off[n_keys]);
    m->cum = (double *)dup_mem(cum, (size_t)row_off[n_keys] * 8);
    m->hsize = 64; while (m->hsize < 4 * (int64_t)n_keys) m->hsize *= 2;
    m->htab = (int32_t *)malloc((size_t)m->hsize * 4);
    for (int64_t i = 0; i < m->hsize; i++) m->htab[i] = -1;
    for (int32_t i = 0; i < n_keys; i++) {
        uint64_t h = str_hash(m->key_chars + key_off[i], key_off[i + 1] - key_off[i]) & (uint64_t)(m->hsize - 1);
        while (m->htab[h] >= 0) h = (h + 1) & (uint64_t)(m->hsize - 1);
        m->htab[h] = i; /* duplicate keys: the dict keeps the last assignment; host de-duplicates before upload */
    }
    return m;
}
BO_EXPORT void bo_qm_destroy(bo_qm *m) {
    if (!m) return;
    free(m->key_chars); free(m->key_off); free(m->row_off); free(m->scores); free(m->cum); free(m->htab); free(m);
}

static int32_t qm_find(const bo_qm *m, const uint8_t *s, int64_t n) {
    uint64_t h = str_hash(s, n) & (uint64_t)(m->hsize - 1);
    while (m->htab[h] >= 0) {
        int32_t i = m->htab[h];
        int64_t len = m->key_off[i + 1] - m->key_off[i];
        if (len == n && memcmp(m->key_chars + m->key_off[i], s, (size_t)n) == 0) return i;
        h = (h + 1) & (uint64_t)(m->hsize - 1);
    }
    return -1;
}

/* ------------------------------------------------------------------------------------------------
 * The hot path
 * ---------------------------------------------------------------------------------------------- */
typedef struct { uint8_t len; uint8_t c[3]; const uint8_t *ext; } slotstr; /* decoded slot string */

static slotstr slot_decode(const bo_em *em, uint32_t s) {
    slotstr r; r.len = (uint8_t)(s & 0xff); r.ext = NULL;
    r.c[0] = (uint8_t)(s >> 8); r.c[1] = (uint8_t)(s >> 16); r.c[2] = (uint8_t)(s >> 24);
    if (r.len > 3) r.ext = em->pool + (s >> 8);
    return r;
}
static inline uint8_t slot_char(const slotstr *s, int i) { return s->ext ? s->ext[i] : s->c[i]; }
static uint32_t slot_inline(int len, uint8_t c0, uint8_t c1) {
    return (uint32_t)len | ((uint32_t)c0 << 8) | ((uint32_t)c1 << 16);
}

/* error_model.add_one_random_change (error_model.py:163-176): returns k encoded slots */
static void add_one_random_change(bo_rng *rng, const uint8_t *kmer, int k, uint32_t *out) {
    for (int j = 0; j < k; j++) out[j] = slot_inline(1, kmer[j], 0);
    uint32_t type = rng_randbelow(rng, 3); /* random.choice(['s','i','d']) */
    uint32_t pos = rng_randbelow(rng, (uint32_t)k); /* random.randint(0, len(kmer)-1) */
    if (type == 0) {
        out[pos] = slot_inline(1, rng_random_different_base(rng, kmer[pos]), 0);
    } else if (type == 1) {
        if (rng_random(rng) < 0.5) { /* random_chance(0.5): base + new */
            uint8_t nb = rng_random_base(rng);
            out[pos] = slot_inline(2, kmer[pos], nb);
        } else {
            uint8_t nb = rng_random_base(rng);
            out[pos] = slot_inline(2, nb, kmer[pos]);
        }
    } else {
        out[pos] = slot_inline(0, 0, 0);
    }
}

/* ErrorModel.add_errors_to_kmer (error_model.py:135-160). Returns 1 when ''.join(new_kmer) == kmer. */
static int add_errors_to_kmer(const bo_em *em, bo_rng *rng, const uint8_t *kmer, uint32_t *out) {
    int k = em->k;
    if (em->type == 0) { add_one_random_change(rng, kmer, k, out); return 0; }
    int64_t idx = 0;
    for (int j = 0; j < k; j++) {
        int c;
        switch (kmer[j]) { case 'A': c = 0; break; case 'C': c = 1; break; case 'G': c = 2; break; case 'T': c = 3; break; default: c = -1; }
        if (c < 0) { idx = -1; break; }
        idx = idx * 4 + c;
    }
    int32_t row = idx < 0 ? -1 : em->kmer_to_row[idx];
    if (row < 0) { add_one_random_change(rng, kmer, k, out); return 0; }
    int32_t e0 = em->row_off[row], ne = em->row_off[row + 1] - e0;
    int pick = rng_choices(rng, em->cum + e0, ne);
    int32_t e = e0 + pick;
    if (em->flags[e] & 2) { add_one_random_change(rng, kmer, k, out); return 0; }
    memcpy(out, em->slots + (int64_t)e * k, (size_t)k * 4);
    return em->flags[e] & 1;
}

typedef struct { uint8_t *p; int64_t n, cap; } bytebuf;
static void bb_reserve(bytebuf *b, int64_t extra) {
    if (b->n + extra > b->cap) {
        while (b->n + extra > b->cap) b->cap = b->cap ? b->cap * 2 : 4096;
        b->p = (uint8_t *)realloc(b->p, (size_t)b->cap);
    }
}

/* ''.join(new_fragment_bases[lo:hi]) */
static void join_slots(const bo_em *em, const uint8_t *frag, const uint32_t *state, int64_t lo, int64_t hi, bytebuf *out) {
    out->n = 0;
    for (int64_t x = lo; x < hi; x++) {
        if (state[x] == SLOT_NONE) { bb_reserve(out, 1); out->p[out->n++] = frag[x]; }
        else {
            slotstr s = slot_decode(em, state[x]);
            bb_reserve(out, s.len);
            for (int c = 0; c < s.len; c++) out->p[out->n++] = slot_char(&s, c);
        }
    }
}

/* QScoreModel.get_qscore (qscore_model.py:273-287) */
static uint8_t get_qscore(const bo_qm *qm, bo_rng *rng, const uint8_t *cigar, int64_t len) {
    for (;;) {
        int32_t key = qm_find(qm, cigar, len);
        if (key >= 0) {
            int32_t e0 = qm->row_off[key], ne = qm->row_off[key + 1] - e0;
            int pick = rng_choices(rng, qm->cum + e0, ne);
            return (uint8_t)(qm->scores[e0 + pick] + 33);
        }
        /* cigar = cigar[1:-1].strip('D') */
        cigar++; len -= 2;
        while (len > 0 && cigar[0] == 'D') { cigar++; len--; }
        while (len > 0 && cigar[len - 1] == 'D') len--;
        if (len <= 0) { fprintf(stderr, "oracle: qscore cigar trimmed to nothing\n"); abort(); }
    }
}

/* qscore_model.get_qscores (qscore_model.py:32-75); identity_by_qscores is a pure function of the returned
 * qual string and is computed by the caller. */
static void get_qscores(const bo_qm *qm, bo_rng *rng, const uint8_t *seq, int64_t seq_len, const uint8_t *frag,
                        int64_t frag_len, uint8_t *qual, int64_t *matches, int64_t *cols) {
    opbuf cg = {0};
    tree_begin(seq, frag);  /* the final alignment (bo_tree_arm) */
    align_path(seq, seq_len, frag, frag_len, &cg, NULL); /* query = mutated read, target = original */
    tree_end();
    identity_counts(&cg, matches, cols);
    int64_t *pos2col = (int64_t *)malloc((size_t)seq_len * 8);
    int64_t i = 0;
    for (int64_t j = 0; j < cg.n; j++)
        if (cg.ops[j] != 'D') pos2col[i++] = j;
    int64_t margins = (qm->kmer_size - 1) / 2;
    for (i = 0; i < seq_len; i++) {
        int64_t start = i - margins, end = i + margins;
        while (start < 0 || end >= seq_len) { start++; end--; }
        int64_t cs = pos2col[start], ce = pos2col[end];
        rng_stream(rng, BO_PURPOSE_QSCORE, (uint32_t)i);
        qual[i] = get_qscore(qm, rng, cg.ops + cs, ce - cs + 1);
    }
    free(pos2col); free(cg.ops);
}

/* Debug capture (tests only): when armed, bo_sequence_fragment leaves copies of the padded fragment and of the
 * untrimmed read here so that a failing device alignment can be replayed in isolation. */
static uint8_t *g_dbg_frag = NULL, *g_dbg_seq = NULL;
static int64_t g_dbg_frag_len = 0, g_dbg_seq_len = 0;
static int g_dbg_armed = 0;
BO_EXPORT void bo_debug_arm(int on) { g_dbg_armed = on; }
BO_EXPORT int64_t bo_debug_get(int which, uint8_t *out, int64_t cap) {
    const uint8_t *p = which == 0 ? g_dbg_frag : g_dbg_seq;
    int64_t n = which == 0 ? g_dbg_frag_len : g_dbg_seq_len;
    if (out && n <= cap && n > 0) memcpy(out, p, (size_t)n);
    return n;
}

#define ALIGNMENT_INTERVAL 25  /* settings.py:24 */
#define ALIGNMENT_SIZE 1000    /* settings.py:25 */

/* simulate.sequence_fragment (simulate.py:256-358).
 * pow_mode 0: estimated_identity ** 1.5 via libm pow (reference fidelity, used with the MT stream);
 * pow_mode 1: x * sqrt(x) (two correctly rounded IEEE operations; what the CUDA path computes).
 * Outputs are malloc'd; *out_len may be 0 (the caller skips such reads, simulate.py:70). */
BO_EXPORT int bo_sequence_fragment(const bo_em *em, const bo_qm *qm, bo_rng *rng, const uint8_t *fragment_in,
                                   int64_t in_len, double target_identity, int pow_mode, uint8_t **seq_out,
                                   uint8_t **qual_out, int64_t *out_len, int64_t *matches_out, int64_t *cols_out,
                                   int64_t *stats /* optional [4]: loop_count, change_count, n_alignments, untrimmed_len */) {
    int k = em->k;
    int64_t frag_len = in_len + 2 * k;
    uint8_t *fragment = (uint8_t *)malloc((size_t)frag_len);
    rng_stream(rng, BO_PURPOSE_PAD, 0);
    for (int j = 0; j < k; j++) fragment[j] = rng_random_base(rng);
    memcpy(fragment + k, fragment_in, (size_t)in_len);
    for (int j = 0; j < k; j++) fragment[k + in_len + j] = rng_random_base(rng);

    uint32_t *state = (uint32_t *)malloc((size_t)frag_len * 4);
    for (int64_t x = 0; x < frag_len; x++) state[x] = SLOT_NONE;

    double errors = 0.0;
    int64_t change_count = 0, loop_count = 0, n_align = 0;
    int64_t max_kmer_index = frag_len - 1 - k;
    double estimated_errors_needed = frag_len * (1.0 - target_identity);
    uint32_t new_kmer[64];
    bytebuf joined = {0};

    for (;;) {
        if (estimated_errors_needed < 0.5) break;
        loop_count++;
        if (loop_count > 100 * frag_len) break;
        if ((double)change_count > 0.9 * (double)frag_len) break;
        double estimated_identity = 1.0 - (errors / (double)frag_len);
        if (estimated_identity <= target_identity) break;

        rng_stream(rng, BO_PURPOSE_LOOP, (uint32_t)(loop_count - 1));
        int64_t i = (int64_t)rng_randbelow(rng, (uint32_t)(max_kmer_index + 1));
        const uint8_t *kmer = fragment + i;
        if (add_errors_to_kmer(em, rng, kmer, new_kmer)) continue;

        for (int j = 0; j < k; j++) {
            uint8_t fragment_base = fragment[i + j];
            slotstr nb = slot_decode(em, new_kmer[j]);
            int differs = !(nb.len == 1 && slot_char(&nb, 0) == fragment_base);
            if (differs && state[i + j] == SLOT_NONE) {
                state[i + j] = new_kmer[j];
                change_count++;
                int new_errors = nb.len < 2 ? 1 : nb.len - 1;
                double scale = pow_mode == 0 ? pow(estimated_identity, 1.5) : estimated_identity * sqrt(estimated_identity);
                errors += (double)new_errors * scale;
                if (change_count % ALIGNMENT_INTERVAL == 0) {
                    opbuf cg = {0};
                    int64_t mt, cl;
                    if (frag_len <= ALIGNMENT_SIZE) {
                        join_slots(em, fragment, state, 0, frag_len, &joined);
                        align_path(fragment, frag_len, joined.p, joined.n, &cg, NULL);
                        identity_counts(&cg, &mt, &cl);
                        double actual_identity = cl ? (double)mt / (double)cl : 0.0;
                        errors = (1.0 - actual_identity) * (double)frag_len;
                    } else {
                        rng_stream(rng, BO_PURPOSE_WINDOW, (uint32_t)n_align);
                        int64_t pos = (int64_t)rng_randbelow(rng, (uint32_t)(frag_len - ALIGNMENT_SIZE + 1));
                        int64_t pos2 = pos + ALIGNMENT_SIZE;
                        join_slots(em, fragment, state, pos, pos2, &joined);
                        align_path(fragment + pos, ALIGNMENT_SIZE, joined.p, joined.n, &cg, NULL);
                        identity_counts(&cg, &mt, &cl);
                        double actual_identity = cl ? (double)mt / (double)cl : 0.0;
                        double estimated_errors = (1.0 - actual_identity) * (double)frag_len;
                        double weight = (double)ALIGNMENT_SIZE / (double)frag_len;
                        errors = (estimated_errors * weight) + (errors * (1 - weight));
                    }
                    free(cg.ops);
                    n_align++;
                }
            }
        }
    }

    int64_t start_trim = 0, end_trim = 0;
    for (int j = 0; j < k; j++) {
        start_trim += state[j] == SLOT_NONE ? 1 : (int64_t)(state[j] & 0xff);
        int64_t x = frag_len - k + j;
        end_trim += state[x] == SLOT_NONE ? 1 : (int64_t)(state[x] & 0xff);
    }
    join_slots(em, fragment, state, 0, frag_len, &joined);
    int64_t seq_len = joined.n;
    if (g_dbg_armed) {
        free(g_dbg_frag); free(g_dbg_seq);
        g_dbg_frag = (uint8_t *)dup_mem(fragment, (size_t)frag_len); g_dbg_frag_len = frag_len;
        g_dbg_seq = (uint8_t *)dup_mem(joined.p, (size_t)seq_len); g_dbg_seq_len = seq_len;
    }
    uint8_t *qual = (uint8_t *)malloc((size_t)(seq_len ? seq_len : 1));
    get_qscores(qm, rng, joined.p, seq_len, fragment, frag_len, qual, matches_out, cols_out);

    int64_t n_out = seq_len - end_trim - start_trim; /* seq[start_trim:-end_trim] */
    if (n_out < 0) n_out = 0;
    *seq_out = (uint8_t *)malloc((size_t)(n_out ? n_out : 1));
    *qual_out = (uint8_t *)malloc((size_t)(n_out ? n_out : 1));
    memcpy(*seq_out, joined.p + start_trim, (size_t)n_out);
    memcpy(*qual_out, qual + start_trim, (size_t)n_out);
    *out_len = n_out;
    if (stats) { stats[0] = loop_count; stats[1] = change_count; stats[2] = n_align; stats[3] = seq_len; }
    free(qual); free(joined.p); free(state); free(fragment);
    return 0;
}

/* get_qscores on its own (qscore_model.py:32): used by tests that mirror test/test_qscore_model.py */
BO_EXPORT int bo_get_qscores(const bo_qm *qm, bo_rng *rng, const uint8_t *seq, int64_t seq_len, const uint8_t *frag,
                             int64_t frag_len, uint8_t *qual, int64_t *matches, int64_t *cols) {
    get_qscores(qm, rng, seq, seq_len, frag, frag_len, qual, matches, cols);
    return 0;
}

BO_EXPORT int bo_add_errors_to_kmer(const bo_em *em, bo_rng *rng, const uint8_t *kmer, uint8_t *out, int32_t *out_off) {
    /* returns the k slot strings concatenated into out with out_off[k+1] offsets (for the error-model tests) */
    uint32_t nk[64];
    int same = add_errors_to_kmer(em, rng, kmer, nk);
    int32_t n = 0;
    for (int j = 0; j < em->k; j++) {
        out_off[j] = n;
        slotstr s = slot_decode(em, nk[j]);
        for (int c = 0; c < s.len; c++) out[n++] = slot_char(&s, c);
    }
    out_off[em->k] = n;
    return same;
}

/* Batch over independent reads in Philox mode, pthread workers pulling read indices from a shared counter —
 * the timed CPU baseline ("port"). frags: concatenated unpadded fragments with frag_off[n+1]; every read's
 * seq/qual are malloc'd (release each with bo_free). Returns the total emitted bases. */
typedef struct {
    const bo_em *em; const bo_qm *qm; uint64_t seed; const uint64_t *read_index; const uint8_t *frags;
    const int64_t *frag_off; int32_t n_reads; const double *target_identity; uint8_t **seq_ptrs;
    uint8_t **qual_ptrs; int64_t *out_len, *matches, *cols; int32_t next;
    int64_t *stats; int64_t **tree_ptrs; int64_t *tree_len;  /* optional (bo_sequence_batch_stats) */
} batch_job;

static void *batch_worker(void *arg) {
    batch_job *jb = (batch_job *)arg;
    for (;;) {
        int32_t r = __atomic_fetch_add(&jb->next, 1, __ATOMIC_RELAXED);
        if (r >= jb->n_reads) break;
        bo_rng *rng = bo_rng_create(BO_RNG_PHILOX, jb->seed, jb->read_index[r]);
        if (jb->tree_ptrs) bo_tree_arm(1);
        bo_sequence_fragment(jb->em, jb->qm, rng, jb->frags + jb->frag_off[r], jb->frag_off[r + 1] - jb->frag_off[r],
                             jb->target_identity[r], 1, &jb->seq_ptrs[r], &jb->qual_ptrs[r], &jb->out_len[r],
                             &jb->matches[r], &jb->cols[r], jb->stats ? jb->stats + 4 * (int64_t)r : NULL);
        if (jb->tree_ptrs) jb->tree_len[r] = bo_tree_take(&jb->tree_ptrs[r]);
        bo_rng_destroy(rng);
    }
    return NULL;
}

static int64_t sequence_batch(batch_job *jb, int n_threads) {
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 256) n_threads = 256;
    pthread_t th[256];
    for (int i = 1; i < n_threads; i++) pthread_create(&th[i], NULL, batch_worker, jb);
    batch_worker(jb);
    for (int i = 1; i < n_threads; i++) pthread_join(th[i], NULL);
    int64_t total = 0;
    for (int32_t r = 0; r < jb->n_reads; r++) total += jb->out_len[r];
    return total;
}

/* bo_sequence_batch that also returns every read's stats[4] (as bo_sequence_fragment's) and the tree of its final
 * alignment (tree_ptrs[r]: tree_len[r] entries of BO_TREE_FIELDS values, release each with bo_free). */
BO_EXPORT int64_t bo_sequence_batch_stats(const bo_em *em, const bo_qm *qm, uint64_t seed, const uint64_t *read_index,
                                          const uint8_t *frags, const int64_t *frag_off, int32_t n_reads,
                                          const double *target_identity, uint8_t **seq_ptrs, uint8_t **qual_ptrs,
                                          int64_t *out_len, int64_t *matches, int64_t *cols, int n_threads,
                                          int64_t *stats, int64_t **tree_ptrs, int64_t *tree_len) {
    batch_job jb = {em, qm, seed, read_index, frags, frag_off, n_reads, target_identity,
                    seq_ptrs, qual_ptrs, out_len, matches, cols, 0, stats, tree_ptrs, tree_len};
    return sequence_batch(&jb, n_threads);
}

BO_EXPORT int64_t bo_sequence_batch(const bo_em *em, const bo_qm *qm, uint64_t seed, const uint64_t *read_index,
                                    const uint8_t *frags, const int64_t *frag_off, int32_t n_reads,
                                    const double *target_identity, uint8_t **seq_ptrs, uint8_t **qual_ptrs,
                                    int64_t *out_len, int64_t *matches, int64_t *cols, int n_threads) {
    batch_job jb = {em, qm, seed, read_index, frags, frag_off, n_reads, target_identity,
                    seq_ptrs, qual_ptrs, out_len, matches, cols, 0, NULL, NULL, NULL};
    return sequence_batch(&jb, n_threads);
}
