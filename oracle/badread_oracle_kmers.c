/*
 * badread_oracle_kmers.c - the CPU oracle for error models whose k-mer index has no dense form: k up to 16, where
 * kmer_to_row[4^k] would take up to 16 GiB.  TEST INFRASTRUCTURE ONLY (front end: oracle/oracle_kmers.py).
 *
 * The unchanged oracle (badread_oracle.c) is compiled into this library as it is; this file adds
 *   bo_em_kmers_create        the model tables with the rows' k-mer codes instead of kmer_to_row: the codes are sorted
 *                             once and a k-mer's row is found by binary search
 *   bo_sequence_fragment_kmers simulate.sequence_fragment (simulate.py:256-358) with that lookup.  It is
 *                             bo_sequence_fragment's loop step for step; only ErrorModel.add_errors_to_kmer
 *                             (error_model.py:135-160) finds the row through the sorted codes
 * Everything else - RNG streams, the aligner, join, get_qscores, the qscore model - is badread_oracle.c's own code.
 */
#include "badread_oracle.c"

typedef struct {
    bo_em em;            /* type 1, kmer_to_row NULL */
    int64_t *codes;      /* the rows' k-mer codes in increasing order ... */
    int32_t *rows;       /* ... and the row of each */
} bo_em_kmers;

BO_EXPORT void bo_em_kmers_destroy(bo_em_kmers *m) {
    if (!m) return;
    free(m->codes); free(m->rows);
    free(m->em.row_off); free(m->em.cum); free(m->em.flags); free(m->em.slots); free(m->em.pool);
    free(m);
}

static const int64_t *g_sort_codes; /* (qsort has no context argument; tables are built from one thread) */
static int cmp_row_by_code(const void *a, const void *b) {
    int64_t x = g_sort_codes[*(const int32_t *)a], y = g_sort_codes[*(const int32_t *)b];
    return x < y ? -1 : x > y ? 1 : 0;
}

/* Row r has the k-mer whose code (base j in bits 2*(k-1-j), A C G T = 0 1 2 3) is kmer_codes[r].  Returns NULL if two
 * rows share a code or k is outside 3..16. */
BO_EXPORT bo_em_kmers *bo_em_kmers_create(int k, int32_t n_rows, const int64_t *kmer_codes, const int32_t *row_off,
                                          const double *cum, const uint8_t *flags, const uint32_t *slots,
                                          const uint8_t *pool, int64_t pool_len) {
    if (k < 3 || k > 16 || n_rows <= 0) return NULL;
    bo_em_kmers *m = (bo_em_kmers *)calloc(1, sizeof(bo_em_kmers));
    int64_t ne = row_off[n_rows];
    m->em.k = k; m->em.type = 1; m->em.n_rows = n_rows; m->em.pool_len = pool_len;
    m->em.row_off = (int32_t *)dup_mem(row_off, (size_t)(n_rows + 1) * 4);
    m->em.cum = (double *)dup_mem(cum, (size_t)ne * 8);
    m->em.flags = (uint8_t *)dup_mem(flags, (size_t)ne);
    m->em.slots = (uint32_t *)dup_mem(slots, (size_t)ne * k * 4);
    m->em.pool = (uint8_t *)dup_mem(pool, (size_t)pool_len);
    m->rows = (int32_t *)malloc((size_t)n_rows * 4);
    m->codes = (int64_t *)malloc((size_t)n_rows * 8);
    for (int32_t r = 0; r < n_rows; r++) m->rows[r] = r;
    g_sort_codes = kmer_codes;
    qsort(m->rows, (size_t)n_rows, 4, cmp_row_by_code);
    for (int32_t i = 0; i < n_rows; i++) {
        m->codes[i] = kmer_codes[m->rows[i]];
        if (i > 0 && m->codes[i] == m->codes[i - 1]) { bo_em_kmers_destroy(m); return NULL; }
    }
    return m;
}

static int32_t kmers_row(const bo_em_kmers *m, int64_t code) {
    int64_t lo = 0, hi = m->em.n_rows;
    while (lo < hi) {
        int64_t mid = (lo + hi) / 2;
        if (m->codes[mid] < code) lo = mid + 1; else hi = mid;
    }
    return lo < m->em.n_rows && m->codes[lo] == code ? m->rows[lo] : -1;
}

/* add_errors_to_kmer with the row found through the sorted codes.  Returns 1 when ''.join(new_kmer) == kmer. */
static int add_errors_to_kmer_kmers(const bo_em_kmers *m, bo_rng *rng, const uint8_t *kmer, uint32_t *out) {
    const bo_em *em = &m->em;
    int k = em->k;
    int64_t idx = 0;
    for (int j = 0; j < k; j++) {
        int c;
        switch (kmer[j]) { case 'A': c = 0; break; case 'C': c = 1; break; case 'G': c = 2; break; case 'T': c = 3; break; default: c = -1; }
        if (c < 0) { idx = -1; break; }
        idx = idx * 4 + c;
    }
    int32_t row = idx < 0 ? -1 : kmers_row(m, idx);
    if (row < 0) { add_one_random_change(rng, kmer, k, out); return 0; }
    int32_t e0 = em->row_off[row], ne = em->row_off[row + 1] - e0;
    int pick = rng_choices(rng, em->cum + e0, ne);
    int32_t e = e0 + pick;
    if (em->flags[e] & 2) { add_one_random_change(rng, kmer, k, out); return 0; }
    memcpy(out, em->slots + (int64_t)e * k, (size_t)k * 4);
    return em->flags[e] & 1;
}

/* bo_sequence_fragment for a bo_em_kmers model: same arguments, same outputs. */
BO_EXPORT int bo_sequence_fragment_kmers(const bo_em_kmers *m, const bo_qm *qm, bo_rng *rng, const uint8_t *fragment_in,
                                         int64_t in_len, double target_identity, int pow_mode, uint8_t **seq_out,
                                         uint8_t **qual_out, int64_t *out_len, int64_t *matches_out, int64_t *cols_out,
                                         int64_t *stats) {
    const bo_em *em = &m->em;
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
        if (add_errors_to_kmer_kmers(m, rng, kmer, new_kmer)) continue;

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
