/*
 * badread_b200.h — C ABI of libbadread_b200.so: the drop-in boundary for Badread's per-read
 * error-injection hot path on NVIDIA H100 (sm_90a).
 *
 * The reference (rrwick/Badread v0.4.2) is pure Python; its only native call on this path is
 * `edlib.align` (third-party).  This ABI is what a ctypes binding inside the reference would bind to replace
 *     simulate.sequence_fragment            badread/simulate.py:256-358
 *     ErrorModel.add_errors_to_kmer         badread/error_model.py:135-176   (table sampling, on device)
 *     qscore_model.get_qscores              badread/qscore_model.py:32-75
 *     QScoreModel.get_qscore                badread/qscore_model.py:273-287
 *     edlib.align(..., task='path')         call sites simulate.py:330,340; qscore_model.py:37; error_model.py:202
 * Plain pointers and sizes only; the caller owns every host buffer, the library owns device memory behind an
 * opaque bb_ctx.  All functions return 0 on success or a negative bb_status; bb_last_error() gives the text.
 * The library never calls exit() and never falls back to a CPU implementation of the hot path.
 */
#ifndef BADREAD_B200_H
#define BADREAD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BB_API __attribute__((visibility("default")))
#else
#define BB_API
#endif

typedef struct bb_ctx bb_ctx;

enum bb_status {
    BB_OK = 0,
    BB_ERR_CUDA = -1,      /* CUDA runtime error (no device, launch failure, out of memory) */
    BB_ERR_ARG = -2,       /* invalid argument */
    BB_ERR_STATE = -3,     /* models / reference not uploaded yet */
    BB_ERR_CAPACITY = -4,  /* caller-provided output buffer too small (required size is reported) */
    BB_ERR_INTERNAL = -5   /* device-side invariant violated (reported with a code in bb_last_error) */
};

/* Segment kinds of a fragment descriptor. A fragment (what simulate.build_fragment returns, simulate.py:91-115)
 * is the concatenation of its segments: slices of the HBM-resident reference (either strand) and literal bytes
 * (adapters, glitch inserts, junk / random reads). */
enum bb_seg_kind {
    BB_SEG_REF_FWD = 0, /* reference bytes [src, src+len) as stored */
    BB_SEG_REF_REV = 1, /* reverse complement (misc.reverse_complement, misc.py:56-71) of reference [src, src+len) */
    BB_SEG_LITERAL = 2  /* bytes [src, src+len) of the literal pool passed with the batch */
};

typedef struct bb_segment {
    int64_t src;   /* offset into the uploaded reference or into the batch's literal pool */
    int32_t len;
    int32_t kind;  /* bb_seg_kind */
} bb_segment;

/* Per-read outputs besides the bases (header fields of simulate.py:73-75 come from these). */
typedef struct bb_read_result {
    int64_t out_off;      /* offset of this read's seq/qual in the output buffers (reads are packed without gaps,
                           * but not necessarily in batch order) */
    int32_t out_len;      /* len(seq) after trimming; 0 => the reference skips the read (simulate.py:70) */
    int32_t frag_len;     /* len(fragment) before padding ("error-free_length") */
    int32_t matches;      /* '=' columns of the final alignment */
    int32_t columns;      /* all columns; read identity = matches / columns (misc.py:228-240) */
    int32_t loop_count;   /* iterations of the k-mer loop (simulate.py:278) */
    int32_t change_count; /* applied slot changes (simulate.py:311) */
    int32_t n_alignments; /* identity re-measurements (simulate.py:325-346) */
    int32_t flags;        /* non-zero: device-side problem for this read (see bb_last_error) */
    int32_t loop_kcycles; /* diagnostics: SM kilo-cycles this read spent in the error loop ... */
    int32_t align_kcycles;/* ... and in the final alignment */
} bb_read_result;

/* ---- lifecycle -------------------------------------------------------------------------------------- */
/* Creates a context on CUDA device `device`. seed is `--seed` (simulate.py:34-36). Fails with BB_ERR_CUDA when
 * there is no usable GPU: there is no CPU path.
 * A context holds BADREAD_B200_SUBBATCHES (environment, default 2, 1..8) workers on the device: large batches are
 * dealt out over them and their kernel chains overlap on separate streams.  Results do not depend on it. */
BB_API int bb_create(bb_ctx **ctx, int device, uint64_t seed);
BB_API int bb_destroy(bb_ctx *ctx);
BB_API const char *bb_last_error(const bb_ctx *ctx); /* ctx may be NULL for creation errors */
BB_API const char *bb_version(void);

/* ---- one-time uploads ------------------------------------------------------------------------------- */
/* Reference contigs concatenated (upper-case ASCII, misc.load_fasta misc.py:122-153). */
BB_API int bb_upload_reference(bb_ctx *ctx, const uint8_t *bases, int64_t n_bases);

/* The reference from a FASTA file parsed on the device, in place of bb_upload_reference: the bases never exist on the host.
 * bb_fasta_parse takes the file's bytes (page-locked memory copies fastest): the FASTA text itself, or with is_bgzf (named
 * for the BGZF files it first took) a gzip stream of it, BGZF or not, inflated on the device as bb_gzip_decompress
 * inflates it.  It drops the context's reference, then parses with the semantics of misc.load_fasta_arrays: a line starting
 * with '>' is a header line; every other byte except '\n', '\r', ' ' and '\t' is kept, 'a'-'z' upper-cased.  It reports
 * the number of header lines, the bytes of their texts and the bytes kept; BB_ERR_ARG names a corrupt gzip member (index
 * and offset) like bb_gzip_decompress, and bb_last_gzip_stats then tells how the stream was inflated.  Device memory peaks
 * at the input plus the text plus the kept bytes, or at the inflater's peak (bb_gzip_decompress).
 * bb_fasta_headers then copies the header table: text[text_off[k] .. text_off[k + 1]) the text of header line k after
 * its '>' (without the newline, otherwise as in the file), kept_off[k] the bytes kept before it and kept_off[n] all of
 * them, so contig k's bases are kept bytes [kept_off[k], kept_off[k + 1]).  BB_ERR_CAPACITY if n_cap or text_cap is
 * smaller than what bb_fasta_parse reported.
 * bb_fasta_reference makes the reference the concatenation of kept bytes [lo[c], hi[c]) for the n_contigs contigs (in
 * place when they are all the kept bytes in order), as bb_upload_reference would, and releases the parse. */
BB_API int bb_fasta_parse(bb_ctx *ctx, const uint8_t *data, int64_t n, int is_bgzf, int32_t *n_headers, int64_t *text_bytes,
                          int64_t *n_kept);
BB_API int bb_fasta_headers(bb_ctx *ctx, char *text, int64_t text_cap, int64_t *text_off, int64_t *kept_off, int32_t n_cap);
/* How the last bb_fasta_parse inflated its gzip stream (all zero for plain text). */
typedef struct bb_gzip_stats bb_gzip_stats;
BB_API int bb_last_gzip_stats(const bb_ctx *ctx, bb_gzip_stats *stats);
BB_API int bb_fasta_reference(bb_ctx *ctx, int32_t n_contigs, const int64_t *lo, const int64_t *hi);
/* Copies bytes [offset, offset + n) of the context's reference to out (for checking what a load left on the device). */
BB_API int bb_download_reference(bb_ctx *ctx, int64_t offset, int64_t n, uint8_t *out);

/* Error model tables (flat form of ErrorModel.alternatives / .probabilities, error_model.py:86-133):
 *  type 0 = 'random' (k = 1, no tables), 1 = 'model'.
 *  kmer_to_row[4^k]: row of each ACGT k-mer or -1; row_off[n_rows+1] entry ranges; per entry: cum (the
 *  list(accumulate(probs)) that random.choices builds), flags (bit0: ''.join(alt)==kmer, bit1: the
 *  "random change" remainder entry appended at error_model.py:151-154), k slot strings encoded as
 *  len | chars<<8 (len<=3) or len | pool_offset<<8. */
BB_API int bb_upload_error_model(bb_ctx *ctx, int k, int type, const int32_t *kmer_to_row, int64_t n_index, int32_t n_rows,
                          const int32_t *row_off, const double *cum, const uint8_t *flags, const uint32_t *slots,
                          const uint8_t *pool, int64_t pool_len);

/* The same tables with the k-mer index as a hash table instead of kmer_to_row[4^k], for any k in 3..16 (k > 12 has no
 *  dense form): row r has the k-mer whose 2-bit code (base j in bits 2*(k-1-j), A C G T = 0 1 2 3) is kmer_codes[r].  A
 *  k-mer without a row, or one holding a non-ACGT base, gets one random change, as with the dense index.  A code outside
 *  0 .. 4^k-1 or one that two rows share is rejected (BB_ERR_ARG, message in bb_last_error). */
BB_API int bb_upload_error_model_kmers(bb_ctx *ctx, int k, int32_t n_rows, const int64_t *kmer_codes, const int32_t *row_off,
                                const double *cum, const uint8_t *flags, const uint32_t *slots, const uint8_t *pool,
                                int64_t pool_len);

/* Qscore model tables (flat form of QScoreModel.scores / .probabilities, qscore_model.py:178-271).
 *  Key i is the CIGAR string key_chars[key_off[i] .. key_off[i+1]) over {=,X,I,D}, of any length;
 *  row_off[n_keys+1]; scores / cum per entry. kmer_size as QScoreModel.kmer_size.  A repeated key keeps its last row
 *  (the dict assignment of QScoreModel.load_from_file).  An empty key or a symbol outside =XID is rejected
 *  (BB_ERR_ARG, message in bb_last_error). */
BB_API int bb_upload_qscore_model_cigars(bb_ctx *ctx, int kmer_size, int32_t n_keys, const uint8_t *key_chars,
                                         const int32_t *key_off, const int32_t *row_off, const uint8_t *scores,
                                         const double *cum);

/* The same tables with keys[n_keys] packed 2 bits per symbol ('='=0, 'X'=1, 'I'=2, 'D'=3) under a leading 1 bit, which
 *  limits a key to 31 symbols; bb_upload_qscore_model_cigars takes keys of any length. */
BB_API int bb_upload_qscore_model(bb_ctx *ctx, int kmer_size, int32_t n_keys, const uint64_t *keys, const int32_t *row_off,
                           const uint8_t *scores, const double *cum);

/* ---- the hot path ----------------------------------------------------------------------------------- */
/* sequence_fragment for a batch of reads (simulate.py:256-358 for each).
 *  read_index[n]: global read ordinal, keys the per-read Philox streams (output is independent of batching and
 *  of the number of GPUs). seg_off[n+1] indexes segs. target_identity[n] as Identities.get_identity().
 *  Outputs: results[n]; seq_out / qual_out receive the trimmed reads back to back (capacity out_cap bytes each);
 *  *out_total = bytes written. If out_cap is too small: returns BB_ERR_CAPACITY with *out_total = required size
 *  (device results are kept; call bb_fetch_last_batch with larger buffers). */
BB_API int bb_sequence_batch(bb_ctx *ctx, int32_t n_reads, const uint64_t *read_index, const int32_t *seg_off,
                      const bb_segment *segs, const uint8_t *literal_pool, int64_t literal_len,
                      const double *target_identity, bb_read_result *results, uint8_t *seq_out, uint8_t *qual_out,
                      int64_t out_cap, int64_t *out_total);
BB_API int bb_fetch_last_batch(bb_ctx *ctx, bb_read_result *results, uint8_t *seq_out, uint8_t *qual_out, int64_t out_cap,
                        int64_t *out_total);

/* Page-locked host memory for the seq / qual output buffers (device-to-host copies into pageable memory go through
 * a staging buffer at a fraction of the link rate).  Optional: any host pointer is accepted by the fetch calls. */
BB_API int bb_host_alloc(void **ptr, int64_t bytes);
BB_API int bb_host_free(void *ptr);

/* Split form used by bench.py to time the device work with inputs already resident in HBM:
 * bb_batch_upload (H2D of descriptors) -> bb_batch_run (kernels only, asynchronous on the ctx stream;
 * may be called repeatedly on the same uploaded batch) -> bb_fetch_last_batch (D2H). */
BB_API int bb_batch_upload(bb_ctx *ctx, int32_t n_reads, const uint64_t *read_index, const int32_t *seg_off,
                    const bb_segment *segs, const uint8_t *literal_pool, int64_t literal_len,
                    const double *target_identity);
BB_API int bb_batch_run(bb_ctx *ctx);
BB_API int bb_synchronize(bb_ctx *ctx);
/* A batch run is enqueued with buffers, error-loop rounds, Hirschberg levels and scratch sized from the fragment lengths.
 * When the device reports that one of them was too small, the fetch raises it and runs the batch again (at most three
 * times; then it fails with "batch did not fit after growing").  Raised limits stay on the context.  This reports the
 * re-runs of the last bb_batch_run, summed over the workers, and the BB_RERUN_* bits of what did not fit; complete once
 * the batch has been fetched.  Environment variables read at bb_create set the starting limits:
 * BADREAD_B200_ROUNDS (1..15, default 3), BADREAD_B200_SLACK (> 0, default 1.25), BADREAD_B200_EXTRA_LEVELS (default 0,
 * may be negative), BADREAD_B200_LR_CAP (split-score rows, default: from the expected edits, at least 4096). */
enum bb_rerun_reason {
    BB_RERUN_ROUNDS = 1,   /* reads still in the error loop after the last round */
    BB_RERUN_SLACK = 2,    /* joined reads longer than the read buffers */
    BB_RERUN_LEVELS = 4,   /* Hirschberg nodes left after the last level */
    BB_RERUN_QUEUES = 8,   /* node queues overflowed */
    BB_RERUN_SCRATCH = 16  /* per-warp alignment scratch too small */
};
BB_API int bb_last_run_retries(const bb_ctx *ctx, int32_t *n_reruns, uint32_t *reasons);
/* Diagnostics: which alignment kernels the last run of the last batch gave work to, summed over the workers and both
 * final-alignment pipelines (the run after any re-runs; complete once the batch has been fetched, BB_ERR_STATE before).
 *  work[BB_WORK_SLOTS]: window alignments by kernel (the 4-word lane kernel takes every window first and passes the
 *    ones beyond its limits on to the 8-word lane kernel, which passes its own on to the warp kernel), summed over the
 *    error-loop rounds; Hirschberg leaves by kernel, all of them and those that were whole roots.
 *  level_nodes[level_cap][BB_NODE_CLASSES]: Hirschberg nodes queued for each level (0: the roots that are not leaves)
 *    by node kernel class; levels the run did not reach hold 0.
 *  *n_levels: Hirschberg levels the run enqueued (at most BB_MAX_LEVELS). */
enum bb_work_slot {
    BB_WORK_WINDOW_LANE4 = 0,     /* bb_k_window_lane_hist<4> (bb_k_window_lane<4> with BADREAD_B200_LOWMEM=1) */
    BB_WORK_WINDOW_LANE8 = 1,     /* bb_k_window_lane_hist<8> / bb_k_window_lane<8> */
    BB_WORK_WINDOW_WARP = 2,      /* bb_k_window_warp */
    BB_WORK_LEAF_LANE = 3,        /* bb_k_leaf_lane_hist / bb_k_leaf_lane */
    BB_WORK_LEAF_WARP = 4,        /* bb_k_leaf_warp */
    BB_WORK_ROOT_LEAF_LANE = 5,   /* ... of BB_WORK_LEAF_LANE: roots (whole reads) */
    BB_WORK_ROOT_LEAF_WARP = 6,   /* ... of BB_WORK_LEAF_WARP: roots */
    BB_WORK_SLOTS = 7
};
/* node classes of level_nodes: bb_k_node_lane<8>, bb_k_node_warp<1>, <2>, <4>, and wide nodes (bb_k_node_pair, or
 * bb_k_node_quad with BADREAD_B200_QUAD=1) */
enum bb_node_class { BB_NODE_LANE8 = 0, BB_NODE_LEAN1 = 1, BB_NODE_LEAN2 = 2, BB_NODE_LEAN4 = 3, BB_NODE_WIDE = 4, BB_NODE_CLASSES = 5 };
#define BB_MAX_LEVELS 48
BB_API int bb_last_run_work(const bb_ctx *ctx, int64_t *work, int64_t *level_nodes, int32_t level_cap, int32_t *n_levels);
/* CUDA-event time (ms) of the last bb_batch_run on the ctx stream, total and per stage
 * (stage_ms[BB_N_STAGES], see bb_stage_name). Synchronizes. */
#define BB_N_STAGES 8
BB_API int bb_last_run_ms(bb_ctx *ctx, float *total_ms, float *stage_ms);
BB_API const char *bb_stage_name(int stage);
/* Number of kernel launches issued by this context so far. */
BB_API int64_t bb_launch_count(const bb_ctx *ctx);
/* Diagnostics: with BADREAD_B200_TRACE=1 in the environment at bb_create, every launch of a run is followed by a CUDA
 * event; this writes the last run's timeline (worker, stream, name, begin_ms, end_ms) as CSV. */
BB_API int bb_trace_dump(bb_ctx *ctx, const char *path);

/* get_qscores(seq, frag, qscore_model) on its own (qscore_model.py:32-75) for one pair; qual_out has seq_len bytes. */
BB_API int bb_get_qscores(bb_ctx *ctx, uint64_t read_index, const uint8_t *seq, int32_t seq_len, const uint8_t *frag,
                   int32_t frag_len, uint8_t *qual_out, int32_t *matches, int32_t *columns);

/* edlib.align(query, target, task='path') on the device for one pair: expanded CIGAR (one of "=XID" per column)
 * into ops_out (capacity ops_cap); *n_ops = columns, *distance = edit distance. Diagnostic / test entry point
 * for the aligner the kernels use. */
BB_API int bb_align_path(bb_ctx *ctx, const uint8_t *query, int32_t q_len, const uint8_t *target, int32_t t_len,
                  uint8_t *ops_out, int64_t ops_cap, int64_t *n_ops, int32_t *distance);

/* ---- BGZF output ------------------------------------------------------------------------------------ */
/* FASTQ text compressed on the device as BGZF (SAM specification §4.1): independent gzip members of BB_BGZF_CHUNK input
 * bytes each (the last one of a stream may be shorter), at fixed offsets of the whole stream, so the bytes do not depend on
 * how the caller splits the stream into calls.  gzip, zlib and htslib read the result.  Each member is entropy coded with
 * its own dynamic Huffman tables per sequence / quality segment (no string matching), or stored if that is not smaller.
 *  bb_bgzf_bound(n): the most bytes compressing n input bytes can give (the end-of-file member not counted).
 *  bb_bgzf_compress: line_mod4 is the index mod 4 of the FASTQ line in[0] belongs to.  Without `final` only the whole
 *  chunks of in[0..n) are compressed and *n_consumed = their length: the caller keeps the rest and passes it again,
 *  followed by more input, in the next call.  With `final` the last partial chunk is compressed as well (*n_consumed = n).
 *  The 28-byte end-of-file member is never written: the caller appends it once the stream is complete.  out_cap must be at
 *  least bb_bgzf_bound(bytes to be consumed), else BB_ERR_CAPACITY with *n_out = that bound.  *n_out = bytes written.
 *  The call runs on a stream and scratch of the context's own: the batch workers' streams and buffers are left alone. */
#define BB_BGZF_CHUNK 65280
BB_API int64_t bb_bgzf_bound(int64_t n);
BB_API int bb_bgzf_compress(bb_ctx *ctx, const uint8_t *in, int64_t n, int line_mod4, int final, uint8_t *out, int64_t out_cap,
                            int64_t *n_out, int64_t *n_consumed);

/* ---- BAM output ------------------------------------------------------------------------------------- */
/* Unaligned BAM records (SAM specification v1.6 §4.2) of the last batch, built on the device from the workers' output
 * buffers, so that with one GPU the bases and qualities never cross PCIe before they are compressed.  A record is
 * refID -1, pos -1, bin 4680, MAPQ 0, FLAG 4, no CIGAR, next_refID -1, next_pos -1, tlen 0, the read name, seq as 4-bit
 * =ACMGRSVTWYHKDBN codes (either case; any other byte is N), qual = the FASTQ quality character - 33, and one CO:Z tag.
 * The records form a record stream (the BAM file after its header) that the context keeps on the device: the records of
 * each bb_bam_build are appended to it.
 *
 *  bb_fetch_last_batch_results: bb_fetch_last_batch without the bases and qualities, which stay on the device for
 *  bb_bam_build.  *out_total = bytes of output the batch holds.
 *
 *  bb_bam_build: appends one record per recs[i] (in order) to the record stream.  recs[i].out_off / out_len are a read's
 *  out_off / out_len in the last fetched batch's results; its name (name_len bytes, at most 254) and its CO text (co_len
 *  bytes) lie back to back at text[recs[i].text_off ..].  Runs on the context's own stream and scratch; the workers'
 *  buffers are only read.  BB_ERR_STATE if no batch was fetched; BB_ERR_ARG for a record outside the batch or the text.
 *
 *  bb_bam_compress_device: compresses the record stream as BGZF members of BB_BGZF_CHUNK bytes at fixed offsets of the
 *  stream, a deflate block starting at every seq or qual field with at least 1024 bytes in the member.  Without `final`
 *  only whole chunks are compressed and the rest (< BB_BGZF_CHUNK bytes) stays on the device for the next call.  out_cap
 *  must be at least bb_bgzf_bound(bytes to be compressed), else BB_ERR_CAPACITY with *n_out = that bound.
 *
 *  bb_bam_fetch_records: copies the records of the last bb_bam_build to the host and takes them off the record stream
 *  (for a record stream merged from several GPUs).  Record i goes to out[dst_off[i] ..], or back to back if dst_off is
 *  NULL; out_cap bounds every write.  *n_bytes = the bytes of the records.  BB_ERR_STATE if the stream was compressed
 *  since that build.
 *
 *  bb_bam_compress: compresses the host bytes in[0..n) of a record stream, in[0] being byte stream_base of the stream,
 *  the way bb_bam_compress_device does: fields[2 * n_fields] are the (stream offset, length) pairs of the seq and qual
 *  fields in stream order (fields outside in[] are ignored).  Consumed bytes, capacity and `final` as bb_bgzf_compress. */
typedef struct bb_bam_record {
    int64_t out_off;   /* the read's out_off in the batch results */
    int64_t text_off;  /* its name, then its CO text, in the text pool */
    int32_t out_len;   /* l_seq */
    int32_t name_len;  /* bytes of the name, without a NUL */
    int32_t co_len;    /* bytes of the CO text, without a NUL */
    int32_t reserved;
} bb_bam_record;
BB_API int bb_fetch_last_batch_results(bb_ctx *ctx, bb_read_result *results, int64_t *out_total);
BB_API int bb_bam_build(bb_ctx *ctx, int32_t n_records, const bb_bam_record *recs, const uint8_t *text, int64_t text_len);
BB_API int bb_bam_compress_device(bb_ctx *ctx, int final, uint8_t *out, int64_t out_cap, int64_t *n_out);
BB_API int bb_bam_fetch_records(bb_ctx *ctx, const int64_t *dst_off, uint8_t *out, int64_t out_cap, int64_t *n_bytes);
BB_API int bb_bam_compress(bb_ctx *ctx, const uint8_t *in, int64_t n, int64_t stream_base, const int64_t *fields,
                           int64_t n_fields, int final, uint8_t *out, int64_t out_cap, int64_t *n_out, int64_t *n_consumed);

/* ---- BGZF input ------------------------------------------------------------------------------------- */
/* Inflates the BGZF stream in[0..n) on `device` (any number of members, the end-of-file member included) into out: one warp
 * per member, all three deflate block types, every member's CRC-32 and ISIZE checked.  Like the model builders' calls it
 * takes a device instead of a bb_ctx, allocates and releases what it needs, and describes failures in bb_model_error().
 *  The host walks the members' BC extra fields (BSIZE) first: *n_out = the inflated size of the stream (the sum of the
 *  ISIZEs); BB_ERR_CAPACITY if out_cap is smaller (out may then be NULL).
 *  BB_ERR_ARG for input that is not BGZF (a gzip member without BC) and for a member that is truncated, holds an invalid
 *  Huffman table or code, a back-reference before its start, or does not match its CRC-32 or ISIZE; the message names the
 *  member (index and offset).  Malformed input never makes the kernel read or write outside the member. */
BB_API int bb_bgzf_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out);

/* Inflates any gzip stream in[0..n) on `device`: one member or several, as gzip, pigz or zlib write them, with what
 * Python's gzip.decompress accepts: NUL padding between and after members, FEXTRA, FNAME, FCOMMENT and FHCRC skipped
 * (the header CRC is not checked).  Unlike Python it refuses a reserved header flag, as RFC 1952 asks.  A stream whose
 * every member is BGZF goes through bb_bgzf_decompress's one warp per member; any other is cut into chunks of
 * chunk_bytes compressed bytes (0: the default, 128 KiB) decoded side by side, each from a block start it finds itself,
 * and stitched where one chunk's decoder stopped at the next one's start (csrc/bb_gunzip.cuh).  The choice is made from
 * the input.  Every member's CRC-32 and ISIZE (mod 2^32) is checked.  Device memory peaks at about 11 bytes per input
 * byte (the input and 16-bit symbol slots of 5 symbols per input byte) plus the output plus 32 KiB per chunk; more if
 * a chunk inflates beyond 5 bytes per input byte, which makes every chunk decode again into larger slots.  The output size is known only once the stream has been inflated: *n_out = it, and BB_ERR_CAPACITY
 * if out_cap is smaller (out may then be NULL), so that the caller asks again with the room.  BB_ERR_ARG for a corrupt
 * stream, the message (bb_model_error()) naming the member by index and input offset.  stats (may be NULL) tells how the
 * stream was inflated. */
struct bb_gzip_stats {
    int64_t members;          /* gzip members */
    int64_t chunks;           /* chunks the deflate data were cut into (0 for BGZF) */
    int64_t absorbed;         /* chunks without a block start, decoded as part of their predecessor */
    int64_t first_candidate;  /* chunks after the first confirmed at the first block start they found */
    int64_t repaired;         /* decodes of a chunk again from where its predecessor stopped, in repair launches */
    int64_t chained;          /* ... and in the final serial chain */
    int64_t reruns;           /* decodes run again with larger output slots */
    int32_t bgzf;             /* 1: every member was BGZF (one warp per member) */
    int32_t reserved;
};
BB_API int bb_gzip_decompress(int device, const uint8_t *in, int64_t n, uint8_t *out, int64_t out_cap, int64_t *n_out,
                              int64_t chunk_bytes, bb_gzip_stats *stats);

/* ---- host-side helpers (no GPU needed) -------------------------------------------------------------- */
/* error_model.align_kmers (error_model.py:179-229) for a batch of (kmer, alt) pairs: kmers is n_alts*k bytes,
 * alts are concatenated with alt_off[n_alts+1]. Writes n_alts*k encoded slots, appends long strings to pool
 * (capacity pool_cap, *pool_len updated) and flags bit0 = (''.join(slots) == kmer). */
BB_API int bb_host_align_kmers(int k, int32_t n_alts, const uint8_t *kmers, const uint8_t *alts, const int32_t *alt_off,
                        uint32_t *slots_out, uint8_t *flags_out, uint8_t *pool, int64_t pool_cap, int64_t *pool_len);
/* edlib.align(query, target, task='path') on the host for SMALL inputs (full matrix; q_len*t_len <= 2^22). */
BB_API int bb_host_align_path(const uint8_t *query, int32_t q_len, const uint8_t *target, int32_t t_len, uint8_t *ops_out,
                       int64_t ops_cap, int64_t *n_ops, int32_t *distance);


/* ---- multi-GPU: the one collective of the path ------------------------------------------------------ */
/* Reads shard over GPUs by read index (GPU g owns indices = g mod G) and never exchange data.  The only value the GPUs
 * have to agree on is the running total of emitted bases that ends the simulation (simulate.py:63): one NCCL
 * all-reduce (SUM, one int64) per batch.  NCCL is loaded at run time (dlopen of libnccl.so.2); bb_nccl_available()
 * says whether that worked.  Two ways to form the communicator:
 *   one process per GPU (torchrun / mpirun): rank 0 calls bb_comm_unique_id, the host program ships the 128 bytes to
 *     the other ranks by whatever means it has, every rank calls bb_comm_init_rank, then bb_allreduce_bases;
 *   one process, several GPUs (`badread simulate --gpus N`): bb_comm_init_all, then bb_allreduce_bases_all. */
typedef struct bb_nccl_id { char internal[128]; } bb_nccl_id;   /* ncclUniqueId */
BB_API int bb_nccl_available(void);
BB_API int bb_comm_unique_id(bb_nccl_id *id);
BB_API int bb_comm_init_rank(bb_ctx *ctx, const bb_nccl_id *id, int rank, int world);
BB_API int bb_comm_init_all(bb_ctx **ctxs, int n);
BB_API int bb_allreduce_bases(bb_ctx *ctx, int64_t local, int64_t *total);
BB_API int bb_allreduce_bases_all(bb_ctx **ctxs, int n, const int64_t *local, int64_t *total);

/* ---- fragment builder and FASTQ assembly on the host (no GPU needed) -------------------------------- */
/* The steps either side of the hot path, as native multi-threaded host code.  bb_planner_plan replaces the per-read
 * Python of build_fragment (badread/simulate.py:91-115), get_fragment / get_real_fragment / get_junk_fragment
 * (:148-253), the adapters (:361-394), add_glitches (:459-482), FragmentLengths.get_fragment_length
 * (fragment_lengths.py:47-64) and Identities.get_identity (identities.py:76-94); it emits fragment DESCRIPTORS in
 * exactly the layout bb_batch_upload / bb_sequence_batch take.  Every read draws from its own random.Random /
 * numpy RandomState keyed by (seed, read index), restated bit for bit. */
typedef struct bb_planner bb_planner;

typedef struct bb_plan_config {
    uint64_t seed;
    /* reference (misc.load_fasta, simulate.py:118-121): contigs in file order */
    int32_t n_contigs;
    const int64_t *contig_len;
    const double *contig_weight;     /* depth * length after adjust_depths (simulate.py:516-536) */
    const uint8_t *contig_flags;     /* bit 0 circular, bit 1 hairpin_left, bit 2 hairpin_right */
    const char *contig_names;        /* concatenated; contig i is [contig_name_off[i], contig_name_off[i+1]) */
    const int64_t *contig_name_off;
    /* fragment lengths (fragment_lengths.py): stdev == 0 => constant */
    double frag_mean, frag_stdev, gamma_k, gamma_t;
    /* identities (identities.py): type 0 beta (mean, max as fractions), 1 normal (mean, stdev as qscores) */
    int32_t identity_type;
    double id_mean, id_stdev, id_max, beta_a, beta_b;
    /* adapters (simulate.py:361-394): rate / amount as fractions */
    const uint8_t *start_adapter; int32_t start_adapter_len; double start_adapter_rate, start_adapter_amount;
    const uint8_t *end_adapter; int32_t end_adapter_len; double end_adapter_rate, end_adapter_amount;
    /* read types (simulate.py:168-180) and chimeras (:101-110), as fractions */
    double junk_rate, random_rate, chimera_rate, chimera_end_adapter_chance, chimera_start_adapter_chance;
    /* glitches (simulate.py:459-482) */
    double glitch_rate, glitch_size, glitch_skip;
} bb_plan_config;

/* The last plan of a planner (pointers stay valid until the next bb_planner_plan / bb_planner_destroy). */
typedef struct bb_plan_view {
    int32_t n_reads;
    const uint64_t *read_index;      /* [n] */
    const int32_t *seg_off;          /* [n+1] */
    const bb_segment *segs;
    const uint8_t *literals;
    int64_t literal_len;
    const double *target_identity;   /* [n] */
    const uint8_t *read_names;       /* [n][16]: uuid.UUID(int=random.getrandbits(128)).bytes (simulate.py:77) */
    const int64_t *info_off;         /* [n+1] into info */
    const char *info;                /* ' '.join(info) of simulate.py:97-113, before the length fields */
    const int32_t *frag_len;         /* [n] len(fragment) */
} bb_plan_view;

BB_API int bb_planner_create(bb_planner **planner, const bb_plan_config *config);
BB_API int bb_planner_destroy(bb_planner *planner);
/* Plans reads first_index, first_index + stride, ... (n_reads of them) with n_threads host threads.
 * BB_ERR_STATE: a read could not be built (the reference exits with bb_planner_error()'s message, simulate.py:164). */
BB_API int bb_planner_plan(bb_planner *planner, uint64_t first_index, uint64_t stride, int32_t n_reads, int32_t n_threads);
BB_API int bb_planner_view(const bb_planner *planner, bb_plan_view *view);
BB_API const char *bb_planner_error(const bb_planner *planner);

/* FASTQ records of simulate.py:70-86 for reads [first, n) of a finished batch in plan order, into out: empty reads
 * are skipped; stops after the read with which bases_so_far + emitted bases reaches target_bases.  *out_len = bytes
 * needed (BB_ERR_CAPACITY if out_cap is smaller), *next_read = first read not consumed. */
BB_API int bb_fastq_format(const bb_plan_view *view, const bb_read_result *results, const uint8_t *seq, const uint8_t *qual,
                    int32_t first, int64_t bases_so_far, int64_t target_bases, int32_t n_threads, uint8_t *out,
                    int64_t out_cap, int64_t *out_len, int32_t *n_emitted, int64_t *bases_emitted, int32_t *next_read);
/* The same for a batch dealt out over n_shards contexts (GPUs): read j of the batch is read j / n_shards of shard
 * j % n_shards (views[g], results[g], seq[g], qual[g]); records come out in read-index order, independent of n_shards. */
BB_API int bb_fastq_format_sharded(int32_t n_shards, const bb_plan_view *const *views, const bb_read_result *const *results,
                            const uint8_t *const *seq, const uint8_t *const *qual, int32_t first, int64_t bases_so_far,
                            int64_t target_bases, int32_t n_threads, uint8_t *out, int64_t out_cap, int64_t *out_len,
                            int32_t *n_emitted, int64_t *bases_emitted, int32_t *next_read);
/* The layout of the BAM records (bb_bam_build) of the same emitted set and cutoff as bb_fastq_format_sharded for the same
 * arguments, the first record starting at byte stream_base of the record stream.  For emitted record e: shard[e] and
 * index[e] (the read's shard and its position in that shard's results), stream_off[e], recs[e] (out_off and out_len from
 * the results; text_off into text) and fields[4 e ..] = stream offset and length of its seq field, then of its qual field.
 * shard, index, stream_off, recs and fields hold an entry for every read of the batch.  The name is the UUID of the FASTQ
 * header and the CO text the rest of its header line ("{info} length=... error-free_length=... read_identity=...%"),
 * formatted by the code that writes the FASTQ header.  *text_len = bytes of text needed (BB_ERR_CAPACITY if text_cap is
 * smaller), *stream_len = bytes of the records. */
BB_API int bb_bam_layout_sharded(int32_t n_shards, const bb_plan_view *const *views, const bb_read_result *const *results,
                                 int32_t first, int64_t bases_so_far, int64_t target_bases, int64_t stream_base,
                                 int32_t *shard, int32_t *index, int64_t *stream_off, bb_bam_record *recs, int64_t *fields,
                                 uint8_t *text, int64_t text_cap, int64_t *text_len, int64_t *stream_len,
                                 int32_t *n_emitted, int64_t *bases_emitted, int32_t *next_read);

/* ---- Model builders: the counting passes of `badread error_model` (badread/error_model.py:31-83) and `badread
 * qscore_model` (badread/qscore_model.py:78-161) on the GPU.  The caller has parsed the inputs and chosen the alignments
 * (badread/alignment.py:79-105) and hands them over flat: for alignment a = 0 .. n_aln-1 the aligned slice of the read
 * read[read_off[a] .. read_off[a+1]) (and its qualities), the aligned slice of the reference ref[ref_off[a] .. ref_off[a+1])
 * already on the read's strand, and the CIGAR runs ops[ops_off[a] .. ops_off[a+1]) in read orientation, each
 * (length << 2) | type with type 0 = M, 1 = I, 2 = D, starting at read offset op_read0[] / reference offset op_ref0[] within
 * the alignment.  A window's content is a 64-bit key; the library returns every distinct key with its count(s) and the first
 * window it occurred in (the reference's dicts keep insertion order and its stable sorts break ties by it), in arbitrary order:
 *   bb_count_kmer_alternatives  key = reference k-mer (2k bits from bit 63 down, A C G T = 0 1 2 3) | read k-mer length
 *                               (6 bits) | read k-mer (2 bits a base from bit 0 up); counts_out: one per key;
 *                               first_out = (alignment << 32) | reference offset of the window.  k <= 12.
 *   bb_count_cigar_qscores      key = CIGAR length (6 bits from bit 63 down) | symbols (2 bits each from bit 0 up, = X I D =
 *                               0 1 2 3, runs of 'D' cut to max_del); counts_out: 94 per key (quality 0 .. 93 of the window's
 *                               middle base); first_out = (alignment << 36) | ((window size - 1) / 2 << 32) | read offset;
 *                               overall_out[94]: the qualities of all bases.  Odd k <= 13: every odd size up to k is counted.
 * Windows that do not fit a key (and quality characters outside '!' .. '~') are not counted but listed: alignment, offset and
 * window size (negative for a bad quality character) in ovf_*; the caller evaluates those itself.  table_cap (a power of two)
 * slots are used on the device and bound the number of distinct keys; BB_ERR_CAPACITY if the table or the overflow list is
 * too small (*n_ovf then holds the required overflow capacity).  bb_model_error() describes the last failure of the calling
 * thread.  No bb_ctx is involved: the calls allocate and release what they need on `device`.  read, qual, ref, ops,
 * op_read0 and op_ref0 may be host memory, copied to the device for the call, or device memory of `device` (a bb_flat_view's
 * arrays), used in place; the three offset arrays are host memory. */
BB_API int bb_count_kmer_alternatives(int device, int k, int32_t n_aln, const uint8_t *read, const int64_t *read_off,
                               const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                               const int32_t *op_ref0, const int64_t *ops_off, int64_t table_cap, uint64_t *keys_out,
                               uint64_t *first_out, uint32_t *counts_out, int64_t *n_entries, int64_t ovf_cap,
                               int32_t *ovf_aln, int32_t *ovf_pos, int32_t *ovf_k, int64_t *n_ovf);
/*   bb_count_kmer_alternatives_wide  the same count for 12 < k <= 16 with a 128-bit key, two words per key in keys_out:
 *                               [2i] = read k-mer (2 bits a base from bit 0 up, at most 32 bases), [2i+1] = (reference k-mer
 *                               << 6) | read k-mer length; first_out and counts_out as above.  Longer read k-mers overflow. */
BB_API int bb_count_kmer_alternatives_wide(int device, int k, int32_t n_aln, const uint8_t *read, const int64_t *read_off,
                                    const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                                    const int32_t *op_ref0, const int64_t *ops_off, int64_t table_cap, uint64_t *keys_out,
                                    uint64_t *first_out, uint32_t *counts_out, int64_t *n_entries, int64_t ovf_cap,
                                    int32_t *ovf_aln, int32_t *ovf_pos, int32_t *ovf_k, int64_t *n_ovf);
BB_API int bb_count_cigar_qscores(int device, int k, int max_del, int32_t n_aln, const uint8_t *read, const uint8_t *qual,
                           const int64_t *read_off, const uint8_t *ref, const int64_t *ref_off, const uint32_t *ops,
                           const int32_t *op_read0, const int32_t *op_ref0, const int64_t *ops_off, int64_t table_cap,
                           uint64_t *keys_out, uint64_t *first_out, uint32_t *counts_out, int64_t *n_entries,
                           uint64_t *overall_out, int64_t ovf_cap, int32_t *ovf_aln, int32_t *ovf_pos, int32_t *ovf_k,
                           int64_t *n_ovf);
BB_API const char *bb_model_error(void);

/* SAM / BAM alignment records for the model builders, parsed on the host (no GPU needed).  data[0..n) is SAM text or, with
 * is_bam, an inflated BAM file (bb_bgzf_decompress).  Mapped records only (FLAG 0x4 and RNAME '*' / refID -1 are skipped),
 * at most max_records of them (<= 0: all).  Per record the fields of the PAF line the reference's builders read:
 *   read_len    the M I S = X H ops            read_start  the leading clip (S + H) on '+', the trailing clip on '-'
 *   read_end    read_start + the M I = X ops   ref_start   POS - 1;   ref_end  ref_start + the M D = X ops
 *   columns     the M I D = X ops              nm          NM:i, or -1 without it;   score  AS:i
 * and the CIGAR runs (length << 4 | BAM op code, SAM order), SEQ (upper case) and QUAL (Phred+33) as stored; a record
 * without SEQ has none, has_qual[i] = 0 without QUAL, full[i] = SEQ present and no H clip.  Reads and references are
 * numbered in order of first appearance (references of a BAM header or of SAM @SQ lines first).
 * BB_ERR_ARG with bb_model_error() = the message to exit with: "Error: no CIGAR string found" (a mapped record with
 * CIGAR '*'), "Error: no alignment score" (no AS:i), an N or P op (names the read), or malformed input.
 * With is_bam = 2 (BB_ALN_PAF) data is PAF text, read as model_builders.load_alignments reads it: '\n', "\r\n" and a lone
 * '\r' end lines, each line is stripped (str.strip()'s ASCII set) and split on '\t', and every line is a record (at most
 * max_records lines are parsed).  read_start / read_end / ref_start / ref_end are columns 3, 4, 8 and 9 as written,
 * columns = column 11, nm = column 11 - column 10, flag 0x10 on strand '-', score = the last AS:i: tag, and the CIGAR the
 * last cg:Z: tag's runs (a digit run followed by a letter or '='; other bytes are skipped) with M I D as BAM's codes and
 * every other letter as 15.  BB_ERR_ARG: "Error: alignment file does not seem to be in PAF format" (fewer than 11
 * columns), "Error: no CIGAR string found", "Error: no alignment score", or a field that is not an integer. */
typedef struct bb_aln_set bb_aln_set;
typedef struct bb_aln_view {
    int64_t n_records;
    int32_t n_refs, n_reads;
    const char *ref_names;  const int64_t *ref_name_off;    /* [n_refs + 1] */
    const char *read_names; const int64_t *read_name_off;   /* [n_reads + 1] */
    const int32_t *read_id, *ref_id, *flag, *score, *nm, *read_len, *read_start, *read_end, *columns;   /* [n_records] */
    const int64_t *ref_start, *ref_end;                     /* [n_records] */
    const uint32_t *cigar;  const int64_t *cigar_off;       /* [n_records + 1] */
    const uint8_t *seq, *qual; const int64_t *seq_off;      /* [n_records + 1] */
    const uint8_t *has_qual, *full;                         /* [n_records] */
} bb_aln_view;
BB_API int bb_aln_parse(const uint8_t *data, int64_t n, int is_bam, int64_t max_records, bb_aln_set **set);
BB_API int bb_aln_view_get(const bb_aln_set *set, bb_aln_view *view);   /* valid until bb_aln_free */
BB_API int bb_aln_free(bb_aln_set *set);
#define BB_ALN_PAF 2

/* The model builders' device route for FASTQ reads (model_builders.DeviceFlat).  bb_device_count: the CUDA devices the
 * library sees (0 when there are none or no driver).
 * bb_fastq_parse: data[0..n) (host memory: the file as it is; is_gzip: a gzip stream, BGZF or not, inflated on the device
 * as bb_gzip_decompress does) parsed on `device` as model_builders.load_fastq parses it (csrc/bb_fastq.cuh).  *first_byte:
 * the first byte of the inflated text (-1 when it is empty); only a text that starts with '@' is parsed, into *n_records
 * records whose name, sequence and quality spans stay on the device and whose names come to the host.  BB_ERR_ARG with
 * bb_model_error() naming the record for a header without a name or a record the file ends in; BB_ERR_CAPACITY naming the
 * stage and the bytes asked for when device memory runs out.  Device memory peaks at the inflater's peak, then at the text
 * plus 56 bytes per record plus 8 per line.
 * bb_flat_build: the flat arrays of bb_count_* on the device for n_aln alignments, records[i] of the bb_aln_view v (PAF):
 * reads joined to FASTQ records by name (a repeated name: its last record), references at contig_at[ref id] of
 * contigs[0..contigs_len) (-1: not loaded), contig_len[ref id] bytes long; the read, quality and reference slices with
 * Python's slice semantics, the reference reverse-complemented on '-', each padded with NUL to the CIGAR's length
 * (model_builders.FlatAlignments).  BB_ERR_ARG with failed[0] = the first alignment whose read (failed[1] = 1) or reference
 * (2) is missing, checked in that order per alignment, or the first whose read holds a byte >= 0x80 in its sequence or
 * qualities (3).  slice_len (may be NULL) gets, per alignment, 3 lengths before any padding or truncation: of the read's
 * sequence slice, of its quality slice and of the reference slice (`badread_b200 plot` refuses alignments whose CIGAR
 * does not fit them).  On success the FASTQ's text and record table are released (its names stay until bb_fastq_free).  Device
 * memory then holds the text and record table plus the flat arrays: 2 bytes per read column, 1 per reference column and 12
 * per CIGAR run, and the uploaded contigs.
 * bb_flat_fetch copies elements [lo, lo + count) of array `which` (0 read, 1 qual, 2 ref, 3 ops, 4 op_read0, 5 op_ref0)
 * to host memory. */
typedef struct bb_fastq_set bb_fastq_set;
typedef struct bb_flat_set bb_flat_set;
typedef struct bb_flat_view {
    int32_t n;                                                   /* alignments */
    const uint8_t *read, *qual, *ref;                            /* device memory */
    const uint32_t *ops; const int32_t *op_read0, *op_ref0;      /* device memory */
    const int64_t *read_off, *ref_off, *ops_off;                 /* host memory, [n + 1] */
} bb_flat_view;
BB_API int bb_device_count(void);
BB_API int bb_fastq_parse(int device, const uint8_t *data, int64_t n, int is_gzip, bb_fastq_set **set, int64_t *n_records,
                          int32_t *first_byte);
BB_API int bb_fastq_free(bb_fastq_set *set);
BB_API int bb_flat_build(bb_fastq_set *fastq, const bb_aln_view *v, int32_t n_aln, const int64_t *records, const int64_t *contig_at,
                         const int64_t *contig_len, const uint8_t *contigs, int64_t contigs_len, bb_flat_set **flat,
                         int64_t *failed, int64_t *slice_len);
BB_API int bb_flat_view_get(const bb_flat_set *flat, bb_flat_view *view);   /* valid until bb_flat_free */
BB_API int bb_flat_fetch(const bb_flat_set *flat, int which, int64_t lo, int64_t count, void *dst);
BB_API int bb_flat_free(bb_flat_set *flat);

/* ---- `badread plot`'s window series (plot_window_identity.get_window_means of the reference; csrc/bb_plot.cuh).
 * bb_window_series: for the alignments first_aln .. first_aln + n_pass - 1 of the flat arrays of bb_count_* (read, qual,
 * ref, ops, op_read0 and op_ref0 host memory, copied for the call, or device memory of `device`, used in place; the
 * offsets [n_aln + 1] host memory), each of read slice length L, the windows i = 0 .. L - window - 1 in order, the
 * alignments one after the other: out_identity[] = 100 * (1 - S / window) with S the errors of read positions
 * [i, i + window) (1 per mismatching M base and per I base, n at the read offset where a D run of n starts), and with
 * want_qual out_qual[] = the sum of (quality byte - 33) over the window / window, both rounded as Python's float
 * operations are.  *n_points = the windows written, sum of max(0, L - window); out_* host memory of that many doubles.
 * The caller has checked every alignment: its M and I runs cover [0, L) exactly, no D run starts at L, its M runs lie
 * inside its reference slice.  Device memory: 8 bytes per read position (16 with want_qual) plus 8 (16) per window, plus
 * the inputs given in host memory.  BB_ERR_ARG for window < 1 or a range outside [0, n_aln); BB_ERR_CAPACITY naming
 * what did not fit in device memory.
 * bb_window_format: the table lines ("name\tposition\t%.4f identity[\t%.4f qscore]\n") of windows [lo, hi) of a
 * series of n_aln alignments: alignment a's name names[name_off[a] .. name_off[a + 1]), its windows [point_off[a],
 * point_off[a + 1]) of identity[] (and qual[], or NULL), at positions pos0[a], pos0[a] + 1, ...  Several host threads
 * format into out; *out_len = the bytes written.  BB_ERR_CAPACITY when cap is less than (hi - lo) times
 * bb_window_line_bound(the longest name), the most one line can take. */
BB_API int bb_window_series(int device, int32_t n_aln, const uint8_t *read, const uint8_t *qual, const uint8_t *ref,
                            const int64_t *read_off, const int64_t *ref_off, const uint32_t *ops, const int32_t *op_read0,
                            const int32_t *op_ref0, const int64_t *ops_off, int64_t window, int want_qual, int32_t first_aln,
                            int32_t n_pass, double *out_identity, double *out_qual, int64_t *n_points);
BB_API int64_t bb_window_line_bound(int64_t name_len);
BB_API int bb_window_format(int32_t n_aln, const char *names, const int64_t *name_off, const int64_t *pos0,
                            const int64_t *point_off, const double *identity, const double *qual, int64_t lo, int64_t hi,
                            char *out, int64_t cap, int64_t *out_len);

#ifdef __cplusplus
}
#endif
#endif /* BADREAD_B200_H */
