"""
ctypes binding of libbadread_b200.so (the C ABI declared in include/badread_b200.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C badread_b200/csrc`. There is no fallback:
if the shared object is missing this module raises, and if no GPU is usable `bb_create` fails.
"""
import ctypes
import os
import pathlib

# every worker of a context drives several CUDA streams; with the default of 8 hardware queues they would serialize
# behind each other (must be set before CUDA is initialized in this process; the library sets the same default)
os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')

_HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB_PATH = _HERE / 'libbadread_b200.so'

BB_OK = 0
BB_ERR_CUDA, BB_ERR_ARG, BB_ERR_STATE, BB_ERR_CAPACITY, BB_ERR_INTERNAL = -1, -2, -3, -4, -5
BB_SEG_REF_FWD, BB_SEG_REF_REV, BB_SEG_LITERAL = 0, 1, 2
BB_N_STAGES = 8
# bb_rerun_reason: what made a batch run again (bb_last_run_retries)
BB_RERUN_ROUNDS, BB_RERUN_SLACK, BB_RERUN_LEVELS, BB_RERUN_QUEUES, BB_RERUN_SCRATCH = 1, 2, 4, 8, 16
# bb_work_slot / bb_node_class: the task counts of bb_last_run_work
WORK_SLOTS = ('window_lane4', 'window_lane8', 'window_warp', 'leaf_lane', 'leaf_warp', 'root_leaf_lane', 'root_leaf_warp')
NODE_CLASSES = ('lane8', 'lean1', 'lean2', 'lean4', 'wide')
BB_MAX_LEVELS = 48
BB_BGZF_CHUNK = 65280   # input bytes per BGZF member (bb_bgzf_compress)


class Segment(ctypes.Structure):
    _fields_ = [('src', ctypes.c_int64), ('len', ctypes.c_int32), ('kind', ctypes.c_int32)]


class ReadResult(ctypes.Structure):
    _fields_ = [('out_off', ctypes.c_int64), ('out_len', ctypes.c_int32), ('frag_len', ctypes.c_int32),
                ('matches', ctypes.c_int32), ('columns', ctypes.c_int32), ('loop_count', ctypes.c_int32),
                ('change_count', ctypes.c_int32), ('n_alignments', ctypes.c_int32), ('flags', ctypes.c_int32),
                ('loop_kcycles', ctypes.c_int32), ('align_kcycles', ctypes.c_int32)]


class BamRecord(ctypes.Structure):
    """bb_bam_record (include/badread_b200.h)."""
    _fields_ = [('out_off', ctypes.c_int64), ('text_off', ctypes.c_int64), ('out_len', ctypes.c_int32),
                ('name_len', ctypes.c_int32), ('co_len', ctypes.c_int32), ('reserved', ctypes.c_int32)]


class GzipStats(ctypes.Structure):
    """bb_gzip_stats (include/badread_b200.h)."""
    _fields_ = [(f, ctypes.c_int64) for f in ('members', 'chunks', 'absorbed', 'first_candidate', 'repaired', 'chained',
                                              'reruns')] + [('bgzf', ctypes.c_int32), ('reserved', ctypes.c_int32)]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f, _ in self._fields_ if f != 'reserved'}


class PlanConfig(ctypes.Structure):
    """bb_plan_config (include/badread_b200.h)."""
    _fields_ = [('seed', ctypes.c_uint64), ('n_contigs', ctypes.c_int32), ('contig_len', ctypes.c_void_p),
                ('contig_weight', ctypes.c_void_p), ('contig_flags', ctypes.c_void_p), ('contig_names', ctypes.c_char_p),
                ('contig_name_off', ctypes.c_void_p),
                ('frag_mean', ctypes.c_double), ('frag_stdev', ctypes.c_double), ('gamma_k', ctypes.c_double),
                ('gamma_t', ctypes.c_double),
                ('identity_type', ctypes.c_int32), ('id_mean', ctypes.c_double), ('id_stdev', ctypes.c_double),
                ('id_max', ctypes.c_double), ('beta_a', ctypes.c_double), ('beta_b', ctypes.c_double),
                ('start_adapter', ctypes.c_char_p), ('start_adapter_len', ctypes.c_int32),
                ('start_adapter_rate', ctypes.c_double), ('start_adapter_amount', ctypes.c_double),
                ('end_adapter', ctypes.c_char_p), ('end_adapter_len', ctypes.c_int32),
                ('end_adapter_rate', ctypes.c_double), ('end_adapter_amount', ctypes.c_double),
                ('junk_rate', ctypes.c_double), ('random_rate', ctypes.c_double), ('chimera_rate', ctypes.c_double),
                ('chimera_end_adapter_chance', ctypes.c_double), ('chimera_start_adapter_chance', ctypes.c_double),
                ('glitch_rate', ctypes.c_double), ('glitch_size', ctypes.c_double), ('glitch_skip', ctypes.c_double)]


class PlanView(ctypes.Structure):
    """bb_plan_view (include/badread_b200.h)."""
    _fields_ = [('n_reads', ctypes.c_int32), ('read_index', ctypes.c_void_p), ('seg_off', ctypes.c_void_p),
                ('segs', ctypes.c_void_p), ('literals', ctypes.c_void_p), ('literal_len', ctypes.c_int64),
                ('target_identity', ctypes.c_void_p), ('read_names', ctypes.c_void_p), ('info_off', ctypes.c_void_p),
                ('info', ctypes.c_void_p), ('frag_len', ctypes.c_void_p)]


class AlnView(ctypes.Structure):
    """bb_aln_view (include/badread_b200.h)."""
    _fields_ = [('n_records', ctypes.c_int64), ('n_refs', ctypes.c_int32), ('n_reads', ctypes.c_int32)] + \
        [(f, ctypes.c_void_p) for f in ('ref_names', 'ref_name_off', 'read_names', 'read_name_off', 'read_id', 'ref_id', 'flag',
                                        'score', 'nm', 'read_len', 'read_start', 'read_end', 'columns', 'ref_start', 'ref_end',
                                        'cigar', 'cigar_off', 'seq', 'qual', 'seq_off', 'has_qual', 'full')]


class FlatView(ctypes.Structure):
    """bb_flat_view (include/badread_b200.h)."""
    _fields_ = [('n', ctypes.c_int32)] + [(f, ctypes.c_void_p) for f in ('read', 'qual', 'ref', 'ops', 'op_read0', 'op_ref0',
                                                                           'read_off', 'ref_off', 'ops_off')]


class EmLoadInfo(ctypes.Structure):
    """bb_em_load_info (include/badread_b200.h)."""
    _fields_ = [('k', ctypes.c_int32), ('index', ctypes.c_int32)] + \
        [(f, ctypes.c_int64) for f in ('n_rows', 'n_entries', 'n_alts', 'pool_bytes', 'text_bytes')] + \
        [('fallback', ctypes.c_uint32), ('reserved', ctypes.c_int32)] + \
        [(f, ctypes.c_double) for f in ('ms_inflate', 'ms_parse', 'ms_align', 'ms_tables', 'ms_index', 'ms_total')]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_ if f != 'reserved'}


# bb_em_fallback: why bb_load_error_model_file left a file to the host loader
EM_FALLBACK = {'number': 1, 'duplicate': 2, 'k': 4, 'base': 8, 'syntax': 16, 'cr': 32, 'long_alt': 64, 'alt_ends': 128,
               'empty_line': 256, 'input': 512, 'size': 1024}


BB_ALN_PAF = 2


class LibraryMissing(RuntimeError):
    pass


_lib = None


def lib():
    """Loads the shared library once. Raises LibraryMissing if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.is_file():
        raise LibraryMissing(f'{LIB_PATH} not found - build it with `python -c "import __graft_entry__ as g; '
                             f'g.build()"` or `make -C badread_b200/csrc` (there is no CPU fallback)')
    L = ctypes.CDLL(str(LIB_PATH))
    c = ctypes
    vp, i32, i64, u64, dbl = c.c_void_p, c.c_int32, c.c_int64, c.c_uint64, c.c_double
    P = c.POINTER
    sigs = {
        'bb_create': (c.c_int, [P(vp), c.c_int, u64]),
        'bb_destroy': (c.c_int, [vp]),
        'bb_last_error': (c.c_char_p, [vp]),
        'bb_version': (c.c_char_p, []),
        'bb_upload_reference': (c.c_int, [vp, vp, i64]),
        'bb_fasta_parse': (c.c_int, [vp, vp, i64, c.c_int, P(i32), P(i64), P(i64)]),
        'bb_fasta_headers': (c.c_int, [vp, vp, i64, vp, vp, i32]),
        'bb_last_gzip_stats': (c.c_int, [vp, P(GzipStats)]),
        'bb_fasta_reference': (c.c_int, [vp, i32, vp, vp]),
        'bb_download_reference': (c.c_int, [vp, i64, i64, vp]),
        'bb_upload_error_model': (c.c_int, [vp, c.c_int, c.c_int, vp, i64, i32, vp, vp, vp, vp, vp, i64]),
        'bb_upload_error_model_kmers': (c.c_int, [vp, c.c_int, i32, vp, vp, vp, vp, vp, vp, i64]),
        'bb_load_error_model_file': (c.c_int, [vp, vp, i64, P(EmLoadInfo)]),
        'bb_download_error_model': (c.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        'bb_upload_qscore_model': (c.c_int, [vp, c.c_int, i32, vp, vp, vp, vp]),
        'bb_upload_qscore_model_cigars': (c.c_int, [vp, c.c_int, i32, vp, vp, vp, vp, vp]),
        'bb_sequence_batch': (c.c_int, [vp, i32, vp, vp, vp, vp, i64, vp, vp, vp, vp, i64, P(i64)]),
        'bb_fetch_last_batch': (c.c_int, [vp, vp, vp, vp, i64, P(i64)]),
        'bb_batch_upload': (c.c_int, [vp, i32, vp, vp, vp, vp, i64, vp]),
        'bb_batch_run': (c.c_int, [vp]),
        'bb_synchronize': (c.c_int, [vp]),
        'bb_last_run_retries': (c.c_int, [vp, P(i32), P(c.c_uint32)]),
        'bb_last_run_work': (c.c_int, [vp, vp, vp, i32, P(i32)]),
        'bb_host_alloc': (c.c_int, [P(vp), i64]),
        'bb_host_free': (c.c_int, [vp]),
        'bb_last_run_ms': (c.c_int, [vp, P(c.c_float), P(c.c_float)]),
        'bb_stage_name': (c.c_char_p, [c.c_int]),
        'bb_launch_count': (i64, [vp]),
        'bb_trace_dump': (c.c_int, [vp, c.c_char_p]),
        'bb_get_qscores': (c.c_int, [vp, u64, vp, i32, vp, i32, vp, P(i32), P(i32)]),
        'bb_align_path': (c.c_int, [vp, vp, i32, vp, i32, vp, i64, P(i64), P(i32)]),
        'bb_host_align_kmers': (c.c_int, [c.c_int, i32, vp, vp, vp, vp, vp, vp, i64, P(i64)]),
        'bb_host_align_path': (c.c_int, [vp, i32, vp, i32, vp, i64, P(i64), P(i32)]),
        'bb_nccl_available': (c.c_int, []),
        'bb_comm_unique_id': (c.c_int, [vp]),
        'bb_comm_init_rank': (c.c_int, [vp, vp, c.c_int, c.c_int]),
        'bb_comm_init_all': (c.c_int, [P(vp), c.c_int]),
        'bb_allreduce_bases': (c.c_int, [vp, i64, P(i64)]),
        'bb_allreduce_bases_all': (c.c_int, [P(vp), c.c_int, P(i64), P(i64)]),
        'bb_planner_create': (c.c_int, [P(vp), P(PlanConfig)]),
        'bb_planner_destroy': (c.c_int, [vp]),
        'bb_planner_plan': (c.c_int, [vp, u64, u64, i32, i32]),
        'bb_planner_view': (c.c_int, [vp, P(PlanView)]),
        'bb_planner_error': (c.c_char_p, [vp]),
        'bb_fastq_format': (c.c_int, [P(PlanView), vp, vp, vp, i32, i64, i64, i32, vp, i64, P(i64), P(i32), P(i64), P(i32)]),
        'bb_fastq_format_sharded': (c.c_int, [i32, vp, vp, vp, vp, i32, i64, i64, i32, vp, i64, P(i64), P(i32), P(i64), P(i32)]),
        'bb_count_kmer_alternatives': (c.c_int, [c.c_int, c.c_int, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp, P(i64),
                                                 i64, vp, vp, vp, P(i64)]),
        'bb_count_kmer_alternatives_wide': (c.c_int, [c.c_int, c.c_int, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp,
                                                      P(i64), i64, vp, vp, vp, P(i64)]),
        'bb_count_cigar_qscores': (c.c_int, [c.c_int, c.c_int, c.c_int, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp,
                                             P(i64), vp, i64, vp, vp, vp, P(i64)]),
        'bb_model_error': (c.c_char_p, []),
        'bb_bgzf_bound': (i64, [i64]),
        'bb_bgzf_compress': (c.c_int, [vp, vp, i64, c.c_int, c.c_int, vp, i64, P(i64), P(i64)]),
        'bb_bgzf_decompress': (c.c_int, [c.c_int, vp, i64, vp, i64, P(i64)]),
        'bb_gzip_decompress': (c.c_int, [c.c_int, vp, i64, vp, i64, P(i64), i64, P(GzipStats)]),
        'bb_fetch_last_batch_results': (c.c_int, [vp, vp, P(i64)]),
        'bb_bam_build': (c.c_int, [vp, i32, vp, vp, i64]),
        'bb_bam_compress_device': (c.c_int, [vp, c.c_int, vp, i64, P(i64)]),
        'bb_bam_fetch_records': (c.c_int, [vp, vp, vp, i64, P(i64)]),
        'bb_bam_compress': (c.c_int, [vp, vp, i64, i64, vp, i64, c.c_int, vp, i64, P(i64), P(i64)]),
        'bb_bam_layout_sharded': (c.c_int, [i32, vp, vp, i32, i64, i64, i64, vp, vp, vp, vp, vp, vp, i64, P(i64), P(i64),
                                            P(i32), P(i64), P(i32)]),
        'bb_aln_parse': (c.c_int, [vp, i64, c.c_int, i64, P(vp)]),
        'bb_aln_view_get': (c.c_int, [vp, P(AlnView)]),
        'bb_aln_free': (c.c_int, [vp]),
        'bb_device_count': (c.c_int, []),
        'bb_fastq_parse': (c.c_int, [c.c_int, vp, i64, c.c_int, P(vp), P(i64), P(i32)]),
        'bb_fastq_free': (c.c_int, [vp]),
        'bb_flat_build': (c.c_int, [vp, P(AlnView), i32, vp, vp, vp, vp, i64, P(vp), vp, vp]),
        'bb_flat_view_get': (c.c_int, [vp, P(FlatView)]),
        'bb_flat_fetch': (c.c_int, [vp, c.c_int, i64, i64, vp]),
        'bb_flat_free': (c.c_int, [vp]),
        'bb_window_series': (c.c_int, [c.c_int, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, c.c_int, i32, i32, vp, vp,
                                       P(i64)]),
        'bb_window_line_bound': (i64, [i64]),
        'bb_window_format': (c.c_int, [i32, vp, vp, vp, vp, vp, vp, i64, i64, vp, i64, P(i64)]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


EXPORTED_SYMBOLS = ['bb_create', 'bb_destroy', 'bb_last_error', 'bb_version', 'bb_upload_reference',
                    'bb_upload_error_model', 'bb_upload_error_model_kmers', 'bb_upload_qscore_model', 'bb_upload_qscore_model_cigars', 'bb_sequence_batch',
                    'bb_fetch_last_batch', 'bb_batch_upload', 'bb_batch_run', 'bb_synchronize', 'bb_last_run_retries',
                    'bb_last_run_work', 'bb_host_alloc', 'bb_host_free',
                    'bb_last_run_ms', 'bb_stage_name', 'bb_launch_count', 'bb_trace_dump', 'bb_get_qscores', 'bb_align_path',
                    'bb_host_align_kmers', 'bb_host_align_path', 'bb_nccl_available', 'bb_comm_unique_id', 'bb_comm_init_rank',
                    'bb_comm_init_all', 'bb_allreduce_bases', 'bb_allreduce_bases_all', 'bb_planner_create', 'bb_planner_destroy',
                    'bb_planner_plan', 'bb_planner_view', 'bb_planner_error', 'bb_fastq_format', 'bb_fastq_format_sharded',
                    'bb_count_kmer_alternatives', 'bb_count_kmer_alternatives_wide', 'bb_count_cigar_qscores', 'bb_model_error',
                    'bb_bgzf_bound', 'bb_bgzf_compress', 'bb_bgzf_decompress', 'bb_aln_parse', 'bb_aln_view_get', 'bb_aln_free',
                    'bb_fetch_last_batch_results', 'bb_bam_build', 'bb_bam_compress_device', 'bb_bam_fetch_records',
                    'bb_bam_compress', 'bb_bam_layout_sharded', 'bb_fasta_parse', 'bb_fasta_headers', 'bb_fasta_reference',
                    'bb_download_reference', 'bb_gzip_decompress', 'bb_last_gzip_stats', 'bb_device_count', 'bb_fastq_parse',
                    'bb_fastq_free', 'bb_flat_build', 'bb_flat_view_get', 'bb_flat_fetch', 'bb_flat_free', 'bb_window_series',
                    'bb_window_line_bound', 'bb_window_format', 'bb_load_error_model_file', 'bb_download_error_model']
