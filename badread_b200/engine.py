"""
Engine - Python owner of one `bb_ctx` (one GPU): uploads the reference and the model tables to HBM once and runs
`sequence_fragment` for batches of fragment descriptors through the C ABI (include/badread_b200.h).
No PyTorch, no CPU path: construction fails when the library or a GPU is missing.
"""
import ctypes
import os
import threading

import numpy as np

from . import _lib
from ._lib import BB_SEG_LITERAL, BB_SEG_REF_FWD, BB_SEG_REF_REV, ReadResult, Segment
from .misc import fasta_contigs


_RESULT_DTYPE = np.dtype([('out_off', np.int64), ('out_len', np.int32), ('frag_len', np.int32), ('matches', np.int32),
                          ('columns', np.int32), ('loop_count', np.int32), ('change_count', np.int32),
                          ('n_alignments', np.int32), ('flags', np.int32), ('loop_kcycles', np.int32),
                          ('align_kcycles', np.int32)])
assert _RESULT_DTYPE.itemsize == ctypes.sizeof(ReadResult)


class EngineError(RuntimeError):
    pass


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _host_alloc(nbytes):
    """nbytes of page-locked memory (bb_host_alloc), so that copies between it and the GPUs run at the link's rate:
    (handle for bb_host_free, uint8 array over the bytes)."""
    p = ctypes.c_void_p()
    if _lib.lib().bb_host_alloc(ctypes.byref(p), nbytes) != 0:
        raise EngineError(f'bb_host_alloc({nbytes}) failed')
    return p, np.ctypeslib.as_array((ctypes.c_uint8 * nbytes).from_address(p.value))


class FragmentBatch(object):
    """Flat fragment descriptors for a batch of reads: per read a run of segments (reference slices on either
    strand and literal bytes), the read's global index and its target identity."""

    def __init__(self):
        self.read_index = []
        self.target_identity = []
        self.seg_off = [0]
        self.seg_src, self.seg_len, self.seg_kind = [], [], []
        self.literals = bytearray()

    def __len__(self):
        return len(self.read_index)

    def add_literal_segment(self, data):
        if isinstance(data, str):
            data = data.encode('latin-1')
        self.seg_src.append(len(self.literals))
        self.seg_len.append(len(data))
        self.seg_kind.append(BB_SEG_LITERAL)
        self.literals += data

    def add_ref_segment(self, src, length, reverse):
        self.seg_src.append(int(src))
        self.seg_len.append(int(length))
        self.seg_kind.append(BB_SEG_REF_REV if reverse else BB_SEG_REF_FWD)

    def end_read(self, read_index, target_identity):
        self.read_index.append(int(read_index))
        self.target_identity.append(float(target_identity))
        self.seg_off.append(len(self.seg_src))

    def add_literal_read(self, read_index, fragment, target_identity):
        self.add_literal_segment(fragment)
        self.end_read(read_index, target_identity)

    def frag_bases(self):
        return sum(self.seg_len)

    def arrays(self):
        """The flat descriptor arrays bb_batch_upload takes (built once per batch state)."""
        key = (len(self.read_index), len(self.seg_src), len(self.literals))
        cached = getattr(self, '_arrays', None)
        if cached is not None and cached[0] == key:
            return cached[1]
        out = self._build_arrays()
        self._arrays = (key, out)
        return out

    def _build_arrays(self):
        n_seg = len(self.seg_src)
        segs = (Segment * max(n_seg, 1))()
        seg_np = np.frombuffer(segs, dtype=np.dtype([('src', np.int64), ('len', np.int32), ('kind', np.int32)]))
        if n_seg:
            seg_np['src'][:n_seg] = self.seg_src
            seg_np['len'][:n_seg] = self.seg_len
            seg_np['kind'][:n_seg] = self.seg_kind
        lit = np.frombuffer(bytes(self.literals), dtype=np.uint8) if self.literals else np.zeros(1, dtype=np.uint8)
        return (np.asarray(self.read_index, dtype=np.uint64), np.asarray(self.seg_off, dtype=np.int32), segs,
                np.ascontiguousarray(lit), len(self.literals), np.asarray(self.target_identity, dtype=np.float64))


class FastaFile(object):
    """The bytes of a FASTA file as Engine.load_fasta takes them, read once for all the engines: the file as it is, in
    page-locked memory (bb_host_alloc) so that it goes to the GPUs at the link's rate.  A gzip file, BGZF or not, is
    inflated on the GPUs.  close() releases the memory."""

    def __init__(self, filename):
        self._lib = _lib.lib()
        self._pinned = None
        with open(filename, 'rb') as f:
            self.gzip = f.read(2) == b'\x1f\x8b'
        size = os.path.getsize(filename)
        self._pinned, data = _host_alloc(max(size, 1))
        self.data = data[:size]
        view, got = memoryview(self.data), 0
        with open(filename, 'rb', buffering=0) as f:
            while got < size:
                n = f.readinto(view[got:got + (1 << 30)])
                if not n:
                    raise EngineError(f'{filename}: file shrank while being read')
                got += n

    def close(self):
        self.data = None
        if self._pinned is not None:
            self._lib.bb_host_free(self._pinned)
            self._pinned = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchResult(object):
    def __init__(self, results, seq, qual, n):
        self.records = results
        self.seq = seq
        self.qual = qual
        self.n = n

    def read(self, i):
        r = self.records[i]
        s = bytes(self.seq[r.out_off:r.out_off + r.out_len]).decode('latin-1')
        q = bytes(self.qual[r.out_off:r.out_off + r.out_len]).decode('latin-1')
        return s, q

    def identity(self, i):
        r = self.records[i]
        return r.matches / r.columns if r.columns else 0.0

    def table(self):
        """The records as a numpy structured array (no copy)."""
        return np.frombuffer(self.records, dtype=_RESULT_DTYPE, count=self.n)

    def total_bases(self):
        return int(self.table()['out_len'].sum()) if self.n else 0


class Engine(object):

    def __init__(self, device=0, seed=0):
        self._lib = _lib.lib()
        self._ctx = ctypes.c_void_p()
        rc = self._lib.bb_create(ctypes.byref(self._ctx), int(device), ctypes.c_uint64(int(seed) & (2 ** 64 - 1)))
        if rc != 0:
            msg = self._lib.bb_last_error(None)
            self._ctx = None
            raise EngineError(f'bb_create failed ({rc}): {msg.decode() if msg else ""}')
        self.device = device
        self.seed = seed
        self.error_model = None
        self.qscore_model = None
        self._out_cap = 0
        self._seq_buf = self._qual_buf = None
        self._pinned = []
        self._bgzf_buf = None

    def close(self):
        if getattr(self, '_ctx', None):
            self._free_out()
            self._lib.bb_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            msg = self._lib.bb_last_error(self._ctx)
            raise EngineError(f'{what} failed ({rc}): {msg.decode() if msg else ""}')

    # ---- uploads
    def upload_reference(self, bases):
        arr = np.frombuffer(bases, dtype=np.uint8) if isinstance(bases, (bytes, bytearray)) else np.ascontiguousarray(bases, dtype=np.uint8)
        self._ref_keepalive = arr
        self._check(self._lib.bb_upload_reference(self._ctx, _ptr(arr), arr.size), 'bb_upload_reference')

    def load_fasta(self, fasta):
        """Makes the reference of this GPU a FASTA file parsed on the GPU (bb_fasta_parse / bb_fasta_headers /
        bb_fasta_reference) in place of upload_reference: the contigs that misc.load_fasta_arrays would give, concatenated,
        without the bases ever being on the host.  fasta: a FastaFile, or a file name.  Returns (names, lengths, depths,
        circular, hairpin_left, hairpin_right), the last four dicts by name as misc.fasta_contigs gives them."""
        own = not isinstance(fasta, FastaFile)
        if own:
            fasta = FastaFile(fasta)
        try:
            n_hdr, n_text, n_kept = ctypes.c_int32(0), ctypes.c_int64(0), ctypes.c_int64(0)
            data = fasta.data
            self._check(self._lib.bb_fasta_parse(self._ctx, _ptr(data) if data.size else None, data.size, int(fasta.gzip),
                                                 ctypes.byref(n_hdr), ctypes.byref(n_text), ctypes.byref(n_kept)),
                        'bb_fasta_parse')
        finally:
            if own:
                fasta.close()
        nh = n_hdr.value
        text = ctypes.create_string_buffer(max(n_text.value, 1))
        text_off = np.zeros(nh + 1, dtype=np.int64)
        kept_off = np.zeros(nh + 1, dtype=np.int64)
        self._check(self._lib.bb_fasta_headers(self._ctx, text, n_text.value, _ptr(text_off), _ptr(kept_off), nh),
                    'bb_fasta_headers')
        raw = text.raw
        headers = [(raw[text_off[k]:text_off[k + 1]].decode('latin-1'), (int(kept_off[k]), int(kept_off[k + 1])))
                   for k in range(nh)]
        names, ranges, depths, circular, hp_left, hp_right = fasta_contigs(headers)
        lo = np.asarray([r[0] for r in ranges] or [0], dtype=np.int64)
        hi = np.asarray([r[1] for r in ranges] or [0], dtype=np.int64)
        self._check(self._lib.bb_fasta_reference(self._ctx, len(ranges), _ptr(lo), _ptr(hi)), 'bb_fasta_reference')
        return names, [b - a for a, b in ranges], depths, circular, hp_left, hp_right

    def last_gzip_stats(self):
        """How the last load_fasta inflated its file (bb_last_gzip_stats), as a dict: all zero for plain text."""
        st = _lib.GzipStats()
        self._check(self._lib.bb_last_gzip_stats(self._ctx, ctypes.byref(st)), 'bb_last_gzip_stats')
        return st.as_dict()

    def download_reference(self, offset=0, n=None):
        """Bytes [offset, offset + n) of this GPU's reference (all from offset when n is None; the length is known to the
        caller, who loaded it) as a uint8 array."""
        out = np.zeros(max(int(n), 1), dtype=np.uint8)
        self._check(self._lib.bb_download_reference(self._ctx, int(offset), int(n), _ptr(out)), 'bb_download_reference')
        return out[:int(n)]

    def set_error_model(self, error_model, index='auto'):
        """index: how the device finds a k-mer's row.  'auto': the dense kmer_to_row[4^k] when the model has one
        (k <= 12), else a hash table of the rows' k-mers; 'hash': the hash table for any k (same reads, for tests and
        measurement)."""
        if index not in ('auto', 'hash'):
            raise ValueError(f"index must be 'auto' or 'hash', not {index!r}")
        t = error_model.to_device_tables()
        if t['type'] == 0:
            rc = self._lib.bb_upload_error_model(self._ctx, 1, 0, None, 0, 0, None, None, None, None, None, 0)
            name = 'bb_upload_error_model'
        elif index == 'auto' and t['index'] == 'dense':
            rc = self._lib.bb_upload_error_model(self._ctx, t['k'], 1, _ptr(t['kmer_to_row']), t['kmer_to_row'].size,
                                                 len(t['row_off']) - 1, _ptr(t['row_off']), _ptr(t['cum']),
                                                 _ptr(t['flags']), _ptr(t['slots']), _ptr(t['pool']), t['pool'].size)
            name = 'bb_upload_error_model'
        else:
            codes = np.ascontiguousarray(t['kmer_codes'], dtype=np.int64)
            rc = self._lib.bb_upload_error_model_kmers(self._ctx, t['k'], len(t['row_off']) - 1, _ptr(codes),
                                                       _ptr(t['row_off']), _ptr(t['cum']), _ptr(t['flags']),
                                                       _ptr(t['slots']), _ptr(t['pool']), t['pool'].size)
            name = 'bb_upload_error_model_kmers'
        self._check(rc, name)
        self.error_model = error_model

    def set_qscore_model(self, qscore_model):
        t = qscore_model.to_device_tables()
        rc = self._lib.bb_upload_qscore_model_cigars(self._ctx, t['kmer_size'], t['n_keys'], _ptr(t['key_chars']),
                                                     _ptr(t['key_off']), _ptr(t['row_off']), _ptr(t['scores']),
                                                     _ptr(t['cum']))
        self._check(rc, 'bb_upload_qscore_model_cigars')
        self.qscore_model = qscore_model

    # ---- batch
    def _ensure_out(self, cap):
        if cap > self._out_cap:
            cap = int(cap * 1.25) + 4096
            # earlier (smaller) buffers stay allocated until close(): BatchResults handed out before still view them
            bufs = []
            for _ in range(2):
                p, buf = _host_alloc(cap)
                self._pinned.append(p)
                bufs.append(buf)
            self._seq_buf, self._qual_buf = bufs
            self._out_cap = cap

    def _free_out(self):
        self._seq_buf = self._qual_buf = self._bgzf_buf = None
        self._out_cap = 0
        for p in self._pinned:
            self._lib.bb_host_free(p)
        self._pinned = []

    def upload_batch(self, batch):
        ri, so, segs, lit, lit_len, ti = batch.arrays()
        self._batch_keepalive = (ri, so, segs, lit, ti)
        self._n = len(batch)
        rc = self._lib.bb_batch_upload(self._ctx, self._n, _ptr(ri), _ptr(so), ctypes.cast(segs, ctypes.c_void_p),
                                       _ptr(lit), lit_len, _ptr(ti))
        self._check(rc, 'bb_batch_upload')

    def run_batch(self):
        self._check(self._lib.bb_batch_run(self._ctx), 'bb_batch_run')

    def synchronize(self):
        self._check(self._lib.bb_synchronize(self._ctx), 'bb_synchronize')

    def last_run_ms(self):
        total = ctypes.c_float(0)
        stages = (ctypes.c_float * _lib.BB_N_STAGES)()
        self._check(self._lib.bb_last_run_ms(self._ctx, ctypes.byref(total), stages), 'bb_last_run_ms')
        names = [self._lib.bb_stage_name(i).decode() for i in range(_lib.BB_N_STAGES)]
        return total.value, dict(zip(names, [float(x) for x in stages]))

    def last_run_retries(self):
        """(re-runs, reason bits) of the last batch: how often a fetch had to run it again because a limit sized from
        the fragment lengths was too small, summed over the workers, and the _lib.BB_RERUN_* bits of those limits."""
        n = ctypes.c_int32(0)
        reasons = ctypes.c_uint32(0)
        self._check(self._lib.bb_last_run_retries(self._ctx, ctypes.byref(n), ctypes.byref(reasons)), 'bb_last_run_retries')
        return int(n.value), int(reasons.value)

    def last_run_work(self):
        """Which alignment kernels the last batch's final run gave work to (bb_last_run_work), summed over the workers:
        window alignments per kernel ('window_lane4', 'window_lane8', 'window_warp'), Hirschberg leaves per kernel
        ('leaf_lane', 'leaf_warp', and 'root_leaf_lane' / 'root_leaf_warp' of them that were whole reads), and
        'levels': for every level the run enqueued, the nodes queued for it per node class, in _lib.NODE_CLASSES
        order.  Available once the batch has been fetched."""
        work = np.zeros(len(_lib.WORK_SLOTS), dtype=np.int64)
        levels = np.zeros((_lib.BB_MAX_LEVELS, len(_lib.NODE_CLASSES)), dtype=np.int64)
        n = ctypes.c_int32(0)
        self._check(self._lib.bb_last_run_work(self._ctx, _ptr(work), _ptr(levels), _lib.BB_MAX_LEVELS, ctypes.byref(n)),
                    'bb_last_run_work')
        out = {name: int(v) for name, v in zip(_lib.WORK_SLOTS, work)}
        out['levels'] = [[int(x) for x in row] for row in levels[:n.value]]
        return out

    def launch_count(self):
        return int(self._lib.bb_launch_count(self._ctx))

    def trace_dump(self, path):
        """Timeline of the last run (needs BADREAD_B200_TRACE=1 in the environment before the Engine is created)."""
        self._check(self._lib.bb_trace_dump(self._ctx, str(path).encode()), 'bb_trace_dump')

    def fetch_batch(self):
        n = self._n
        results = (ReadResult * n)()
        total = ctypes.c_int64(0)
        rc = self._lib.bb_fetch_last_batch(self._ctx, results, _ptr(self._seq_buf) if self._seq_buf is not None else None,
                                           _ptr(self._qual_buf) if self._qual_buf is not None else None,
                                           self._out_cap, ctypes.byref(total))
        if rc == _lib.BB_ERR_CAPACITY:
            self._ensure_out(total.value)
            rc = self._lib.bb_fetch_last_batch(self._ctx, results, _ptr(self._seq_buf), _ptr(self._qual_buf),
                                               self._out_cap, ctypes.byref(total))
        self._check(rc, 'bb_fetch_last_batch')
        return BatchResult(results, self._seq_buf, self._qual_buf, n), int(total.value)

    def sequence_batch(self, batch):
        """bb_sequence_batch (upload + run + fetch in one call: with several workers each block is copied out while
        the other workers still compute); returns (BatchResult, total_bases)."""
        ri, so, segs, lit, lit_len, ti = batch.arrays()
        self._batch_keepalive = (ri, so, segs, lit, ti)
        self._n = n = len(batch)
        if self._seq_buf is None:
            self._ensure_out(int(1.1 * batch.frag_bases()) + 4096)
        results = (ReadResult * n)()
        total = ctypes.c_int64(0)
        rc = self._lib.bb_sequence_batch(self._ctx, n, _ptr(ri), _ptr(so), ctypes.cast(segs, ctypes.c_void_p), _ptr(lit),
                                         lit_len, _ptr(ti), results, _ptr(self._seq_buf), _ptr(self._qual_buf),
                                         self._out_cap, ctypes.byref(total))
        if rc == _lib.BB_ERR_CAPACITY:
            self._ensure_out(total.value)
            rc = self._lib.bb_fetch_last_batch(self._ctx, results, _ptr(self._seq_buf), _ptr(self._qual_buf),
                                               self._out_cap, ctypes.byref(total))
        self._check(rc, 'bb_sequence_batch')
        return BatchResult(results, self._seq_buf, self._qual_buf, n), int(total.value)

    # ---- BGZF output
    def bgzf_compress(self, buf, line_mod4=0, final=False):
        """BGZF members of FASTQ text on this GPU (bb_bgzf_compress): buf is any bytes-like object, line_mod4 the index
        mod 4 of the FASTQ line its first byte belongs to.  Without `final` only the whole chunks of _lib.BB_BGZF_CHUNK bytes
        are compressed.  Returns (members, bytes of buf consumed); members is a uint8 array in page-locked memory that the
        next call reuses.  The end-of-file member is not included (badread_b200.bgzf.EOF_MEMBER)."""
        data = np.frombuffer(buf, dtype=np.uint8)
        buf_out = self._members_buf(int(self._lib.bb_bgzf_bound(data.size)))
        n_out, n_used = ctypes.c_int64(0), ctypes.c_int64(0)
        rc = self._lib.bb_bgzf_compress(self._ctx, _ptr(data) if data.size else None, data.size, int(line_mod4), int(bool(final)),
                                        _ptr(buf_out), buf_out.size, ctypes.byref(n_out), ctypes.byref(n_used))
        self._check(rc, 'bb_bgzf_compress')
        return buf_out[:n_out.value], int(n_used.value)

    # ---- BAM output (badread_b200/bam.py)
    def run_batch_results(self, batch):
        """Uploads, runs and fetches a batch like sequence_batch, but leaves the bases and qualities on the device for
        bam_build (bb_fetch_last_batch_results); returns (BatchResult without seq / qual, total_bases)."""
        self.upload_batch(batch)
        self.run_batch()
        n = self._n
        results = (ReadResult * n)()
        total = ctypes.c_int64(0)
        self._check(self._lib.bb_fetch_last_batch_results(self._ctx, results, ctypes.byref(total)), 'bb_fetch_last_batch_results')
        return BatchResult(results, None, None, n), int(total.value)

    def bam_build(self, recs, text):
        """Appends BAM records of the last batch to this GPU's record stream (bb_bam_build): recs is an array of
        planner.BAM_RECORD_DTYPE, text the pool their text_off index."""
        recs = np.ascontiguousarray(recs)
        text = np.ascontiguousarray(np.frombuffer(text, dtype=np.uint8) if isinstance(text, (bytes, bytearray)) else text)
        self._check(self._lib.bb_bam_build(self._ctx, len(recs), _ptr(recs) if len(recs) else None,
                                           _ptr(text) if text.size else None, text.size), 'bb_bam_build')

    def _members_buf(self, need):
        """The page-locked buffer the compressors write members to, grown to at least `need` bytes."""
        if self._bgzf_buf is None or self._bgzf_buf.size < need:
            p, self._bgzf_buf = _host_alloc(max(need + need // 8, 1 << 20))
            self._pinned.append(p)
        return self._bgzf_buf

    def bam_compress_device(self, final=False):
        """BGZF members of the whole chunks of the record stream (all of it with `final`); the rest stays on the device.
        Returns a uint8 array in page-locked memory that the next call reuses."""
        n_out = ctypes.c_int64(0)
        buf = self._bgzf_buf
        rc = self._lib.bb_bam_compress_device(self._ctx, int(bool(final)), _ptr(buf) if buf is not None else None,
                                              buf.size if buf is not None else 0, ctypes.byref(n_out))
        if rc == _lib.BB_ERR_CAPACITY:
            buf = self._members_buf(n_out.value)
            rc = self._lib.bb_bam_compress_device(self._ctx, int(bool(final)), _ptr(buf), buf.size, ctypes.byref(n_out))
        self._check(rc, 'bb_bam_compress_device')
        return buf[:n_out.value] if n_out.value else np.zeros(0, np.uint8)

    def bam_fetch_records(self, out, dst_off=None):
        """Copies the records of the last bam_build into the uint8 array out (record i at dst_off[i], or back to back) and
        takes them off the record stream; returns their size in bytes."""
        n = ctypes.c_int64(0)
        off = np.ascontiguousarray(dst_off, dtype=np.int64) if dst_off is not None else None
        self._check(self._lib.bb_bam_fetch_records(self._ctx, _ptr(off) if off is not None and off.size else None,
                                                   _ptr(out) if out.size else None, out.size, ctypes.byref(n)),
                    'bb_bam_fetch_records')
        return int(n.value)

    def bam_compress(self, buf, stream_base, fields, final=False):
        """BGZF members of host bytes of a record stream (bb_bam_compress): buf starts at byte stream_base of the stream,
        fields is an (n, 2) int64 array of the (stream offset, length) of its seq and qual fields.  Returns (members, bytes
        of buf consumed) like bgzf_compress."""
        data = np.frombuffer(buf, dtype=np.uint8)
        f = np.ascontiguousarray(fields, dtype=np.int64).reshape(-1, 2)
        buf_out = self._members_buf(int(self._lib.bb_bgzf_bound(data.size)))
        n_out, n_used = ctypes.c_int64(0), ctypes.c_int64(0)
        rc = self._lib.bb_bam_compress(self._ctx, _ptr(data) if data.size else None, data.size, int(stream_base),
                                       _ptr(f) if len(f) else None, len(f), int(bool(final)), _ptr(buf_out), buf_out.size,
                                       ctypes.byref(n_out), ctypes.byref(n_used))
        self._check(rc, 'bb_bam_compress')
        return buf_out[:n_out.value], int(n_used.value)

    # ---- the one collective: SUM of emitted bases over the GPUs (stop condition, simulate.py:63)
    def comm_init_rank(self, unique_id, rank, world):
        """One process per GPU: joins the NCCL communicator identified by `unique_id` (128 bytes from
        `comm_unique_id()` on rank 0, shipped to the other ranks by the host program)."""
        buf = ctypes.create_string_buffer(bytes(unique_id), 128)
        self._check(self._lib.bb_comm_init_rank(self._ctx, buf, int(rank), int(world)), 'bb_comm_init_rank')

    def allreduce_bases(self, local):
        total = ctypes.c_int64(0)
        self._check(self._lib.bb_allreduce_bases(self._ctx, int(local), ctypes.byref(total)), 'bb_allreduce_bases')
        return int(total.value)

    # ---- single pair helpers
    def get_qscores(self, seq, frag, read_index=0):
        s = np.frombuffer(seq.encode('latin-1'), dtype=np.uint8)
        f = np.frombuffer(frag.encode('latin-1'), dtype=np.uint8)
        qual = np.empty(len(s), dtype=np.uint8)
        m, c = ctypes.c_int32(0), ctypes.c_int32(0)
        rc = self._lib.bb_get_qscores(self._ctx, ctypes.c_uint64(read_index), _ptr(s), len(s), _ptr(f), len(f), _ptr(qual),
                                      ctypes.byref(m), ctypes.byref(c))
        self._check(rc, 'bb_get_qscores')
        return bytes(qual).decode('latin-1'), m.value, c.value

    def align_path(self, query, target):
        """edlib.align(query, target, task='path') on the GPU -> (expanded ops string, edit distance)."""
        q = np.frombuffer(query.encode('latin-1') if isinstance(query, str) else bytes(query), dtype=np.uint8)
        t = np.frombuffer(target.encode('latin-1') if isinstance(target, str) else bytes(target), dtype=np.uint8)
        ops = np.empty(len(q) + len(t) + 16, dtype=np.uint8)
        n_ops, dist = ctypes.c_int64(0), ctypes.c_int32(0)
        rc = self._lib.bb_align_path(self._ctx, _ptr(q), len(q), _ptr(t), len(t), _ptr(ops), ops.size,
                                     ctypes.byref(n_ops), ctypes.byref(dist))
        self._check(rc, 'bb_align_path')
        return bytes(ops[:n_ops.value]).decode('ascii'), dist.value


def nccl_available():
    return bool(_lib.lib().bb_nccl_available())


def comm_unique_id():
    """128 bytes identifying a new NCCL communicator (ncclGetUniqueId)."""
    buf = ctypes.create_string_buffer(128)
    rc = _lib.lib().bb_comm_unique_id(buf)
    if rc != 0:
        raise EngineError(f'bb_comm_unique_id failed ({rc}): NCCL not available')
    return buf.raw


def comm_init_all(engines):
    """One process, several GPUs: one communicator over the engines' devices."""
    arr = (ctypes.c_void_p * len(engines))(*[e._ctx for e in engines])
    rc = _lib.lib().bb_comm_init_all(arr, len(engines))
    if rc != 0:
        msg = _lib.lib().bb_last_error(engines[0]._ctx)
        raise EngineError(f'bb_comm_init_all failed ({rc}): {msg.decode() if msg else ""}')


def run_each(n, work):
    """work(k) for k < n, one host thread each when n > 1 (inline when n == 1).  Every call finishes before the exception
    of the lowest k that raised one is re-raised on the caller's thread."""
    errors = [None] * n

    def run(k):
        try:
            work(k)
        except BaseException as e:
            errors[k] = e

    if n == 1:
        run(0)
    else:
        threads = [threading.Thread(target=run, args=(k,)) for k in range(n)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    for e in errors:
        if e is not None:
            raise e


def allreduce_bases_all(engines, local):
    """SUM of the engines' emitted-base counts through one NCCL group call."""
    arr = (ctypes.c_void_p * len(engines))(*[e._ctx for e in engines])
    loc = (ctypes.c_int64 * len(engines))(*[int(x) for x in local])
    total = ctypes.c_int64(0)
    rc = _lib.lib().bb_allreduce_bases_all(arr, len(engines), loc, ctypes.byref(total))
    if rc != 0:
        msg = _lib.lib().bb_last_error(engines[0]._ctx)
        raise EngineError(f'bb_allreduce_bases_all failed ({rc}): {msg.decode() if msg else ""}')
    return int(total.value)


# ---- module-level default engine for the single-read convenience functions ---------------------------
_default = {'engine': None, 'seed': None, 'next_read': 0}


def set_seed(seed):
    """Seed of the per-read Philox streams used by the module-level convenience functions."""
    _default['seed'] = seed
    _default['next_read'] = 0
    if _default['engine'] is not None:
        _default['engine'].close()
        _default['engine'] = None


def default_engine(error_model=None, qscore_model=None):
    if _default['engine'] is None:
        seed = _default['seed']
        if seed is None:
            seed = int.from_bytes(os.urandom(8), 'little')
            _default['seed'] = seed
        _default['engine'] = Engine(device=int(os.environ.get('BADREAD_B200_DEVICE', '0')), seed=seed)
    eng = _default['engine']
    if error_model is not None and eng.error_model is not error_model:
        eng.set_error_model(error_model)
    if qscore_model is not None and eng.qscore_model is not qscore_model:
        eng.set_qscore_model(qscore_model)
    return eng


def next_read_index():
    i = _default['next_read']
    _default['next_read'] = i + 1
    return i
