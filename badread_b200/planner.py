"""
planner - the fragment builder and the FASTQ assembly as native host code (csrc/bb_planner.cpp) behind the C ABI.

`NativePlanner` is what `simulate()` and bench.py use: it plans whole batches of reads (build_fragment and friends,
/root/reference/badread/simulate.py:91-253,361-394,459-482; fragment lengths and identities) on all host threads and
hands the resulting descriptor arrays to `Engine` without touching them from Python.  Its per-read random streams
and every draw are identical to `simulate.ReadPlanner` (the readable Python statement of the same planner, kept as
the pin for tests/test_planner.py).
"""
import ctypes
import os
import sys

import numpy as np

from . import _lib, settings
from ._lib import PlanConfig, PlanView, ReadResult, Segment

_SEG_DTYPE = np.dtype([('src', np.int64), ('len', np.int32), ('kind', np.int32)])


def _as_array(ptr, n, ctype):
    if n <= 0 or not ptr:
        return np.zeros(0, dtype=np.dtype(ctype))
    return np.ctypeslib.as_array((ctype * n).from_address(ptr))


class PlannedBatch(object):
    """The last plan of a NativePlanner as zero-copy numpy views (valid until the planner plans again)."""

    def __init__(self, view, keepalive):
        self.view = view
        self._keepalive = keepalive
        n = view.n_reads
        self.n = n
        self.read_index = _as_array(view.read_index, n, ctypes.c_uint64)
        self.seg_off = _as_array(view.seg_off, n + 1, ctypes.c_int32)
        n_seg = int(self.seg_off[n]) if n else 0
        self.segs = np.frombuffer((ctypes.c_uint8 * (16 * n_seg)).from_address(view.segs), dtype=_SEG_DTYPE) if n_seg else \
            np.zeros(0, dtype=_SEG_DTYPE)
        self.literal_len = int(view.literal_len)
        self.literals = _as_array(view.literals, max(self.literal_len, 1), ctypes.c_uint8)
        self.target_identity = _as_array(view.target_identity, n, ctypes.c_double)
        self.names = _as_array(view.read_names, 16 * n, ctypes.c_uint8).reshape(n, 16) if n else np.zeros((0, 16), np.uint8)
        self.info_off = _as_array(view.info_off, n + 1, ctypes.c_int64)
        self.info = _as_array(view.info, int(self.info_off[n]) if n else 0, ctypes.c_uint8)
        self.frag_len = _as_array(view.frag_len, n, ctypes.c_int32)

    def __len__(self):
        return self.n

    def detach(self):
        """A copy that owns its arrays (the planner can plan the next batch while this one is still in use)."""
        own = {k: np.array(getattr(self, k), copy=True) for k in ('read_index', 'seg_off', 'segs', 'literals',
                                                                  'target_identity', 'names', 'info_off', 'info', 'frag_len')}
        v = PlanView()
        v.n_reads = self.n
        v.literal_len = self.literal_len
        for field, key in (('read_index', 'read_index'), ('seg_off', 'seg_off'), ('segs', 'segs'), ('literals', 'literals'),
                           ('target_identity', 'target_identity'), ('read_names', 'names'), ('info_off', 'info_off'),
                           ('info', 'info'), ('frag_len', 'frag_len')):
            setattr(v, field, own[key].ctypes.data if own[key].size else None)
        return PlannedBatch(v, own)

    def arrays(self):
        """(read_index, seg_off, segs, literals, literal_len, target_identity) as bb_batch_upload takes them."""
        return (self.read_index, self.seg_off, ctypes.c_void_p(self.view.segs), self.literals, self.literal_len,
                self.target_identity)

    def frag_bases(self):
        return int(self.frag_len.sum())

    def h2d_bytes(self):
        return int(self.read_index.nbytes + self.seg_off.nbytes + self.segs.nbytes + self.literal_len +
                   self.target_identity.nbytes)

    def info_str(self, i):
        return bytes(self.info[self.info_off[i]:self.info_off[i + 1]]).decode('latin-1')

    def name_str(self, i):
        h = bytes(self.names[i]).hex()
        return f'{h[:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:]}'

    def fragment(self, i, ref_concat):
        """The fragment of read i as a str (tests and the oracle-side checks; the GPU gathers it itself)."""
        from .misc import reverse_complement
        out = []
        for s in self.segs[self.seg_off[i]:self.seg_off[i + 1]]:
            src, ln, kind = int(s['src']), int(s['len']), int(s['kind'])
            if kind == _lib.BB_SEG_LITERAL:
                out.append(bytes(self.literals[src:src + ln]))
            elif kind == _lib.BB_SEG_REF_FWD:
                out.append(ref_concat[src:src + ln].tobytes())
            else:
                out.append(reverse_complement(ref_concat[src:src + ln].tobytes()))
        return b''.join(out).decode('latin-1')


class NativePlanner(object):

    def __init__(self, args, ref, frag_lengths, identities, seed, n_threads=None):
        from .simulate import adapter_parameters
        self._lib = _lib.lib()
        self.ref = ref
        self.n_threads = int(n_threads or os.cpu_count() or 1)
        start_rate, start_amount = adapter_parameters(args.start_adapter)
        end_rate, end_amount = adapter_parameters(args.end_adapter)
        n = len(ref.names)
        self._len = np.asarray(ref.lengths, dtype=np.int64)
        self._weight = np.asarray([d * l for d, l in zip(ref.depths, ref.lengths)], dtype=np.float64)
        self._flags = np.asarray([(1 if ref.circular[i] else 0) | (2 if ref.left_hairpin[i] else 0) |
                                  (4 if ref.right_hairpin[i] else 0) for i in range(n)], dtype=np.uint8)
        names = [nm.encode('latin-1') for nm in ref.names]
        self._names = b''.join(names)
        self._name_off = np.concatenate([[0], np.cumsum([len(x) for x in names])]).astype(np.int64)
        self._start = (args.start_adapter_seq or '').encode('latin-1')
        self._end = (args.end_adapter_seq or '').encode('latin-1')
        c = PlanConfig()
        c.seed = int(seed) & (2 ** 64 - 1)
        c.n_contigs = n
        c.contig_len = self._len.ctypes.data
        c.contig_weight = self._weight.ctypes.data
        c.contig_flags = self._flags.ctypes.data
        c.contig_names = self._names
        c.contig_name_off = self._name_off.ctypes.data
        c.frag_mean = float(frag_lengths.mean)
        c.frag_stdev = float(frag_lengths.stdev)
        c.gamma_k = float(frag_lengths.gamma_k or 0.0)
        c.gamma_t = float(frag_lengths.gamma_t or 0.0)
        c.identity_type = 0 if identities.type == 'beta' else 1
        c.id_mean = float(identities.mean)
        c.id_stdev = float(identities.stdev)
        c.id_max = float(identities.max_identity if identities.max_identity is not None else 0.0)
        c.beta_a = float(identities.beta_a or 0.0)
        c.beta_b = float(identities.beta_b or 0.0)
        c.start_adapter, c.start_adapter_len = self._start, len(self._start)
        c.start_adapter_rate, c.start_adapter_amount = start_rate, start_amount
        c.end_adapter, c.end_adapter_len = self._end, len(self._end)
        c.end_adapter_rate, c.end_adapter_amount = end_rate, end_amount
        c.junk_rate, c.random_rate = args.junk_reads / 100, args.random_reads / 100
        c.chimera_rate = args.chimeras / 100
        c.chimera_end_adapter_chance = settings.CHIMERA_END_ADAPTER_CHANCE
        c.chimera_start_adapter_chance = settings.CHIMERA_START_ADAPTER_CHANCE
        c.glitch_rate, c.glitch_size, c.glitch_skip = float(args.glitch_rate), float(args.glitch_size), float(args.glitch_skip)
        self._cfg = c
        self._h = ctypes.c_void_p()
        rc = self._lib.bb_planner_create(ctypes.byref(self._h), ctypes.byref(c))
        if rc != 0:
            raise RuntimeError(f'bb_planner_create failed ({rc})')

    def close(self):
        if getattr(self, '_h', None):
            self._lib.bb_planner_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def plan(self, first_index, n_reads, stride=1):
        """Plans reads first_index, first_index + stride, ...; returns a PlannedBatch (views into the planner)."""
        rc = self._lib.bb_planner_plan(self._h, ctypes.c_uint64(first_index), ctypes.c_uint64(stride), int(n_reads),
                                       self.n_threads)
        if rc == _lib.BB_ERR_STATE:
            sys.exit(self._lib.bb_planner_error(self._h).decode())
        if rc != 0:
            raise RuntimeError(f'bb_planner_plan failed ({rc}): {self._lib.bb_planner_error(self._h).decode()}')
        v = PlanView()
        self._lib.bb_planner_view(self._h, ctypes.byref(v))
        return PlannedBatch(v, self)


def fastq_format(planned, results, seq_buf, qual_buf, first, bases_so_far, target_bases, n_threads=None, out=None):
    """bb_fastq_format: FASTQ records (simulate.py:70-86) of reads [first, n) of a finished batch.
    Returns (buffer view of the records, n_emitted, bases_emitted, next_read, out_buffer)."""
    return fastq_format_sharded([planned], [results], [seq_buf], [qual_buf], first, bases_so_far, target_bases,
                                n_threads=n_threads, out=out)


def fastq_format_sharded(planned, results, seq_bufs, qual_bufs, first, bases_so_far, target_bases, n_threads=None,
                         out=None):
    """bb_fastq_format_sharded: the batch was dealt out over len(planned) GPUs (read j -> shard j % G)."""
    L = _lib.lib()
    G = len(planned)
    n_threads = int(n_threads or os.cpu_count() or 1)
    views = (ctypes.c_void_p * G)(*[ctypes.addressof(p.view) for p in planned])
    res = (ctypes.c_void_p * G)(*[ctypes.addressof(r) for r in results])
    seqs = (ctypes.c_void_p * G)(*[b.ctypes.data for b in seq_bufs])
    quals = (ctypes.c_void_p * G)(*[b.ctypes.data for b in qual_bufs])
    need, n_emit, bases, nxt = ctypes.c_int64(0), ctypes.c_int32(0), ctypes.c_int64(0), ctypes.c_int32(0)

    def call(o):
        return L.bb_fastq_format_sharded(G, views, res, seqs, quals, int(first), int(bases_so_far), int(target_bases),
                                         n_threads, o.ctypes.data_as(ctypes.c_void_p) if o is not None else None,
                                         o.size if o is not None else 0, ctypes.byref(need), ctypes.byref(n_emit),
                                         ctypes.byref(bases), ctypes.byref(nxt))
    rc = call(out)
    if rc == _lib.BB_ERR_CAPACITY:
        out = np.empty(int(need.value * 1.1) + 4096, dtype=np.uint8)
        rc = call(out)
    if rc != 0:
        raise RuntimeError(f'bb_fastq_format_sharded failed ({rc})')
    return (out[:need.value] if out is not None else np.zeros(0, np.uint8)), n_emit.value, bases.value, nxt.value, out


BAM_RECORD_DTYPE = np.dtype([('out_off', np.int64), ('text_off', np.int64), ('out_len', np.int32), ('name_len', np.int32),
                             ('co_len', np.int32), ('reserved', np.int32)])
assert BAM_RECORD_DTYPE.itemsize == ctypes.sizeof(_lib.BamRecord)


class BamLayout(object):
    """bb_bam_layout_sharded: where the BAM records of a batch's emitted reads go.  Per emitted record e: shard[e] and
    index[e] (the read's shard and position in that shard's results), stream_off[e] (its offset in the record stream),
    recs[e] (a bb_bam_record, text_off into text) and fields[2 e], fields[2 e + 1] (stream offset, length) of its seq and
    qual field.  stream_len: bytes of the records."""

    def __init__(self, shard, index, stream_off, recs, fields, text, stream_len, n_emitted, bases, next_read):
        self.shard, self.index, self.stream_off, self.recs, self.fields, self.text = shard, index, stream_off, recs, fields, text
        self.stream_len, self.n_emitted, self.bases, self.next_read = stream_len, n_emitted, bases, next_read


def bam_layout_sharded(planned, results, first, bases_so_far, target_bases, stream_base=0):
    """The BAM records (bb_bam_build) of the reads fastq_format_sharded would emit for the same arguments."""
    L = _lib.lib()
    G = len(planned)
    n = sum(len(p) for p in planned)
    views = (ctypes.c_void_p * G)(*[ctypes.addressof(p.view) for p in planned])
    res = (ctypes.c_void_p * G)(*[ctypes.addressof(r) for r in results])
    shard, index = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.int32)
    stream_off = np.empty(max(n, 1), np.int64)
    recs = np.empty(max(n, 1), BAM_RECORD_DTYPE)
    fields = np.empty((max(n, 1) * 2, 2), np.int64)
    text_len, stream_len = ctypes.c_int64(0), ctypes.c_int64(0)
    n_emit, bases, nxt = ctypes.c_int32(0), ctypes.c_int64(0), ctypes.c_int32(0)
    text = np.empty(n * 192 + 1, np.uint8)

    def call(t):
        return L.bb_bam_layout_sharded(G, views, res, int(first), int(bases_so_far), int(target_bases), int(stream_base),
                                       shard.ctypes.data, index.ctypes.data, stream_off.ctypes.data, recs.ctypes.data,
                                       fields.ctypes.data, t.ctypes.data, t.size, ctypes.byref(text_len),
                                       ctypes.byref(stream_len), ctypes.byref(n_emit), ctypes.byref(bases), ctypes.byref(nxt))
    rc = call(text)
    if rc == _lib.BB_ERR_CAPACITY:
        text = np.empty(text_len.value + 1, np.uint8)
        rc = call(text)
    if rc != 0:
        raise RuntimeError(f'bb_bam_layout_sharded failed ({rc})')
    e = n_emit.value
    return BamLayout(shard[:e], index[:e], stream_off[:e], recs[:e], fields[:2 * e], text[:text_len.value], stream_len.value,
                     e, bases.value, nxt.value)
