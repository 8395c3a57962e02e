"""
model_builders.py - `badread error_model` and `badread qscore_model` (SURVEY.md 8f row f4) with the counting on the GPU.

Mirrors badread/error_model.py:31-83 (make_error_model), badread/qscore_model.py:78-175 (make_qscore_model,
print_qscore_fractions) and badread/alignment.py:23-100 (PAF records, best alignment per read): same arguments, same
messages, byte-identical model files (tests/test_model_builders.py compares with outputs of the unmodified reference).
The host parses the three input files and flattens the chosen alignments; libbadread_b200.so counts the windows
(csrc/bb_tu_models.cu: one CTA per alignment, one thread per window, 64-bit keys in an open-addressing table with the
first occurrence of every key); the host sorts and prints.  Windows whose content does not fit a key come back in an
overflow list and are evaluated here, exactly, from the same flat arrays.

The alignments may also be SAM (plain or gzipped) or BAM, told apart from PAF by their content (alignment_format).  A
BAM's BGZF members are inflated on the GPU (bgzf.decompress); native host code (csrc/bb_bam.cpp) turns the records of
either into the fields of the PAF line the reference would read, and the best alignment per read is chosen here with
the rules of load_alignments, over arrays.  Without --reads the sequences and qualities come from the records.

With PAF alignments, --reads and a CUDA device (device_route) the FASTQ is parsed on the GPU, the PAF by bb_aln_parse and
the aligned slices are gathered on the GPU into a DeviceFlat (csrc/bb_tu_fastq.cu), which the counting kernels read in
place; the same messages, progress text and model files as the host route above.
"""
import collections
import ctypes
import gzip
import re
import sys

import numpy as np

from . import _lib, bgzf
from .misc import float_to_str, get_compression_type, get_open_func, load_fasta, reverse_complement

_CIGAR_RUN = re.compile(r'(\d+)([A-Za-z=])')
_OP_CODE = {'M': 0, 'I': 1, 'D': 2}
_SYM = '=XID'
N_Q = 94


# ---------------------------------------------------------------------------------------------------- inputs
def load_fastq(filename, output=sys.stderr, dot_interval=1000):
    """misc.load_fastq (misc.py:97-119): {name: (upper-case sequence, qualities)}; name = first token of the header."""
    reads = {}
    print('Loading reads', end='', file=output, flush=True)
    with get_open_func(filename)(filename, 'rb') as handle:
        first = handle.read(1)
        if first != b'@':
            sys.exit('Error: {} is not FASTQ format'.format(filename))
        handle.seek(0)
        n = 0
        for line in handle:
            line = line.strip()
            if not line.startswith(b'@'):
                continue
            name = line[1:].split()[0].decode()
            seq = next(handle).strip().upper().decode()
            next(handle)
            qual = next(handle).strip().decode()
            reads[name] = (seq, qual)
            n += 1
            if n % dot_interval == 0:
                print('.', end='', file=output, flush=True)
    print('', file=output, flush=True)
    return reads


class Alignment(object):
    """One PAF line (alignment.py:23-76).  `runs` = the CIGAR runs in READ orientation (reversed for '-' strand hits)."""

    def __init__(self, paf_line):
        f = paf_line.strip().split('\t')
        if len(f) < 11:
            sys.exit('Error: alignment file does not seem to be in PAF format')
        self.read_name, self.read_start, self.read_end, self.strand = f[0], int(f[2]), int(f[3]), f[4]
        self.ref_name, self.ref_start, self.ref_end = f[5], int(f[7]), int(f[8])
        self.matching_bases, self.num_bases = int(f[9]), int(f[10])
        self.percent_identity = 100.0 * self.matching_bases / self.num_bases
        self.cigar, self.alignment_score = None, None
        for part in f:
            if part.startswith('cg:Z:'):
                self.cigar = part[5:]
            if part.startswith('AS:i:'):
                self.alignment_score = int(part[5:])
        if self.cigar is None:
            sys.exit('Error: no CIGAR string found')
        if self.alignment_score is None:
            sys.exit('Error: no alignment score')
        self.runs = [(int(n), t) for n, t in _CIGAR_RUN.findall(self.cigar)]
        self.max_indel = max([n for n, t in self.runs if t in 'ID'], default=0)
        if self.strand == '-':
            self.runs.reverse()

    def __repr__(self):
        return '%s:%d-%d(%s),%s:%d-%d(%.3f%%)' % (self.read_name, self.read_start, self.read_end, self.strand,
                                                   self.ref_name, self.ref_start, self.ref_end, self.percent_identity)


def load_alignments(filename, max_alignments=None, output=sys.stderr, dot_interval=1000):
    """alignment.py:79-105: the highest-scoring alignment of every read (the last one among equals), kept if it has
    more than 100 columns and more than 80 % identity; reads in order of first appearance."""
    print('Loading alignments', end='', file=output, flush=True)
    per_read = collections.OrderedDict()
    with get_open_func(filename)(filename, 'rt') as paf:
        for n, line in enumerate(paf, start=1):
            a = Alignment(line)
            per_read.setdefault(a.read_name, []).append(a)
            if n % dot_interval == 0:
                print('.', end='', file=output, flush=True)
            if n == max_alignments:
                break
    print('', file=output, flush=True)
    print('Choosing best alignment per read', end='', file=output, flush=True)
    chosen = []
    for alns in per_read.values():
        best = alns[0]
        for a in alns[1:]:
            if a.alignment_score >= best.alignment_score:
                best = a
        if best.num_bases > 100 and best.percent_identity > 80.0:
            chosen.append(best)
            if len(chosen) % dot_interval == 0:
                print('.', end='', file=output, flush=True)
    print('', file=output, flush=True)
    return chosen


_SAM_CIGAR = re.compile(r'(\d+[MIDNSHP=X])+')
_inflate = bgzf.decompress      # BAM's BGZF, inflated on the GPU


def alignment_format(filename):
    """'bam', 'sam' or 'paf', from the content: BGZF whose first inflated bytes are BAM's magic is BAM; a first line that
    starts with '@', or that has SAM's 11 columns with integer FLAG, POS and MAPQ and a CIGAR or '*' in column 6, is SAM
    (plain or gzipped); anything else is PAF."""
    try:
        with open(filename, 'rb') as f:
            magic = f.read(4)
        with (gzip.open if magic[:2] == b'\x1f\x8b' else open)(filename, 'rb') as f:
            head = f.read(4)
            line = head + (f.readline() if not head.endswith(b'\n') else b'')
    except (OSError, EOFError):
        return 'paf'    # (unreadable: the PAF path reports it as it always has)
    if magic == b'\x1f\x8b\x08\x04' and head == b'BAM\x01':
        return 'bam'
    if line.startswith(b'@'):
        return 'sam'
    f = line.rstrip(b'\r\n').split(b'\t')
    if len(f) >= 11 and all(re.fullmatch(rb'-?\d+', f[i]) for i in (1, 3, 4)) and \
            (f[5] == b'*' or _SAM_CIGAR.fullmatch(f[5].decode('latin-1'))):
        return 'sam'
    return 'paf'


class SamAlignment(object):
    """The chosen alignment of a read from a SAM / BAM record: the attributes of Alignment that FlatAlignments reads, and
    its identity for Alignment's repr."""
    __slots__ = ('read_name', 'read_start', 'read_end', 'strand', 'ref_name', 'ref_start', 'ref_end', 'runs',
                 'percent_identity')

    def __init__(self, read_name, read_start, read_end, strand, ref_name, ref_start, ref_end, runs, percent_identity):
        self.read_name, self.read_start, self.read_end, self.strand = read_name, read_start, read_end, strand
        self.ref_name, self.ref_start, self.ref_end, self.runs = ref_name, ref_start, ref_end, runs
        self.percent_identity = percent_identity

    __repr__ = Alignment.__repr__


def _view_array(ptr, n, dtype):
    if n == 0:
        return np.zeros(0, dtype=dtype)
    return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(n,)).copy()


def _names(blob_ptr, off):
    blob = ctypes.string_at(blob_ptr, int(off[-1])) if off[-1] else b''
    return [blob[a:b].decode() for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


def _parse_records(filename, fmt, max_alignments):
    """bb_aln_parse of a SAM, BAM or PAF file (a BAM's BGZF and a gzipped PAF inflated on the GPU): its handle (bb_aln_free
    it)."""
    with (open if fmt in ('bam', 'paf') else get_open_func(filename))(filename, 'rb') as handle:
        data = handle.read()
    if fmt == 'bam':
        try:
            data = _inflate(data)
        except ValueError as e:
            sys.exit(f'\nError: {filename} is not a valid BAM file ({e})')
    elif fmt == 'paf' and get_compression_type(filename) == 'gz':
        try:
            data = bgzf.gunzip(data)[0]
        except ValueError as e:
            sys.exit(f'\nError: {filename} could not be inflated ({e})')
    L = _lib.lib()
    buf = np.frombuffer(memoryview(data).cast('B'), dtype=np.uint8)
    handle = ctypes.c_void_p()
    rc = L.bb_aln_parse(buf.ctypes.data_as(ctypes.c_void_p) if buf.size else None, buf.size,
                        {'sam': 0, 'bam': 1, 'paf': _lib.BB_ALN_PAF}[fmt], max_alignments or 0, ctypes.byref(handle))
    if rc != _lib.BB_OK:      # (load_alignments' messages end its unfinished line; bb_aln_parse's SAM / BAM ones break it)
        sys.exit(('' if fmt == 'paf' else '\n') + L.bb_model_error().decode(errors='replace'))
    return handle


def _record_arrays(handle):
    """(bb_aln_view, records, reference names, read names, {field: array}) of a bb_aln_parse handle."""
    v = _lib.AlnView()
    _lib.lib().bb_aln_view_get(handle, ctypes.byref(v))
    n = v.n_records
    ref_names = _names(v.ref_names, _view_array(v.ref_name_off, v.n_refs + 1, np.int64))
    read_names = _names(v.read_names, _view_array(v.read_name_off, v.n_reads + 1, np.int64))
    a = {f: _view_array(getattr(v, f), n, t) for f, t in
         (('read_id', np.int32), ('ref_id', np.int32), ('flag', np.int32), ('score', np.int32), ('nm', np.int32),
          ('read_start', np.int32), ('read_end', np.int32), ('columns', np.int32), ('ref_start', np.int64),
          ('ref_end', np.int64), ('has_qual', np.uint8), ('full', np.uint8))}
    return v, n, ref_names, read_names, a


def _best_per_read(a, n):
    """Per read the record with the highest score, the last among equals; reads in order of first appearance."""
    order = np.lexsort((np.arange(n), a['score'], a['read_id']))           # per read: by score, then by position
    last = np.flatnonzero(np.append(a['read_id'][order][1:] != a['read_id'][order][:-1], True)) if n else order
    return order[last]


def _usable(best, columns, matches):
    """The records of `best` with more than 100 columns and more than 80 % identity (Alignment.percent_identity's two
    operations)."""
    cols = columns.astype(np.int64)
    with np.errstate(divide='ignore', invalid='ignore'):
        return best[(cols > 100) & (100.0 * matches / cols > 80.0)]


def load_sam_alignments(filename, fmt, max_alignments, reads, refs, need_qual, output=sys.stderr, dot_interval=1000):
    """The alignments of a SAM or BAM file, chosen as load_alignments chooses them: per read the record with the highest
    AS:i (the last among equals), kept with more than 100 columns and more than 80 % identity, reads in order of first
    appearance; --max_alignments counts mapped records.  The identity is (columns - NM:i) / columns, the matching bases
    counted from the sequences only for a record without NM.  reads: the FASTQ's {name: (seq, qual)}, or None to take
    every chosen read's sequence and qualities from a record of it that holds the whole read (SEQ not '*', no H clip),
    turned back to the read's own orientation.  Returns (alignments, reads)."""
    print('Loading alignments', end='', file=output, flush=True)
    L = _lib.lib()
    handle = _parse_records(filename, fmt, max_alignments)
    try:
        v, n, ref_names, read_names, a = _record_arrays(handle)
        cigar_off = _view_array(v.cigar_off, n + 1, np.int64)
        cigar = _view_array(v.cigar, int(cigar_off[-1]), np.uint32)
        seq_off = _view_array(v.seq_off, n + 1, np.int64)
        seq = ctypes.string_at(v.seq, int(seq_off[-1])) if seq_off[-1] else b''
        qual = ctypes.string_at(v.qual, int(seq_off[-1])) if seq_off[-1] else b''
    finally:
        L.bb_aln_free(handle)
    print('.' * (n // dot_interval), file=output, flush=True)

    print('Choosing best alignment per read', end='', file=output, flush=True)
    best = _best_per_read(a, n)

    def whole_read(i):
        """The read of record i's own orientation from the record of it that holds the whole read."""
        rid = int(a['read_id'][i])
        name = read_names[rid]
        if reads is not None:
            return reads.get(name)
        j = full_of.get(rid)
        if j is None:
            sys.exit(f'\nError: no record of read {name} holds its whole sequence (SEQ not * and no hard clips): '
                     f'give the reads with --reads')
        if need_qual and not a['has_qual'][j]:
            sys.exit(f'\nError: the record of read {name} has no qualities (QUAL is *): give the reads with --reads')
        s = seq[seq_off[j]:seq_off[j + 1]].decode('latin-1')
        q = qual[seq_off[j]:seq_off[j + 1]].decode('latin-1') if a['has_qual'][j] else ''
        if a['flag'][j] & 16:
            s, q = reverse_complement(s), q[::-1]
        return s, q

    full_idx = np.flatnonzero(a['full'])
    _, first_full = np.unique(a['read_id'][full_idx], return_index=True)
    full_of = dict(zip(a['read_id'][full_idx][first_full].tolist(), full_idx[first_full].tolist()))
    matches = a['columns'][best].astype(np.int64) - a['nm'][best]
    own_reads = {} if reads is None else reads
    for k in np.flatnonzero(a['nm'][best] < 0).tolist():                    # no NM:i: count from the sequences
        i = int(best[k])
        matches[k] = _count_matches(i, a, cigar, cigar_off, whole_read(i), refs.get(ref_names[a['ref_id'][i]]))
    keep = _usable(best, a['columns'][best], matches)
    with np.errstate(divide='ignore', invalid='ignore'):
        identity_of = dict(zip(best.tolist(), (100.0 * matches / a['columns'][best].astype(np.int64)).tolist()))
    chosen = []
    for i in keep.tolist():
        name = read_names[a['read_id'][i]]
        if reads is None and name not in own_reads:
            own_reads[name] = whole_read(i)
        runs = [(c >> 4, 'MIDNSHPMM'[c & 15]) for c in cigar[cigar_off[i]:cigar_off[i + 1]].tolist() if (c & 15) not in (4, 5)]
        strand = '-' if a['flag'][i] & 16 else '+'
        if strand == '-':
            runs.reverse()
        chosen.append(SamAlignment(name, int(a['read_start'][i]), int(a['read_end'][i]), strand, ref_names[a['ref_id'][i]],
                                   int(a['ref_start'][i]), int(a['ref_end'][i]), runs, identity_of[i]))
        if len(chosen) % dot_interval == 0:
            print('.', end='', file=output, flush=True)
    print('', file=output, flush=True)
    return chosen, own_reads


def _count_matches(i, a, cigar, cigar_off, read, ref):
    """Matching bases of record i without NM:i: its M = X columns where the read (in the reference's orientation) and the
    reference agree."""
    if read is None or ref is None:
        return 0        # (FlatAlignments reports the missing read or reference)
    seq = read[0]
    s = reverse_complement(seq) if a['flag'][i] & 16 else seq
    rp, fp, m = 0, int(a['ref_start'][i]), 0
    for c in cigar[cigar_off[i]:cigar_off[i + 1]].tolist():
        op, n = c & 15, c >> 4
        if op in (0, 7, 8):
            m += sum(x == y for x, y in zip(s[rp:rp + n], ref[fp:fp + n]))
            rp += n
            fp += n
        elif op in (1, 4, 5):     # (the whole read holds the hard-clipped bases too)
            rp += n
        elif op == 2:
            fp += n
    return m


def load_inputs(args, refs, output, need_qual):
    """(reads, chosen alignments) of the builders' --reads and --alignment, whichever alignment format it is (--reads may
    be None for SAM and BAM only)."""
    fmt = alignment_format(args.alignment)
    reads = load_fastq(args.reads, output=output) if args.reads is not None else None
    if fmt == 'paf':
        return reads, load_alignments(args.alignment, args.max_alignments, output=output)
    alignments, reads = load_sam_alignments(args.alignment, fmt, args.max_alignments, reads, refs, need_qual, output=output)
    return reads, alignments


class FlatAlignments(object):
    """The chosen alignments as the flat arrays bb_count_* take: per alignment the aligned slice of the read (+ its
    qualities), the aligned slice of the reference on the read's strand, and the CIGAR runs in read orientation with the
    offsets they start at."""

    def __init__(self, alignments, reads, refs, output, dot_interval):
        read_parts, qual_parts, ref_parts, ops, p0, r0 = [], [], [], [], [], []
        self.read_off, self.ref_off, self.ops_off = [0], [0], [0]
        print('Processing alignments', end='', file=output, flush=True)
        for n, a in enumerate(alignments, start=1):
            if a.read_name not in reads:
                sys.exit(f'\nError: could not find read {a.read_name}\nare you sure your read file and alignment file match?')
            if a.ref_name not in refs:
                sys.exit(f'\nError: could not find reference {a.ref_name}\nare you sure your reference file and '
                         f'alignment file match?')
            seq, qual = reads[a.read_name]
            read_seq, read_qual = seq[a.read_start:a.read_end], qual[a.read_start:a.read_end]
            ref_seq = refs[a.ref_name][a.ref_start:a.ref_end]
            if a.strand == '-':
                ref_seq = reverse_complement(ref_seq)
            rp = fp = 0
            for count, kind in a.runs:
                if kind not in _OP_CODE:
                    continue        # (alignment.align_sequences ignores every other CIGAR letter)
                ops.append((count << 2) | _OP_CODE[kind]); p0.append(rp); r0.append(fp)
                if kind != 'D':
                    rp += count
                if kind != 'I':
                    fp += count
            # the CIGAR may cover less than the slices (or more: the reference's slicing silently truncates, so do we)
            read_parts.append(read_seq[:rp].ljust(rp, '\0')); qual_parts.append(read_qual[:rp].ljust(rp, '\0'))
            ref_parts.append(ref_seq[:fp].ljust(fp, '\0'))
            self.read_off.append(self.read_off[-1] + rp)
            self.ref_off.append(self.ref_off[-1] + fp)
            self.ops_off.append(len(ops))
            if n % dot_interval == 0:
                print('.', end='', file=output, flush=True)
        print('', file=output, flush=True)
        self.n = len(alignments)
        self.read = np.frombuffer(''.join(read_parts).encode('latin-1') or b'\0', dtype=np.uint8)
        self.qual = np.frombuffer(''.join(qual_parts).encode('latin-1') or b'\0', dtype=np.uint8)
        self.ref = np.frombuffer(''.join(ref_parts).encode('latin-1') or b'\0', dtype=np.uint8)
        self.read_off = np.asarray(self.read_off, dtype=np.int64)
        self.ref_off = np.asarray(self.ref_off, dtype=np.int64)
        self.ops_off = np.asarray(self.ops_off, dtype=np.int64)
        self.ops = np.asarray(ops or [0], dtype=np.uint32)
        self.op_read0 = np.asarray(p0 or [0], dtype=np.int32)
        self.op_ref0 = np.asarray(r0 or [0], dtype=np.int32)

    # exact host evaluation of single windows (the overflow list)
    def columns(self, a):
        """Per read base of alignment a: symbol and the number of 'D' columns behind it; per reference base: the read
        offset at its column and whether that column holds a read base."""
        lo, hi = int(self.ops_off[a]), int(self.ops_off[a + 1])
        return _columns(self.read[self.read_off[a]:self.read_off[a + 1]], self.ref[self.ref_off[a]:self.ref_off[a + 1]],
                        self.ops[lo:hi], self.op_read0[lo:hi], self.op_ref0[lo:hi])

    def quals(self, a):
        """The quality slice of alignment a."""
        return self.qual[self.read_off[a]:self.read_off[a + 1]]


def _columns(read, ref, ops, op_read0, op_ref0):
    """FlatAlignments.columns of one alignment's slices and runs."""
    sym = np.zeros(len(read), dtype=np.uint8)
    dcount = np.zeros(len(read), dtype=np.int64)
    rp_at = np.zeros(len(ref), dtype=np.int64)
    is_m = np.zeros(len(ref), dtype=bool)
    lead = 0
    for o in range(len(ops)):
        count, kind, p, r = int(ops[o]) >> 2, int(ops[o]) & 3, int(op_read0[o]), int(op_ref0[o])
        if kind == 0:
            sym[p:p + count] = (read[p:p + count] != ref[r:r + count]).astype(np.uint8)
            rp_at[r:r + count] = np.arange(p, p + count); is_m[r:r + count] = True
        elif kind == 1:
            sym[p:p + count] = 2
        else:
            rp_at[r:r + count] = p
            if p > 0:
                dcount[p - 1] += count
            else:
                lead += count
    return read, ref, sym, dcount, rp_at, is_m, lead


# ---------------------------------------------------------------------------------------------------- device route
def device_route(args, fmt):
    """The route hook: True when a builder takes the device route - PAF alignments with --reads, and the library sees a
    CUDA device.  The FASTQ is then parsed on the GPU and the aligned slices gathered there (csrc/bb_tu_fastq.cu), the
    PAF parsed by native code (bb_aln_parse), and the counting kernels take the flat arrays where they lie (DeviceFlat).
    Otherwise the host route: load_fastq, load_alignments / load_sam_alignments and FlatAlignments."""
    if fmt != 'paf' or args.reads is None:
        return False
    try:
        return _lib.lib().bb_device_count() > 0
    except (_lib.LibraryMissing, OSError):
        return False


class DeviceFlat(object):
    """FlatAlignments in device memory (bb_flat_build): the same attributes and dtypes, the offsets on the host and the
    other arrays copied to the host on first access; columns(a) fetches alignment a's slices only; device_pointers are
    what _count passes to the counting kernels.  close() releases the device memory."""
    _ARRAYS = {'read': (0, np.uint8, 'read_off'), 'qual': (1, np.uint8, 'read_off'), 'ref': (2, np.uint8, 'ref_off'),
               'ops': (3, np.uint32, 'ops_off'), 'op_read0': (4, np.int32, 'ops_off'), 'op_ref0': (5, np.int32, 'ops_off')}

    def __init__(self, handle):
        self._handle = handle
        v = _lib.FlatView()
        _lib.lib().bb_flat_view_get(handle, ctypes.byref(v))
        self.n = v.n
        self.read_off = _view_array(v.read_off, self.n + 1, np.int64)
        self.ref_off = _view_array(v.ref_off, self.n + 1, np.int64)
        self.ops_off = _view_array(v.ops_off, self.n + 1, np.int64)
        self.device_pointers = [ctypes.c_void_p(getattr(v, f)) for f in ('read', 'qual', 'ref', 'ops', 'op_read0', 'op_ref0')]

    def _fetch(self, name, lo, count, size=None):
        which, dtype, _ = self._ARRAYS[name]
        out = np.zeros(count if size is None else size, dtype=dtype)
        L = _lib.lib()
        if count and L.bb_flat_fetch(self._handle, which, lo, count, _ptr(out)) != _lib.BB_OK:
            raise RuntimeError('model builder: ' + L.bb_model_error().decode(errors='replace'))
        return out

    def __getattr__(self, name):
        if name not in DeviceFlat._ARRAYS or self.__dict__.get('_handle') is None:
            raise AttributeError(name)
        total = int(getattr(self, self._ARRAYS[name][2])[-1])
        arr = self._fetch(name, 0, total, max(total, 1))       # (one NUL / zero when empty, as FlatAlignments)
        self.__dict__[name] = arr
        return arr

    def columns(self, a):
        """FlatAlignments.columns, from alignment a's slices."""
        r0, r1, f0, f1 = int(self.read_off[a]), int(self.read_off[a + 1]), int(self.ref_off[a]), int(self.ref_off[a + 1])
        o0, o1 = int(self.ops_off[a]), int(self.ops_off[a + 1])
        return _columns(self._fetch('read', r0, r1 - r0), self._fetch('ref', f0, f1 - f0), self._fetch('ops', o0, o1 - o0),
                        self._fetch('op_read0', o0, o1 - o0), self._fetch('op_ref0', o0, o1 - o0))

    def quals(self, a):
        """FlatAlignments.quals, fetched for alignment a only."""
        r0, r1 = int(self.read_off[a]), int(self.read_off[a + 1])
        return self._fetch('qual', r0, r1 - r0)

    def close(self):
        if self._handle is not None:
            _lib.lib().bb_flat_free(self._handle)
            self._handle = None


def _fastq_on_device(filename, output, dot_interval=1000):
    """load_fastq's parse on the GPU (bb_fastq_parse) with its progress text and messages: the handle (bb_fastq_free)."""
    from .engine import FastaFile
    L = _lib.lib()
    print('Loading reads', end='', file=output, flush=True)
    get_compression_type(filename)      # (bzip2 and zip exit with its messages)
    f = FastaFile(filename)
    handle, n_rec, first = ctypes.c_void_p(), ctypes.c_int64(0), ctypes.c_int32(-1)
    try:
        rc = L.bb_fastq_parse(0, _ptr(f.data) if f.data.size else None, f.data.size, int(f.gzip), ctypes.byref(handle),
                              ctypes.byref(n_rec), ctypes.byref(first))
    finally:
        f.close()
    if rc != _lib.BB_OK:      # (the message names the record or the stage: "Error: ..."; the file goes in front of it)
        msg = L.bb_model_error().decode(errors='replace')
        sys.exit(f'\nError: {filename}: {msg[len("Error: "):]}' if msg.startswith('Error: ') else f'\nError: {filename}: {msg}')
    if first.value != ord('@'):
        L.bb_fastq_free(handle)
        sys.exit('Error: {} is not FASTQ format'.format(filename))
    print('.' * (n_rec.value // dot_interval), file=output, flush=True)
    return handle


def _touched_contigs(ref_ids, ref_names, refs):
    """The contigs of reference ids ref_ids, concatenated once each: (offset of each id or -1 when refs lacks it, length
    of each id, the bytes, their total)."""
    contig_at = np.full(max(len(ref_names), 1), -1, dtype=np.int64)
    contig_len = np.zeros(max(len(ref_names), 1), dtype=np.int64)
    parts, pos = [], 0
    for rid in np.unique(ref_ids).tolist():
        seq = refs.get(ref_names[rid])
        if seq is not None:
            parts.append(seq.encode('latin-1'))
            contig_at[rid], contig_len[rid] = pos, len(parts[-1])
            pos += len(parts[-1])
    return contig_at, contig_len, np.frombuffer(b''.join(parts) or b'\0', dtype=np.uint8), pos


class _HostInputs(object):
    """A builder's reads and chosen alignments on the host route."""

    def __init__(self, reads, alignments, refs):
        self.reads, self.alignments, self.refs, self.n = reads, alignments, refs, len(alignments)

    def flatten(self, output, dot_interval):
        return FlatAlignments(self.alignments, self.reads, self.refs, output, dot_interval)

    def close(self):
        pass


class _DeviceInputs(object):
    """A builder's reads (parsed on the GPU) and chosen PAF records on the device route, with load_fastq's and
    load_alignments' progress text and messages; flatten() gathers the DeviceFlat.  close() releases everything."""

    def __init__(self, args, refs, output, dot_interval=1000):
        self.refs, self.fastq, self.records, self.flat = refs, None, None, None
        try:
            self.fastq = _fastq_on_device(args.reads, output)
            print('Loading alignments', end='', file=output, flush=True)
            self.records = _parse_records(args.alignment, 'paf', args.max_alignments)
            self.view, n, self.ref_names, self.read_names, self.a = _record_arrays(self.records)
            print('.' * (n // dot_interval), file=output, flush=True)
            print('Choosing best alignment per read', end='', file=output, flush=True)
            best = _best_per_read(self.a, n)
            self.chosen = _usable(best, self.a['columns'][best], self.a['columns'][best].astype(np.int64) - self.a['nm'][best])
            print('.' * (len(self.chosen) // dot_interval), file=output, flush=True)
            self.n = len(self.chosen)
        except BaseException:
            self.close()
            raise

    def flatten(self, output, dot_interval, slice_len=None):
        """The DeviceFlat of the chosen alignments; slice_len (an int64 array (n, 3), or None) gets the lengths of
        each alignment's sequence, quality and reference slices before they are fitted to its CIGAR."""
        L, a, chosen = _lib.lib(), self.a, self.chosen.astype(np.int64)
        print('Processing alignments', end='', file=output, flush=True)
        contig_at, contig_len, contigs, pos = _touched_contigs(a['ref_id'][chosen], self.ref_names, self.refs)
        handle, failed = ctypes.c_void_p(), np.zeros(2, dtype=np.int64)
        rc = L.bb_flat_build(self.fastq, ctypes.byref(self.view), len(chosen), _ptr(chosen), _ptr(contig_at), _ptr(contig_len),
                             _ptr(contigs), pos, ctypes.byref(handle), _ptr(failed),
                             None if slice_len is None else _ptr(slice_len))
        if rc != _lib.BB_OK:
            i, kind = int(failed[0]), int(failed[1])
            if kind == 0:
                sys.exit('\n' + L.bb_model_error().decode(errors='replace'))
            print('.' * (i // dot_interval), end='', file=output, flush=True)
            read, ref = self.read_names[a['read_id'][chosen[i]]], self.ref_names[a['ref_id'][chosen[i]]]
            if kind == 1:
                sys.exit(f'\nError: could not find read {read}\nare you sure your read file and alignment file match?')
            if kind == 2:
                sys.exit(f'\nError: could not find reference {ref}\nare you sure your reference file and alignment file match?')
            sys.exit(f'\nError: read {read} has bytes outside ASCII in its sequence or qualities')
        self.flat = DeviceFlat(handle)
        L.bb_fastq_free(self.fastq)
        self.fastq = None
        print('.' * (self.n // dot_interval), file=output, flush=True)
        return self.flat

    def close(self):
        L = _lib.lib()
        if self.flat is not None:
            self.flat.close()
            self.flat = None
        if self.fastq is not None:
            L.bb_fastq_free(self.fastq)
            self.fastq = None
        if self.records is not None:
            L.bb_aln_free(self.records)
            self.records = None


def _inputs(args, refs, output, need_qual):
    """A builder's inputs on the route device_route chooses."""
    if device_route(args, alignment_format(args.alignment)):
        return _DeviceInputs(args, refs, output)
    reads, alignments = load_inputs(args, refs, output, need_qual)
    return _HostInputs(reads, alignments, refs)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _count(which, flat, k, max_del=0, device=0, cap=None, ovf_cap=None):
    """Runs bb_count_kmer_alternatives ('kmers'), bb_count_kmer_alternatives_wide ('kmers_wide': keys come back as
    (n, 2) words, read k-mer and reference k-mer << 6 | length) or bb_count_cigar_qscores ('cigars'), growing the table
    (from `cap` slots, a power of two >= 16) and the overflow list (from `ovf_cap` entries) until they fit."""
    L = _lib.lib()
    per_slot = N_Q if which == 'cigars' else 1
    key_words = 2 if which == 'kmers_wide' else 1
    if cap is None:
        cap = 1 << 18       # slots; doubled until the distinct keys fit (k-mer pairs: at most one per window)
        while which != 'cigars' and cap < min(2 * int(flat.ref_off[-1]) + 16, 1 << 22):
            cap <<= 1
    if ovf_cap is None:
        ovf_cap = 1 << 16
    while True:
        keys = np.empty(cap * key_words, dtype=np.uint64); first = np.empty(cap, dtype=np.uint64)
        counts = np.empty(cap * per_slot, dtype=np.uint32)
        ovf = [np.empty(ovf_cap, dtype=np.int32) for _ in range(3)]
        overall = np.zeros(N_Q, dtype=np.uint64)
        n_entries, n_ovf = ctypes.c_int64(0), ctypes.c_int64(0)
        if isinstance(flat, DeviceFlat):
            read, qual, ref, ops, p0, r0 = flat.device_pointers
        else:
            read, qual, ref, ops, p0, r0 = (_ptr(x) for x in (flat.read, flat.qual, flat.ref, flat.ops, flat.op_read0, flat.op_ref0))
        common = [ref, _ptr(flat.ref_off), ops, p0, r0, _ptr(flat.ops_off), cap, _ptr(keys), _ptr(first), _ptr(counts),
                  ctypes.byref(n_entries)]
        tail = [ovf_cap, _ptr(ovf[0]), _ptr(ovf[1]), _ptr(ovf[2]), ctypes.byref(n_ovf)]
        if which == 'kmers':
            rc = L.bb_count_kmer_alternatives(device, k, flat.n, read, _ptr(flat.read_off), *common, *tail)
        elif which == 'kmers_wide':
            rc = L.bb_count_kmer_alternatives_wide(device, k, flat.n, read, _ptr(flat.read_off), *common, *tail)
        else:
            rc = L.bb_count_cigar_qscores(device, k, max_del, flat.n, read, qual, _ptr(flat.read_off), *common, _ptr(overall),
                                          *tail)
        if rc == _lib.BB_ERR_CAPACITY:
            if n_ovf.value > ovf_cap:
                ovf_cap = int(n_ovf.value) + 16
            else:
                cap <<= 1
            continue
        if rc != _lib.BB_OK:
            raise RuntimeError('model builder: ' + L.bb_model_error().decode(errors='replace'))
        n, m = int(n_entries.value), int(n_ovf.value)
        keys = keys[:n * key_words].reshape(n, 2) if key_words == 2 else keys[:n]
        return keys, first[:n], counts[:n * per_slot].reshape(n, per_slot), overall, [o[:m] for o in ovf]


# ---------------------------------------------------------------------------------------------------- error model
MAX_K_DENSE = 12    # 64-bit keys and dense per-k-mer arrays (4^k entries)
MAX_K_WIDE = 16     # 128-bit keys, aggregated over the reference k-mers that occur


def _overflow_alternatives(flat, ovf, k):
    """Read k-mers too long for a key (the overflow list), counted here, exactly:
    {reference k-mer code: {read k-mer: [count, first occurrence]}}."""
    long_alts, cache = collections.defaultdict(dict), {}
    for a, r, _ in zip(*(o.tolist() for o in ovf)):
        if a not in cache:
            cache[a] = flat.columns(a)
        read, ref, _, _, rp_at, is_m, _ = cache[a]
        p_lo = 0 if r == 0 else int(rp_at[r])
        p_hi = int(rp_at[r + k - 1]) + int(is_m[r + k - 1])
        read_kmer = bytes(read[p_lo:p_hi]).decode('latin-1')
        if set(read_kmer) <= set('ACGT'):
            code = 0
            for c in bytes(ref[r:r + k]):
                code = code * 4 + b'ACGT'.index(c)
            entry = long_alts[code].setdefault(read_kmer, [0, (a << 32) | r])
            entry[0] += 1
            entry[1] = min(entry[1], (a << 32) | r)
    return long_alts


def _error_model_lines_sparse(args, flat, k):
    """The model file for 12 < k <= 16 from 128-bit keys: the same lines as the dense path below, aggregated over the
    reference k-mers that occur (np.unique) instead of arrays of 4^k entries."""
    keys, first, counts, _, ovf = _count('kmers_wide', flat, k)
    counts = counts[:, 0].astype(np.int64)
    read_bits, hi = keys[:, 0], keys[:, 1]
    refcode = (hi >> np.uint64(6)).astype(np.int64)
    lens = (hi & np.uint64(63)).astype(np.int64)
    long_alts = _overflow_alternatives(flat, ovf, k)
    codes = np.unique(np.concatenate([refcode, np.fromiter(long_alts, dtype=np.int64, count=len(long_alts))]))
    group_of = np.searchsorted(codes, refcode)            # entry -> index of its reference k-mer in `codes`
    totals = np.bincount(group_of, weights=counts, minlength=codes.size).astype(np.int64)
    for code, alts in long_alts.items():
        totals[np.searchsorted(codes, code)] += sum(c for c, _ in alts.values())
    same = np.zeros(refcode.size, dtype=np.uint64)        # the read bits of the unchanged k-mer: base j at bits 2j
    rc = refcode.astype(np.uint64)
    for j in range(k):
        same |= ((rc >> np.uint64(2 * (k - 1 - j))) & np.uint64(3)) << np.uint64(2 * j)
    is_identity = (lens == k) & (read_bits == same)
    unchanged = np.zeros(codes.size, dtype=np.int64)
    unchanged[group_of[is_identity]] = counts[is_identity]
    alt = np.flatnonzero(~is_identity)
    order = alt[np.lexsort((first[alt], -counts[alt], refcode[alt]))]
    group = refcode[order]
    starts = np.flatnonzero(np.concatenate([[True], group[1:] != group[:-1]])) if order.size else np.zeros(0, dtype=np.int64)
    rank = np.arange(order.size) - np.repeat(starts, np.diff(np.concatenate([starts, [order.size]])))
    # (a reference k-mer with alternatives in the overflow list keeps all of its entries: they are merged below)
    crowded = np.isin(group, np.fromiter(long_alts, dtype=np.int64, count=len(long_alts)))
    kept = order[(rank < args.max_alt) | crowded]
    kept_lens = lens[kept]
    width = int(kept_lens.max()) if kept.size else 1
    letters = np.frombuffer(b'ACGT', dtype=np.uint8)[((read_bits[kept][:, None] >> (np.uint64(2) * np.arange(width, dtype=np.uint64))) &
                                                    np.uint64(3)).astype(np.int64)].tobytes()
    kept_code, kept_count, kept_first = refcode[kept].tolist(), counts[kept].tolist(), first[kept].tolist()
    per_code = collections.defaultdict(list)
    for i, n in enumerate(kept_lens.tolist()):
        per_code[kept_code[i]].append((letters[i * width:i * width + n].decode(), kept_count[i], kept_first[i]))
    out = []
    for code, total, n_same in zip(codes.tolist(), totals.tolist(), unchanged.tolist()):
        kmer = ''.join('ACGT'[(code >> (2 * (k - 1 - j))) & 3] for j in range(k))
        alts = per_code.get(code, [])
        if code in long_alts:
            alts = sorted(alts + [(a, c, s) for a, (c, s) in long_alts[code].items()], key=lambda x: (-x[1], x[2]))
        line = [f'{kmer},{n_same / total:.6f};']
        line.extend(f'{a},{c / total:.6f};' for a, c, _ in alts[:args.max_alt])
        out.append(''.join(line))
    return '\n'.join(out)


def make_error_model(args, output=sys.stderr, dot_interval=1000):
    """error_model.py:31-83."""
    refs = load_fasta(args.reference)[0]
    inputs = _inputs(args, refs, output, need_qual=False)
    try:
        _error_model(args, inputs, output, dot_interval)
    finally:
        inputs.close()


def _error_model(args, inputs, output, dot_interval):
    if inputs.n == 0:
        sys.exit('Error: no usable alignments')
    k = args.k_size
    if k > MAX_K_WIDE:
        sys.exit(f'Error: error models with k > {MAX_K_WIDE} are not supported by badread_b200')
    flat = inputs.flatten(output, dot_interval)
    if k > MAX_K_DENSE:
        print(_error_model_lines_sparse(args, flat, k))
        return
    keys, first, counts, _, ovf = _count('kmers', flat, k)
    counts = counts[:, 0].astype(np.int64)
    shift_ref, shift_len = np.uint64(64 - 2 * k), np.uint64(58 - 2 * k)
    long_alts = _overflow_alternatives(flat, ovf, k)
    # per reference k-mer: total, the count of the unchanged k-mer, and the alternatives by (count, first occurrence) -
    # the order of the reference's stable sort by fraction over its insertion-ordered dict
    refcode = (keys >> shift_ref).astype(np.int64)
    totals = np.bincount(refcode, weights=counts, minlength=4 ** k).astype(np.int64)
    for code, alts in long_alts.items():
        totals[code] += sum(c for c, _ in alts.values())
    same = np.zeros(4 ** k, dtype=np.uint64)        # the read part of the key of an unchanged k-mer: base j at bits 2j
    codes = np.arange(4 ** k, dtype=np.uint64)
    for j in range(k):
        same |= ((codes >> np.uint64(2 * (k - 1 - j))) & np.uint64(3)) << np.uint64(2 * j)
    identity_key = (codes << shift_ref) | (np.uint64(k) << shift_len) | same
    is_identity = keys == identity_key[refcode]
    unchanged = np.zeros(4 ** k, dtype=np.int64)
    unchanged[refcode[is_identity]] = counts[is_identity]
    alt = np.flatnonzero(~is_identity)
    order = alt[np.lexsort((first[alt], -counts[alt], refcode[alt]))]
    group = refcode[order]
    starts = np.flatnonzero(np.concatenate([[True], group[1:] != group[:-1]])) if order.size else np.zeros(0, dtype=np.int64)
    rank = np.arange(order.size) - np.repeat(starts, np.diff(np.concatenate([starts, [order.size]])))
    # (a reference k-mer with alternatives in the overflow list keeps all of its entries: they are merged below)
    crowded = np.zeros(4 ** k, dtype=bool)
    crowded[list(long_alts)] = True
    kept = order[(rank < args.max_alt) | crowded[group]]
    lens = ((keys[kept] >> shift_len) & np.uint64(63)).astype(np.int64)
    width = int(lens.max()) if kept.size else 1
    letters = np.frombuffer(b'ACGT', dtype=np.uint8)[((keys[kept][:, None] >> (np.uint64(2) * np.arange(width, dtype=np.uint64))) &
                                                   np.uint64(3)).astype(np.int64)].tobytes()
    kept_code, kept_count, kept_first = refcode[kept].tolist(), counts[kept].tolist(), first[kept].tolist()
    per_code = collections.defaultdict(list)
    for i, n in enumerate(lens.tolist()):
        per_code[kept_code[i]].append((letters[i * width:i * width + n].decode(), kept_count[i], kept_first[i]))
    out = []
    totals_l, unchanged_l = totals.tolist(), unchanged.tolist()
    for code in np.flatnonzero(totals).tolist():
        kmer = ''.join('ACGT'[(code >> (2 * (k - 1 - j))) & 3] for j in range(k))
        total = totals_l[code]
        alts = per_code.get(code, [])
        if code in long_alts:
            alts = sorted(alts + [(a, c, s) for a, (c, s) in long_alts[code].items()], key=lambda x: (-x[1], x[2]))
        line = [f'{kmer},{unchanged_l[code] / total:.6f};']
        line.extend(f'{a},{c / total:.6f};' for a, c, _ in alts[:args.max_alt])
        out.append(''.join(line))
    print('\n'.join(out))


# ---------------------------------------------------------------------------------------------------- qscore model
def print_qscore_fractions(cigar, qscores, min_occur):
    """qscore_model.py:164-174; qscores: {quality value: count}."""
    total = sum(qscores.values())
    if total < min_occur:
        return
    fracs = ''.join(f'{q}:{float_to_str(qscores[q] / total, decimals=6, trim_zeros=True)},' for q in sorted(qscores))
    print(f'{cigar};{total};{fracs}')


def make_qscore_model(args, output=sys.stderr, dot_interval=1000):
    """qscore_model.py:78-161."""
    refs = load_fasta(args.reference)[0]
    inputs = _inputs(args, refs, output, need_qual=True)
    try:
        _qscore_model(args, inputs, output, dot_interval)
    finally:
        inputs.close()


def _qscore_model(args, inputs, output, dot_interval):
    if inputs.n == 0:
        sys.exit('Error: no usable alignments')
    assert args.k_size % 2 == 1     # an odd size has a middle base to take the qscore from
    flat = inputs.flatten(output, dot_interval)
    keys, first, counts, overall, ovf = _count('cigars', flat, args.k_size, args.max_del)
    table = {}          # cigar -> [histogram, first occurrence]
    for key, stamp, hist in zip(keys.tolist(), first.tolist(), counts):
        n = key >> 58
        table[''.join(_SYM[(key >> (2 * j)) & 3] for j in range(n))] = [hist.astype(np.int64), stamp]
    overall = overall.astype(np.int64)
    cache = {}
    for a, i, kk in zip(*(o.tolist() for o in ovf)):    # CIGARs longer than a key holds (or odd quality characters)
        if a not in cache:
            cache[a] = flat.columns(a), flat.quals(a)
        (_, _, sym, dcount, _, _, lead), quals = cache[a]
        odd_quality = kk < 0
        kk = abs(kk)
        parts = ['D' * min(lead, args.max_del)] if i == 0 else []
        for j in range(kk):
            parts.append(_SYM[sym[i + j]])
            if j + 1 < kk:
                parts.append('D' * min(int(dcount[i + j]), args.max_del))
        cigar = ''.join(parts)
        q = int(quals[i + (kk - 1) // 2]) - 33
        if odd_quality:
            sys.exit(f'Error: quality character {chr(q + 33)!r} outside the Phred+33 range')
        stamp = (a << 36) | (((kk - 1) // 2) << 32) | i
        entry = table.setdefault(cigar, [np.zeros(N_Q, dtype=np.int64), stamp])
        entry[0][q] += 1
        entry[1] = min(entry[1], stamp)
    print_qscore_fractions('overall', {q: int(c) for q, c in enumerate(overall) if c}, 0)
    order = sorted(table, key=lambda c: table[c][1])                       # insertion order of the reference's dict ...
    order.sort(key=lambda c: int(table[c][0].sum()), reverse=True)        # ... then stably by how common the CIGAR is
    for n, cigar in enumerate(order, start=1):
        print_qscore_fractions(cigar, {q: int(c) for q, c in enumerate(table[cigar][0]) if c}, args.min_occur)
        if n >= args.max_output:
            break
