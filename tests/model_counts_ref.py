"""
model_counts_ref.py - what `error_model` and `qscore_model` count, from the definition, and seeded inputs for it.
TEST INFRASTRUCTURE (a module the tests import, not a conftest).

The count (DESIGN.md section 4, model builders; the docstrings of csrc/bb_models.cuh):
  an alignment is two gapped column strings, the read's and the reference's.
  error model   the window of reference base r runs from r's column (column 0 for r = 0) to the column of reference base
                r + k - 1; its two strings without their gaps are the reference k-mer and the read k-mer.  Counted if the
                read k-mer has more than one base, both are ACGT only and they agree in their first and last base.
  qscore model  for kk = 1, 3, ..., K the window of read base i runs from i's column (column 0 for i = 0) to the column of
                read base i + kk - 1; its CIGAR is one of = X I D per column with every run of D cut to max_del, its
                quality that of the middle read base.  Every kk = 1 window also counts into `overall`.
Strings are strings here: no packed keys, no length limits, no overflow list.  Dicts keep insertion order, which is the
order of first occurrence (alignment, then window size, then position) that breaks every tie in the model files.

The generators at the bottom make reads, references and PAF lines in memory from a seed.
"""
import collections
import hashlib
import math
import os
import re
import types

import numpy as np

_ACGT = b'ACGT'
_COMP = bytes.maketrans(b'ACGTN', b'TGCAN')


# ---------------------------------------------------------------------------------------------------- columns
def columns(aln, reads, refs):
    """(read columns, reference columns, read qualities without gaps) of one chosen alignment; b'-' is a gap."""
    seq, qual = reads[aln.read_name]
    read = seq[aln.read_start:aln.read_end].encode('latin-1')
    qual = qual[aln.read_start:aln.read_end].encode('latin-1')
    ref = refs[aln.ref_name][aln.ref_start:aln.ref_end].encode('latin-1')
    if aln.strand == '-':
        ref = ref.translate(_COMP)[::-1]
    read_cols, ref_cols, p, r = [], [], 0, 0
    for n, kind in aln.runs:
        if kind == 'M':
            read_cols.append(read[p:p + n]); ref_cols.append(ref[r:r + n]); p += n; r += n
        elif kind == 'I':
            read_cols.append(read[p:p + n]); ref_cols.append(b'-' * n); p += n
        elif kind == 'D':
            read_cols.append(b'-' * n); ref_cols.append(ref[r:r + n]); r += n
    return b''.join(read_cols), b''.join(ref_cols), qual[:p]


def _base_columns(cols):
    return np.flatnonzero(np.frombuffer(cols, dtype=np.uint8) != ord('-')).tolist()


def error_windows(read_cols, ref_cols, k):
    """[(reference k-mer, read k-mer)] of the windows r = 0, 1, ... of one alignment, counted or not."""
    at = _base_columns(ref_cols)
    if len(at) < k:
        return []
    starts, ends = [0] + at[1:len(at) - k + 1], [c + 1 for c in at[k - 1:]]
    return [(ref_cols[s:e].replace(b'-', b''), read_cols[s:e].replace(b'-', b'')) for s, e in zip(starts, ends)]


def error_window_counts(pair):
    ref_kmer, read_kmer = pair
    return len(read_kmer) > 1 and read_kmer[0] == ref_kmer[0] and read_kmer[-1] == ref_kmer[-1] and \
        not ref_kmer.translate(None, _ACGT) and not read_kmer.translate(None, _ACGT)


def cigar_columns(read_cols, ref_cols):
    a, b = np.frombuffer(read_cols, dtype=np.uint8), np.frombuffer(ref_cols, dtype=np.uint8)
    gap = ord('-')
    return np.where(a == gap, ord('D'), np.where(b == gap, ord('I'), np.where(a == b, ord('='), ord('X')))).astype(np.uint8).tobytes()


def qscore_windows(read_cols, ref_cols, qual, kk, max_del):
    """[(CIGAR, quality character code)] of the windows i = 0, 1, ... of kk read bases of one alignment."""
    at = _base_columns(read_cols)
    if len(at) < kk:
        return []
    cig = cigar_columns(read_cols, ref_cols)
    long_run, cut = re.compile(b'D{%d,}' % (max_del + 1)), b'D' * max_del
    starts, ends = [0] + at[1:len(at) - kk + 1], [c + 1 for c in at[kk - 1:]]
    mid = (kk - 1) // 2
    return [(long_run.sub(cut, cig[s:e]), qual[i + mid]) for i, (s, e) in enumerate(zip(starts, ends))]


def _first_positions(keys):
    n = len(keys)
    return dict(zip(reversed(keys), range(n - 1, -1, -1)))


# ---------------------------------------------------------------------------------------------------- counts
def count_error_model(alignments, reads, refs, k):
    """-> (counts {reference k-mer: {read k-mer: count}}, first {(reference k-mer, read k-mer): (alignment, r)},
    windows looked at).  Keys are str."""
    counts, first, n_windows = {}, {}, 0
    for a, aln in enumerate(alignments):
        read_cols, ref_cols, _ = columns(aln, reads, refs)
        wins = error_windows(read_cols, ref_cols, k)
        n_windows += len(wins)
        pos = _first_positions(wins)
        for pair, n in collections.Counter(w for w in wins if error_window_counts(w)).items():
            ref_kmer, read_kmer = pair[0].decode(), pair[1].decode()
            alts = counts.setdefault(ref_kmer, {})
            alts[read_kmer] = alts.get(read_kmer, 0) + n
            first.setdefault((ref_kmer, read_kmer), (a, pos[pair]))
    return counts, first, n_windows


def count_qscore_model(alignments, reads, refs, k, max_del):
    """-> (hist {CIGAR: {quality: count}}, first {CIGAR: (alignment, window size, i)}, overall {quality: count},
    windows looked at).  A quality is the character code minus 33, whatever the character."""
    hist, first, overall, n_windows = {}, {}, collections.Counter(), 0
    for a, aln in enumerate(alignments):
        read_cols, ref_cols, qual = columns(aln, reads, refs)
        for kk in range(1, k + 1, 2):
            wins = qscore_windows(read_cols, ref_cols, qual, kk, max_del)
            n_windows += len(wins)
            if kk == 1:
                overall.update(q - 33 for _, q in wins)
            for cigar, i in _first_positions([c for c, _ in wins]).items():
                first.setdefault(cigar.decode(), (a, kk, i))
            for (cigar, q), n in collections.Counter(wins).items():
                h = hist.setdefault(cigar.decode(), {})
                h[q - 33] = h.get(q - 33, 0) + n
    return hist, first, dict(overall), n_windows


# ---------------------------------------------------------------------------------------------------- model files
def error_model_text(counts, max_alt):
    """One line per reference k-mer in ACGT order: its own fraction, then the other read k-mers by count (stable, so ties
    stay in order of first occurrence), at most max_alt of them; six decimals."""
    lines = []
    for kmer in sorted(counts):
        alts = counts[kmer]
        total = sum(alts.values())
        others = sorted(((a, c) for a, c in alts.items() if a != kmer), key=lambda x: -x[1])[:max_alt]
        lines.append(f'{kmer},{alts.get(kmer, 0) / total:.6f};' + ''.join(f'{a},{c / total:.6f};' for a, c in others))
    return ''.join(line + '\n' for line in lines)


def _fraction(v):
    return str(int(v)) if v == int(v) else ('%.6f' % v).rstrip('0')


def _qscore_line(cigar, h):
    total = sum(h.values())
    return f'{cigar};{total};' + ''.join(f'{q}:{_fraction(h[q] / total)},' for q in sorted(h)) + '\n'


def qscore_model_text(hist, overall, min_occur, max_output):
    """'overall', then the CIGARs by total (stable): the first max_output of them, those below min_occur left out."""
    out = [_qscore_line('overall', overall)]
    order = sorted(hist, key=lambda c: -sum(hist[c].values()))
    for cigar in order[:max_output]:
        if sum(hist[cigar].values()) >= min_occur:
            out.append(_qscore_line(cigar, hist[cigar]))
    return ''.join(out)


# ---------------------------------------------------------------------------------------------------- inputs from a seed
class Dataset(object):
    """refs {name: sequence}, reads [(name, sequence, qualities)], paf [line]; one alignment per read, all of them kept by
    load_alignments (more than 100 columns; the matching-bases column of the PAF line, which only that filter reads, is
    never below 81 % of the columns)."""

    def __init__(self):
        self.refs, self.reads, self.paf = {}, [], []

    def add(self, name, ctg, start, strand, script, qual, head='', tail=''):
        """One alignment of a new read against refs[ctg][start:...].  script, in read orientation: ('M', n) copies n
        reference bases, ('X', n) changes them, ('N', n) reads them as N, ('I', bases) inserts, ('D', n) deletes; every
        item is a CIGAR run of its own except neighbouring M / X / N.  qual: a function of the read length."""
        n_ref = sum(x for op, x in script if op != 'I')
        seg = self.refs[ctg][start:start + n_ref]
        assert len(seg) == n_ref
        if strand == '-':
            seg = seg.encode().translate(_COMP)[::-1].decode()
        out, runs, r, matches = [], [], 0, 0
        for op, x in script:
            if op == 'I':
                out.append(x); runs.append([len(x), 'I'])
                continue
            if op == 'D':
                runs.append([x, 'D']); r += x
                continue
            piece = seg[r:r + x]
            if op == 'X':
                piece = piece.translate(str.maketrans('ACGTN', 'CGTAA'))
            elif op == 'N':
                piece = 'N' * x
            else:
                matches += x
            out.append(piece); r += x
            if runs and runs[-1][1] == 'M':
                runs[-1][0] += x
            else:
                runs.append([x, 'M'])
        aligned = ''.join(out)
        cols = sum(n for n, _ in runs)
        assert cols > 100, (name, cols)
        if strand == '-':
            runs = runs[::-1]
        read = head + aligned + tail
        matches = max(matches, math.ceil(0.81 * cols))
        self.reads.append((name, read, qual(len(read))))
        self.paf.append('\t'.join([name, str(len(read)), str(len(head)), str(len(head) + len(aligned)), strand, ctg,
                                   str(len(self.refs[ctg])), str(start), str(start + n_ref), str(matches), str(cols), '60',
                                   'tp:A:P', f'AS:i:{2 * matches - cols}', 'cg:Z:' + ''.join(f'{n}{t}' for n, t in runs)]))

    def extend(self, other):
        self.refs.update(other.refs); self.reads.extend(other.reads); self.paf.extend(other.paf)
        return self

    def write(self, directory):
        """ref.fasta, reads.fastq and reads.paf in `directory` -> the builders' arguments for them."""
        with open(os.path.join(directory, 'ref.fasta'), 'w') as f:
            for name, seq in self.refs.items():
                f.write(f'>{name}\n{seq}\n')
        with open(os.path.join(directory, 'reads.fastq'), 'w') as f:
            for name, seq, qual in self.reads:
                f.write(f'@{name}\n{seq}\n+\n{qual}\n')
        with open(os.path.join(directory, 'reads.paf'), 'w') as f:
            f.write('\n'.join(self.paf) + '\n')
        return types.SimpleNamespace(reference=os.path.join(directory, 'ref.fasta'), reads=os.path.join(directory, 'reads.fastq'),
                                     alignment=os.path.join(directory, 'reads.paf'), max_alignments=None)


def _dna(rs, n):
    return np.frombuffer(_ACGT, dtype=np.uint8)[rs.randint(0, 4, n)].tobytes().decode()


def _quals(rs, lo='!', hi='~'):
    return lambda n: (rs.randint(ord(lo), ord(hi) + 1, n).astype(np.uint8)).tobytes().decode()


def edges(seed=11, bad_quality=False):
    """One hand-built alignment per edge the golden data does not reach (the test docstrings list them).  bad_quality
    adds one read with a blank, which is not a Phred+33 character, among its qualities."""
    rs = np.random.RandomState(seed)
    d = Dataset()
    d.refs['edge'] = _dna(rs, 40000)
    q, at = _quals(rs, '"', 'I'), iter(range(0, 40000, 700))

    def add(name, script, qual=q, strand='+'):
        d.add('edge_' + name, 'edge', next(at), strand, script, qual, head=_dna(rs, 7), tail=_dna(rs, 3))
    # read k-mers of exactly max_len / max_len + 1 bases: an insertion of L bases makes every window over it k + L long
    for lo in (5, 15, 16, 19, 23):          # 17/18 at k = 12; 22/23 at k = 7; 32/33 at k = 16; 32/33 at k = 13; 26/27 at k = 3
        add(f'ins{lo}_{lo + 1}', [('M', 60), ('I', _dna(rs, lo)), ('M', 60), ('I', _dna(rs, lo + 1)), ('M', 60)])
    # CIGAR windows of exactly 29 and 30 symbols: 9 read bases over 20 / 21 'D' (max_del 6), 13 over 16 / 17 (max_del 2)
    add('cigar29', [('M', 100)] + [('D', 7), ('M', 1)] * 3 + [('D', 2), ('M', 100)])
    add('cigar30', [('M', 100)] + [('D', 7), ('M', 1)] * 3 + [('D', 3), ('M', 100)])
    add('cigar29_k13', [('M', 100)] + [('D', 2), ('M', 1)] * 8 + [('M', 100)])
    add('cigar30_k13', [('M', 100)] + [('D', 2), ('M', 1)] * 8 + [('D', 1), ('M', 100)])
    add('q_ends', [('M', 60), ('X', 1), ('M', 30), ('I', 'AC'), ('M', 30)], qual=lambda n: ('!~' * n)[:n])
    add('n_in_read', [('M', 50), ('N', 1), ('M', 30), ('N', 3), ('M', 40)])
    add('few_ref_bases', [('M', 5), ('I', _dna(rs, 95)), ('M', 5)])
    add('few_read_bases', [('M', 4), ('D', 95), ('M', 4)])
    add('starts_with_i', [('I', 'ACGTT'), ('M', 110)])
    add('ends_with_i', [('M', 110), ('I', 'GGTCA')])
    add('starts_with_d', [('D', 4), ('M', 110)])
    add('ends_with_d', [('M', 110), ('D', 4)])
    add('d_then_i', [('M', 60), ('D', 3), ('I', 'TG'), ('M', 60)])
    add('i_then_d', [('M', 60), ('I', 'CA'), ('D', 3), ('M', 60)])
    add('two_d_runs', [('M', 60), ('D', 2), ('D', 3), ('M', 60)])
    add('minus_strand', [('M', 40), ('I', 'A'), ('M', 40), ('D', 2), ('X', 2), ('M', 40)], strand='-')
    if bad_quality:
        add('bad_quality', [('M', 120)], qual=lambda n: 'I' * 20 + ' ' + 'I' * (n - 21))
    return d


def hot(n_alignments=3000, seed=12):
    """Error-free alignments of 200 bases over homopolymers and dinucleotide repeats, one quality value: a handful of
    keys take every increment.  Among them, alignments inside the poly-A stretch with one inserted base: a C in every
    10th alignment from the start, a G in every 5th of the second half, equally many of each.  Every window over such an
    insertion is a read k-mer (and a CIGAR) seen once per alignment, so the C and G alternatives of AAA..A have equal counts,
    and the order of their lines is that of their first occurrences, which lie in alignments far apart."""
    rs = np.random.RandomState(seed)
    d = Dataset()
    d.refs['low'] = 'A' * 3000 + 'AC' * 1000 + 'T' * 2000 + 'GA' * 1000 + 'C' * 1500 + 'TG' * 750
    n_tie = n_alignments // 10
    c_at = set(range(3, n_alignments, 10)[:n_tie])
    g_at = set(range(n_alignments // 2 + 1, n_alignments, 5)[:n_tie])
    assert len(c_at) == len(g_at) == n_tie
    for i in range(n_alignments):
        if i in c_at or i in g_at:
            left = int(rs.randint(40, 160))
            script = [('M', left), ('I', 'C' if i in c_at else 'G'), ('M', 200 - left)]
            d.add(f'hot{i:05d}', 'low', int(rs.randint(0, 2700)), '+', script, lambda n: '5' * n)
        else:
            d.add(f'hot{i:05d}', 'low', int(rs.randint(0, len(d.refs['low']) - 200)), '+', [('M', 200)], lambda n: '5' * n)
    return d


def _noisy_script(rs, seg, rate):
    """Columns drawn one by one: substitutions, deletion and insertion runs (1-3 long, one in ten 5-12), N in the read."""
    script, j, x = [], 0, rs.rand(2 * len(seg) + 16)
    n = 0
    while j < len(seg):
        u = x[n]; n += 1
        if u < rate * 0.4:
            script.append(('X', 1)); j += 1
        elif u < rate:
            run = int(rs.randint(1, 4)) if rs.rand() < 0.9 else int(rs.randint(5, 13))
            if u < rate * 0.7:
                run = min(run, len(seg) - j)
                script.append(('D', run)); j += run
            else:
                script.append(('I', _dna(rs, run)))
        elif u > 0.998:
            script.append(('N', 1)); j += 1
        else:
            script.append(('M', 1)); j += 1
    merged = []
    for op, v in script:        # (neighbouring M columns as one item: the script stays short)
        if op == 'M' and merged and merged[-1][0] == 'M':
            merged[-1] = ('M', merged[-1][1] + v)
        else:
            merged.append((op, v))
    return merged


def diverse(n_alignments=300, length=1250, seed=13, name='div', aligned_ends=False):
    """Noisy alignments of both strands: 25-30 % of the columns are errors, indel runs up to 12, N in reads and
    reference, qualities over the whole '!'..'~' range; they start and end with whatever column was drawn (aligned_ends:
    with an aligned column)."""
    rs = np.random.RandomState(seed)
    d = Dataset()
    ctg = name + '_ctg'
    ref = np.frombuffer(_dna(rs, 60000).encode(), dtype=np.uint8).copy()
    ref[rs.rand(ref.size) < 0.002] = ord('N')
    d.refs[ctg] = ref.tobytes().decode()
    q = _quals(rs)
    for i in range(n_alignments):
        start, strand = int(rs.randint(0, ref.size - length)), '+-'[int(rs.randint(0, 2))]
        seg = d.refs[ctg][start:start + length]
        script = _noisy_script(rs, seg, 0.25 + 0.05 * rs.rand())
        while aligned_ends and script[0][0] in 'ID':
            script.pop(0)
        while aligned_ends and script[-1][0] in 'ID':
            script.pop()
        d.add(f'{name}{i:05d}', ctg, start, strand, script, q, head=_dna(rs, int(rs.randint(0, 30))))
    return d


def long_alignment(seed=14):
    """One alignment of 150 kb: 25 kb of noisy columns, a single M run of 100 kb, 25 kb of noisy columns."""
    rs = np.random.RandomState(seed)
    d = Dataset()
    d.refs['long_ctg'] = _dna(rs, 150000)
    seg = d.refs['long_ctg']
    script = _noisy_script(rs, seg[:25000], 0.1) + [('D', 1), ('M', 100000), ('I', 'T')] + _noisy_script(rs, seg[125001:], 0.1)
    d.add('long', 'long_ctg', 0, '+', script, _quals(rs, '#', 'Z'))
    assert '100000M' in d.paf[0]
    return d


def many(n_alignments=70000, seed=15):
    """Short alignments (102-105 columns, one substitution and one single-base indel each), more of them than a 16-bit
    index counts."""
    rs = np.random.RandomState(seed)
    d = Dataset()
    d.refs['many_ctg'] = _dna(rs, 20000)
    starts, cut, kind = rs.randint(0, 19800, n_alignments), rs.randint(10, 90, n_alignments), rs.randint(0, 2, n_alignments)
    extra = rs.randint(0, 4, n_alignments)
    q = _quals(rs, '+', 'K')
    for i in range(n_alignments):
        c = int(cut[i])
        indel = ('I', 'ACGT'[int(extra[i])]) if kind[i] else ('D', 1)
        d.add(f'm{i:05d}', 'many_ctg', int(starts[i]), '+', [('M', c), ('X', 1), ('M', 5), indel, ('M', 95 + int(extra[i]) - c)], q)
    return d


# the mix oracle/make_golden_model_stress.py runs the unmodified reference on (tests/golden/golden_model_stress.json)
STRESS_LEFT_OUT = ('edge_starts_with_i', 'edge_starts_with_d', 'edge_ends_with_d')
STRESS_MODELS = [('error_model_k7', 'error', dict(k_size=7, max_alt=25)), ('error_model_k12', 'error', dict(k_size=12, max_alt=25)),
                 ('qscore_model_k9', 'qscore', dict(k_size=9, max_del=6, min_occur=1, max_output=10000))]


def stress_mix():
    """400 hot alignments, 60 diverse ones of 600 reference bases that start and end on an aligned column, and the edges without
    STRESS_LEFT_OUT."""
    d = hot(400).extend(diverse(60, 600, name='mix', aligned_ends=True))
    e = edges()
    keep = [i for i, (name, _, _) in enumerate(e.reads) if name not in STRESS_LEFT_OUT]
    d.refs.update(e.refs)
    d.reads.extend(e.reads[i] for i in keep)
    d.paf.extend(e.paf[i] for i in keep)
    return d


def stress_digest(text):
    lines = text.splitlines()
    return {'sha256': hashlib.sha256(text.encode()).hexdigest(), 'lines': len(lines), 'first': lines[:3], 'last': lines[-3:]}


def load(args):
    """(chosen alignments, reads, references) of written inputs, through the builders' own loaders."""
    import io
    from badread_b200 import model_builders as mb
    from badread_b200.misc import load_fasta
    sink = io.StringIO()
    return mb.load_alignments(args.alignment, None, output=sink), mb.load_fastq(args.reads, output=sink), load_fasta(args.reference)[0]
