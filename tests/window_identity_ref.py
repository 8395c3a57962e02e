"""A restatement of `badread plot`'s window series from its definition, pinned to tests/golden/golden_plot.json (which
the unmodified reference wrote) and used where the reference cannot finish or the data is too large to store.  It
shares no code with badread_b200's kernel.  TEST INFRASTRUCTURE.

For an aligned read slice of length L: e[p] = 1 for an M base whose read and reference bases differ and for an I base,
plus n at the read offset where a D run of n starts; other CIGAR letters are skipped.  For i in range(L - w): position
read_start + i + w // 2, identity 100.0 * (1.0 - S / w) and mean qscore Q / w, with S and Q the integer sums of e and of
(ord(q) - 33) over [i, i + w).  numpy's float64 operations round as Python's do, so the values are bit-identical."""
import re

import numpy as np

_COMP = str.maketrans('ACGTacgtNn', 'TGCAtgcaNn')


def errors_per_position(read_seq, ref_seq, runs):
    """e[0..len(read_seq)) of an alignment whose runs [(count, letter)] are in read orientation and ref_seq is on the
    read's strand."""
    e = np.zeros(len(read_seq), dtype=np.int64)
    read = np.frombuffer(read_seq.encode('latin-1'), dtype=np.uint8)
    ref = np.frombuffer(ref_seq.encode('latin-1'), dtype=np.uint8)
    rp = fp = 0
    for count, letter in runs:
        if letter == 'M':
            e[rp:rp + count] += read[rp:rp + count] != ref[fp:fp + count]
            rp += count
            fp += count
        elif letter == 'I':
            e[rp:rp + count] += 1
            rp += count
        elif letter == 'D':
            e[rp] += count
            fp += count
    return e


def window_means(values, window, read_start):
    """get_window_means of integer values: (positions, means) as int64 / float64 arrays; S / w in float64."""
    values = np.asarray(values, dtype=np.int64)
    n = max(len(values) - window, 0)
    s = np.concatenate([[0], np.cumsum(values)])
    sums = s[window:window + n] - s[:n]
    return read_start + np.arange(n, dtype=np.int64) + window // 2, sums / np.float64(window)


def series(read_seq, read_qual, ref_seq, runs, read_start, window, qual=False):
    """(positions, identities, mean qscores or None) of one alignment."""
    pos, mean = window_means(errors_per_position(read_seq, ref_seq, runs), window, read_start)
    identity = 100.0 * (1.0 - mean)
    mq = None
    if qual:
        q = np.frombuffer(read_qual.encode('latin-1'), dtype=np.uint8).astype(np.int64) - 33
        mq = window_means(q, window, read_start)[1]
    return pos, identity, mq


def reverse_complement(s):
    return s.translate(_COMP)[::-1]


def paf_runs(cigar, strand):
    runs = [(int(n), t) for n, t in re.findall(r'(\d+)([A-Za-z=])', cigar)]
    return runs[::-1] if strand == '-' else runs


def alignment_series(aln, reads, refs, window, qual=False):
    """series() of an alignment with read_name, read_start, read_end, strand, ref_name, ref_start, ref_end and runs (read
    orientation), against reads {name: (seq, qual)} and refs {name: seq}."""
    seq, q = reads[aln.read_name]
    ref = refs[aln.ref_name][aln.ref_start:aln.ref_end]
    if aln.strand == '-':
        ref = reverse_complement(ref)
    return series(seq[aln.read_start:aln.read_end], q[aln.read_start:aln.read_end], ref, aln.runs, aln.read_start, window,
                  qual)
