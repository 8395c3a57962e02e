"""
`badread_b200 plot` on the CPU: the command line and its refusals, the restatement of the window series
(window_identity_ref.py) against the reference's golden series (tests/golden/golden_plot.json, oracle/make_golden_plot.py),
and the series kernel (csrc/bb_plot.cuh) under the warp emulator against both, with tiles small enough that windows and D
runs straddle tile edges at every offset.  The --no_plot run needs no kernel, so its stdout is checked here too.
"""
import hashlib
import json
import os
import random
import subprocess
import sys
import types

import numpy as np
import pytest

import window_identity_ref as W
from emu import emu_plot as EP

HERE = os.path.dirname(os.path.realpath(__file__))
ROOT = os.path.join(HERE, '..')
DATA = os.path.join(HERE, 'golden', 'models')
GOLDEN = json.load(open(os.path.join(HERE, 'golden', 'golden_plot.json')))
CASES = [(c['window'], c['qual']) for c in GOLDEN['cases']]


def _sha(values, dtype):
    return hashlib.sha256(np.asarray(values, dtype=dtype).tobytes()).hexdigest()


def _golden_inputs():
    import io
    from badread_b200 import misc
    from badread_b200 import model_builders as mb
    sink = io.StringIO()
    reads = mb.load_fastq(os.path.join(DATA, 'reads.fastq'), output=sink)
    refs = misc.load_fasta(os.path.join(DATA, 'ref.fasta'))[0]
    alns = mb.load_alignments(os.path.join(DATA, 'reads.paf'), output=sink)
    return reads, refs, alns


def _case(window, qual):
    return next(c for c in GOLDEN['cases'] if c['window'] == window and c['qual'] == qual)


def _run(*argv, cwd=ROOT):
    return subprocess.run([sys.executable, '-m', 'badread_b200', 'plot', *argv], cwd=cwd, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True)


def _golden_args(*extra):
    return ['--reference', os.path.join(DATA, 'ref.fasta'), '--reads', os.path.join(DATA, 'reads.fastq'),
            '--alignment', os.path.join(DATA, 'reads.paf'), *extra]


# ------------------------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize('window,qual', CASES)
def test_restatement_equals_the_reference(window, qual):
    reads, refs, alns = _golden_inputs()
    c = _case(window, qual)
    parts = [W.alignment_series(a, reads, refs, window, qual) for a in alns]
    assert [len(p[0]) for p in parts] == c['counts']
    assert _sha(np.concatenate([p[0] for p in parts]), np.int64) == c['positions_sha256']
    assert _sha(np.concatenate([p[1] for p in parts]), np.float64) == c['identity_sha256']
    for a, j, pos, value in c['samples']:
        assert (int(parts[a][0][j]), float(parts[a][1][j])) == (pos, float.fromhex(value))
    if qual:
        assert _sha(np.concatenate([p[2] for p in parts]), np.float64) == c['qual_sha256']


def test_golden_covers_negative_and_empty_series():
    assert float.fromhex(_case(7, False)['min_identity']) < 0
    assert sum(_case(2500, False)['counts']) == 0


# ------------------------------------------------------------------------------------------------ the command line
def test_no_plot_stdout_equals_the_reference():
    p = _run(*_golden_args('--no_plot'))
    assert p.returncode == 0, p.stderr[-500:]
    assert p.stdout == GOLDEN['stdout']


def test_no_plot_takes_the_window_and_qual_flags():
    p = _run(*_golden_args('--no_plot', '--qual', '--window', '7'))
    assert p.returncode == 0, p.stderr[-500:]
    assert p.stdout == GOLDEN['stdout']


def test_drawing_is_refused_before_loading():
    p = _run('--reference', 'missing.fasta', '--reads', 'missing.fastq', '--alignment', 'missing.paf')
    assert p.returncode != 0
    assert p.stderr.startswith('Error: ') and '--windows' in p.stderr and '--no_plot' in p.stderr
    assert p.stdout == ''


@pytest.mark.parametrize('window', ['0', '-5'])
def test_window_below_one_is_an_argument_error(window):
    p = _run(*_golden_args('--no_plot', '--window', window))
    assert p.returncode == 2
    assert 'argument --window' in p.stderr and 'must be at least 1' in p.stderr


@pytest.mark.parametrize('missing', ['--reference', '--reads', '--alignment'])
def test_required_arguments(missing):
    argv = _golden_args('--no_plot')
    i = argv.index(missing)
    p = _run(*(argv[:i] + argv[i + 2:]))
    assert p.returncode == 2 and 'required' in p.stderr


# ------------------------------------------------------------------------------------------------ refusals
def _write_set(tmp_path, reads, paf_lines, contigs=None):
    """ref.fasta (contigs {name: seq}), reads.fastq (reads {name: (seq, qual)}) and aln.paf in tmp_path."""
    contigs = contigs or {}
    (tmp_path / 'ref.fasta').write_text(''.join(f'>{n}\n{s}\n' for n, s in contigs.items()))
    (tmp_path / 'reads.fastq').write_text(''.join(f'@{n}\n{s}\n+\n{q}\n' for n, (s, q) in reads.items()))
    (tmp_path / 'aln.paf').write_text(''.join(line + '\n' for line in paf_lines))
    return ['--reference', str(tmp_path / 'ref.fasta'), '--reads', str(tmp_path / 'reads.fastq'), '--alignment',
            str(tmp_path / 'aln.paf')]


def _paf(name, rlen, rs, re_, ctg, clen, fs, fe, cigar, strand='+', matches=None, cols=None):
    cols = cols or 200
    matches = cols if matches is None else matches
    return f'{name}\t{rlen}\t{rs}\t{re_}\t{strand}\t{ctg}\t{clen}\t{fs}\t{fe}\t{matches}\t{cols}\t60\tAS:i:100\tcg:Z:{cigar}'


_RND = random.Random(5)
CTG = ''.join(_RND.choice('ACGT') for _ in range(1000))
READ = CTG[100:300]


def _refused(tmp_path, paf_line, qual=None, extra=()):
    ok = _paf('good', 200, 0, 200, 'c', 1000, 100, 300, '200M')
    argv = _write_set(tmp_path, {'good': (READ, 'I' * 200), 'bad': (READ, qual or 'I' * 200)}, [ok, paf_line], {'c': CTG})
    return _run(*argv, '--no_plot', *extra)


@pytest.mark.parametrize('line,why', [
    (_paf('bad', 200, 0, 210, 'c', 1000, 100, 310, '210M'), 'covers 210 read bases but the aligned part of the read has 200'),
    (_paf('bad', 200, 0, 200, 'c', 1000, 100, 250, '150M'), 'covers 150 read bases but the aligned part of the read has 200'),
    (_paf('bad', 200, 0, 200, 'c', 1000, 900, 1100, '200M'), 'reaches past the aligned part of the reference (100 bases)'),
    (_paf('bad', 200, 0, 200, 'c', 1000, 100, 305, '200M5D'), 'has a deletion after the last aligned read base'),
], ids=['read_end_past_the_read', 'cigar_short_of_the_slice', 'ref_end_past_the_contig', 'deletion_at_the_end'])
def test_alignments_the_reference_cannot_plot_are_refused(tmp_path, line, why):
    p = _refused(tmp_path, line)
    assert p.returncode != 0
    assert p.stderr.strip().splitlines()[-1].startswith('Error: alignment bad:0-'), p.stderr
    assert 'of read bad: its CIGAR ' + why in p.stderr
    assert 'good:0-200' not in p.stdout    # nothing is written before every alignment is checked


def test_short_qualities_are_refused_with_qual_only(tmp_path):
    line = _paf('bad', 200, 0, 200, 'c', 1000, 100, 300, '200M')
    p = _refused(tmp_path, line, qual='I' * 150, extra=('--qual',))
    assert p.returncode != 0 and 'the read has fewer qualities (150) than bases (200)' in p.stderr
    p = _refused(tmp_path, line, qual='I' * 150)
    assert p.returncode == 0, p.stderr
    assert p.stdout.splitlines()[-2:] == ['good:0-200(+),c:100-300(100.000%)', 'bad:0-200(+),c:100-300(100.000%)']


def test_missing_read_and_reference_give_the_builders_messages(tmp_path):
    p = _refused(tmp_path, _paf('other', 200, 0, 200, 'c', 1000, 100, 300, '200M'))
    assert p.returncode != 0 and 'Error: could not find read other' in p.stderr
    p = _refused(tmp_path, _paf('bad', 200, 0, 200, 'nowhere', 1000, 100, 300, '200M'))
    assert p.returncode != 0 and 'Error: could not find reference nowhere' in p.stderr


# ------------------------------------------------------------------------------------------------ the kernel, emulated
def _flat(alns, reads, refs):
    import io
    from badread_b200 import model_builders as mb
    return mb.FlatAlignments(alns, reads, refs, io.StringIO(), 1000)


def _expected(alns, reads, refs, window, qual):
    parts = [W.alignment_series(a, reads, refs, window, qual) for a in alns]
    return (np.concatenate([p[1] for p in parts]) if parts else np.zeros(0),
            np.concatenate([p[2] for p in parts]) if qual and parts else None)


@pytest.mark.parametrize('items', [1, 3, 8])
@pytest.mark.parametrize('window,qual', CASES)
def test_emulated_kernel_equals_the_reference(window, qual, items):
    reads, refs, alns = _golden_inputs()
    ident, mq = EP.window_series(_flat(alns, reads, refs), window, qual, items)
    c = _case(window, qual)
    assert ident.size == sum(c['counts'])
    assert _sha(ident, np.float64) == c['identity_sha256']
    if qual:
        assert _sha(mq, np.float64) == c['qual_sha256']


def _aln(name, runs, read_start=0, strand='+', ref_start=0):
    rp = sum(n for n, t in runs if t in 'MI')
    fp = sum(n for n, t in runs if t in 'MD')
    return types.SimpleNamespace(read_name=name, read_start=read_start, read_end=read_start + rp, strand=strand,
                                 ref_name='c', ref_start=ref_start, ref_end=ref_start + fp, runs=runs)


def _edge_set(rnd, n_ref=4000):
    ref = ''.join(rnd.choice('ACGT') for _ in range(n_ref))
    shapes = {
        'leading_d': [(4, 'D'), (60, 'M'), (2, 'I'), (50, 'M')],
        'adjacent_d': [(30, 'M'), (3, 'D'), (5, 'D'), (40, 'M'), (1, 'D'), (1, 'D'), (1, 'D'), (35, 'M')],
        'empty_runs': [(20, 'M'), (7, 'D'), (0, 'I'), (0, 'M'), (30, 'M'), (0, 'D'), (2, 'I'), (60, 'M')],
        'long_d': [(40, 'M'), (300, 'D'), (70, 'M')],
        'eq_x_letters': [(50, 'M'), (10, '='), (5, 'X'), (60, 'M')],
        'insertions': [(10, 'I'), (90, 'M'), (25, 'I'), (15, 'M')],
    }
    reads, alns = {}, []
    for name, runs in shapes.items():
        for strand in '+-':
            a = _aln(f'{name}{strand}', runs, read_start=3, strand=strand, ref_start=rnd.randrange(0, n_ref - 600))
            seg = ref[a.ref_start:a.ref_end]
            if strand == '-':
                seg = W.reverse_complement(seg)
            body, fp = [], 0
            for n, t in runs:
                if t == 'M':
                    body.append(''.join(c if rnd.random() > 0.2 else rnd.choice('ACGT') for c in seg[fp:fp + n]))
                    fp += n
                elif t == 'I':
                    body.append(''.join(rnd.choice('ACGT') for _ in range(n)))
                elif t == 'D':
                    fp += n
            seq = 'GGG' + ''.join(body) + 'TT'
            reads[a.read_name] = (seq, ''.join(chr(33 + rnd.randrange(0, 94)) for _ in seq))
            alns.append(a)
    return reads, {'c': ref}, alns


@pytest.mark.parametrize('items', [1, 2, 5])
@pytest.mark.parametrize('window', [1, 2, 3, 7, 31, 64, 65, 129])
def test_emulated_kernel_on_edge_cigars(window, items):
    reads, refs, alns = _edge_set(random.Random(11))
    flat = _flat(alns, reads, refs)
    ident, mq = EP.window_series(flat, window, True, items)
    exp_i, exp_q = _expected(alns, reads, refs, window, True)
    assert ident.tobytes() == exp_i.tobytes()
    assert mq.tobytes() == exp_q.tobytes()


def test_emulated_kernel_at_windows_around_the_length():
    reads, refs, alns = _edge_set(random.Random(12))
    flat = _flat(alns, reads, refs)
    for a in range(flat.n):
        L = int(flat.read_off[a + 1] - flat.read_off[a])
        one = types.SimpleNamespace(n=1, read=flat.read[flat.read_off[a]:flat.read_off[a + 1]],
                                    qual=flat.qual[flat.read_off[a]:flat.read_off[a + 1]],
                                    ref=flat.ref[flat.ref_off[a]:flat.ref_off[a + 1]] if flat.ref_off[a + 1] > flat.ref_off[a] else flat.ref[:1],
                                    read_off=np.array([0, L], np.int64),
                                    ref_off=np.array([0, flat.ref_off[a + 1] - flat.ref_off[a]], np.int64),
                                    ops=flat.ops[flat.ops_off[a]:flat.ops_off[a + 1]],
                                    op_read0=flat.op_read0[flat.ops_off[a]:flat.ops_off[a + 1]],
                                    op_ref0=flat.op_ref0[flat.ops_off[a]:flat.ops_off[a + 1]],
                                    ops_off=np.array([0, flat.ops_off[a + 1] - flat.ops_off[a]], np.int64))
        for window in (L - 1, L, L + 1):
            ident, _ = EP.window_series(one, window, False, 3)
            exp = _expected([alns[a]], reads, refs, window, False)[0]
            assert ident.size == max(L - window, 0)
            assert ident.tobytes() == exp.tobytes()


def test_emulated_kernel_on_noisy_reads():
    rnd = random.Random(21)
    ref = ''.join(rnd.choice('ACGT') for _ in range(20000))
    reads, alns = {}, []
    for i in range(12):
        runs, n_read = [], 0
        while n_read < rnd.randrange(150, 1500):
            t = rnd.choices('MID', weights=(70, 15, 15))[0]
            n = rnd.randrange(1, 4) if t == 'M' or rnd.random() < 0.8 else rnd.randrange(5, 40)
            if not runs and t == 'D' and rnd.random() < 0.5:
                n = 1
            runs.append((n, t))
            n_read += n if t != 'D' else 0
        while runs[-1][1] == 'D':
            runs.pop()
        a = _aln(f'r{i}', runs, read_start=rnd.randrange(0, 50), strand=rnd.choice('+-'), ref_start=rnd.randrange(0, 15000))
        seq = ''.join(rnd.choice('ACGT') for _ in range(a.read_end))
        reads[a.read_name] = (seq, ''.join(chr(33 + rnd.randrange(0, 60)) for _ in seq))
        alns.append(a)
    flat = _flat(alns, reads, {'c': ref})
    for window, items in ((1, 1), (5, 2), (40, 3), (100, 8)):
        ident, mq = EP.window_series(flat, window, True, items)
        exp_i, exp_q = _expected(alns, reads, {'c': ref}, window, True)
        assert ident.tobytes() == exp_i.tobytes() and mq.tobytes() == exp_q.tobytes()
