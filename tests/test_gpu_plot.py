"""
`badread_b200 plot` on the GPU: the device route (FASTQ parsed and slices gathered on the GPU, series by
bb_window_series) prints the reference's --no_plot stdout, and its --windows table, plain and BGZF, holds '%.4f' of the
reference's series (tests/golden/golden_plot.json) and of the restatement (window_identity_ref.py).  The series
themselves equal the restatement bit for bit on the golden set, on seeded noisy sets, on one alignment of 1 Mb and over
many passes of a small position budget.  SAM and BAM versions of the golden PAF give the same stdout and table.
"""
import argparse
import gzip
import io
import os
import random

import numpy as np
import pytest

import window_identity_ref as W
from test_model_builders_alignments import inputs  # noqa: F401 (fixture)
from test_plot import CASES, DATA, GOLDEN, _case, _golden_args, _run, _sha

pytestmark = pytest.mark.gpu


def _host_inputs(ref, reads, paf):
    from badread_b200 import misc
    from badread_b200 import model_builders as mb
    sink = io.StringIO()
    return (mb.load_fastq(reads, output=sink), misc.load_fasta(ref)[0], mb.load_alignments(paf, output=sink))


def _device_series(ref, reads, paf, window, qual, budget=None):
    """plot.window_series of the device route's DeviceFlat."""
    from badread_b200 import misc, plot
    from badread_b200 import model_builders as mb
    args = argparse.Namespace(reference=ref, reads=reads, alignment=paf, max_alignments=None)
    inp = mb._DeviceInputs(args, misc.load_fasta(ref)[0], io.StringIO())
    try:
        flat = inp.flatten(io.StringIO(), 1000, np.zeros((inp.n, 3), np.int64))
        assert isinstance(flat, mb.DeviceFlat)
        kw = {} if budget is None else {'budget': budget}
        return plot.window_series(flat, inp.a['read_start'][inp.chosen], window, qual, **kw)
    finally:
        inp.close()


def _expected(ref, reads, paf, window, qual):
    r, f, alns = _host_inputs(ref, reads, paf)
    parts = [W.alignment_series(a, r, f, window, qual) for a in alns]
    return alns, parts


def _table(alns, parts, qual):
    lines = []
    for a, (pos, ident, mq) in zip(alns, parts):
        for j in range(len(pos)):
            lines.append(f'{a.read_name}\t{pos[j]}\t{ident[j]:.4f}' + (f'\t{mq[j]:.4f}' if qual else '') + '\n')
    return ''.join(lines)


def _golden_paths():
    return os.path.join(DATA, 'ref.fasta'), os.path.join(DATA, 'reads.fastq'), os.path.join(DATA, 'reads.paf')


def test_no_plot_stdout_on_the_device_route():
    p = _run(*_golden_args('--no_plot'))
    assert p.returncode == 0, p.stderr[-500:]
    assert p.stdout == GOLDEN['stdout']


@pytest.mark.parametrize('window,qual', CASES)
def test_device_series_equal_the_reference(window, qual):
    point_off, pos, ident, mq = _device_series(*_golden_paths(), window, qual)
    c = _case(window, qual)
    assert np.diff(point_off).tolist() == c['counts']
    assert _sha(pos, np.int64) == c['positions_sha256']
    assert _sha(ident, np.float64) == c['identity_sha256']
    if qual:
        assert _sha(mq, np.float64) == c['qual_sha256']


@pytest.mark.parametrize('gz', [False, True], ids=['plain', 'bgzf'])
@pytest.mark.parametrize('window,qual', [(100, True), (7, False), (1, True), (2500, True)])
def test_windows_table(tmp_path, window, qual, gz):
    out = tmp_path / ('w.tsv.gz' if gz else 'w.tsv')
    p = _run(*_golden_args('--window', str(window), '--windows', str(out), *(['--qual'] if qual else [])))
    assert p.returncode == 0, p.stderr[-500:]
    assert p.stdout == GOLDEN['stdout']
    text = (gzip.open(out, 'rt') if gz else open(out)).read()
    alns, parts = _expected(*_golden_paths(), window, qual)
    assert text == _table(alns, parts, qual)
    c = _case(window, qual)
    assert text.count('\n') == sum(c['counts'])
    for a, j, _, value in c['samples']:
        line = text.splitlines()[sum(c['counts'][:a]) + j]
        assert line.split('\t')[2] == '%.4f' % float.fromhex(value)


def _noisy_set(tmp_path, seed, n_reads, length, error=0.28, long_indels=True):
    """A seeded set with error-dense CIGARs and indel runs up to 60, both strands; the PAF's identity columns are set
    so that every alignment is chosen."""
    rnd = random.Random(seed)
    ctg = ''.join(rnd.choice('ACGT') for _ in range(length * 2 + 1000))
    fq, paf = [], []
    for i in range(n_reads):
        n = length if n_reads == 1 else rnd.randrange(length // 4, length)
        fs = rnd.randrange(0, len(ctg) - 2 * n)
        runs, body, rp, fp = [], [], 0, 0
        while rp < n:
            r = rnd.random()
            if r < 1 - error:
                k, t = rnd.randrange(1, 12), 'M'
            elif r < 1 - error / 2:
                k, t = (rnd.randrange(10, 60) if long_indels and rnd.random() < 0.05 else rnd.randrange(1, 4)), 'I'
            else:
                k, t = (rnd.randrange(10, 60) if long_indels and rnd.random() < 0.05 else rnd.randrange(1, 4)), 'D'
            if t == 'D' and rp == 0 and rnd.random() < 0.7:
                continue
            runs.append((k, t))
            rp += k if t != 'D' else 0
            fp += k if t != 'I' else 0
        strand = rnd.choice('+-')
        seg = ctg[fs:fs + fp]
        if strand == '-':
            seg = W.reverse_complement(seg)
        q = 0
        for k, t in runs:
            if t == 'M':
                body.append(''.join(c if rnd.random() > error else rnd.choice('ACGT') for c in seg[q:q + k]))
                q += k
            elif t == 'I':
                body.append(''.join(rnd.choice('ACGT') for _ in range(k)))
            else:
                q += k
        lead, trail = rnd.randrange(0, 30), rnd.randrange(0, 30)
        seq = ''.join(rnd.choice('ACGT') for _ in range(lead)) + ''.join(body) + 'A' * trail
        qual = ''.join(chr(33 + rnd.randrange(2, 40)) for _ in seq)
        fq.append(f'@n{i} x\n{seq}\n+\n{qual}\n')
        cigar_runs = runs[::-1] if strand == '-' else runs
        cigar = ''.join(f'{k}{t}' for k, t in cigar_runs)
        cols = rp + sum(k for k, t in runs if t == 'D')
        paf.append(f'n{i}\t{len(seq)}\t{lead}\t{lead + rp}\t{strand}\tc\t{len(ctg)}\t{fs}\t{fs + fp}\t{int(cols * 0.9)}\t{cols}\t60'
                   f'\tAS:i:{rnd.randrange(100, 1000)}\tcg:Z:{cigar}\n')
    (tmp_path / 'ref.fasta').write_text(f'>c\n{ctg}\n')
    (tmp_path / 'reads.fastq').write_text(''.join(fq))
    (tmp_path / 'aln.paf').write_text(''.join(paf))
    return str(tmp_path / 'ref.fasta'), str(tmp_path / 'reads.fastq'), str(tmp_path / 'aln.paf')


def _compare(paths, window, qual, budget=None):
    point_off, pos, ident, mq = _device_series(*paths, window, qual, budget)
    alns, parts = _expected(*paths, window, qual)
    assert np.diff(point_off).tolist() == [len(p[0]) for p in parts]
    assert pos.tobytes() == np.concatenate([p[0] for p in parts]).astype(np.int64).tobytes()
    assert ident.tobytes() == np.concatenate([p[1] for p in parts]).tobytes()
    if qual:
        assert mq.tobytes() == np.concatenate([p[2] for p in parts]).tobytes()
    return point_off


@pytest.mark.parametrize('seed', [1, 2, 3])
@pytest.mark.parametrize('window', [1, 10, 100, 1000])
def test_noisy_sets_equal_the_restatement(tmp_path, seed, window):
    _compare(_noisy_set(tmp_path, seed, 40, 6000), window, True)


def test_one_megabase_alignment(tmp_path):
    paths = _noisy_set(tmp_path, 7, 1, 1_000_000)
    for window in (100, 5000):
        point_off = _compare(paths, window, True)
        assert point_off[-1] > 900_000


def test_many_passes_of_a_small_budget(tmp_path):
    paths = _noisy_set(tmp_path, 9, 120, 3000)
    point_off = _compare(paths, 50, True, budget=4000)       # (about 2 alignments per pass)
    assert len(point_off) == 121
    _compare(paths, 50, False, budget=1)                     # (one alignment per pass: the longest sets the budget)


@pytest.mark.parametrize('fmt', ['sam', 'bam'])
def test_sam_and_bam_give_the_paf_output(tmp_path, inputs, fmt):  # noqa: F811
    argv = ['--reference', os.path.join(DATA, 'ref.fasta'), '--reads', os.path.join(DATA, 'reads.fastq'),
            '--alignment', str(inputs.dir / f'reads.{fmt}'), '--qual', '--window', '50']
    ours, paf = tmp_path / 'a.tsv', tmp_path / 'p.tsv'
    p = _run(*argv, '--windows', str(ours))
    assert p.returncode == 0, p.stderr[-500:]
    assert p.stdout == GOLDEN['stdout']
    q = _run(*_golden_args('--qual', '--window', '50', '--windows', str(paf)))
    assert q.returncode == 0, q.stderr[-500:]
    assert ours.read_bytes() == paf.read_bytes() and paf.stat().st_size > 0
