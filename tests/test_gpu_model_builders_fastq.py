"""The model builders' device route on the GPU (FASTQ parsed on the device, PAF parsed by bb_aln_parse, the aligned slices
gathered on the device): the golden model files from plain, gzip and BGZF FASTQ and a gzipped PAF with the host route's
loaders patched to fail, the same progress text; DeviceFlat equal to FlatAlignments array by array on the golden set and
the data sets of tests/model_counts_ref.py; load_fastq's edge cases; the host route's error messages."""
import contextlib
import gzip
import io
import os
import subprocess
import sys
import types

import numpy as np
import pytest

import model_counts_ref as R
from test_model_builders import _golden
from test_model_builders_alignments import MODELS, bgzf

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.realpath(__file__))
DATA = os.path.join(HERE, 'golden', 'models')
ARRAYS = ('read', 'qual', 'ref', 'read_off', 'ref_off', 'ops_off', 'ops', 'op_read0', 'op_ref0')


@pytest.fixture(scope='module')
def mb():
    from badread_b200 import model_builders
    return model_builders


@pytest.fixture(scope='module')
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp('fastq')
    raw = open(os.path.join(DATA, 'reads.fastq'), 'rb').read()
    (d / 'reads.fastq.gz').write_bytes(gzip.compress(raw, 6))
    (d / 'reads.bgzf.fastq.gz').write_bytes(bgzf(raw, sizes=[7000, 65280]))
    (d / 'reads.paf.gz').write_bytes(gzip.compress(open(os.path.join(DATA, 'reads.paf'), 'rb').read(), 6))
    return types.SimpleNamespace(dir=d, fastq={'plain': os.path.join(DATA, 'reads.fastq'), 'gzip': str(d / 'reads.fastq.gz'),
                                              'bgzf': str(d / 'reads.bgzf.fastq.gz')})


def _args(reads, alignment, reference=os.path.join(DATA, 'ref.fasta'), **kw):
    return types.SimpleNamespace(reference=reference, reads=reads, alignment=alignment, **kw)


def _run(fn, args):
    out, err = io.StringIO(), io.StringIO()
    with contextlib.redirect_stdout(out):
        fn(args, output=err)
    return out.getvalue(), err.getvalue()


def _fail(*a, **kw):
    raise AssertionError('the host route ran')


def _host_route(mb, fn, args):
    mb_route = mb.device_route
    mb.device_route = lambda args, fmt: False
    try:
        return _run(fn, args)
    finally:
        mb.device_route = mb_route


@pytest.mark.parametrize('fastq', ['plain', 'gzip', 'bgzf'])
@pytest.mark.parametrize('name,kw', MODELS, ids=[m[0] for m in MODELS])
def test_golden_models_on_the_device_route(mb, files, fastq, name, kw):
    fn = mb.make_error_model if name.startswith('error') else mb.make_qscore_model
    paf = str(files.dir / 'reads.paf.gz') if fastq == 'bgzf' else os.path.join(DATA, 'reads.paf')
    host = _host_route(mb, fn, _args(files.fastq[fastq], paf, **kw))
    saved = {n: getattr(mb, n) for n in ('device_route', 'load_fastq', 'load_alignments', 'FlatAlignments')}
    try:
        mb.device_route = lambda args, fmt: fmt == 'paf'
        mb.load_fastq = mb.load_alignments = mb.FlatAlignments = _fail
        got = _run(fn, _args(files.fastq[fastq], paf, **kw))
    finally:
        for n, f in saved.items():
            setattr(mb, n, f)
    assert got[0] == _golden(name)
    assert got == host


def test_command_line_from_a_gzipped_fastq(files):
    cmd = [sys.executable, '-m', 'badread_b200', 'error_model', '--reference', os.path.join(DATA, 'ref.fasta'), '--reads',
           files.fastq['gzip'], '--alignment', os.path.join(DATA, 'reads.paf')]
    p = subprocess.run(cmd, cwd=os.path.join(HERE, '..'), stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert p.returncode == 0, p.stderr.decode()[-500:]
    assert p.stdout.decode() == _golden('error_model_k7')
    assert b'Loading reads' in p.stderr and b'Processing alignments' in p.stderr


def _flats(mb, reads, paf, reference, max_alignments=None):
    """(DeviceFlat, FlatAlignments) of one input, both routes forced through the route hook."""
    refs = mb.load_fasta(reference)[0]
    args = _args(reads, paf, reference, max_alignments=max_alignments)
    sink = io.StringIO()
    host = mb.load_inputs(args, refs, sink, True)
    want = mb.FlatAlignments(host[1], host[0], refs, sink, 1000)
    inputs = mb._DeviceInputs(args, refs, sink)
    return inputs, inputs.flatten(sink, 1000), want


def _same_arrays(got, want):
    assert got.n == want.n
    for f in ARRAYS:
        g, w = getattr(got, f), getattr(want, f)
        assert g.dtype == w.dtype and np.array_equal(g, w), f


def _write_case(tmp_path, d):
    """A model_counts_ref data set as FASTQ / PAF / FASTA files."""
    (tmp_path / 'reads.fastq').write_text(''.join(f'@{n}\n{s}\n+\n{q}\n' for n, s, q in d.reads))
    (tmp_path / 'reads.paf').write_text(''.join(line if line.endswith('\n') else line + '\n' for line in d.paf))
    (tmp_path / 'ref.fasta').write_text(''.join(f'>{n}\n{s}\n' for n, s in d.refs.items()))
    return str(tmp_path / 'reads.fastq'), str(tmp_path / 'reads.paf'), str(tmp_path / 'ref.fasta')


def test_device_flat_equals_flat_alignments_on_the_golden_set(mb):
    inputs, got, want = _flats(mb, os.path.join(DATA, 'reads.fastq'), os.path.join(DATA, 'reads.paf'), os.path.join(DATA, 'ref.fasta'))
    try:
        _same_arrays(got, want)
        for a in range(0, got.n, 7):
            for x, y in zip(got.columns(a), want.columns(a)):
                assert np.array_equal(x, y)
        for which, k, max_del in (('kmers', 7, 0), ('kmers_wide', 14, 0), ('cigars', 9, 6)):
            for cap, ovf_cap in ((None, None), (16, 0)):
                g, w = mb._count(which, got, k, max_del, cap=cap, ovf_cap=ovf_cap), mb._count(which, want, k, max_del, cap=cap, ovf_cap=ovf_cap)
                gi, wi = np.lexsort(g[1][None, :]), np.lexsort(w[1][None, :])
                for x, y in zip(g[:3], w[:3]):
                    assert np.array_equal(x[gi], y[wi])
                assert np.array_equal(g[3], w[3])
                assert sorted(zip(*(o.tolist() for o in g[4]))) == sorted(zip(*(o.tolist() for o in w[4])))
    finally:
        inputs.close()


@pytest.mark.parametrize('name', ['edges', 'hot', 'diverse', 'long', 'many'])
def test_device_flat_equals_flat_alignments_on_the_count_sets(mb, tmp_path, name):
    d = {'edges': R.edges, 'hot': R.hot, 'diverse': lambda: R.diverse(400), 'long': R.long_alignment, 'many': R.many}[name]()
    inputs, got, want = _flats(mb, *_write_case(tmp_path, d))
    try:
        _same_arrays(got, want)
    finally:
        inputs.close()


# load_fastq's semantics: every case has records a PAF names, so that the gathered slices show the parse
FASTQ_CASES = {
    'crlf': b'@r1 x\r\nACGTAC\r\n+\r\nIIIIII\r\n@r2\r\nGGAC\r\n+\r\n!!!!\r\n',
    'blank_lines': b'@r1\nACGTAC\n+\nIIIIII\n\n\n  \n@r2\nGGAC\n+\n!!!!\n',
    'at_in_fields': b'@r1\n@CGTAC\n+\n@IIIII\n@r2\nGGAC\n@\n@@@@\n',
    'spaces': b'@r0\nA\n+\nI\n \t@r1\x0b rest\x0c\n \tacgTAC\x0b\n+ \n \x0cIIIIII \n@r2\nGGAC\n+\n!!!!\n',
    'name_after_spaces': b'@  r1 rest\nACGTAC\n+\nIIIIII\n@r2\tz\nGGAC\n+\n!!!!\n',
    'empty_fields': b'@r1\n\n+\n\n@r2\nGGAC\n+\n\n',
    'repeated': b'@r1\nAAAAAA\n+\n!!!!!!\n@r2\nGGAC\n+\n!!!!\n@r1\nACGTAC\n+\nIIIIII\n',
    'no_final_newline': b'@r1\nACGTAC\n+\nIIIIII\n@r2\nGGAC\n+\n!!!!',
    'long_line': b'@r1\n' + b'ACGT' * 20000 + b'\n+\n' + b'I' * 80000 + b'\n@r2\nGGAC\n+\n!!!!\n',
    'junk_between': b'@r1\nACGTAC\n+\nIIIIII\nnot a header\n+\n@r2\nGGAC\n+\n!!!!\n',
}


@pytest.mark.parametrize('case', sorted(FASTQ_CASES))
@pytest.mark.parametrize('gz', [False, True], ids=['plain', 'gzip'])
def test_fastq_cases(mb, tmp_path, case, gz):
    raw = FASTQ_CASES[case]
    fq = tmp_path / ('reads.fastq.gz' if gz else 'reads.fastq')
    fq.write_bytes(gzip.compress(raw) if gz else raw)
    ref = 'ACGTACGGACTTGACCATGACGATCAGGACTAGG' * 4
    (tmp_path / 'ref.fasta').write_text(f'>c\n{ref}\n')
    lines = [f'{n}\t0\t{a}\t{b}\t{s}\tc\t{len(ref)}\t{f}\t{g}\t200\t200\t60\tAS:i:1\tcg:Z:{cg}\n'
             for n, a, b, s, f, g, cg in (('r1', 1, -1, '+', 3, 9, '2M1I2M3D1M'), ('r2', -3, 99, '-', 5, 40, '1M1D2M'),
                                          ('r1', 0, 80000, '-', 0, 144, '3M2D200I9M'))]
    (tmp_path / 'reads.paf').write_text(''.join(lines))
    inputs, got, want = _flats(mb, str(fq), str(tmp_path / 'reads.paf'), str(tmp_path / 'ref.fasta'))
    try:
        _same_arrays(got, want)
    finally:
        inputs.close()


def _exit_message(mb, fn, args):
    with pytest.raises(SystemExit) as e:
        _run(fn, args)
    return str(e.value.code)


@pytest.mark.parametrize('case', ['missing_read', 'missing_contig', 'not_fastq', 'bz2', 'short_line', 'no_cigar', 'no_score',
                                  'no_usable'])
def test_error_messages_equal_the_host_route(mb, tmp_path, case):
    fq, paf, ref = tmp_path / 'reads.fastq', tmp_path / 'reads.paf', tmp_path / 'ref.fasta'
    fq.write_text('@r1\n' + 'ACGT' * 50 + '\n+\n' + 'I' * 200 + '\n')
    ref.write_text('>c\n' + 'ACGT' * 100 + '\n')
    line = 'r1\t200\t0\t150\t+\tc\t400\t0\t150\t150\t150\t60\tAS:i:1\tcg:Z:150M\n'
    if case == 'missing_read':
        line = line + line.replace('r1', 'r9')
    elif case == 'missing_contig':
        line = line.replace('\tc\t', '\tc2\t')
    elif case == 'not_fastq':
        fq.write_text('>r1\nACGT\n')
    elif case == 'bz2':
        fq.write_bytes(b'BZh91AY&SY' + b'\0' * 20)
    elif case == 'short_line':
        line = line + 'r2\t1\t2\n'
    elif case == 'no_cigar':
        line = line.replace('\tcg:Z:150M', '')
    elif case == 'no_score':
        line = line.replace('\tAS:i:1', '')
    elif case == 'no_usable':
        line = line.replace('\t150\t150\t60', '\t100\t150\t60')
    paf.write_text(line)
    args = _args(str(fq), str(paf), str(ref), k_size=7, max_alt=25, max_alignments=None)
    saved = mb.device_route
    try:
        mb.device_route = lambda args, fmt: False
        want = _exit_message(mb, mb.make_error_model, args)
        mb.device_route = lambda args, fmt: fmt == 'paf'
        got = _exit_message(mb, mb.make_error_model, args)
    finally:
        mb.device_route = saved
    assert got == want


@pytest.mark.parametrize('text,words', [(b'@r1\nACGT\n+\nIIII\n@\nAC\n+\nII\n', 'record 2 has no read name'),
                                        (b'@r1\nACGT\n+\nIIII\n@r2\nAC\n+\n', 'record 2 (r2) is truncated'),
                                        (b'@r1\nAC\xc3\xa9GT\n+\nIIIII\n', 'read r1 has bytes outside ASCII')])
def test_fastq_errors_name_the_record(mb, tmp_path, text, words):
    fq, paf, ref = tmp_path / 'reads.fastq', tmp_path / 'reads.paf', tmp_path / 'ref.fasta'
    fq.write_bytes(text)
    ref.write_text('>c\n' + 'ACGT' * 100 + '\n')
    paf.write_text('r1\t200\t0\t150\t+\tc\t400\t0\t150\t150\t150\t60\tAS:i:1\tcg:Z:150M\n')
    saved = mb.device_route
    try:
        mb.device_route = lambda args, fmt: fmt == 'paf'
        msg = _exit_message(mb, mb.make_error_model, _args(str(fq), str(paf), str(ref), k_size=7, max_alt=25, max_alignments=None))
    finally:
        mb.device_route = saved
    assert msg.startswith('\nError: ') and words in msg
