"""The model builders' device route off the GPU: the FASTQ parser (csrc/bb_fastq.cuh) under the warp emulator against
model_builders.load_fastq - the edge cases, tile sizes 1, 7, 64 and the device's with records straddling tile edges at
every offset, a line longer than a tile, gzip and BGZF through the emulated inflaters, a seeded fuzz - and the slice
gather with the library's host planning (fq_plan) against FlatAlignments on the golden set and the edges, hot and long
sets of tests/model_counts_ref.py."""
import gzip
import io
import os
import random

import numpy as np
import pytest

import model_counts_ref as R
from emu import emu_fastq as EF
from emu import emu_gunzip as EG
from emu import emu_inflate as EI
from test_model_builders_alignments import bgzf

HERE = os.path.dirname(os.path.realpath(__file__))
DATA = os.path.join(HERE, 'golden', 'models')
ARRAYS = ('read', 'qual', 'ref', 'read_off', 'ref_off', 'ops_off', 'ops', 'op_read0', 'op_ref0')
TILES = [(1, 1), (7, 1), (64, 2), (EF.TILE, EF.LPT)]        # (bytes per tile, lines per thread)

CASES = {
    'crlf': b'@r1 x\r\nACGTAC\r\n+\r\nIIIIII\r\n@r2\r\nGGAC\r\n+\r\n!!!!\r\n',
    'blank_lines': b'@r1\nACGTAC\n+\nIIIIII\n\n\n  \n@r2\nGGAC\n+\n!!!!\n',
    'at_in_fields': b'@r1\n@CGTAC\n+\n@IIIII\n@r2\nGGAC\n@\n@@@@\n',
    'spaces': b'@r0\nA\n+\nI\n \t@r1\x0b rest\x0c\n \tacgTAC\x0b\n+ \n \x0cIIIIII \n\x0b@r2\nGGAC\n+\n!!!!\n',
    'name_after_spaces': b'@  r1 rest\nACGTAC\n+\nIIIIII\n@r2\tz\nGGAC\n+\n!!!!\n',
    'lower_case': b'@r1\nacgtnx\n+\nabcdef\n',
    'empty_fields': b'@r1\n\n+\n\n@r2\nGGAC\n+\n\n',
    'repeated': b'@r1\nAAAAAA\n+\n!!!!!!\n@r2\nGGAC\n+\n!!!!\n@r1\nACGTAC\n+\nIIIIII\n',
    'no_final_newline': b'@r1\nACGTAC\n+\nIIIIII\n@r2\nGGAC\n+\n!!!!',
    'long_line': b'@r1\n' + b'ACGT' * 5000 + b'\n+\n' + b'I' * 20000 + b'\n@r2\nGGAC\n+\n!!!!\n',
    'junk_between': b'@r1\nACGTAC\n+\nIIIIII\nnot a header\n+\n@r2\nGGAC\n+\n!!!!\n',
}


def host(text, tmp_path, name='reads.fastq'):
    from badread_b200.model_builders import load_fastq
    p = tmp_path / name
    p.write_bytes(text)
    return load_fastq(str(p), output=io.StringIO())


@pytest.mark.parametrize('tile,lpt', TILES)
@pytest.mark.parametrize('case', sorted(CASES))
def test_cases(tmp_path, case, tile, lpt):
    if tile == 1 and case == 'long_line':
        pytest.skip('one CTA per byte: covered by the other tiles')
    assert EF.load(CASES[case], tile, lpt) == host(CASES[case], tmp_path)


def test_records_straddle_tiles_at_every_offset(tmp_path):
    """Three records behind a prefix of every length up to 70 bytes: every record edge falls on every tile offset."""
    body = b'@a x\nACgT\n+\nIIII\n \n@b\n\nxx+\n!!\n@c\tq\nN\n+\n~'
    for k in range(71):
        text = b'@p\n' + b'C' * k + b'\n+\n' + b'I' * k + b'\n' + body
        want = host(text, tmp_path)
        for tile, lpt in TILES[:3]:
            assert EF.load(text, tile, lpt) == want, (k, tile)


def test_scan_ctas_take_several_tiles(tmp_path):
    """More line tiles than the scan CTAs have threads (16 here, 1 024 on the device): each thread composes a run of
    tiles, from every start state."""
    rnd = random.Random(3)
    parts = []
    for i in range(700):
        parts.append(b'\n' * rnd.randrange(0, 3) + b'@r%d junk\n' % i + b'ACGT'[:rnd.randrange(0, 4)] + b'\n+\n' + b'I' * rnd.randrange(0, 4) + b'\n')
    text = b''.join(parts)
    want = host(text, tmp_path)
    for tile, lpt in ((1, 1), (64, 1), (100, 3)):
        assert EF.load(text, tile, lpt) == want


@pytest.mark.parametrize('kind', ['gzip', 'bgzf'])
def test_compressed_through_the_emulated_inflaters(tmp_path, kind):
    raw = open(os.path.join(DATA, 'reads.fastq'), 'rb').read()
    stream = gzip.compress(raw, 6) if kind == 'gzip' else bgzf(raw, sizes=[7000, 65280])
    text = bytes(EG.gunzip(stream)[0] if kind == 'gzip' else EI.decompress(stream))
    assert text == raw
    assert EF.load(text, 64, 2) == host(stream, tmp_path, 'reads.fastq.gz')


def test_fuzz(tmp_path):
    """Seeded FASTQ over '@ + A c N I ! \\n \\r \\t space', compared wherever load_fastq does not raise; where it raises
    (a header without a name, a truncated last record) the parse fails too."""
    rnd = random.Random(5)
    alphabet = [b'@', b'+', b'A', b'c', b'N', b'I', b'!', b'\n', b'\r', b'\t', b' ']
    compared = failed = 0
    for _ in range(400):
        text = b'@' + b''.join(rnd.choice(alphabet) for _ in range(rnd.randrange(1, 300)))
        try:
            want = host(text, tmp_path)
        except (IndexError, StopIteration):
            with pytest.raises(EF.ParseError):
                EF.parse(text, rnd.choice([1, 7, 64]), rnd.choice([1, 2]))
            failed += 1
            continue
        tile, lpt = rnd.choice(TILES)
        assert EF.load(text, tile, lpt) == want, text
        compared += 1
    assert compared > 100 and failed > 20


@pytest.mark.parametrize('text,why', [(b'@r1\nACGT\n+\nIIII\n@\nAC\n+\nII\n', ('name', 1)),
                                      (b'@r1\nACGT\n+\nIIII\n  @ \t\nAC\n+\nII\n', ('name', 1)),
                                      (b'@r1\nACGT\n+\nIIII\n@r2\nAC\n+\n', ('truncated', 1)),
                                      (b'@r1\nACGT', ('truncated', 0))])
def test_parse_errors_name_the_record(text, why):
    with pytest.raises(EF.ParseError) as e:
        EF.parse(text, 7, 1)
    assert e.value.args[0] == why


# ------------------------------------------------------------------------------------------------ the gather
def _same(got, want):
    assert got.n == want.n
    for f in ARRAYS:
        g, w = getattr(got, f), getattr(want, f)
        assert g.dtype == w.dtype and np.array_equal(g, w), f


def _host_flat(fastq, paf, refs):
    from badread_b200 import model_builders as mb
    sink = io.StringIO()
    return mb.FlatAlignments(mb.load_alignments(str(paf), None, output=sink), mb.load_fastq(str(fastq), output=sink), refs, sink, 1000)


def test_gather_equals_flat_alignments_on_the_golden_set():
    from badread_b200.misc import load_fasta
    refs = load_fasta(os.path.join(DATA, 'ref.fasta'))[0]
    fastq, paf = os.path.join(DATA, 'reads.fastq'), os.path.join(DATA, 'reads.paf')
    want = _host_flat(fastq, paf, refs)
    for tile, lpt in ((64, 2), (EF.TILE, EF.LPT)):
        _same(EF.flat(open(fastq, 'rb').read(), paf, refs, tile, lpt), want)


@pytest.mark.parametrize('name', ['edges', 'hot', 'long'])
def test_gather_equals_flat_alignments_on_the_count_sets(tmp_path, name):
    d = {'edges': R.edges, 'hot': R.hot, 'long': R.long_alignment}[name]()
    text = ''.join(f'@{n}\n{s}\n+\n{q}\n' for n, s, q in d.reads).encode()
    (tmp_path / 'reads.fastq').write_bytes(text)
    (tmp_path / 'reads.paf').write_text(''.join(line if line.endswith('\n') else line + '\n' for line in d.paf))
    _same(EF.flat(text, tmp_path / 'reads.paf', d.refs), _host_flat(tmp_path / 'reads.fastq', tmp_path / 'reads.paf', d.refs))


def test_gather_slices_and_failures(tmp_path):
    """Python slice semantics on the read, on the qualities (shorter than the read) and on the reference, both strands;
    a repeated name takes its last record; a missing read, a missing reference and a non-ASCII read fail in
    FlatAlignments' order."""
    refs = {'c': 'ACGTACGGACTTGACCATGACGATCAGGACTAGG' * 4}
    text = b'@r1\nAAAA\n+\n!!!!\n@r2\nggacNN\n+\n!!!\n@r1\nACGTACGGAC\n+\nIIIIII\n@r3\nAC\xc3\xa9\n+\nIII\n'
    (tmp_path / 'reads.fastq').write_bytes(text)
    lines = [f'{n}\t0\t{a}\t{b}\t{s}\t{c}\t136\t{f}\t{g}\t200\t200\t60\tAS:i:1\tcg:Z:{cg}\n'
             for n, a, b, s, c, f, g, cg in (('r1', 1, -1, '+', 'c', 3, 9, '2M1I2M3D1M'), ('r2', -3, 99, '-', 'c', -20, 400, '1M1D2M9I'),
                                             ('r1', 0, 80000, '-', 'c', 0, 144, '3M2D20I9M'))]
    paf = tmp_path / 'reads.paf'
    paf.write_text(''.join(lines))
    _same(EF.flat(text, paf, refs), _host_flat(tmp_path / 'reads.fastq', paf, refs))
    paf.write_text(lines[1] + lines[0].replace('r1', 'r9') + lines[0].replace('\tc\t', '\tz\t'))
    assert EF.flat(text, paf, refs) == ('read', 1)
    paf.write_text(lines[1] + lines[0].replace('\tc\t', '\tz\t') + lines[0].replace('r1', 'r9'))
    assert EF.flat(text, paf, refs) == ('reference', 1)
    paf.write_text(lines[1] + lines[0].replace('r1', 'r3'))
    assert EF.flat(text, paf, refs) == ('ascii', 1)
