"""PAF through bb_aln_parse (host code, no GPU): the bb_aln_view of a PAF file equals model_builders.Alignment line by
line - on the golden set and on crafted lines (line ends, repeated tags, tags in the first columns, junk in CIGARs) - the
failing lines give Alignment's messages, and a seeded CIGAR fuzz equals _CIGAR_RUN.findall."""
import ctypes
import os
import random

import numpy as np
import pytest

HERE = os.path.dirname(os.path.realpath(__file__))
PAF = os.path.join(HERE, 'golden', 'models', 'reads.paf')


@pytest.fixture(scope='module')
def mb():
    from badread_b200 import model_builders
    return model_builders


def parse(data, max_alignments=0):
    """(records as dicts, error message or None) of PAF bytes."""
    from badread_b200 import _lib
    from badread_b200.model_builders import _record_arrays, _view_array
    L = _lib.lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    handle = ctypes.c_void_p()
    rc = L.bb_aln_parse(buf.ctypes.data_as(ctypes.c_void_p) if buf.size else None, buf.size, _lib.BB_ALN_PAF, max_alignments,
                        ctypes.byref(handle))
    if rc != _lib.BB_OK:
        return None, L.bb_model_error().decode()
    try:
        v, n, ref_names, read_names, a = _record_arrays(handle)
        cigar_off = _view_array(v.cigar_off, n + 1, np.int64)
        cigar = _view_array(v.cigar, int(cigar_off[-1]), np.uint32)
    finally:
        L.bb_aln_free(handle)
    out = []
    for i in range(n):
        runs = [(int(c) >> 4, int(c) & 15) for c in cigar[cigar_off[i]:cigar_off[i + 1]]]
        out.append(dict(read_name=read_names[a['read_id'][i]], ref_name=ref_names[a['ref_id'][i]],
                        strand='-' if a['flag'][i] & 16 else '+', read_start=int(a['read_start'][i]),
                        read_end=int(a['read_end'][i]), ref_start=int(a['ref_start'][i]), ref_end=int(a['ref_end'][i]),
                        num_bases=int(a['columns'][i]), matching_bases=int(a['columns'][i]) - int(a['nm'][i]),
                        alignment_score=int(a['score'][i]), runs=runs))
    return out, None


def expected(mb, text, max_alignments=None):
    """What load_alignments' loop makes of the text (read in text mode), as parse() reports it."""
    import io
    out = []
    try:
        for n, line in enumerate(io.StringIO(text, newline=None), start=1):
            x = mb.Alignment(line)
            runs = [(int(c), {'M': 0, 'I': 1, 'D': 2}.get(t, 15)) for c, t in mb._CIGAR_RUN.findall(x.cigar)]
            out.append(dict(read_name=x.read_name, ref_name=x.ref_name, strand='-' if x.strand == '-' else '+',
                            read_start=x.read_start, read_end=x.read_end, ref_start=x.ref_start, ref_end=x.ref_end,
                            num_bases=x.num_bases, matching_bases=x.matching_bases, alignment_score=x.alignment_score,
                            runs=[(c if t != 15 else 0, t) for c, t in runs]))
            if n == max_alignments:
                break
    except SystemExit as e:
        return None, str(e)
    return out, None


def test_golden_paf(mb):
    data = open(PAF, 'rb').read()
    got = parse(data)
    assert got == expected(mb, data.decode())
    assert len(got[0]) > 100
    assert parse(data, 50)[0] == got[0][:50]


LINE = 'r1\t500\t10\t400\t{strand}\tctg\t9000\t100\t495\t350\t{cols}\t60{tags}'


@pytest.mark.parametrize('text', [
    LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:390M5D') + '\r\n' + LINE.format(strand='-', cols=410, tags='\tcg:Z:3M\tAS:i:9') + '\r',
    LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:390M5D') + '\r' + LINE.format(strand='-', cols=401, tags='\tcg:Z:3M\tAS:i:9'),
    LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:390M5D\x1c') + '\n' + LINE.format(strand='-', cols=400, tags='\tAS:i:-2 ') + '\tcg:Z:1=2X3M\n',
    LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:390M5D\tAS:i:8\tcg:Z:4I5M') + '\n',          # repeated tags: the last
    'cg:Z:5M\tAS:i:3\t1\t6\t+\tc\t10\t0\t5\t5\t6\tx\n',                                              # tags among the first columns
    LINE.format(strand='*', cols=400, tags='\tAS:i:1\tcg:Z:#12M3=4X 5D12x7S99!8I3H0M007N') + '\n',
    ' \t' + LINE.format(strand='+', cols=400, tags='\tAS:i:+4\tcg:Z:10M') + ' \x0b\n',
    '',
])
def test_crafted_lines(mb, text):
    assert parse(text.encode()) == expected(mb, text)


@pytest.mark.parametrize('text', [
    '\n',                                                                              # a blank line
    'a\tb\tc\n',                                                                       # fewer than 11 columns
    LINE.format(strand='+', cols=400, tags='\tAS:i:7') + '\n',                         # no CIGAR
    LINE.format(strand='+', cols=400, tags='\tcg:Z:10M') + '\n',                       # no score
    LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:10M') + '\n' + 'bad line\n',
])
def test_failing_lines(mb, text):
    want = expected(mb, text)
    assert want[0] is None
    assert parse(text.encode()) == want


def test_max_alignments_stops_before_a_bad_line(mb):
    good = LINE.format(strand='+', cols=400, tags='\tAS:i:7\tcg:Z:10M') + '\n'
    text = good * 3 + 'not PAF\n'
    assert parse(text.encode(), 3) == expected(mb, text, 3)
    assert parse(text.encode(), 3)[1] is None


@pytest.mark.parametrize('text', [LINE.format(strand='+', cols='4x0', tags='\tAS:i:7\tcg:Z:10M') + '\n',
                                  LINE.format(strand='+', cols=400, tags='\tAS:i:7.5\tcg:Z:10M') + '\n'])
def test_bad_integers_exit_with_an_error(text):
    records, msg = parse(text.encode())
    assert records is None and msg.startswith('Error: ')


def test_cigar_fuzz(mb):
    rnd = random.Random(11)
    alphabet = '0123456789MIDX=SHNmid#* '
    for _ in range(400):
        cg = ''.join(rnd.choice(alphabet) for _ in range(rnd.randrange(0, 40)))
        text = LINE.format(strand=rnd.choice('+-'), cols=400, tags=f'\tAS:i:1\tcg:Z:{cg}') + '\n'
        assert parse(text.encode()) == expected(mb, text), cg
