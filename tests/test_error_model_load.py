"""The device error model loader (badread_b200/csrc/bb_em_load.cuh) under the warp emulator against the host loader
(ErrorModel(file)._tables): the golden models and seeded synthetic ones, bit for bit, with text tiles small enough that
lines straddle every kind of tile edge; its fast-path float parser against float(); its restatement of CPython's sum()
against sum(); and every input that must leave the file to the host loader, flagged with its reason."""
import gzip
import io
import pathlib
import random
import struct

import numpy as np
import pytest

from badread_b200 import _lib
from badread_b200.error_model import ErrorModel

GOLDEN = pathlib.Path(__file__).resolve().parent / 'golden' / 'models'
MODELS = sorted(p.name for p in GOLDEN.glob('error_model_*.txt.gz'))
FB = _lib.EM_FALLBACK
TABLE_KEYS = ('row_off', 'cum', 'flags', 'slots', 'pool', 'probs', 'kmer_codes', 'kmer_to_row')


def _emu():
    from emu import emu_em_load
    return emu_em_load


def _host(tmp_path, text, name='model.txt'):
    path = tmp_path / name
    path.write_bytes(text)
    return ErrorModel(str(path), io.StringIO())


def _assert_tables(got, want):
    assert set(got) == set(want)
    for key in TABLE_KEYS:
        if key in want:
            assert got[key].dtype == want[key].dtype, key
            assert got[key].tobytes() == want[key].tobytes(), key


def _assert_rowinfo(rowinfo, t):
    ro, cum, flags = t['row_off'], t['cum'], t['flags']
    e0, e1 = ro[:-1].astype(np.int64), ro[1:].astype(np.int64)
    assert np.array_equal(rowinfo[:, 0], cum[e1 - 1])
    assert np.array_equal(rowinfo[:, 1], cum[e0])
    assert np.array_equal(rowinfo[:, 2], e0)
    assert np.array_equal(rowinfo[:, 3], e1 - e0)
    assert np.array_equal(rowinfo[:, 4], (flags[e0] == 1).astype(np.float64))


def synthetic_model(k, n_rows, seed, max_alts=4, long_alts=False):
    """Model text in the builders' form (kmer,p;alt,p;...;) over n_rows distinct random k-mers: each row the k-mer and
    up to max_alts alternatives made by substitutions, insertions and deletions that keep the first and last base."""
    rnd = random.Random(seed)
    kmers = set()
    while len(kmers) < n_rows:
        kmers.add(''.join(rnd.choice('ACGT') for _ in range(k)))
    lines = []
    for kmer in sorted(kmers, key=lambda _: rnd.random()):
        alts = [kmer]
        for _ in range(rnd.randint(0, max_alts)):
            inner = list(kmer[1:-1])
            for _ in range(rnd.randint(1, 3)):
                op = rnd.random()
                pos = rnd.randint(0, len(inner))
                if op < 0.4 and inner:
                    inner[min(pos, len(inner) - 1)] = rnd.choice('ACGT')
                elif op < 0.7 and inner:
                    del inner[min(pos, len(inner) - 1)]
                else:
                    inner.insert(pos, ''.join(rnd.choice('ACGT') for _ in range(rnd.randint(1, 30 if long_alts else 5))))
            alt = kmer[0] + ''.join(inner)[:62] + kmer[-1]
            if alt not in alts:
                alts.append(alt)
        probs = [rnd.random() for _ in alts]
        scale = rnd.choice([1.0, 0.9, 1.1]) / sum(probs)
        lines.append(''.join(f'{a},{p * scale:.6f};' for a, p in zip(alts, probs)))
    return ('\n'.join(lines) + '\n').encode()


@pytest.mark.parametrize('tile', [16384, 1000, 7, 1])
@pytest.mark.parametrize('name', MODELS)
def test_golden_models(name, tile):
    if tile < 1000 and name not in ('error_model_k4_max50.txt.gz', 'error_model_k5_alt3.txt.gz'):
        pytest.skip('tiny tiles on the small models only')
    text = gzip.open(GOLDEN / name, 'rb').read()
    info, t, rowinfo = _emu().load(text, tile=tile)
    assert info['fallback'] == 0 and info['capacity'] == 0
    want = ErrorModel(str(GOLDEN / name), io.StringIO())
    _assert_tables(t, want._tables)
    _assert_rowinfo(rowinfo, t)
    assert info['k'] == want.kmer_size


@pytest.mark.parametrize('name', ['error_model_k5_alt3.txt.gz', 'error_model_k13.txt.gz'])
def test_golden_gzip_through_the_emulated_inflater(name):
    from emu import emu_gunzip
    data = (GOLDEN / name).read_bytes()
    text, _ = emu_gunzip.gunzip(data)
    info, t, _ = _emu().load(text)
    assert info['fallback'] == 0
    _assert_tables(t, ErrorModel(str(GOLDEN / name), io.StringIO())._tables)


@pytest.mark.parametrize('k,seed', [(3, 1), (4, 2), (7, 3), (12, 4), (13, 5), (16, 6)])
def test_synthetic_models(tmp_path, k, seed):
    text = synthetic_model(k, min(4 ** k // 2, 1500), seed, long_alts=True)
    info, t, rowinfo = _emu().load(text, tile=4096)
    assert info['fallback'] == 0
    _assert_tables(t, _host(tmp_path, text)._tables)
    _assert_rowinfo(rowinfo, t)


def test_hash_index_build_has_no_dense_table(tmp_path):
    text = synthetic_model(7, 300, 9)
    info, t, _ = _emu().load(text, dense=False)
    want = dict(_host(tmp_path, text)._tables)
    del want['kmer_to_row']
    _assert_tables(t, want)


def test_last_line_without_newline_and_trailing_separator(tmp_path):
    text = b'AAAA,0.5;ACCA,0.25\nCCCC,1;CC,0\nGGGG,.5;GTG,0.;GAAAAAAAAAG,0.125;'
    info, t, _ = _emu().load(text)
    assert info['fallback'] == 0
    _assert_tables(t, _host(tmp_path, text)._tables)


def test_parse_prob_matches_float():
    emu = _emu()
    rnd = random.Random(11)
    bad = []
    for i in range(1_000_000):
        r = rnd.random()
        s = f'{r * rnd.choice((1.0, 1e-3, 1e-6, 10.0)):.6f}' if i % 4 else f'{rnd.randint(0, 10 ** 9) / 10 ** rnd.randint(0, 9):.{rnd.randint(0, 12)}f}'
        got = emu.parse_prob(s)
        if got is None and int(s.replace('.', '')) >= 2 ** 53:   # off the fast path: the host loader's
            continue
        if got is None or struct.pack('<d', got) != struct.pack('<d', float(s)):
            bad.append(s)
            if len(bad) > 5:
                break
    assert not bad, bad


@pytest.mark.parametrize('s', ['0', '1', '0.0', '1.000000', '.5', '5.', '007.250', '9007199254740991',
                               '0.9007199254740991', '0.' + '0' * 20 + '11', '0.' + '0' * 21 + '1', '123456789.0123456',
                               '0.1', '0.3', '2.225073858507201', '4503599627370497'])
def test_parse_prob_edges(s):
    got = _emu().parse_prob(s)
    assert got is not None and struct.pack('<d', got) == struct.pack('<d', float(s))


@pytest.mark.parametrize('s', ['9007199254740992', '0.' + '1' * 23, '1e5', '1E-3', '-1', '+1', 'inf', 'nan', '', '.',
                               '1_0', '0x1', '1.2.3', '99999999999999999999', '2.2250738585072014'])
def test_parse_prob_off_the_fast_path(s):
    assert _emu().parse_prob(s) is None


def test_pysum_matches_cpython():
    emu = _emu()
    rnd = random.Random(5)
    for _ in range(20000):
        n = rnd.randint(1, 30)
        kind = rnd.random()
        if kind < 0.4:
            xs = [float(f'{rnd.random():.6f}') for _ in range(n)]
        elif kind < 0.7:   # cancelling magnitudes
            xs = [rnd.choice((1.0, -1.0)) * 10.0 ** rnd.randint(-20, 20) * rnd.random() for _ in range(n)]
        else:
            xs = [rnd.choice((1e16, -1e16, 1.0, 0.1, 1e-16, 3.0)) for _ in range(n)]
        assert struct.pack('<d', emu.pysum(xs)) == struct.pack('<d', sum(xs)), xs


FALLBACKS = {
    'exponent': (b'AAAA,1e-1;\n', 'number'),
    'sign': (b'AAAA,-0.1;\n', 'number'),
    'inf': (b'AAAA,inf;\n', 'number'),
    'too_many_digits': (b'AAAA,0.' + b'1' * 23 + b';\n', 'number'),
    'significand_2_53': (b'AAAA,9007199254740992;\n', 'number'),
    'duplicate': (b'AAAA,0.5;\nCCCC,1;\nAAAA,0.25;ACCA,0.5;\n', 'duplicate'),
    'mixed_k': (b'AAAA,0.5;\nCCCCC,1;\n', 'k'),
    'k_2': (b'AA,0.5;\n', 'k'),
    'k_17': (b'A' * 17 + b',0.5;\n', 'k'),
    'non_acgt_kmer': (b'AAAA,0.5;\nACNA,1;\n', 'base'),
    'lowercase': (b'aaaa,0.5;\n', 'base'),
    'non_acgt_alt': (b'AAAA,0.5;ANNA,0.1;\n', 'base'),
    'empty_line': (b'AAAA,0.5;\n\nCCCC,1;\n', 'empty_line'),
    'empty_file': (b'', 'empty_line'),
    'stray_semicolon': (b'AAAA,0.5;;ACCA,0.1;\n', 'syntax'),
    'stray_comma': (b'AAAA,0.5,;\n', 'syntax'),
    'missing_probability': (b'AAAA;\n', 'k'),
    'crlf': (b'AAAA,0.5;\r\nCCCC,1;\r\n', 'cr'),
    'space': (b'AAAA,0.5; \n', 'syntax'),
    'long_alt': (b'AAAA,0.5;A' + b'C' * 64 + b'A,0.1;\n', 'long_alt'),
    'alt_first_base': (b'AAAA,0.5;CAAA,0.1;\n', 'alt_ends'),
    'alt_one_base': (b'AAAA,0.5;A,0.1;\n', 'alt_ends'),
}


@pytest.mark.parametrize('case', sorted(FALLBACKS))
def test_fallbacks_are_flagged(tmp_path, case):
    text, reason = FALLBACKS[case]
    info, t, _ = _emu().load(text)
    assert info['fallback'] & FB[reason], (info, reason)
    assert t is None


def test_pool_offsets_follow_file_order(tmp_path):
    # every alternative pools long slots: the pool is the host's append order byte for byte
    rnd = random.Random(3)
    kmers = sorted({''.join(rnd.choice('ACGT') for _ in range(7)) for _ in range(200)})
    lines = [f'{km},0.5;{km[0]}{"ACGT"[i % 4] * (4 + i % 50)}{km[1:]},0.2;{km[:3]}{"T" * (i % 9)}{km[3:]},0.1;'
             for i, km in enumerate(kmers)]
    text = ('\n'.join(lines) + '\n').encode()
    info, t, _ = _emu().load(text, tile=333)
    assert info['fallback'] == 0 and info['pool_bytes'] > 0
    _assert_tables(t, _host(tmp_path, text)._tables)
