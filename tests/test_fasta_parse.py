"""The device FASTA parser (badread_b200/csrc/bb_fasta.cuh) under the warp emulator against misc.load_fasta_arrays: names,
bases, depths and flags on hand-built files and on seeded byte soups, with tiles small enough that every kind of tile
edge occurs."""
import random

import numpy as np
import pytest

from badread_b200.misc import load_fasta_arrays

_DEVICE_TILE = 16384   # FASTA_TILE

CASES = {
    'plain': b'>chr1 circular=true\nACGTACGT\nacgtnn\n>chr2 depth=2.5\nGGGG\n',
    'crlf': b'>a depth=3\r\nACGT\r\nacgt\r\n\r\n>b hairpin_left=true hairpin_right=true\r\nTTTT\r\n',
    'blank_lines': b'\n\n>a\n\nAC\n\n\nGT\n\n>b\n\n',
    'lowercase': b'>x\nacgtrykmswbdhvnz\n',
    'whitespace_in_sequence': b'>x\nAC GT\tAC\x0bGT\x0c\xa0\xffAC \t\n',
    'before_first_header': b'JUNK junk\nmore\n>a\nACGT\n',
    'empty_header': b'>a\nACGT\n>\nTTTT\n>b\nGG\n> \t\r\nCCCC\n',
    'headers_only': b'>a\n>b\n>c',
    'no_trailing_newline': b'>a\nACGT\n>b\nGGCC',
    'empty_file': b'',
    'no_header': b'ACGT\nACGT\n',
    'repeated_names': b'>a first\nAAAA\n>b\nCC\n>a second depth=4 circular=true\nGGG\n>c\nT\n',
    'gt_mid_line': b'>a\nAC>GT\n >x\n>b\nA>\n',
    'header_at_end_without_newline': b'>a\nACGT\n>last depth=2',
    'gt_alone': b'>',
    'newline_only': b'\n',
    'depth_unparseable': b'>a depth=.\nAC\n>b depth=1.2.3\nGG\n>c DEPTH=7\nTT\n',
}


def _long_line_case(tile):
    rs = np.random.RandomState(3)
    seq = bytes(np.frombuffer(b'ACGTacgt', np.uint8)[rs.randint(0, 8, 3 * tile + 17)])
    hdr = b'>long ' + b'x' * (2 * tile + 5) + b' depth=2'
    return hdr + b'\n' + seq + b'\n>short\n' + seq[:tile] + b'\n' + seq


def _newline_last_in_tile(tile):
    """Every tile ends on a newline: lines of exactly `tile` bytes with the newline."""
    body = b'A' * (tile - 1) + b'\n'
    hdr = b'>' + b'h' * (tile - 2) + b'\n'
    return hdr + body * 3 + hdr + body + (b'>' + b'\n') + body


def _load_file(tmp_path, data):
    p = tmp_path / 'ref.fasta'
    p.write_bytes(data)
    return load_fasta_arrays(str(p))


def _comparable(loaded):
    names, seqs, depths, circular, hp_left, hp_right = loaded
    return names, [bytes(s) for s in seqs], depths, circular, hp_left, hp_right


def _assert_same(got, want, what=None):
    assert _comparable(got) == _comparable(want), what


@pytest.mark.parametrize('tile', [1, 2, 3, 7, 64, _DEVICE_TILE])
@pytest.mark.parametrize('case', sorted(CASES))
def test_cases_match_host_loader(tmp_path, case, tile):
    from emu import emu_fasta
    data = CASES[case]
    _assert_same(emu_fasta.load(data, tile), _load_file(tmp_path, data))


@pytest.mark.parametrize('tile', [5, 16, 64, 100])
def test_lines_longer_than_a_tile(tmp_path, tile):
    from emu import emu_fasta
    data = _long_line_case(tile)
    _assert_same(emu_fasta.load(data, tile), _load_file(tmp_path, data))


@pytest.mark.parametrize('tile', [4, 16, 65])
def test_newline_as_a_tiles_last_byte(tmp_path, tile):
    from emu import emu_fasta
    data = _newline_last_in_tile(tile)
    _assert_same(emu_fasta.load(data, tile), _load_file(tmp_path, data))


def test_parse_table_against_definition():
    """The raw header table: every header line's start, end and the bytes kept before it, from a line-by-line count."""
    from emu import emu_fasta
    data = CASES['empty_header'] + CASES['before_first_header'] + CASES['no_trailing_newline']
    kept, start, end, kept_off = emu_fasta.parse(data, 3)
    pos, n_kept, want = 0, 0, []
    for line in data.split(b'\n'):
        if line.startswith(b'>'):
            want.append((pos, pos + len(line), n_kept))
        else:
            n_kept += sum(c not in b'\r \t' for c in line)
        pos += len(line) + 1
    assert list(zip(start.tolist(), end.tolist(), kept_off.tolist())) == want
    assert kept.size == n_kept


_SOUP = [b'A', b'C', b'G', b'T', b'a', b'c', b'g', b't', b'N', b'>', b'\n', b'\r', b' ', b'\t', b'\x0b', b'\xa0']


def test_random_byte_soups(tmp_path):
    """Seeded soups over the alphabet that matters to the parser, in tiles of 1 to 12 bytes."""
    from emu import emu_fasta
    for seed in range(300):
        rnd = random.Random(seed)
        n = rnd.randint(0, 160)
        weights = [rnd.random() for _ in _SOUP]
        weights[_SOUP.index(b'>')] *= 0.5
        data = b''.join(rnd.choices(_SOUP, weights=weights, k=n))
        tile = rnd.randint(1, 12)
        _assert_same(emu_fasta.load(data, tile), _load_file(tmp_path, data), (seed, tile, data))
