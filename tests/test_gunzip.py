"""The gzip inflater of csrc/bb_gunzip.cuh (one deflate stream decoded in parallel chunks) under the warp emulator: its
output equals zlib's byte for byte over zlib's settings, data shapes and member shapes, at the default chunk size and at
small ones that make many chunks; a planted false block start is repaired; corrupt streams are refused with the member
named by index and offset.  CORPUS and REFUSALS are shared with tests/test_gpu_gunzip.py."""
import gzip
import os
import struct
import zlib

import numpy as np
import pytest

import deflate_ref as D
from emu import emu_gunzip

GOLDEN_FASTA = os.path.join(os.path.dirname(__file__), 'golden', 'models', 'ref.fasta')


def gz(data, level=6, wbits=15, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0):
    """One gzip member of data from zlib; flush_every: a sync flush (a block boundary, window kept) every that many bytes."""
    co = zlib.compressobj(level, zlib.DEFLATED, 16 + wbits, mem, strategy)
    if not flush_every:
        return co.compress(data) + co.flush()
    out = b''.join(co.compress(data[i:i + flush_every]) + co.flush(zlib.Z_SYNC_FLUSH) for i in range(0, len(data), flush_every))
    return out + co.flush()


def header(flags=0, extra=b'', name=b'', comment=b''):
    h = b'\x1f\x8b\x08' + bytes([flags]) + b'\0\0\0\0\0\xff'
    if flags & 4:
        h += struct.pack('<H', len(extra)) + extra
    if flags & 8:
        h += name + b'\0'
    if flags & 16:
        h += comment + b'\0'
    if flags & 2:
        h += struct.pack('<H', zlib.crc32(h) & 0xffff)
    return h


def member(raw, data, hdr=None):
    """A gzip member around raw deflate data."""
    return (hdr or header()) + raw + struct.pack('<II', zlib.crc32(data), len(data) & 0xffffffff)


def raw_deflate(data, level=6):
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    return co.compress(data) + co.flush()


def _data():
    rs = np.random.RandomState(3)
    acgt = np.frombuffer(b'ACGT', np.uint8)[rs.randint(0, 4, 120000)].tobytes()
    fasta = b'>r\n' + b'\n'.join(acgt[i:i + 60] for i in range(0, len(acgt), 60)) + b'\n'
    with open(GOLDEN_FASTA, 'rb') as f:
        golden = f.read()
    rnd = rs.randint(0, 256, 40000).astype(np.uint8).tobytes()
    runs = b''.join(bytes([65 + k % 4]) * int(n) for k, n in enumerate(rs.randint(1, 3000, 120)))
    block = rs.randint(0, 256, 32768).astype(np.uint8).tobytes()
    far = (block + acgt[:5000]) * 3   # matches at distance 32768 + 5000 > 32 KiB are not made; 32768 exactly are
    return dict(fasta=fasta, golden=golden, random=rnd, runs=runs, far=block * 2 + acgt[:3000] + block, repeats=block * 6,
                acgt=acgt, far_mixed=far)


DATA = _data()


def _corpus():
    c, f = {}, DATA['fasta']
    for level in (1, 6, 9):
        c[f'level{level}'] = (gz(f, level), f)
    for name, s in (('filtered', zlib.Z_FILTERED), ('huffman', zlib.Z_HUFFMAN_ONLY), ('rle', zlib.Z_RLE), ('fixed', zlib.Z_FIXED)):
        c[f'strategy_{name}'] = (gz(f, 6, strategy=s), f)
    c['wbits9'] = (gz(f, 9, wbits=9), f)
    c['mem1'] = (gz(f, 6, mem=1), f)
    c['mem9'] = (gz(f, 6, mem=9), f)
    for name in ('golden', 'random', 'runs', 'far', 'far_mixed'):
        c[name] = (gz(DATA[name], 6), DATA[name])
    c['repeats_flushed'] = (gz(DATA['repeats'], 9, flush_every=3000), DATA['repeats'])
    c['empty_input'] = (b'', b'')
    c['empty_member'] = (gzip.compress(b''), b'')
    parts = [DATA['acgt'][:40000], b'', DATA['random'][:9000], DATA['runs'][:50000], b'x']
    c['multi_member'] = (b''.join(gzip.compress(p, lvl) for p, lvl in zip(parts, (1, 9, 6, 0, 6))), b''.join(parts))
    hdr = header(4 | 8 | 16 | 2, extra=b'AB\x03\x00xyz', name=b'ref.fa', comment=b'a comment')
    c['header_fields'] = (member(raw_deflate(f), f, hdr) + member(raw_deflate(b'tail'), b'tail', header(8, name=b'n')), f + b'tail')
    c['nul_padding'] = (gzip.compress(f[:30000]) + b'\0' * 7 + gzip.compress(b'more') + b'\0' * 100, f[:30000] + b'more')
    bg = b''.join(D.member(raw_deflate(f[i:i + 60000]), f[i:i + 60000]) for i in range(0, len(f), 60000))
    c['bgzf'] = (bg + bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000'), f)
    return c


CORPUS = _corpus()


def planted_false_candidate():
    """(stream, data, chunk_bytes): a stored block whose payload is itself a valid non-final dynamic block (and an empty
    stored block, so that it ends byte-aligned), with chunk 1 starting exactly at the payload.  Chunk 0 stops after the
    stored block; chunk 1's decoder takes the payload's block for a block start, and has to be repaired."""
    rs = np.random.RandomState(9)
    lits = [int(x) for x in np.frombuffer(b'ACGT', np.uint8)[rs.randint(0, 4, 6000)]]
    fake = D.deflate([{'type': 'dynamic', 'tokens': [67, 65, 84] * 50, 'final': False}, {'type': 'stored', 'data': b'', 'final': False}])
    program = [{'type': 'dynamic', 'tokens': lits[:3000]}, {'type': 'stored', 'data': fake},
               {'type': 'dynamic', 'tokens': lits[3000:]}, {'type': 'dynamic', 'tokens': lits[:2000]}]
    raw, data = D.deflate(program), D.program_output(program)
    stream = member(raw, data)
    at = raw.find(fake)
    assert at > 0 and raw.find(fake, at + 1) < 0
    return stream, data, at   # (chunk 1 starts at data0 + chunk_bytes = 10 + at)


def _fixed_distance_too_far():
    raw = D.deflate([{'type': 'fixed', 'tokens': [65, 66, (3, 5)]}])
    return member(raw, b'ABABA')


def _refusals():
    ok = gzip.compress(DATA['fasta'][:50000])
    two = ok + gzip.compress(b'second')
    r = {}
    r['truncated'] = (ok[:-30], 0, 0, 'truncated deflate data')
    bad = bytearray(two)
    bad[len(ok) - 8] ^= 1
    r['bad_crc'] = (bytes(bad), 0, 0, 'CRC-32 mismatch')
    bad = bytearray(two)
    bad[-1] ^= 1
    r['bad_isize'] = (bytes(bad), 1, len(ok), 'ISIZE does not match')
    r['block_type_3'] = (ok + member(b'\x07\x00', b''), 1, len(ok), 'invalid block type')
    r['distance_before_member'] = (ok + _fixed_distance_too_far(), 1, len(ok), 'back-reference before the start')
    r['trailing_garbage'] = (ok + b'\0\0garbage', 1, len(ok) + 2, 'bytes after the last member that are neither NUL padding nor a gzip member')
    r['other_method'] = (ok + b'\x1f\x8b\x07' + ok[3:], 1, len(ok), 'compression method other than deflate')
    r['reserved_flag'] = (ok[:3] + b'\x20' + ok[4:], 0, 0, 'reserved header flag')
    r['not_gzip'] = (b'hello', 0, 0, 'not a gzip stream')
    return r


REFUSALS = _refusals()


@pytest.mark.parametrize('chunk', [0, 2048])
@pytest.mark.parametrize('case', sorted(CORPUS))
def test_equals_zlib(case, chunk):
    stream, data = CORPUS[case]
    if stream:
        assert gzip.decompress(stream) == data
    out, stats = emu_gunzip.gunzip(stream, chunk)
    assert out == data
    assert stats['chained'] == 0


def repeats_stream():
    """32 KiB of random bytes, then dynamic blocks that each copy the 32 KiB before them (length 256, distance 32768):
    every chunk after the first is made of markers that reach through the chunks before it."""
    rs = np.random.RandomState(4)
    block = rs.randint(0, 256, 32768).astype(np.uint8).tobytes()
    program = [{'type': 'stored', 'data': block[i:i + 16384]} for i in (0, 16384)]
    program += [{'type': 'dynamic', 'tokens': [(256, 32768)] * 128 + [int(block[k])]} for k in range(12)]
    raw, data = D.deflate(program), D.program_output(program)
    return member(raw, data), data


def test_many_chunks_and_markers():
    stream, data = repeats_stream()
    out, stats = emu_gunzip.gunzip(stream, 256)
    assert out == data
    assert stats['chunks'] - stats['absorbed'] >= 10 and stats['chained'] == 0


def test_members_counted():
    assert emu_gunzip.gunzip(*CORPUS['multi_member'][:1], 1500)[1]['members'] == 5
    assert emu_gunzip.gunzip(CORPUS['empty_input'][0])[1]['members'] == 0


def test_planted_false_candidate_is_repaired():
    stream, data, chunk = planted_false_candidate()
    assert zlib.decompress(stream, 31) == data
    out, stats = emu_gunzip.gunzip(stream, chunk)
    assert out == data
    assert stats['repaired'] >= 1


@pytest.mark.parametrize('case', sorted(REFUSALS))
def test_refusals(case):
    stream, idx, at, why = REFUSALS[case]
    if case != 'reserved_flag':   # (Python's gzip module ignores reserved flags; RFC 1952 and zlib refuse them)
        with pytest.raises((OSError, EOFError, zlib.error)):
            gzip.decompress(stream)
    for chunk in (0, 2048):
        with pytest.raises(ValueError, match=rf'member {idx} \(offset {at}\): {why}'):
            emu_gunzip.gunzip(stream, chunk)


@pytest.mark.parametrize('case', ['fixed', 'stored'])
def test_long_decode_moves_its_bit_reader(case):
    """A build whose bit readers cover 128 KiB and move after 64 KiB: a Z_FIXED stream (no dynamic block to start a
    chunk at) and a stored one (random bytes) are each decoded by one decoder that reads far past the move."""
    rs = np.random.RandomState(21)
    if case == 'fixed':
        data = np.frombuffer(b'ACGT', np.uint8)[rs.randint(0, 4, 1_500_000)].tobytes()
        stream = gz(data, 6, strategy=zlib.Z_FIXED)
    else:
        data = rs.randint(0, 256, 600_000).astype(np.uint8).tobytes()
        stream = gz(data, 6)
    assert len(stream) > 4 * (1 << 16)
    out, stats = emu_gunzip.gunzip(stream, 1 << 15, defines=emu_gunzip.SMALL_SPAN)
    assert out == data
    assert stats['chunks'] - stats['absorbed'] == 1 and stats['chained'] == 0
