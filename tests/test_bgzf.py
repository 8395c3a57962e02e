"""BGZF output (`simulate --gzip`): the compressor's device code (csrc/bb_bgzf.cuh) under the warp emulator, checked with
zlib: every member a valid BGZF member that inflates on its own to its chunk, chunks at fixed offsets of the stream,
and on FASTQ of oracle reads no larger than zlib level 6 on the same chunks.  The writer (badread_b200/bgzf.py) runs
here with engines whose compressor is the emulator."""
import gzip
import io
import os
import random
import struct
import threading
import uuid
import zlib

import numpy as np
import pytest

from emu import emu_bgzf as B

CHUNK = 65280
EOF = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')


def members(stream):
    """Splits a BGZF stream into its members, checking every header and trailer field against the inflated chunk."""
    out, pos = [], 0
    while pos < len(stream):
        hdr = stream[pos:pos + 18]
        assert hdr[:4] == b'\x1f\x8b\x08\x04', hdr      # magic, deflate, FLG.FEXTRA
        xlen, si, slen, bsize = struct.unpack('<H2sHH', hdr[10:18])
        assert (xlen, si, slen) == (6, b'BC', 2)
        size = bsize + 1
        assert size <= 65536 and pos + size <= len(stream)
        m = stream[pos:pos + size]
        d = zlib.decompressobj(-15)
        data = d.decompress(m[18:-8]) + d.flush()
        assert d.eof and d.unused_data == b''
        crc, isize = struct.unpack('<II', m[-8:])
        assert crc == zlib.crc32(data) and isize == len(data)
        out.append((m, data))
        pos += size
    return out


def check(data, comp):
    """comp: the members of data (no end-of-file member) - chunk i of the member list is data[i * CHUNK ...]."""
    ms = members(comp)
    assert len(ms) == -(-len(data) // CHUNK)
    for i, (_, chunk) in enumerate(ms):
        assert chunk == data[i * CHUNK:(i + 1) * CHUNK]
    assert gzip.decompress(comp + EOF) == data
    return ms


def fasta_like(rnd, n):
    return ''.join(rnd.choice('ACGT') for _ in range(n)).encode()


# ------------------------------------------------------------------------------------------------ FASTQ of oracle reads
_FASTQ = {}


def oracle_fastq(error_name, qscore_name, n_reads=48):
    """Records in the simulator's layout, reads from the oracle's sequence_fragment with the given models."""
    if (error_name, qscore_name) in _FASTQ:
        return _FASTQ[(error_name, qscore_name)]
    from conftest import load_models
    from oracle import oracle as O
    em, qm = load_models(error_name, qscore_name)
    rnd = random.Random(17)
    ref = fasta_like(rnd, 120000).decode()
    frags, idents, info = [], [], []
    for _ in range(n_reads):
        n = rnd.randint(300, 12000)
        start = rnd.randint(0, len(ref) - n)
        frags.append(ref[start:start + n])
        idents.append(rnd.uniform(0.85, 0.98))
        info.append(f'{uuid.UUID(int=rnd.getrandbits(128))} chr1,+strand,{start}-{start + n}')
    reads, _ = O.Oracle(em, qm).sequence_batch(frags, idents, 5, list(range(n_reads)), n_threads=os.cpu_count() or 1)
    out = io.StringIO()
    for (s, q, m, c), f, h in zip(reads, frags, info):
        if s:
            out.write(f'@{h} length={len(s)} error-free_length={len(f)} read_identity={100.0 * m / c:.3f}%\n{s}\n+\n{q}\n')
    _FASTQ[(error_name, qscore_name)] = out.getvalue().encode('latin-1')
    return _FASTQ[(error_name, qscore_name)]


MODEL_PAIRS = [('nanopore2023', 'nanopore2023'), ('nanopore2020', 'nanopore2020'), ('pacbio2021', 'pacbio2021')]


def cases():
    """The inputs the GPU tier compares with the emulator byte for byte: (name, data, line_mod4)."""
    rnd = random.Random(3)
    dna = fasta_like(rnd, 3 * CHUNK + 17)
    one_line = b'@r\n' + fasta_like(rnd, 150000) + b'\n+\n' + bytes(rnd.randint(33, 80) for _ in range(150000)) + b'\n'
    return [('empty', b'', 0), ('one_byte', b'A', 0), ('chunk', dna[:CHUNK], 0), ('chunk_plus_1', dna[:CHUNK + 1], 0),
            ('three_chunks_plus_17', dna, 0), ('single_value', b'G' * (2 * CHUNK + 5), 0),
            ('random_bytes', np.random.RandomState(4).randint(0, 256, 2 * CHUNK + 100, dtype=np.uint8).tobytes(), 0),
            ('line_longer_than_a_chunk', one_line, 0)]


@pytest.mark.parametrize('name,data,line_mod4', cases(), ids=[c[0] for c in cases()])
def test_members_round_trip(name, data, line_mod4):
    comp, used = B.compress(data, line_mod4, final=True)
    assert used == len(data)
    ms = check(data, comp)
    btypes = [(m[18] >> 1) & 3 for m, _ in ms]
    if name in ('random_bytes', 'one_byte'):
        assert btypes == [0] * len(ms)                  # stored: random bytes and tiny inputs do not code smaller
        assert all(len(m) == len(c) + 31 for m, c in ms)
    if name in ('single_value', 'three_chunks_plus_17', 'line_longer_than_a_chunk'):
        assert all(b == 2 for b, (_, c) in zip(btypes, ms) if len(c) > 100)   # dynamic Huffman (17 bytes: stored)
        assert len(comp) < len(data) // 2
    if name == 'single_value':                          # two literal codes (the byte, end-of-block) of one bit each
        assert all(len(m) < 26 + 40 + len(c) // 8 for m, c in ms if len(c) > 100)


@pytest.mark.parametrize('error_name,qscore_name', MODEL_PAIRS)
def test_oracle_fastq_smaller_than_zlib_level_6(error_name, qscore_name):
    """Reads of three model pairs (pacbio2021's qualities reach 93), the stream started at each line index mod 4: valid
    BGZF, the same bytes twice, and no larger than zlib level 6 on the same chunks."""
    fastq = oracle_fastq(error_name, qscore_name)
    lines = fastq.split(b'\n')
    assert len(fastq) > 4 * CHUNK
    for mod4 in range(4):
        data = b'\n'.join(lines[mod4:])
        comp, _ = B.compress(data, mod4, final=True)
        check(data, comp)
        assert B.compress(data, mod4, final=True)[0] == comp
        level6 = sum(len(zlib.compress(data[i:i + CHUNK], 6)) + 31 - 6 for i in range(0, len(data), CHUNK))
        assert len(comp) <= level6, (len(comp), level6)


def test_line_mod4_selects_the_block_starts():
    """Sequence and quality lines (index 1 and 3 mod 4) of at least 1024 bytes start their own deflate block; header and
    '+' lines do not: the same bytes read as starting at another line give other blocks."""
    fastq = oracle_fastq(*MODEL_PAIRS[0])[:CHUNK]
    outs = {B.compress(fastq, mod4, final=True)[0] for mod4 in range(4)}
    assert len(outs) > 1
    for comp in outs:
        check(fastq, comp)


def test_calls_split_anywhere_give_the_same_stream():
    """Without `final` only whole chunks are compressed and consumed: a caller that carries the rest into the next call
    (with the line index mod 4 of its first byte) gets the members of a single call."""
    data = oracle_fastq(*MODEL_PAIRS[1])
    whole, _ = B.compress(data, 0, final=True)
    rnd = random.Random(9)
    got, pos = [], 0
    for cut in sorted(rnd.sample(range(1, len(data)), 5)) + [len(data)]:
        mod4 = data[:pos].count(b'\n') & 3
        comp, used = B.compress(data[pos:cut], mod4, final=cut == len(data))
        assert used == (cut - pos if cut == len(data) else (cut - pos) // CHUNK * CHUNK)
        got.append(comp)
        pos += used
    assert b''.join(got) == whole


class _EmuEngine(object):
    """An engine whose compressor is the device code under the emulator (one emulated CTA at a time: the writer's threads
    take turns)."""
    lock = threading.Lock()

    def __init__(self):
        self.calls = 0

    def bgzf_compress(self, buf, line_mod4=0, final=False):
        self.calls += 1
        with self.lock:
            return B.compress(bytes(buf), line_mod4, final)


@pytest.mark.parametrize('n_engines', [1, 2, 3])
def test_writer_stream_independent_of_batches_and_engines(n_engines):
    """BGZFWriter: records in batches of any size, dealt out over the engines, give the members of one call over the
    whole FASTQ, then the end-of-file member."""
    from badread_b200.bgzf import EOF_MEMBER, BGZFWriter
    assert EOF_MEMBER == EOF
    data = oracle_fastq(*MODEL_PAIRS[2])
    lines = data.split(b'\n')[:-1]
    records = [b'\n'.join(lines[i:i + 4]) + b'\n' for i in range(0, len(lines), 4)]
    assert b''.join(records) == data
    whole, _ = B.compress(data, 0, final=True)
    rnd = random.Random(n_engines)
    out = io.BytesIO()
    engines = [_EmuEngine() for _ in range(n_engines)]
    w = BGZFWriter(engines, out)
    w.write(b''.join(records[:3]))
    i = 3
    while i < len(records):
        k = rnd.choice([1, 2, 7, len(records) // 2]) if i > 3 else len(records) // 2   # (three chunks and more)
        w.write(b''.join(records[i:i + k]))
        i += k
    w.close()
    assert out.getvalue() == whole + EOF
    assert all(e.calls for e in engines)
    assert gzip.decompress(out.getvalue()) == data


def test_writer_empty_stream():
    from badread_b200.bgzf import BGZFWriter
    out = io.BytesIO()
    BGZFWriter([_EmuEngine()], out).close()
    assert out.getvalue() == EOF and gzip.decompress(out.getvalue()) == b''


def test_gzip_flag():
    from badread_b200.__main__ import parse_args
    base = ['simulate', '--reference', 'r.fa', '--quantity', '1x']
    assert parse_args(base).gzip is False
    assert parse_args(base + ['--gzip']).gzip is True
