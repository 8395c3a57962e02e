"""
The model builders with SAM and BAM alignments (CPU tier).  The golden data set (tests/golden/models: reads.fastq,
reads.paf) is turned into SAM and BAM here: soft clips from the PAF coordinates, SEQ reverse-complemented on '-', AS:i
copied, NM:i = columns - matches, the secondary (tp:A:S) lines as FLAG 256 without SEQ (some of them before their primary
record), and the BAM's BGZF written with Python's zlib.  Built from either, with or without --reads, the seven model files
equal the reference's for the PAF; the BAM is inflated by the device code under the warp emulator (tests/emu/
emu_inflate.cpp), which is checked against zlib on its own: every compression level and strategy, member sizes from 0 to
65 280 bytes, the end-of-file member, the project's own compressor, and corrupt members, which give a clean error.
"""
import contextlib
import gzip
import io
import os
import random
import struct
import types
import zlib

import numpy as np
import pytest

from emu import emu_inflate as EI
from test_model_builders import _golden, _host_count

HERE = os.path.dirname(os.path.realpath(__file__))
DATA = os.path.join(HERE, 'golden', 'models')
CHUNK = 65280
EOF = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')
_COMP = bytes.maketrans(b'ACGTN', b'TGCAN')

# the parameters of oracle/make_golden_models.py
MODELS = [('error_model_k7', dict(k_size=7, max_alt=25, max_alignments=None)),
          ('error_model_k5_alt3', dict(k_size=5, max_alt=3, max_alignments=None)),
          ('error_model_k4_max50', dict(k_size=4, max_alt=25, max_alignments=50)),
          ('qscore_model_k9', dict(k_size=9, max_del=6, min_occur=3, max_output=10000, max_alignments=None)),
          ('qscore_model_k5_del3', dict(k_size=5, max_del=3, min_occur=1, max_output=10000, max_alignments=None)),
          ('qscore_model_k9_max40', dict(k_size=9, max_del=6, min_occur=100, max_output=40, max_alignments=None)),
          ('qscore_model_k9_all', dict(k_size=9, max_del=6, min_occur=1, max_output=1000000, max_alignments=None))]


# ------------------------------------------------------------------------------------------------ PAF + FASTQ -> SAM / BAM
def revcomp(s):
    return s.encode().translate(_COMP)[::-1].decode()


def read_fastq(path):
    lines = open(path).read().split('\n')
    return {lines[i][1:].split()[0]: (lines[i + 1], lines[i + 3]) for i in range(0, len(lines) - 3, 4)}


def read_refs(path):
    refs, name = {}, None
    for line in open(path):
        line = line.strip()
        if line.startswith('>'):
            name = line[1:].split()[0]
            refs[name] = []
        elif line:
            refs[name].append(line)
    return {k: ''.join(v) for k, v in refs.items()}


def paf_to_records(paf_lines, reads):
    """SAM records (lists of 11+ columns) of PAF lines."""
    out = []
    for line in paf_lines:
        f = line.rstrip('\n').split('\t')
        name, qlen, qs, qe, strand, ctg, ts = f[0], int(f[1]), int(f[2]), int(f[3]), f[4], f[5], int(f[7])
        tags = dict((t[:2], t) for t in f[12:])
        cg = tags['cg'][5:]
        secondary = tags.get('tp') == 'tp:A:S'
        lead, trail = (qs, qlen - qe) if strand == '+' else (qlen - qe, qs)
        cigar = (f'{lead}S' if lead else '') + cg + (f'{trail}S' if trail else '')
        seq, qual = reads[name]
        if strand == '-':
            seq, qual = revcomp(seq), qual[::-1]
        flag = (16 if strand == '-' else 0) | (256 if secondary else 0)
        if secondary:
            seq = qual = '*'
        out.append([name, str(flag), ctg, str(ts + 1), '60', cigar, '*', '0', '0', seq, qual,
                    tags['AS'], f'NM:i:{int(f[10]) - int(f[9])}'])
    return out


def sam_text(records, refs, header=True):
    head = '@HD\tVN:1.6\tSO:unsorted\n' + ''.join(f'@SQ\tSN:{n}\tLN:{len(s)}\n' for n, s in refs.items()) if header else ''
    return head + ''.join('\t'.join(r) + '\n' for r in records)


_OPS = 'MIDNSHP=X'


def bam_bytes(records, refs):
    """The uncompressed BAM (SAM specification §4.2) of SAM records."""
    ids = {n: i for i, n in enumerate(refs)}
    text = sam_text([], refs).encode()
    out = [b'BAM\x01', struct.pack('<i', len(text)), text, struct.pack('<i', len(refs))]
    for n, s in refs.items():
        out.append(struct.pack('<i', len(n) + 1) + n.encode() + b'\0' + struct.pack('<i', len(s)))
    for r in records:
        name, flag, ctg, pos, mapq, cigar, seq, qual = r[0], int(r[1]), r[2], int(r[3]) - 1, int(r[4]), r[5], r[9], r[10]
        runs = [] if cigar == '*' else [(int(n), _OPS.index(o)) for n, o in __import__('re').findall(r'(\d+)([MIDNSHP=X])', cigar)]
        seq = '' if seq == '*' else seq
        packed = bytearray((len(seq) + 1) // 2)
        for i, c in enumerate(seq):
            packed[i // 2] |= '=ACMGRSVTWYHKDBN'.index(c) << (4 if i % 2 == 0 else 0)
        q = bytes(ord(c) - 33 for c in qual) if qual != '*' else b'\xff' * len(seq)
        tags = b''
        for t in r[11:]:
            tags += t[:2].encode() + b'i' + struct.pack('<i', int(t[5:]))
        rid = ids.get(ctg, -1)
        body = struct.pack('<iiBBHHHiiii', rid, pos, len(name) + 1, mapq, 4680, len(runs), flag, len(seq), -1, -1, 0) + \
            name.encode() + b'\0' + b''.join(struct.pack('<I', (n << 4) | o) for n, o in runs) + bytes(packed) + q + tags
        out.append(struct.pack('<i', len(body)) + body)
    return b''.join(out)


def bgzf_member(raw, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    d = c.compress(raw) + c.flush()
    return b'\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0' + struct.pack('<H', len(d) + 25) + d + \
        struct.pack('<II', zlib.crc32(raw), len(raw))


SETTINGS = [(0, zlib.Z_DEFAULT_STRATEGY), (1, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_DEFAULT_STRATEGY), (9, zlib.Z_DEFAULT_STRATEGY),
            (6, zlib.Z_FIXED), (6, zlib.Z_RLE), (6, zlib.Z_HUFFMAN_ONLY)]


def bgzf(raw, sizes=None, eof=True):
    """BGZF of raw in members of the given sizes (cycled; default: full chunks), levels and strategies cycling through
    SETTINGS."""
    sizes = sizes or [CHUNK]
    out, pos, k = [], 0, 0
    while pos < len(raw):
        n = sizes[k % len(sizes)]
        out.append(bgzf_member(raw[pos:pos + n], *SETTINGS[k % len(SETTINGS)]))
        pos += n
        k += 1
    return b''.join(out) + (EOF if eof else b'')


@pytest.fixture(scope='module')
def inputs(tmp_path_factory):
    """SAM (plain and gzipped, the latter without a header) and BAM of the golden data set; the BAM's members are 9 000
    to 40 000 bytes, so records straddle them."""
    d = tmp_path_factory.mktemp('aln')
    reads = read_fastq(os.path.join(DATA, 'reads.fastq'))
    refs = read_refs(os.path.join(DATA, 'ref.fasta'))
    records = paf_to_records(open(os.path.join(DATA, 'reads.paf')).read().splitlines(), reads)
    (d / 'reads.sam').write_text(sam_text(records, refs))
    with gzip.open(d / 'reads.sam.gz', 'wt') as f:
        f.write(sam_text(records, refs, header=False))
    raw = bam_bytes(records, refs)
    (d / 'reads.bam').write_bytes(bgzf(raw, sizes=[9000, 40000, 23456]))
    return types.SimpleNamespace(dir=d, raw_bam=raw, records=records, refs=refs, reads=reads)


def _args(alignment, reads=True, **kw):
    return types.SimpleNamespace(reference=os.path.join(DATA, 'ref.fasta'),
                                 reads=os.path.join(DATA, 'reads.fastq') if reads else None, alignment=str(alignment), **kw)


def _run(fn, args, stderr=None):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        fn(args, output=stderr if stderr is not None else io.StringIO())
    return out.getvalue()


@pytest.fixture
def emulated(monkeypatch):
    """The builders with the BAM inflated by the emulated device code and the windows counted by the restated kernels."""
    from badread_b200 import model_builders as mb
    calls = []

    def inflate(data):
        calls.append(len(data))
        return EI.decompress(data)
    monkeypatch.setattr(mb, '_inflate', inflate)
    monkeypatch.setattr(mb, '_count', _host_count)
    return mb, calls


# ------------------------------------------------------------------------------------------------ the golden model files
@pytest.mark.parametrize('fmt', ['sam', 'sam.gz', 'bam'])
@pytest.mark.parametrize('with_reads', [True, False], ids=['reads', 'no_reads'])
@pytest.mark.parametrize('name,kw', MODELS, ids=[m[0] for m in MODELS])
def test_golden_models_from_sam_and_bam(inputs, emulated, fmt, with_reads, name, kw):
    mb, calls = emulated
    fn = mb.make_error_model if name.startswith('error') else mb.make_qscore_model
    assert mb.alignment_format(str(inputs.dir / f'reads.{fmt}')) == fmt.split('.')[0]
    assert _run(fn, _args(inputs.dir / f'reads.{fmt}', with_reads, **kw)) == _golden(name)
    assert bool(calls) == (fmt == 'bam')


def test_flat_alignments_equal_the_paf_path(inputs, emulated):
    """What the counting kernels receive from a BAM without --reads is exactly what they receive from the PAF + FASTQ, and
    the progress lines are the PAF path's."""
    mb, _ = emulated
    refs = read_refs(os.path.join(DATA, 'ref.fasta'))
    sink = io.StringIO()
    reads, alns = mb.load_inputs(_args(inputs.dir / 'reads.bam', False, max_alignments=None), refs, sink, need_qual=True)
    flat = mb.FlatAlignments(alns, reads, refs, io.StringIO(), 1000)
    paf_alns = mb.load_alignments(os.path.join(DATA, 'reads.paf'), None, output=io.StringIO())
    want = mb.FlatAlignments(paf_alns, mb.load_fastq(os.path.join(DATA, 'reads.fastq'), output=io.StringIO()), refs,
                             io.StringIO(), 1000)
    assert [a.read_name for a in alns] == [a.read_name for a in paf_alns]
    for f in ('read', 'qual', 'ref', 'read_off', 'ref_off', 'ops_off', 'ops', 'op_read0', 'op_ref0'):
        assert np.array_equal(getattr(flat, f), getattr(want, f)), f
    assert 'Loading alignments' in sink.getvalue() and 'Choosing best alignment per read' in sink.getvalue()


# ------------------------------------------------------------------------------------------------ the inflater vs zlib
@pytest.mark.parametrize('level,strategy', SETTINGS, ids=['level0', 'level1', 'level6', 'level9', 'fixed', 'rle', 'huffman_only'])
def test_inflate_equals_zlib(level, strategy):
    """Member sizes from 1 byte to a whole chunk, an empty member, and the end-of-file member, on DNA-like text (long
    matches) and random bytes (mostly literals)."""
    rnd = random.Random(level * 10 + strategy)
    text = ''.join(rnd.choice(['ACGT', 'AC', 'G', 'TTTTTTTT', 'ACGTTGCA\n']) for _ in range(40000)).encode()
    noise = bytes(rnd.getrandbits(8) for _ in range(70000))
    for raw in (text, noise):
        members, want = [], b''
        for n in (1, 2, 7, 258, 259, 1000, 32768, 32769, 65280, 0, 5000):
            chunk = raw[:n]
            members.append(bgzf_member(chunk, level, strategy))
            want += chunk
        stream = b''.join(members) + EOF
        assert gzip.decompress(stream) == want
        assert bytes(EI.decompress(stream)) == want


def test_inflate_records_straddling_members(inputs):
    for sizes in ([CHUNK], [1, 333, 65280, 4097], [100]):
        assert bytes(EI.decompress(bgzf(inputs.raw_bam, sizes))) == inputs.raw_bam


def test_inflate_of_the_projects_own_compressor():
    from emu import emu_bgzf as B
    from test_bgzf import oracle_fastq
    data = oracle_fastq('nanopore2023', 'nanopore2023')
    comp, _ = B.compress(data, 0, final=True)
    assert bytes(EI.decompress(comp + EOF)) == data
    assert EI.decompress(b'') == bytearray() and EI.decompress(EOF) == bytearray()


# ------------------------------------------------------------------------------------------------ corrupt input
class BitWriter(object):
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits.extend((v >> i) & 1 for i in range(n))

    def put_code(self, code, n):      # Huffman codes go most significant bit first
        self.bits.extend((code >> (n - 1 - i)) & 1 for i in range(n))

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + j] << j for j in range(8)) for i in range(0, len(b), 8))


def raw_member(deflate, isize, crc):
    return b'\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0' + struct.pack('<H', len(deflate) + 25) + deflate + \
        struct.pack('<II', crc, isize)


def fixed_literal(w, c):   # fixed Huffman code of a literal byte < 144
    w.put_code(0x30 + c, 8)


def corrupt_cases():
    """(name, stream): every one must fail with ValueError naming the member."""
    good = bgzf_member(b'ACGT' * 1000, 6)
    cases = [('not_bgzf', gzip.compress(b'ACGT' * 100)), ('not_gzip', b'@read\nACGT\n+\nIIII\n' * 3),
             ('truncated_member', good + good[:len(good) // 2]), ('truncated_header', good + good[:10]),
             ('bad_crc', good[:-8] + bytes([good[-8] ^ 1]) + good[-7:]),
             ('isize_too_large', good[:-4] + struct.pack('<I', 5000)),
             ('isize_too_small', good[:-4] + struct.pack('<I', 3000)),
             ('isize_beyond_64k', good[:-4] + struct.pack('<I', 70000))]
    # deflate data cut short inside the member (BSIZE consistent)
    d = zlib.compressobj(6, zlib.DEFLATED, -15)
    data = d.compress(b'ACGTTGCA' * 500) + d.flush()
    cases.append(('truncated_deflate', raw_member(data[:len(data) // 2], 4000, zlib.crc32(b'ACGTTGCA' * 500))))
    w = BitWriter()                   # block type 3
    w.put(1, 1); w.put(3, 2)
    cases.append(('bad_block_type', raw_member(w.bytes() + b'\0' * 4, 0, 0)))
    w = BitWriter()                   # stored block whose NLEN is not the complement of LEN
    w.put(1, 1); w.put(0, 2)
    cases.append(('bad_stored_length', raw_member(w.bytes() + struct.pack('<HH', 4, 4) + b'ACGT', 4, zlib.crc32(b'ACGT'))))
    w = BitWriter()                   # fixed block: a back-reference at the member's first byte
    w.put(1, 1); w.put(1, 2)
    w.put_code(1, 7)                  # length symbol 257 (3 bytes)
    w.put_code(0, 5)                  # distance 1
    w.put_code(0, 7)                  # end of block
    cases.append(('distance_before_start', raw_member(w.bytes(), 3, zlib.crc32(b'AAA'))))
    w = BitWriter()                   # fixed block: a literal then a distance of 2 (one byte too far back)
    w.put(1, 1); w.put(1, 2)
    fixed_literal(w, ord('A'))
    w.put_code(1, 7); w.put_code(1, 5)
    w.put_code(0, 7)
    cases.append(('distance_one_too_far', raw_member(w.bytes(), 4, zlib.crc32(b'AAAA'))))
    w = BitWriter()                   # dynamic block whose code-length code is over-subscribed
    w.put(1, 1); w.put(2, 2); w.put(0, 5); w.put(0, 5); w.put(15, 4)
    for _ in range(19):
        w.put(1, 3)
    cases.append(('bad_huffman_table', raw_member(w.bytes() + b'\0' * 8, 1, 0)))
    w = BitWriter()                   # fixed block: more bytes than ISIZE
    w.put(1, 1); w.put(1, 2)
    for c in b'ACGTACGT':
        fixed_literal(w, c)
    w.put_code(0, 7)
    cases.append(('more_than_isize', raw_member(w.bytes(), 4, zlib.crc32(b'ACGT'))))
    w = BitWriter()                   # fixed block: literal/length symbol 286 (no such code)
    w.put(1, 1); w.put(1, 2)
    w.put_code(0xc6, 8)
    cases.append(('bad_huffman_code', raw_member(w.bytes() + b'\0', 0, 0)))
    # a corrupt member after good ones is named by its index
    cases.append(('third_member_bad', good + good + good[:-8] + bytes([good[-8] ^ 0x80]) + good[-7:] + EOF))
    return cases


@pytest.mark.parametrize('name,stream', corrupt_cases(), ids=[c[0] for c in corrupt_cases()])
def test_corrupt_members_give_a_clean_error(name, stream):
    with pytest.raises(ValueError) as e:
        EI.decompress(stream)
    msg = str(e.value)
    assert msg.startswith('bb_bgzf_decompress: member '), msg
    if name == 'third_member_bad':
        assert 'member 2 ' in msg and 'CRC' in msg
    if name == 'not_bgzf':
        assert 'BC' in msg
    if name.startswith('distance'):
        assert 'before the start' in msg


def test_bam_that_is_not_bgzf_exits(inputs, emulated, tmp_path):
    mb, _ = emulated
    bam = tmp_path / 'x.bam'
    bam.write_bytes(bgzf(inputs.raw_bam)[:-200])     # the last member cut short
    with pytest.raises(SystemExit) as e:
        _run(mb.make_error_model, _args(bam, False, k_size=5, max_alt=3, max_alignments=None))
    assert 'not a valid BAM file' in str(e.value) and 'truncated' in str(e.value)


# ------------------------------------------------------------------------------------------------ record rules, small cases
REF = {'ctg': ''.join(random.Random(5).choice('ACGT') for _ in range(3000))}


def _small(tmp_path, lines, fmt='sam', refs=REF):
    fa = tmp_path / 'ref.fasta'
    fa.write_text(''.join(f'>{n}\n{s}\n' for n, s in refs.items()))
    path = tmp_path / ('x.' + fmt)
    if fmt == 'sam':
        path.write_text(sam_text([l.split('\t') for l in lines], refs))
    else:
        path.write_bytes(bgzf(bam_bytes([l.split('\t') for l in lines], refs)))
    return str(fa), str(path)


def _load(mb, fa, path, need_qual=True, max_alignments=None):
    refs = read_refs(fa)
    args = types.SimpleNamespace(reference=fa, reads=None, alignment=path, max_alignments=max_alignments)
    return mb.load_inputs(args, refs, io.StringIO(), need_qual)


@pytest.mark.parametrize('fmt', ['sam', 'bam'])
def test_minus_strand_and_hard_clips(tmp_path, emulated, fmt):
    """'-': the read starts at the trailing clip, SEQ comes back reverse-complemented and QUAL reversed, the runs in read
    orientation; an H-clipped record gives coordinates but not the sequence, which comes from the read's other record."""
    mb, _ = emulated
    ref = REF['ctg']
    read = 'GGGGG' + revcomp(ref[100:300]) + 'TTT'                # 5 + 200 + 3 bases, aligned on '-'
    qual = ''.join(chr(33 + i % 40) for i in range(len(read)))
    sam_seq, sam_qual = revcomp(read), qual[::-1]                 # SAM orientation: 3 clipped, 200 aligned, 5 clipped
    lines = ['r1\t16\tctg\t101\t60\t3S100M2D98M2I5S\t*\t0\t0\t' + sam_seq[:201] + sam_seq[201:] + '\t' + sam_qual + '\tAS:i:300\tNM:i:4',
             'r1\t2064\tctg\t101\t60\t3H100M2D98M2I5H\t*\t0\t0\t' + sam_seq[3:-5] + '\t' + sam_qual[3:-5] + '\tAS:i:300\tNM:i:4']
    fa, path = _small(tmp_path, lines, fmt)
    reads, alns = _load(mb, fa, path)
    a = alns[0]
    assert (a.read_name, a.strand, a.read_start, a.read_end, a.ref_start, a.ref_end) == ('r1', '-', 5, 205, 100, 300)
    assert a.runs == [(2, 'I'), (98, 'M'), (2, 'D'), (100, 'M')]
    assert reads['r1'] == (read, qual)
    # hard clips alone: the whole read is nowhere
    fa, path = _small(tmp_path, lines[1:], fmt)
    with pytest.raises(SystemExit) as e:
        _load(mb, fa, path)
    assert 'r1' in str(e.value) and 'whole sequence' in str(e.value)


@pytest.mark.parametrize('fmt', ['sam', 'bam'])
def test_match_and_mismatch_runs_count_as_m(tmp_path, emulated, fmt):
    mb, _ = emulated
    ref = REF['ctg']
    read = ref[10:60] + ('A' if ref[60] != 'A' else 'C') + ref[61:200]
    fa, path = _small(tmp_path, ['x\t0\tctg\t11\t60\t50=1X139=\t*\t0\t0\t' + read + '\t' + 'I' * 190 + '\tAS:i:200'], fmt)
    reads, alns = _load(mb, fa, path)
    assert alns[0].runs == [(50, 'M'), (1, 'M'), (139, 'M')]
    assert (alns[0].read_start, alns[0].read_end, alns[0].ref_end) == (0, 190, 200)
    flat = mb.FlatAlignments(alns, reads, REF, io.StringIO(), 1000)
    fa, path = _small(tmp_path, ['x\t0\tctg\t11\t60\t190M\t*\t0\t0\t' + read + '\t' + 'I' * 190 + '\tAS:i:200'], fmt)
    reads_m, alns_m = _load(mb, fa, path)
    flat_m = mb.FlatAlignments(alns_m, reads_m, REF, io.StringIO(), 1000)
    for which, k in (('kmers', 5), ('cigars', 5)):     # the same windows as one M run
        got, want = _host_count(which, flat, k), _host_count(which, flat_m, k)
        assert sorted(zip(got[0].tolist(), got[2].tolist())) == sorted(zip(want[0].tolist(), want[2].tolist()))
    # no NM:i: the matching bases are counted from the sequences (189 of 190 columns)
    fa, path = _small(tmp_path, ['x\t0\tctg\t11\t60\t190M\t*\t0\t0\t' + read + '\t*\tAS:i:200'], fmt)
    _, alns = _load(mb, fa, path, need_qual=False)
    assert len(alns) == 1
    with pytest.raises(SystemExit) as e:                        # qscore_model needs the qualities
        _load(mb, fa, path, need_qual=True)
    assert 'QUAL' in str(e.value)
    # 150 mismatches of 190: below the 80 % identity filter
    bad = ''.join('A' if c != 'A' else 'C' for c in read[:150]) + read[150:]
    fa, path = _small(tmp_path, ['x\t0\tctg\t11\t60\t190M\t*\t0\t0\t' + bad + '\t*\tAS:i:200'], fmt)
    assert _load(mb, fa, path, need_qual=False)[1] == []


@pytest.mark.parametrize('fmt', ['sam', 'bam'])
def test_best_alignment_unmapped_and_max_alignments(tmp_path, emulated, fmt):
    """Unmapped records (FLAG 0x4, RNAME '*') are skipped; the highest AS wins, the later among equals; --max_alignments
    counts mapped records."""
    mb, _ = emulated
    ref = REF['ctg']
    seq = ref[0:150]
    rec = 'a\t{f}\t{c}\t{p}\t60\t150M\t*\t0\t0\t' + seq + '\t' + 'I' * 150 + '\tAS:i:{s}\tNM:i:0'
    lines = [rec.format(f=4, c='ctg', p=1, s=999), rec.format(f=0, c='ctg', p=1, s=10), rec.format(f=256, c='ctg', p=5, s=50),
             rec.format(f=256, c='ctg', p=9, s=50), rec.format(f=256, c='ctg', p=13, s=20)]
    if fmt == 'sam':
        lines.append('a\t0\t*\t0\t0\t*\t*\t0\t0\t*\t*')
    fa, path = _small(tmp_path, lines, fmt)
    _, alns = _load(mb, fa, path)
    assert [a.ref_start for a in alns] == [8]
    _, alns = _load(mb, fa, path, max_alignments=2)
    assert [a.ref_start for a in alns] == [4]


@pytest.mark.parametrize('fmt', ['sam', 'bam'])
def test_missing_score_cigar_and_unsupported_ops(tmp_path, emulated, fmt):
    mb, _ = emulated
    seq = REF['ctg'][:150]
    base = 'r7\t0\tctg\t1\t60\t{cig}\t*\t0\t0\t' + seq + '\t*'
    for cig, tags, msg in [('150M', '', 'Error: no alignment score'), ('*', '\tAS:i:5', 'Error: no CIGAR string found'),
                           ('70M5N80M', '\tAS:i:5', 'r7'), ('70M2P80M', '\tAS:i:5', 'r7')]:
        fa, path = _small(tmp_path, [base.format(cig=cig) + tags], fmt)
        with pytest.raises(SystemExit) as e:
            _load(mb, fa, path)
        assert msg in str(e.value), (cig, str(e.value))


def test_format_detection(tmp_path, inputs):
    from badread_b200.model_builders import alignment_format
    paf = os.path.join(DATA, 'reads.paf')
    assert alignment_format(paf) == 'paf'
    gz = tmp_path / 'reads.paf.gz'
    gz.write_bytes(gzip.compress(open(paf, 'rb').read()))
    assert alignment_format(str(gz)) == 'paf'
    bgz = tmp_path / 'reads.paf.bgz'          # BGZF, but not BAM
    bgz.write_bytes(bgzf(open(paf, 'rb').read()))
    assert alignment_format(str(bgz)) == 'paf'
    headerless = tmp_path / 'x.txt'           # SAM without a header, by its columns; the file name does not matter
    headerless.write_text(sam_text(inputs.records[:3], inputs.refs, header=False))
    assert alignment_format(str(headerless)) == 'sam'
    assert alignment_format(str(inputs.dir / 'reads.bam')) == 'bam'
    assert alignment_format(str(tmp_path / 'missing')) == 'paf'


def test_reads_optional_for_sam_and_bam_only(inputs, capsys):
    from badread_b200.__main__ import parse_args
    for fmt in ('sam', 'bam'):
        a = parse_args(['error_model', '--reference', 'r.fa', '--alignment', str(inputs.dir / f'reads.{fmt}')])
        assert a.reads is None
    with pytest.raises(SystemExit) as e:
        parse_args(['qscore_model', '--reference', 'r.fa', '--alignment', os.path.join(DATA, 'reads.paf')])
    assert e.value.code == 2
    assert 'the following arguments are required: --reads' in capsys.readouterr().err
