"""Unaligned BAM output (`simulate --bam`) on the CPU: the record kernel (csrc/bb_bam_out.cuh) and the compressor's BAM
mode (bgzf_k_compress_bam, csrc/bb_bgzf.cuh) under the warp emulator, behind the native record layout
(bb_bam_layout_sharded).  Decoded by tests/bam_ref.py, an independent reader, the records give back the FASTQ that
bb_fastq_format_sharded writes for the same batch; every member inflates to its chunk, and its deflate blocks start where
the field rule says."""
import os
import random

import numpy as np
import pytest

import bam_ref
import deflate_ref
from emu import emu_bam as E

CHUNK = 65280
MIN_SEG = 1024


class _Planned(object):
    """The parts of a PlannedBatch that the FASTQ and BAM layouts read, built from arrays."""

    def __init__(self, names, infos, frag_len):
        from badread_b200._lib import PlanView
        self.n = len(names)
        self.names = np.frombuffer(b''.join(names), np.uint8).copy() if names else np.zeros(1, np.uint8)
        info = [s.encode('latin-1') for s in infos]
        self.info = np.frombuffer(b''.join(info) + b'\0', np.uint8).copy()
        self.info_off = np.concatenate([[0], np.cumsum([len(s) for s in info])]).astype(np.int64)
        self.frag_len = np.asarray(frag_len, np.int32)
        v = PlanView()
        v.n_reads = self.n
        v.read_names, v.info_off, v.info = self.names.ctypes.data, self.info_off.ctypes.data, self.info.ctypes.data
        v.frag_len = self.frag_len.ctypes.data if self.n else None
        self.view = v

    def __len__(self):
        return self.n


def make_batch(reads, n_shards, rnd):
    """reads: [(seq, qual, frag_len, matches, columns)] in batch order.  Deals them out over n_shards as a --gpus run
    does (read j -> shard j % n_shards), each shard's output packed in reverse read order.  Returns (planned, results,
    seq buffers, qual buffers)."""
    from badread_b200._lib import ReadResult
    planned, results, seqs, quals = [], [], [], []
    for g in range(n_shards):
        mine = reads[g::n_shards]
        names = [rnd.getrandbits(128).to_bytes(16, 'big') for _ in mine]
        infos = [f'chr{g},+strand,{i}-{i + len(r[0])}' + (' chimera junk_seq' if i % 5 == 3 else '') for i, r in enumerate(mine)]
        planned.append(_Planned(names, infos, [r[2] for r in mine]))
        res = (ReadResult * max(1, len(mine)))()
        seq, qual, at = bytearray(), bytearray(), 0
        for i in reversed(range(len(mine))):
            s, q, frag, m, c = mine[i]
            res[i].out_off, res[i].out_len, res[i].frag_len, res[i].matches, res[i].columns = at, len(s), frag, m, c
            seq += s
            qual += q
            at += len(s)
        seqs.append(np.frombuffer(bytes(seq) + b'\0', np.uint8))
        quals.append(np.frombuffer(bytes(qual) + b'\0', np.uint8))
        results.append(res)
    return planned, results, seqs, quals


def emulated_records(planned, results, seqs, quals, first, so_far, target, stream_base, split_sources=True):
    """The record stream of a batch as the GPUs build it: the native layout, each shard's records built by the record
    kernel under the emulator from its output (split into two worker buffers), merged at their stream offsets.  Returns
    (layout, record bytes), and checks the fields the kernel reports against the layout's."""
    from badread_b200.planner import bam_layout_sharded
    lay = bam_layout_sharded(planned, results, first, so_far, target, stream_base)
    merged = bytearray(lay.stream_len)
    for g in range(len(planned)):
        mine = np.nonzero(lay.shard == g)[0]
        if not len(mine):
            continue
        s, q = seqs[g], quals[g]
        cut = int(results[g][len(planned[g]) // 2].out_off) if split_sources and len(planned[g]) > 1 else s.size
        sources = [(s[:cut], q[:cut]), (s[cut:], q[cut:])] if 0 < cut < s.size else [(s, q)]
        recs = lay.recs[mine]
        data, fields = E.records(recs, lay.text, sources, stream_base=0)
        sizes = [E.record_size(int(r['name_len']), int(r['out_len']), int(r['co_len'])) for r in recs]
        local = np.concatenate([[0], np.cumsum(sizes)])[:-1]
        for k, e in enumerate(mine):
            at = int(lay.stream_off[e]) - stream_base
            merged[at:at + sizes[k]] = data[local[k]:local[k] + sizes[k]]
            shift = int(lay.stream_off[e]) - int(local[k])
            assert (fields[2 * k:2 * k + 2, 0] + shift == lay.fields[2 * e:2 * e + 2, 0]).all()
            assert (fields[2 * k:2 * k + 2, 1] == lay.fields[2 * e:2 * e + 2, 1]).all()
    return lay, bytes(merged)


def expected_fastq(planned, results, seqs, quals, first, so_far, target):
    from badread_b200.planner import fastq_format_sharded
    buf, n_emit, bases, nxt, _ = fastq_format_sharded(planned, results, seqs, quals, first, so_far, target)
    lines = bytes(buf).decode('latin-1').split('\n')
    for i in range(1, len(lines), 4):
        lines[i] = bam_ref.n_rule(lines[i])
    return '\n'.join(lines).encode('latin-1'), n_emit, bases, nxt


def check_batch(reads, n_shards, target=None, first=0, so_far=0, stream_base=0, seed=1):
    rnd = random.Random(seed)
    planned, results, seqs, quals = make_batch(reads, n_shards, rnd)
    target = target if target is not None else so_far + sum(len(r[0]) for r in reads) + 1
    want, n_emit, bases, nxt = expected_fastq(planned, results, seqs, quals, first, so_far, target)
    lay, data = emulated_records(planned, results, seqs, quals, first, so_far, target, stream_base)
    assert (lay.n_emitted, lay.bases, lay.next_read) == (n_emit, bases, nxt)
    recs = bam_ref.records_only(data)
    assert len(recs) == n_emit
    assert bam_ref.to_fastq(recs) == want
    return lay, data


# ------------------------------------------------------------------------------------------------ inputs
_ORACLE = {}


def oracle_reads(error_name, qscore_name, n_reads=40):
    """Reads of the oracle's sequence_fragment with the given models: [(seq, qual, frag_len, matches, columns)]."""
    if (error_name, qscore_name) not in _ORACLE:
        from conftest import load_models
        from oracle import oracle as O
        em, qm = load_models(error_name, qscore_name)
        rnd = random.Random(23)
        ref = ''.join(rnd.choice('ACGT') for _ in range(60000))
        frags, idents = [], []
        for _ in range(n_reads):
            n = rnd.randint(200, 6000)
            start = rnd.randint(0, len(ref) - n)
            frags.append(ref[start:start + n])
            idents.append(rnd.uniform(0.85, 0.98))
        reads, _ = O.Oracle(em, qm).sequence_batch(frags, idents, 5, list(range(n_reads)), n_threads=os.cpu_count() or 1)
        _ORACLE[(error_name, qscore_name)] = [(s.encode('latin-1'), q.encode('latin-1'), len(f), m, c)
                                              for (s, q, m, c), f in zip(reads, frags)]
    return _ORACLE[(error_name, qscore_name)]


MODEL_PAIRS = [('nanopore2023', 'nanopore2023'), ('nanopore2020', 'nanopore2020'), ('pacbio2021', 'pacbio2021')]


def synthetic(lengths, rnd, alphabet='ACGT'):
    out = []
    for n in lengths:
        s = ''.join(rnd.choice(alphabet) for _ in range(n)).encode('latin-1')
        q = bytes(rnd.randint(33, 126) for _ in range(n))
        c = n + rnd.randint(0, 9)
        out.append((s, q, n + rnd.randint(0, 50), max(0, n - rnd.randint(0, 9)), c))
    return out


@pytest.mark.parametrize('pair', MODEL_PAIRS, ids=[p[0] for p in MODEL_PAIRS])
@pytest.mark.parametrize('n_shards', [1, 2, 3])
def test_records_decode_to_the_fastq_oracle_reads(pair, n_shards):
    check_batch(oracle_reads(*pair), n_shards, stream_base=12345)


@pytest.mark.parametrize('n_shards', [1, 2, 3])
def test_records_decode_to_the_fastq_edge_lengths(n_shards):
    """Reads of 1 and 2 bases, odd and even lengths, a 150 kb read, and empty reads (skipped, as the FASTQ skips them)."""
    rnd = random.Random(n_shards)
    reads = synthetic([1, 2, 3, 4, 0, 5, 150000, 0, 7, 8, 1, 0, 999, 1000], rnd)
    lay, _ = check_batch(reads, n_shards)
    assert lay.n_emitted == 11


def test_records_iupac_and_letters_outside_the_alphabet():
    """IUPAC codes, '=', lower case and letters outside =ACMGRSVTWYHKDBN (those become N)."""
    rnd = random.Random(4)
    reads = synthetic([1, 17, 300, 2], rnd, alphabet='ACGTRYKMSWBDHVN=acgtrnXZ*.')
    check_batch(reads, 2)
    assert bam_ref.n_rule('AcX=z*') == 'ACN=NN'


@pytest.mark.parametrize('n_shards', [1, 3])
def test_records_stop_at_the_target(n_shards):
    """A cutoff mid-batch: the records stop after the read that reaches the target, as the FASTQ does; and a batch
    continued from a later read."""
    rnd = random.Random(9)
    reads = synthetic([rnd.randint(1, 3000) for _ in range(60)], rnd)
    total = sum(len(r[0]) for r in reads[:25])
    lay, _ = check_batch(reads, n_shards, target=1000 + total - 5, so_far=1000)
    assert lay.n_emitted == 25 and lay.next_read == 25
    lay, _ = check_batch(reads, n_shards, first=7, target=10 ** 9)
    assert lay.n_emitted == 53


def test_layout_record_sizes_match_the_kernel():
    rnd = random.Random(2)
    reads = synthetic([1, 2, 10, 11], rnd)
    lay, data = check_batch(reads, 1, stream_base=70000)
    assert lay.stream_len == len(data)
    assert list(np.diff(np.concatenate([lay.stream_off, [70000 + lay.stream_len]]))) == \
        [E.record_size(int(r['name_len']), int(r['out_len']), int(r['co_len'])) for r in lay.recs]
    assert all(int(r['name_len']) == 36 for r in lay.recs)


# ------------------------------------------------------------------------------------------------ compressor
def record_stream(n_reads=400, seed=3):
    """A record stream of oracle-like reads (several chunks): (bytes, fields)."""
    rnd = random.Random(seed)
    reads = synthetic([rnd.choice([rnd.randint(1, 900), rnd.randint(900, 12000)]) for _ in range(n_reads)], rnd)
    planned, results, seqs, quals = make_batch(reads, 1, rnd)
    lay, data = emulated_records(planned, results, seqs, quals, 0, 0, 10 ** 12, 0)
    return data, lay.fields


def expected_starts(fields, cs, length):
    """Block starts of the chunk [cs, cs + length) of the stream: 0, and every field that starts after cs with at least
    MIN_SEG bytes in the chunk."""
    starts = [0]
    for off, ln in fields:
        if cs < off and min(off + ln, cs + length) - off >= MIN_SEG:
            starts.append(int(off - cs))
    return starts


def test_bam_members_inflate_and_blocks_start_at_the_fields():
    data, fields = record_stream()
    assert len(data) > 4 * CHUNK
    for base in (0, 5000):   # the same bytes read as starting at another stream offset: other blocks
        comp, used = E.compress(data, base, fields + [base, 0], final=True)
        assert used == len(data)
        ms = bam_ref.members(comp)
        assert len(ms) == -(-len(data) // CHUNK)
        n_dynamic = 0
        for i, (m, chunk) in enumerate(ms):
            assert chunk == data[i * CHUNK:(i + 1) * CHUNK]
            p = deflate_ref.parse_member(m)
            if p['blocks'][0]['type'] == 'stored':
                assert len(p['blocks']) == 1
                continue
            n_dynamic += 1
            starts = [b['out'][0] for b in p['blocks']]
            assert starts == expected_starts(fields + [base, 0], base + i * CHUNK, len(chunk))
        assert n_dynamic == len(ms)
        assert len(comp) < 0.8 * len(data)   # (uniform random qualities: about 6.6 bits each)


def test_bam_calls_split_anywhere_give_the_same_stream():
    """Without `final` only whole chunks are compressed: a caller that carries the rest (and its stream offset) gets the
    members of a single call."""
    data, fields = record_stream(seed=5)
    whole, _ = E.compress(data, 0, fields, final=True)
    rnd = random.Random(9)
    got, pos = [], 0
    for cut in sorted(rnd.sample(range(1, len(data)), 5)) + [len(data)]:
        comp, used = E.compress(data[pos:cut], pos, fields, final=cut == len(data))
        assert used == (cut - pos if cut == len(data) else (cut - pos) // CHUNK * CHUNK)
        got.append(comp)
        pos += used
    assert b''.join(got) == whole


def test_bam_compress_header_member():
    from badread_b200.bam import header_bytes
    from badread_b200.version import __version__
    h = header_bytes()
    comp, _ = E.compress(h, 0, np.zeros((0, 2), np.int64), final=True)
    text, refs, recs, ms, end = bam_ref.read_bam(comp + bam_ref.EOF_MEMBER)
    assert text == f'@HD\tVN:1.6\tSO:unknown\n@PG\tID:badread\tPN:badread\tVN:{__version__}\n'
    assert refs == [] and recs == [] and end == len(h)


# ------------------------------------------------------------------------------------------------ command line
def test_bam_flag_and_gzip_conflict(tmp_path):
    from badread_b200.__main__ import check_simulate_args, parse_args
    ref = tmp_path / 'r.fa'
    ref.write_text('>a\nACGT\n')
    base = ['simulate', '--reference', str(ref), '--quantity', '1x']
    assert parse_args(base).bam is False
    assert parse_args(base + ['--bam']).bam is True
    with pytest.raises(SystemExit) as e:
        check_simulate_args(parse_args(base + ['--bam', '--gzip']))
    assert str(e.value) == 'Error: --bam and --gzip cannot be used together (BAM is always compressed)'
