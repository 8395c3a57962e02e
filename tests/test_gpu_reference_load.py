"""Loading the simulate reference on the GPU (Engine.load_fasta: BGZF inflated and the FASTA parsed on the device) against
the host loader, misc.load_fasta_arrays, on plain, gzip and BGZF files; and `simulate` on the three giving the same reads."""
import gzip
import io
import struct
import zlib

import numpy as np
import pytest

from test_fasta_parse import CASES, _long_line_case, _newline_last_in_tile

pytestmark = pytest.mark.gpu


def bgzf(data, cuts):
    """BGZF of data with members ending at the offsets `cuts` (zlib raw deflate, BC extra field), then the EOF member."""
    out = bytearray()
    bounds = [0] + sorted(c for c in set(cuts) if 0 < c < len(data)) + [len(data)]
    for a, b in zip(bounds[:-1], bounds[1:]):
        if a == b:
            continue
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        body = co.compress(data[a:b]) + co.flush()
        out += b'\x1f\x8b\x08\x04' + b'\0' * 4 + b'\0\xff' + struct.pack('<HBBHH', 6, 66, 67, 2, len(body) + 25)
        out += body + struct.pack('<II', zlib.crc32(data[a:b]), b - a)
    out += bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')
    return bytes(out)


def _cuts(data):
    """Member ends inside every header line, between every '\\r' and its '\\n', and every 5 bytes."""
    cuts = set(range(5, len(data), 5))
    for i in range(len(data)):
        if data[i:i + 2] == b'\r\n':
            cuts.add(i + 1)
        if data[i:i + 1] == b'>':
            cuts.update((i + 1, i + 2))
    return cuts


def _files(tmp_path, name, data):
    plain, gz, bz = tmp_path / f'{name}.fa', tmp_path / f'{name}.fa.gz', tmp_path / f'{name}.bgzf.fa.gz'
    plain.write_bytes(data)
    gz.write_bytes(gzip.compress(data))
    bz.write_bytes(bgzf(data, _cuts(data)))
    return plain, gz, bz


def _host(path):
    from badread_b200.misc import load_fasta_arrays
    names, seqs, depths, circular, left, right = load_fasta_arrays(str(path))
    return names, [int(s.size) for s in seqs], depths, circular, left, right, b''.join(bytes(s) for s in seqs)


ALL_CASES = dict(CASES, long_lines=_long_line_case(20000), newline_last_in_tile=_newline_last_in_tile(16384))


@pytest.mark.parametrize('case', sorted(ALL_CASES))
def test_cases_plain_gzip_bgzf(engine, tmp_path, case):
    data = ALL_CASES[case]
    (tmp_path / 'x.fa').write_bytes(data)
    want = _host(tmp_path / 'x.fa')
    for path in _files(tmp_path, case, data):
        got = engine.load_fasta(str(path))
        assert tuple(got) == want[:6], path.name
        assert bytes(engine.download_reference(0, sum(got[1]))) == want[6], path.name


def test_reference_equals_host_reference(engine, tmp_path):
    """A reference of a few Mb with 60-column lines, lowercase stretches, CRLF, a repeated name and an empty header:
    the context's reference is Reference(path).concat."""
    from badread_b200 import simulate as S
    rs = np.random.RandomState(7)
    parts = []
    for i in range(6):
        seq = np.frombuffer(b'ACGTNacgtn', np.uint8)[rs.randint(0, 10, int(rs.randint(1, 900000)))].tobytes()
        lines = [seq[j:j + 60] for j in range(0, len(seq), 60)]
        eol = b'\r\n' if i % 2 else b'\n'
        name = b'dup' if i in (1, 4) else b'c%d' % i
        parts.append(b'>' + name + b' depth=%d circular=true' % (i + 1) + eol + eol.join(lines) + eol)
    parts.insert(3, b'>\nACGT\n')
    data = b''.join(parts)
    for path in _files(tmp_path, 'big', data):
        ref = S.Reference(str(path), io.StringIO())
        got = engine.load_fasta(str(path))
        assert got[0] == ref.names and got[1] == ref.lengths
        assert np.array_equal(engine.download_reference(0, ref.size), ref.concat)


def test_input_beyond_2_gib(engine, tmp_path):
    """A plain file of more than 2^31 bytes from two known contigs (a block of 60-column lines repeated), so the
    expected bases need no host loader."""
    rs = np.random.RandomState(5)
    block = np.frombuffer(b'ACGTacgt', np.uint8)[rs.randint(0, 8, 60 * 17476)].tobytes()
    text = b'\n'.join(block[j:j + 60] for j in range(0, len(block), 60)) + b'\n'
    reps = 1060
    path = tmp_path / 'huge.fa'
    with open(path, 'wb') as f:
        for name in (b'>first', b'>second depth=3'):
            f.write(name + b'\n')
            for _ in range(reps):
                f.write(text)
    assert path.stat().st_size > 2 ** 31
    names, lengths, depths, circular, _, _ = engine.load_fasta(str(path))
    assert names == ['first', 'second'] and lengths == [len(block) * reps] * 2 and depths['second'] == 3.0
    upper = block.upper()
    step = len(block) * 64
    total = 2 * len(block) * reps
    for off in range(0, total, step):
        n = min(step, total - off)
        got = engine.download_reference(off, n)
        assert off % len(block) == 0 and bytes(got) == (upper * 64)[:n], off


def test_corrupt_member_is_named(engine, tmp_path):
    from badread_b200.engine import EngineError
    data = CASES['plain'] * 50
    z = bytearray(bgzf(data, range(100, len(data), 100)))
    at = 0
    for _ in range(3):   # the fourth member's CRC-32
        at += struct.unpack('<H', z[at + 16:at + 18])[0] + 1
    bsize = struct.unpack('<H', z[at + 16:at + 18])[0] + 1
    z[at + bsize - 8] ^= 0xff
    path = tmp_path / 'bad.fa.gz'
    path.write_bytes(bytes(z))
    with pytest.raises(EngineError, match=rf'member 3 \(offset {at}\): CRC-32 mismatch'):
        engine.load_fasta(str(path))
    (tmp_path / 'ok.fa').write_bytes(data)
    assert engine.load_fasta(str(tmp_path / 'ok.fa'))[0] == ['chr1', 'chr2']   # the context loads again after the error


def _simulate(path, extra=()):
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.simulate import simulate
    args = parse_args(['simulate', '--reference', str(path), '--quantity', '4x', '--length', '2500,1500', '--seed', '5',
                       '--glitches', '2000,20,20', '--chimeras', '5'] + list(extra))
    check_simulate_args(args)
    out, err = io.TextIOWrapper(io.BytesIO(), encoding='latin-1'), io.StringIO()
    simulate(args, output=err, stdout=out)
    out.flush()
    return args, out.buffer.getvalue(), err.getvalue()


def _reference_text():
    rs = np.random.RandomState(11)
    acgt = np.frombuffer(b'ACGTacgt', np.uint8)
    a = acgt[rs.randint(0, 8, 40000)].tobytes()
    b = acgt[rs.randint(0, 4, 15000)].tobytes()
    wrap = lambda s: b'\r\n'.join(s[i:i + 70] for i in range(0, len(s), 70))   # noqa: E731
    return b'>chr circular=true\r\n' + wrap(a) + b'\r\n\n>lin depth=2\n' + wrap(b) + b'\n'


def _two_gpus():
    from badread_b200.engine import Engine, EngineError
    try:
        Engine(device=1, seed=0).close()
        return True
    except EngineError:
        return False


@pytest.mark.parametrize('mode', ['fastq', 'bam'])
def test_simulate_same_reads_from_plain_gzip_bgzf(tmp_path, mode):
    from badread_b200 import simulate as S
    from badread_b200.error_model import ErrorModel
    from badread_b200.fragment_lengths import FragmentLengths
    from badread_b200.identities import Identities
    from badread_b200.qscore_model import QScoreModel
    from oracle import oracle as O
    extra = ['--bam'] if mode == 'bam' else []
    outs = {}
    for path in _files(tmp_path, 'ref', _reference_text()):
        args, out, err = _simulate(path, extra)
        outs[path.name] = out
        assert f'Loading reference from {path}' in err and 'chr: 40,000 bp, circular' in err and 'total size: 55,000 bp' in err
    if _two_gpus():
        outs['two_gpus'] = _simulate(path, extra + ['--gpus', '2'])[1]
    assert len(set(outs.values())) == 1, {k: len(v) for k, v in outs.items()}
    if mode == 'bam':
        return
    lines = next(iter(outs.values())).decode().strip().split('\n')
    records = {lines[i][1:].split(' ')[0]: (lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    sink = io.StringIO()
    ref = S.Reference(args.reference, sink)
    fl = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, sink)
    S.adjust_depths(ref, fl, args, np.random.RandomState(5))
    planner = S.ReadPlanner(args, ref, fl, Identities(args.mean_identity, args.identity_stdev, args.max_identity, sink), 5)
    orc = O.Oracle(ErrorModel(args.error_model, sink), QScoreModel(args.qscore_model, sink))
    checked = 0
    for idx in range(len(records) + 50):
        pieces, info, ident, name = planner.plan(idx)
        rec = records.get(str(name))
        if rec is None:
            continue
        seq, qual, _ = orc.sequence_fragment(planner.materialise(pieces), ident, 5, read_index=idx)
        assert rec == (seq, qual)
        checked += 1
    assert checked == len(records) >= 20
