"""The gzip inflater on the GPU (bb_gzip_decompress, bgzf.gunzip): zlib's bytes and the emulator's stats on the corpus of
tests/test_gunzip.py, the parallel path doing the work on a level-6 FASTA, a member past 4 GiB, and the simulate
reference loaded from plain gzip without the host inflating it."""
import gzip
import zlib

import numpy as np
import pytest

from test_gunzip import CORPUS, REFUSALS, emu_gunzip, planted_false_candidate, repeats_stream

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('chunk', [0, 2048])
@pytest.mark.parametrize('case', sorted(CORPUS))
def test_device_equals_zlib_and_emulator(case, chunk):
    from badread_b200.bgzf import gunzip
    stream, data = CORPUS[case]
    out, stats = gunzip(stream, chunk_bytes=chunk)
    assert bytes(out) == data
    if case == 'bgzf':   # every member BGZF: one warp per member
        assert stats['bgzf'] == 1 and stats['chunks'] == 0
        return
    assert stats == emu_gunzip.gunzip(stream, chunk)[1]


def test_planted_false_candidate_and_markers():
    from badread_b200.bgzf import gunzip
    stream, data, chunk = planted_false_candidate()
    out, stats = gunzip(stream, chunk_bytes=chunk)
    assert bytes(out) == data and stats['repaired'] >= 1 and stats == emu_gunzip.gunzip(stream, chunk)[1]
    stream, data = repeats_stream()
    out, stats = gunzip(stream, chunk_bytes=256)
    assert bytes(out) == data and stats == emu_gunzip.gunzip(stream, 256)[1]


@pytest.mark.parametrize('case', sorted(REFUSALS))
def test_refusals(case):
    from badread_b200.bgzf import gunzip
    stream, idx, at, why = REFUSALS[case]
    for chunk in (0, 2048):
        with pytest.raises(ValueError, match=rf'member {idx} \(offset {at}\): {why}'):
            gunzip(stream, chunk_bytes=chunk)


def test_level6_fasta_runs_in_parallel():
    from badread_b200.bgzf import gunzip
    rs = np.random.RandomState(12)
    bases = np.frombuffer(b'ACGTacgt', np.uint8)[rs.randint(0, 8, 30_000_000)].tobytes()
    text = b'>big\n' + b'\n'.join(bases[i:i + 60] for i in range(0, len(bases), 60)) + b'\n'
    stream = gzip.compress(text, 6)
    out, stats = gunzip(stream)
    assert bytes(out) == text
    assert stats['chunks'] > 1 and stats['chunks'] - stats['absorbed'] > 1 and stats['chained'] == 0, stats


def test_member_past_4_gib():
    """One member of 4.3 GB: a 4 MiB piece compressed once with a full flush (independent, byte-aligned, non-final
    blocks), repeated, then an empty final block.  ISIZE wraps and every offset needs 64 bits."""
    from badread_b200.bgzf import gunzip
    rs = np.random.RandomState(13)
    piece = np.frombuffer(b'ACGT', np.uint8)[rs.randint(0, 4, 1 << 22)].tobytes()
    co = zlib.compressobj(1, zlib.DEFLATED, -15)
    body = co.compress(piece) + co.flush(zlib.Z_FULL_FLUSH)
    reps = 1030
    crc = 0
    for _ in range(reps):
        crc = zlib.crc32(piece, crc)
    total = reps * len(piece)
    assert total > 2 ** 32
    stream = b'\x1f\x8b\x08\0\0\0\0\0\0\xff' + body * reps + b'\x03\x00' + (crc.to_bytes(4, 'little') +
                                                                          (total & 0xffffffff).to_bytes(4, 'little'))
    out, stats = gunzip(stream)
    assert len(out) == total and stats['members'] == 1 and stats['chained'] == 0
    view = memoryview(out)
    for k in range(reps):
        assert view[k * len(piece):(k + 1) * len(piece)] == piece, k


def test_load_fasta_from_gzip_equals_host(engine, tmp_path):
    from test_gpu_reference_load import _host, _reference_text
    from test_gunzip import header, member, raw_deflate
    text = _reference_text() * 20
    files = {'plain_gzip.fa.gz': gzip.compress(text, 6),
             'members.fa.gz': b''.join(gzip.compress(text[i:i + 70001], 1 + i % 9) for i in range(0, len(text), 70001)),
             'fields.fa.gz': member(raw_deflate(text), text, header(4 | 8 | 16 | 2, b'xy\x01\x00z', b'ref.fa', b'note'))}
    (tmp_path / 'x.fa').write_bytes(text)
    want = _host(tmp_path / 'x.fa')
    for name, blob in files.items():
        path = tmp_path / name
        path.write_bytes(blob)
        got = engine.load_fasta(str(path))
        assert tuple(got) == want[:6], name
        assert bytes(engine.download_reference(0, sum(got[1]))) == want[6], name
        st = engine.last_gzip_stats()
        assert st['bgzf'] == 0 and st['chunks'] >= 1 and st['members'] >= 1, (name, st)


def test_simulate_from_plain_gzip_never_inflates_on_the_host(tmp_path, monkeypatch):
    from test_gpu_reference_load import _reference_text, _simulate
    text = _reference_text()
    plain, gz = tmp_path / 'ref.fa', tmp_path / 'ref.fa.gz'
    plain.write_bytes(text)
    gz.write_bytes(gzip.compress(text, 6))
    want = _simulate(plain)[1]

    def refuse(*a, **k):
        raise AssertionError('the host inflated the reference')
    for name in ('open', 'decompress', 'GzipFile'):
        monkeypatch.setattr(gzip, name, refuse)
    assert _simulate(gz)[1] == want
