"""Error model files loaded on the GPU (Engine.load_error_model_file / DeviceErrorModel) against the host loader: the
tables bit for bit on the golden models (plain, gzip and BGZF) and on seeded synthetic models of every index kind, hash
lookups, reads simulated with either model, the oracle's reads, the fallbacks and `simulate` end to end."""
import gzip
import io
import pathlib
import random
import subprocess
import sys
import types

import numpy as np
import pytest

from badread_b200 import _lib
from badread_b200.error_model import DeviceErrorModel, ErrorModel, load_error_model

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parent.parent
GOLDEN = ROOT / 'tests' / 'golden' / 'models'
MODELS = sorted(p.name for p in GOLDEN.glob('error_model_*.txt.gz'))
TABLE_KEYS = ('row_off', 'cum', 'flags', 'slots', 'pool', 'probs', 'kmer_codes', 'kmer_to_row')


def _synthetic(k, n_rows, seed):
    """Model text in the builders' form over n_rows distinct k-mers (drawn from a seeded permutation of codes)."""
    rng = np.random.default_rng(seed)
    codes = rng.choice(4 ** k, size=n_rows, replace=False) if 4 ** k < 2 ** 40 else None
    shifts = 2 * np.arange(k - 1, -1, -1, dtype=np.int64)
    letters = np.frombuffer(b'ACGT', np.uint8)
    kmers = letters[(codes[:, None] >> shifts) & 3]
    rnd = random.Random(seed)
    out = []
    for row in kmers:
        km = row.tobytes().decode()
        alts = [km]
        for _ in range(rnd.randint(0, 3)):
            i = rnd.randint(1, k - 2)
            kind = rnd.random()
            alt = km[:i] + (rnd.choice('ACGT') * rnd.randint(1, 6) if kind < 0.5 else '') + km[i + (kind >= 0.3):]
            if len(alt) >= 2 and alt not in alts:
                alts.append(alt)
        ps = [rnd.random() for _ in alts]
        s = rnd.choice((1.0, 0.95)) / sum(ps)
        out.append(''.join(f'{a},{p * s:.6f};' for a, p in zip(alts, ps)))
    return ('\n'.join(out) + '\n').encode()


@pytest.fixture(scope='module')
def engine():
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=5)
    yield eng
    eng.close()


def _write(tmp_path, name, text, form, engine=None):
    path = tmp_path / name
    if form == 'plain':
        path.write_bytes(text)
    elif form == 'gzip':
        path.write_bytes(gzip.compress(text))
    else:   # BGZF, compressed on the GPU by bgzf.py
        from badread_b200.bgzf import BGZFWriter
        buf = io.BytesIO()
        w = BGZFWriter([engine], buf)
        w.write(text)
        w.close()
        path.write_bytes(buf.getvalue())
    return path


def _assert_same(engine, path, index_kind=None):
    info = engine.load_error_model_file(str(path))
    assert info['fallback'] == 0, info
    want = ErrorModel(str(path), io.StringIO())
    got = engine.download_error_model(info)
    assert set(got) == set(want._tables)
    for key in TABLE_KEYS:
        if key in want._tables:
            assert got[key].dtype == want._tables[key].dtype, key
            assert got[key].tobytes() == want._tables[key].tobytes(), key
    if index_kind is not None:
        assert info['index'] == index_kind
    return info, want


@pytest.mark.parametrize('form', ['plain', 'gzip', 'bgzf'])
@pytest.mark.parametrize('name', MODELS)
def test_golden_models(engine, tmp_path, name, form):
    text = gzip.open(GOLDEN / name, 'rb').read()
    _assert_same(engine, _write(tmp_path, name.replace('.gz', ''), text, form, engine))


@pytest.mark.parametrize('k,n_rows,index_kind', [(12, 200_000, 1), (13, 200_000, 2), (16, 1_000_000, 2)])
def test_synthetic_models(engine, tmp_path, k, n_rows, index_kind):
    path = _write(tmp_path, f'k{k}.txt', _synthetic(k, n_rows, k), 'gzip')
    info, want = _assert_same(engine, path, index_kind)
    assert info['n_rows'] == n_rows


def test_hash_lookups(engine, tmp_path):
    """Every row's code finds its row through the device-built model's hash table, and absent codes find none: reads
    simulated through the device-loaded hash index equal reads through an upload of the host tables' hash index."""
    from badread_b200.engine import FragmentBatch
    path = _write(tmp_path, 'k13.txt', _synthetic(13, 50_000, 3), 'plain')
    dm = DeviceErrorModel.load(str(path), [engine], io.StringIO())
    assert dm is not None and dm.info['index'] == 2
    hm = ErrorModel(str(path), io.StringIO())
    from badread_b200.qscore_model import QScoreModel
    engine.set_qscore_model(QScoreModel('nanopore2023', io.StringIO()))
    rnd = random.Random(1)
    codes = dm._tables['kmer_codes']
    kmers = [''.join('ACGT'[(int(c) >> (2 * (12 - j))) & 3] for j in range(13)) for c in codes[:2000]]
    batch = FragmentBatch()
    for i in range(60):   # fragments made of the model's k-mers and of random ones
        frag = ''.join(rnd.choice(kmers) if rnd.random() < 0.7 else ''.join(rnd.choice('ACGT') for _ in range(13))
                       for _ in range(rnd.randint(20, 200)))
        batch.add_literal_read(i, frag, 0.9)
    engine.load_error_model_file(str(path), owner=dm)
    a, _ = engine.sequence_batch(batch)
    ra = [a.read(i) for i in range(60)]
    engine.set_error_model(hm, index='hash')
    b, _ = engine.sequence_batch(batch)
    assert ra == [b.read(i) for i in range(60)]


@pytest.mark.parametrize('name', ['error_model_k7.txt.gz', 'error_model_k16.txt.gz'])
def test_reads_equal_host_model_and_oracle(engine, name):
    from badread_b200.engine import FragmentBatch
    from badread_b200.qscore_model import QScoreModel
    from oracle.oracle_kmers import make_oracle
    sink = io.StringIO()
    qm = QScoreModel('nanopore2023', sink)
    engine.set_qscore_model(qm)
    dm = DeviceErrorModel.load(str(GOLDEN / name), [engine], sink)
    hm = ErrorModel(str(GOLDEN / name), sink)
    rnd = random.Random(7)
    frags = [''.join(rnd.choice('ACGT') for _ in range(rnd.randint(200, 3000))) for _ in range(300)]
    batch = FragmentBatch()
    for i, f in enumerate(frags):
        batch.add_literal_read(i, f, 0.9)
    engine.set_error_model(dm)   # (already installed: nothing is uploaded)
    got, _ = engine.sequence_batch(batch)
    dev = [got.read(i) for i in range(len(frags))]
    orc = make_oracle(dm, qm)   # (dm's tables come from the engine, so before it installs hm's)
    engine.set_error_model(hm)
    ref, _ = engine.sequence_batch(batch)
    assert dev == [ref.read(i) for i in range(len(frags))]
    for i in range(0, len(frags), 30):
        s, q, _ = orc.sequence_fragment(frags[i], 0.9, 5, read_index=i)
        assert dev[i] == (s, q)


def test_set_error_model_does_not_upload_again(engine, monkeypatch):
    dm = DeviceErrorModel.load(str(GOLDEN / 'error_model_k5_alt3.txt.gz'), [engine], io.StringIO())
    calls = []
    lib = engine._lib
    monkeypatch.setattr(engine, '_lib', types.SimpleNamespace(
        bb_upload_error_model=lambda *a: calls.append(a) or 0, bb_upload_error_model_kmers=lambda *a: calls.append(a) or 0,
        bb_last_error=lib.bb_last_error))
    engine.set_error_model(dm)
    assert calls == [] and engine.error_model is dm


def test_messages_and_lazy_tables(engine, tmp_path):
    path = GOLDEN / 'error_model_k13.txt.gz'
    a, b = io.StringIO(), io.StringIO()
    dm = load_error_model(str(path), [engine], a)
    hm = ErrorModel(str(path), b)
    assert isinstance(dm, DeviceErrorModel)
    assert a.getvalue() == b.getvalue()
    assert dm.alternatives == hm.alternatives and dm.probabilities == hm.probabilities
    dm.save_tables(tmp_path / 'd.npz')
    hm.save_tables(tmp_path / 'h.npz')
    with np.load(tmp_path / 'd.npz') as x, np.load(tmp_path / 'h.npz') as y:
        assert sorted(x.files) == sorted(y.files) and all(np.array_equal(x[f], y[f]) for f in x.files)


@pytest.mark.parametrize('text,reason', [(b'AAAA,1e-1;\n', 'number'), (b'AAAA,0.5;\nAAAA,0.5;\n', 'duplicate'),
                                         (b'AAAA,0.5;\r\n', 'cr'), (b'AAAA,0.5;\n\nCCCC,1;\n', 'empty_line'),
                                         (b'AAAA,0.5;ANNA,0.5;\n', 'base')])
def test_fallback_uses_the_host_loader(engine, tmp_path, text, reason):
    path = tmp_path / 'm.txt'
    path.write_bytes(text)
    info = engine.load_error_model_file(str(path))
    assert info['fallback'] & _lib.EM_FALLBACK[reason]
    a, b = io.StringIO(), io.StringIO()
    try:
        want = ErrorModel(str(path), b)
    except BaseException as e:   # the host loader's error, raised the same way
        with pytest.raises(type(e)):
            load_error_model(str(path), [engine], a)
    else:
        got = load_error_model(str(path), [engine], a)
        assert type(got) is ErrorModel and a.getvalue() == b.getvalue()
        assert all(np.array_equal(got._tables[k], want._tables[k]) for k in want._tables)


def test_duplicate_in_a_hash_model_falls_back(engine, tmp_path):
    text = _synthetic(13, 1000, 4)
    lines = text.split(b'\n')
    path = tmp_path / 'dup.txt'
    path.write_bytes(b'\n'.join(lines[:-1] + [lines[3]]) + b'\n')
    assert engine.load_error_model_file(str(path))['fallback'] & _lib.EM_FALLBACK['duplicate']


@pytest.mark.parametrize('gpus', [1, 2])
def test_simulate_cli_routes_agree(tmp_path, gpus):
    from badread_b200.engine import _lib as L
    if gpus > L.lib().bb_device_count():
        pytest.skip('needs 2 GPUs')
    model = GOLDEN / 'error_model_k7.txt.gz'
    base = [sys.executable, '-m', 'badread_b200', 'simulate', '--reference', str(GOLDEN / 'ref.fasta'), '--quantity', '20x',
            '--error_model', str(model), '--qscore_model', 'nanopore2023', '--seed', '1', '--gpus', str(gpus)]
    dev = subprocess.run(base, capture_output=True, cwd=ROOT, check=True)
    patch = ('import sys, runpy; import badread_b200.error_model as m; '
             'm.DeviceErrorModel.load = classmethod(lambda cls, *a, **k: None); '
             'sys.argv = ["badread_b200"] + sys.argv[1:]; runpy.run_module("badread_b200", run_name="__main__")')
    host = subprocess.run([sys.executable, '-c', patch] + base[3:], capture_output=True, cwd=ROOT, check=True)
    assert dev.stdout == host.stdout and len(dev.stdout) > 0
    assert dev.stderr == host.stderr
