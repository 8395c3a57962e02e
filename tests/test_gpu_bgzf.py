"""BGZF output on the GPU: `simulate --gzip` inflates to the FASTQ of the same run without it, the compressed bytes do not
depend on the batch size or the number of GPUs, Engine.bgzf_compress splits anywhere over a large buffer, and the
device gives the emulator's bytes (tests/test_bgzf.py checks those against zlib)."""
import gzip
import io
import random

import numpy as np
import pytest

from emu import emu_bgzf as B
from test_bgzf import CHUNK, EOF, MODEL_PAIRS, cases, check, oracle_fastq

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engine():
    """A context of this module's own, released when the module is done: the batch below allocates its workers' scratch,
    which the session-wide context would keep for the GPU tests that come after (several of them create contexts of
    their own, with up to four workers)."""
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=1234)
    yield eng
    eng.close()

# the parameter sets of test_gpu_cli.py: its default run and its three config variants
VARIANTS = [
    [],
    ['--quantity', '2x', '--error_model', 'nanopore2020', '--qscore_model', 'nanopore2020', '--identity', '90,98,5',
     '--glitches', '1000,100,100'],
    ['--quantity', '2x', '--error_model', 'pacbio2021', '--qscore_model', 'pacbio2021', '--chimeras', '10'],
    ['--quantity', '2x', '--error_model', 'random', '--qscore_model', 'ideal', '--identity', '12,3', '--junk_reads', '10',
     '--random_reads', '10'],
]


def _run(tmp_path, extra=(), batch_reads=16384, gz=False):
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.simulate import simulate
    rs = np.random.RandomState(11)
    ref = tmp_path / 'ref.fasta'
    if not ref.exists():
        ref.write_text('>chr circular=true\n' + bytes(np.frombuffer(b'ACGT', dtype=np.uint8)[rs.randint(0, 4, 40000)]).decode() +
                       '\n>lin depth=2\n' + bytes(np.frombuffer(b'ACGT', dtype=np.uint8)[rs.randint(0, 4, 15000)]).decode() + '\n')
    args = parse_args(['simulate', '--reference', str(ref), '--quantity', '6x', '--length', '2500,1500', '--seed', '5',
                       '--glitches', '2000,20,20', '--chimeras', '5', '--batch_reads', str(batch_reads)] + list(extra) +
                      (['--gzip'] if gz else []))
    check_simulate_args(args)
    out = io.BytesIO() if gz else io.StringIO()
    simulate(args, output=io.StringIO(), stdout=out)
    return out.getvalue()


@pytest.mark.parametrize('extra', VARIANTS, ids=['default', 'nanopore2020', 'pacbio2021', 'random_ideal'])
def test_simulate_gzip_inflates_to_the_fastq(tmp_path, extra):
    fastq = _run(tmp_path, extra).encode('latin-1')
    comp = _run(tmp_path, extra, gz=True)
    assert comp.endswith(EOF)
    assert gzip.decompress(comp) == fastq
    check(fastq, comp[:-len(EOF)])
    assert len(comp) < len(fastq) / 1.5


def test_simulate_gzip_independent_of_batches_and_gpus(tmp_path):
    comp = _run(tmp_path, gz=True)
    assert _run(tmp_path, batch_reads=100, gz=True) == comp
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU: --gpus 2 not compared')
    assert _run(tmp_path, ['--gpus', '2'], gz=True) == comp


def _synthetic_fastq(n_bytes, seed=1):
    """FASTQ records of random reads (500 .. 30 000 bases, qualities '!' .. 'Z'), built in numpy."""
    rs = np.random.RandomState(seed)
    parts, total, i = [], 0, 0
    acgt = np.frombuffer(b'ACGT', dtype=np.uint8)
    while total < n_bytes:
        n = int(rs.randint(500, 30000))
        rec = b'@%032x length=%d\n' % (int(rs.randint(0, 2 ** 62)) * (i + 1), n) + acgt[rs.randint(0, 4, n)].tobytes() + \
            b'\n+\n' + (rs.randint(33, 91, n).astype(np.uint8)).tobytes() + b'\n'
        parts.append(rec)
        total += len(rec)
        i += 1
    return b''.join(parts)


def test_engine_compress_split_anywhere_large_buffer(engine):
    """256 MB through Engine.bgzf_compress: one call, and calls split at random points (the caller carries the rest and
    the line index mod 4 of its first byte), give the same bytes; the stream inflates back.  Covers the passes of 2048
    chunks and the compaction of thousands of members."""
    data = _synthetic_fastq(256 << 20)
    whole = bytes(engine.bgzf_compress(data, 0, final=True)[0])
    assert gzip.decompress(whole + EOF) == data
    rnd = random.Random(2)
    got, pos = [], 0
    view = memoryview(data)
    for cut in sorted(rnd.sample(range(1, len(data)), 6)) + [len(data)]:
        mod4 = data.count(b'\n', 0, pos) & 3
        comp, used = engine.bgzf_compress(view[pos:cut], mod4, final=cut == len(data))
        got.append(bytes(comp))
        pos += used
    assert pos == len(data) and b''.join(got) == whole


@pytest.mark.parametrize('name,data,line_mod4', cases(), ids=[c[0] for c in cases()])
def test_device_bytes_equal_the_emulator(engine, name, data, line_mod4):
    got = bytes(engine.bgzf_compress(data, line_mod4, final=True)[0])
    assert got == B.compress(data, line_mod4, final=True)[0]


@pytest.mark.parametrize('pair', MODEL_PAIRS, ids=[p[0] for p in MODEL_PAIRS])
def test_device_bytes_equal_the_emulator_on_oracle_fastq(engine, pair):
    fastq = oracle_fastq(*pair)
    lines = fastq.split(b'\n')
    for mod4 in range(4):
        data = b'\n'.join(lines[mod4:])
        got = bytes(engine.bgzf_compress(data, mod4, final=True)[0])
        assert got == B.compress(data, mod4, final=True)[0]
        check(data, got)


def test_compress_leaves_the_batch_workers_alone(engine):
    """A compress call between batches does not disturb the workers: the next batch still equals the oracle."""
    from badread_b200.engine import FragmentBatch
    from conftest import load_models, random_dna
    from oracle import oracle as O
    em, qm = load_models('nanopore2023', 'nanopore2023')
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    rnd = random.Random(8)
    frags = [random_dna(rnd, 1000 + 500 * i) for i in range(4)]
    batch = FragmentBatch()
    for i, f in enumerate(frags):
        batch.add_literal_read(i, f, 0.9)
    engine.bgzf_compress(_synthetic_fastq(3 * CHUNK), 0, final=True)
    res, _ = engine.sequence_batch(batch)
    engine.bgzf_compress(_synthetic_fastq(5 * CHUNK, seed=2), 0, final=True)
    orc = O.Oracle(em, qm)
    for i, f in enumerate(frags):
        s, q, _ = orc.sequence_fragment(f, 0.9, engine.seed, read_index=i)
        assert res.read(i) == (s, q)
