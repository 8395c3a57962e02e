"""Unaligned BAM output on the GPU: `simulate --bam` decodes (tests/bam_ref.py) to the FASTQ of the same run without it,
its bytes do not depend on the batch size or the number of GPUs, the device's records and members equal the emulator's,
the model builders' BAM parser accepts the file, and a batch run after a BAM build still equals the oracle."""
import ctypes
import gzip
import io
import random

import numpy as np
import pytest

import bam_ref
from emu import emu_bam as E
from test_bam_output import _Planned, synthetic
from test_gpu_bgzf import VARIANTS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engine():
    """A context of this module's own, released when the module is done (its batches allocate worker scratch)."""
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=4321)
    yield eng
    eng.close()


def _run(tmp_path, extra=(), batch_reads=16384, bam=False):
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.simulate import simulate
    rs = np.random.RandomState(11)
    ref = tmp_path / 'ref.fasta'
    if not ref.exists():
        ref.write_text('>chr circular=true\n' + bytes(np.frombuffer(b'ACGT', dtype=np.uint8)[rs.randint(0, 4, 40000)]).decode() +
                       '\n>lin depth=2\n' + bytes(np.frombuffer(b'ACGT', dtype=np.uint8)[rs.randint(0, 4, 15000)]).decode() + '\n')
    args = parse_args(['simulate', '--reference', str(ref), '--quantity', '6x', '--length', '2500,1500', '--seed', '5',
                       '--glitches', '2000,20,20', '--chimeras', '5', '--batch_reads', str(batch_reads)] + list(extra) +
                      (['--bam'] if bam else []))
    check_simulate_args(args)
    out = io.BytesIO() if bam else io.StringIO()
    simulate(args, output=io.StringIO(), stdout=out)
    return out.getvalue()


def check_bam_file(bam, fastq):
    from badread_b200.bam import header_bytes
    text, refs, recs, ms, header_end = bam_ref.read_bam(bam)
    assert ms[0][1] == header_bytes() and header_end == len(ms[0][1])   # the header in a member of its own
    assert ms[-1][0] == bam_ref.EOF_MEMBER and all(len(d) for _, d in ms[:-1])
    assert bam_ref.to_fastq(recs) == fastq
    return recs


@pytest.mark.parametrize('extra', VARIANTS, ids=['default', 'nanopore2020', 'pacbio2021', 'random_ideal'])
def test_simulate_bam_decodes_to_the_fastq(tmp_path, extra):
    fastq = _run(tmp_path, extra).encode('latin-1')
    bam = _run(tmp_path, extra, bam=True)
    recs = check_bam_file(bam, fastq)
    assert len(recs) == fastq.count(b'\n') // 4
    assert len(bam) < len(fastq) / 1.5


def test_simulate_bam_independent_of_batches_and_gpus(tmp_path, monkeypatch):
    bam = _run(tmp_path, bam=True)
    assert _run(tmp_path, batch_reads=100, bam=True) == bam
    import torch
    if torch.cuda.device_count() >= 2:
        assert _run(tmp_path, ['--gpus', '2'], bam=True) == bam
    # the merge path of --gpus 2 on two contexts of device 0, without NCCL
    import badread_b200.engine as engine_mod
    import badread_b200.simulate as sim
    real = engine_mod.Engine
    monkeypatch.setattr(sim, 'Engine', lambda device=0, seed=0: real(device=0, seed=seed))
    monkeypatch.setattr(engine_mod, 'nccl_available', lambda: False)
    assert _run(tmp_path, ['--gpus', '2'], bam=True) == bam
    assert _run(tmp_path, ['--gpus', '3'], batch_reads=100, bam=True) == bam


def test_model_builder_parser_accepts_the_file(tmp_path):
    """bb_aln_parse(is_bam=1) takes the inflated file (inflated on the GPU) and finds no mapped record in it."""
    from badread_b200 import _lib
    from badread_b200.bgzf import decompress
    bam = _run(tmp_path, bam=True)
    raw = decompress(bam)
    assert bytes(raw) == gzip.decompress(bam)
    L = _lib.lib()
    buf = np.frombuffer(raw, dtype=np.uint8)
    handle = ctypes.c_void_p()
    assert L.bb_aln_parse(buf.ctypes.data_as(ctypes.c_void_p), buf.size, 1, 0, ctypes.byref(handle)) == _lib.BB_OK
    v = _lib.AlnView()
    L.bb_aln_view_get(handle, ctypes.byref(v))
    assert v.n_records == 0 and v.n_refs == 0
    L.bb_aln_free(handle)


def _batch(engine, n_reads, seed):
    """A batch of literal reads large enough to be split over the context's workers; returns (BatchResult, planned)."""
    from badread_b200.engine import FragmentBatch
    from conftest import load_models, random_dna
    em, qm = load_models('nanopore2023', 'nanopore2023')
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    rnd = random.Random(seed)
    batch = FragmentBatch()
    frags = [random_dna(rnd, rnd.choice([1, 2, 3, rnd.randint(50, 3000)])) for _ in range(n_reads)]
    for i, f in enumerate(frags):
        batch.add_literal_read(i, f, 0.9)
    res, total = engine.sequence_batch(batch)
    planned = _Planned([rnd.getrandbits(128).to_bytes(16, 'big') for _ in frags], [f'r{i}' for i in range(n_reads)],
                       [len(f) for f in frags])
    return res, total, planned, frags


def test_device_records_and_members_equal_the_emulator(engine):
    from badread_b200.planner import bam_layout_sharded
    res, total, planned, _ = _batch(engine, 300, 1)
    lay = bam_layout_sharded([planned], [res.records], 0, 0, 10 ** 12, 0)
    seq, qual = np.array(res.seq[:total]), np.array(res.qual[:total])
    want, want_fields = E.records(lay.recs, lay.text, [(seq, qual)])
    assert (want_fields == lay.fields).all()
    engine.bam_build(lay.recs, lay.text)
    got = np.zeros(lay.stream_len, np.uint8)
    assert engine.bam_fetch_records(got) == lay.stream_len
    assert got.tobytes() == want
    # several builds on the device stream, compressed in whole chunks with the rest carried, then the rest
    data, fields, members = b'', [], []
    for k in range(3):
        lay = bam_layout_sharded([planned], [res.records], 0, 0, 10 ** 12, len(data))
        engine.bam_build(lay.recs, lay.text)
        members.append(bytes(engine.bam_compress_device(final=False)))
        data += want
        fields.append(lay.fields)
    members.append(bytes(engine.bam_compress_device(final=True)))
    fields = np.concatenate(fields)
    whole, _ = E.compress(data, 0, fields, final=True)
    assert b''.join(members) == whole
    assert bam_ref.members(whole)[0][1] == data[:E.CHUNK]
    # host bytes through bb_bam_compress, split at a point that is not a chunk boundary
    cut = 3 * E.CHUNK + 1234
    a, used = engine.bam_compress(data[:cut], 0, fields, final=False)
    a = bytes(a)   # (the members are a view of a buffer the next call reuses)
    b, _ = engine.bam_compress(data[used:], used, fields, final=True)
    assert used == 3 * E.CHUNK and a + bytes(b) == whole


def test_batch_after_bam_build_equals_the_oracle(engine):
    from badread_b200.engine import FragmentBatch
    from badread_b200.planner import bam_layout_sharded
    from conftest import load_models, random_dna
    from oracle import oracle as O
    res, total, planned, _ = _batch(engine, 150, 2)
    lay = bam_layout_sharded([planned], [res.records], 0, 0, 10 ** 12, 0)
    engine.bam_build(lay.recs, lay.text)
    engine.bam_compress_device(final=True)
    em, qm = load_models('nanopore2023', 'nanopore2023')
    rnd = random.Random(8)
    frags = [random_dna(rnd, 1000 + 500 * i) for i in range(4)]
    batch = FragmentBatch()
    for i, f in enumerate(frags):
        batch.add_literal_read(i, f, 0.9)
    res, _ = engine.sequence_batch(batch)
    orc = O.Oracle(em, qm)
    for i, f in enumerate(frags):
        s, q, _ = orc.sequence_fragment(f, 0.9, engine.seed, read_index=i)
        assert res.read(i) == (s, q)


def test_build_needs_a_fetched_batch_and_valid_records(engine):
    from badread_b200.engine import EngineError, FragmentBatch
    from badread_b200.planner import BAM_RECORD_DTYPE
    res, total, planned, _ = _batch(engine, 4, 3)
    bad = np.zeros(1, BAM_RECORD_DTYPE)
    bad['out_off'], bad['out_len'], bad['name_len'] = total - 1, 2, 1
    with pytest.raises(EngineError, match='outside the batch output'):
        engine.bam_build(bad, b'x')
    batch = FragmentBatch()
    batch.add_literal_read(0, 'ACGT' * 50, 0.9)
    engine.upload_batch(batch)
    bad['out_off'], bad['out_len'] = 0, 1
    with pytest.raises(EngineError, match='no fetched batch'):
        engine.bam_build(bad, b'x')
    engine.run_batch_results(batch)
    engine.bam_build(bad, b'x')
    out = np.zeros(200, np.uint8)
    assert engine.bam_fetch_records(out) == E.record_size(1, 1, 0)
