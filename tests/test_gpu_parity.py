"""
GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle in Philox mode on the same
seeded inputs. Integer / byte / index work: the bar is bit-exact sequences, quality strings and alignment counts.
"""
import random

import pytest

from conftest import load_models, mutate, random_dna

pytestmark = pytest.mark.gpu


def _oracle(em, qm):
    from oracle import oracle as O
    return O, O.Oracle(em, qm)


def test_align_path_matches_oracle(engine):
    from oracle import oracle as O
    rnd = random.Random(11)
    cases = []
    for _ in range(60):
        n = rnd.randint(1, 1500)
        a = random_dna(rnd, n)
        b = mutate(rnd, a, rnd.choice([0.0, 0.02, 0.1, 0.3])) if rnd.random() < 0.8 else random_dna(rnd, rnd.randint(1, 900), 'ACGTN')
        cases.append((a, b))
    # sizes beyond edlib's 1 MiB traceback estimate -> Hirschberg; multi-strip queries
    for n, rate in ((2500, 0.05), (4000, 0.1), (6000, 0.02), (3000, 0.3)):
        a = random_dna(rnd, n)
        cases.append((a, mutate(rnd, a, rate)))
        cases.append((mutate(rnd, a, rate), a))
    cases.append((random_dna(rnd, 3000), random_dna(rnd, 700)))   # tall leaf: 3 strips, few columns
    cases.append((random_dna(rnd, 40), random_dna(rnd, 30000)))   # wide leaf
    for a, b in cases:
        want_ops, want_d = O.align_path(a, b)
        got_ops, got_d = engine.align_path(a, b)
        assert got_d == want_d
        assert got_ops == want_ops


@pytest.mark.parametrize('error_name,qscore_name', [('random', 'ideal'), ('random', 'random'),
                                                    ('nanopore2023', 'nanopore2023'),
                                                    ('nanopore2020', 'nanopore2020'),
                                                    ('pacbio2021', 'pacbio2021')])
def test_sequence_batch_matches_oracle(engine, error_name, qscore_name):
    from badread_b200.engine import FragmentBatch
    em, qm = load_models(error_name, qscore_name)
    O, orc = _oracle(em, qm)
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    import zlib
    rnd = random.Random(zlib.crc32((error_name + qscore_name).encode()))
    lengths = [1, 2, 5, 30, 200, 985, 986, 987, 1000, 1400, 3000, 5000, 9000, 20000]
    batch = FragmentBatch()
    frags, idents = [], []
    for i, n in enumerate(lengths * 2):
        frag = random_dna(rnd, n, 'ACGT' if i % 5 else 'ACGTN')
        ident = rnd.choice([1.0, 0.99, 0.95, 0.9, 0.8, 0.6]) if i >= len(lengths) else 0.93
        frags.append(frag)
        idents.append(ident)
        batch.add_literal_read(1000 + i, frag, ident)
    res, total = engine.sequence_batch(batch)
    assert total == sum(res.records[i].out_len for i in range(len(frags)))
    for i, (frag, ident) in enumerate(zip(frags, idents)):
        s, q, identity, st = orc.sequence_fragment(frag, ident, engine.seed, read_index=1000 + i, with_stats=True)
        gs, gq = res.read(i)
        rec = res.records[i]
        assert (rec.loop_count, rec.change_count, rec.n_alignments) == (st['loop_count'], st['change_count'], st['n_alignments']), (i, len(frag), ident)
        assert gs == s, (i, len(frag), ident)
        assert gq == q, (i, len(frag), ident)
        assert (rec.matches, rec.columns) == (st['matches'], st['columns'])
        assert rec.frag_len == len(frag)


def test_large_batch_split_over_workers_matches_oracle(engine):
    """A batch big enough to be dealt out over the context's sub-batch workers (>= 64 reads per worker): every read,
    wherever it ran and wherever its block landed in the output buffers, equals the oracle's."""
    _check_large_split_batch(engine)


def test_head_batch_matches_oracle(monkeypatch):
    """The same batch on a context of three workers: worker 0 then carries a head batch of the 43 longest reads (3 or
    more workers and at least 16 reads of >= 0.6x the longest), run by bb_k_mutate_chain on high-priority streams."""
    from badread_b200.engine import Engine
    monkeypatch.setenv('BADREAD_B200_SUBBATCHES', '3')
    monkeypatch.setenv('BADREAD_B200_HEAD_WORKER', '1')
    eng = Engine(device=0, seed=1234)
    try:
        _check_large_split_batch(eng)
    finally:
        eng.close()


def _check_large_split_batch(engine):
    from badread_b200.engine import FragmentBatch
    em, qm = load_models('nanopore2023', 'nanopore2023')
    O, orc = _oracle(em, qm)
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    rnd = random.Random(20260924)
    n_reads = 700
    batch = FragmentBatch()
    frags, idents = [], []
    for i in range(n_reads):
        n = rnd.choice([1, 40, 300, 900, 1500, 2600, 4000]) + rnd.randrange(0, 50)
        frag = random_dna(rnd, n, 'ACGT' if i % 11 else 'ACGTN')
        ident = rnd.choice([1.0, 0.98, 0.93, 0.88, 0.8])
        frags.append(frag)
        idents.append(ident)
        batch.add_literal_read(5000 + 3 * i, frag, ident)
    res, total = engine.sequence_batch(batch)
    assert total == sum(res.records[i].out_len for i in range(n_reads))
    spans = sorted((res.records[i].out_off, res.records[i].out_len) for i in range(n_reads) if res.records[i].out_len)
    assert spans[0][0] == 0 and all(a + la == b for (a, la), (b, _) in zip(spans, spans[1:]))   # packed, no overlap
    assert spans[-1][0] + spans[-1][1] == total
    outs, _ = orc.sequence_batch(frags, idents, engine.seed, [5000 + 3 * i for i in range(n_reads)], n_threads=8)
    for i in range(n_reads):
        gs, gq = res.read(i)
        assert (gs, gq) == (outs[i][0], outs[i][1]), (i, len(frags[i]), idents[i])
        rec = res.records[i]
        assert rec.frag_len == len(frags[i])
        assert (rec.matches, rec.columns) == (outs[i][2], outs[i][3])


def test_output_buffers_grow_on_capacity_error(engine):
    """bb_sequence_batch with buffers that are too small reports BB_ERR_CAPACITY and the needed size; the fetch is
    repeated with larger buffers (single-worker and split batches), and the reads are unchanged."""
    from badread_b200.engine import FragmentBatch
    em, qm = load_models('random', 'ideal')
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    rnd = random.Random(77)
    for n_reads in (5, 300):
        batch = FragmentBatch()
        for i in range(n_reads):
            batch.add_literal_read(i, random_dna(rnd, rnd.randrange(2000, 3000)), 0.9)
        ref, total = engine.sequence_batch(batch)
        want = [ref.read(i) for i in range(n_reads)]
        engine._seq_buf = engine._qual_buf = None
        engine._out_cap = 0
        engine._ensure_out(16)                      # far too small for the batch
        assert engine._out_cap < total
        got, total2 = engine.sequence_batch(batch)
        assert total2 == total and engine._out_cap >= total
        assert [got.read(i) for i in range(n_reads)] == want


def _np_dna(seed, n):
    import numpy as np
    return np.frombuffer(b'ACGT', dtype=np.uint8)[np.random.RandomState(seed).randint(0, 4, n)].tobytes().decode('ascii')


# Long reads: the regime that carries most of the benchmark's bases (58 % of configs[1] sits in reads > 20 kb; the
# longest is ~150 kb) and all of config 5.  Lengths x identities are chosen to reach both final-alignment pipelines
# (lean single-warp nodes; wide roots by warp pairs with 8-, 16- and 32-word chunks) and the strip fallback
# (a + b > 30 * 1024 rows: 150 kb at identity 0.75).
LONG_CASES = [(25000, 0.95), (25000, 0.8), (40000, 0.9), (40000, 0.95), (60000, 0.95), (60000, 0.8), (100000, 0.9),
              (100000, 0.95), (150000, 0.95), (150000, 0.9), (150000, 0.8), (150000, 0.75), (131072, 0.99), (33000, 1.0)]


@pytest.mark.parametrize('error_name,qscore_name', [('nanopore2023', 'nanopore2023'), ('nanopore2020', 'nanopore2020')])
def test_long_reads_match_oracle(engine, error_name, qscore_name):
    from badread_b200.engine import FragmentBatch
    em, qm = load_models(error_name, qscore_name)
    O, orc = _oracle(em, qm)
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    batch = FragmentBatch()
    frags, idents, ridx = [], [], []
    for i, (n, ident) in enumerate(LONG_CASES):
        frags.append(_np_dna(977 + i, n))
        idents.append(ident)
        ridx.append(90000 + 7 * i)
        batch.add_literal_read(ridx[-1], frags[-1], ident)
    res, total = engine.sequence_batch(batch)
    outs, _ = orc.sequence_batch(frags, idents, engine.seed, ridx, n_threads=max(1, min(16, len(frags))))
    for i in range(len(frags)):
        gs, gq = res.read(i)
        rec = res.records[i]
        assert rec.flags == 0
        assert gs == outs[i][0], (i, LONG_CASES[i])
        assert gq == outs[i][1], (i, LONG_CASES[i])
        assert (rec.matches, rec.columns) == (outs[i][2], outs[i][3]), (i, LONG_CASES[i])
    assert total == sum(len(o[0]) for o in outs)


def test_long_reads_in_a_split_batch_match_oracle(engine):
    """Long reads inside a batch that is dealt out over the sub-batch workers (>= 64 reads per worker): the wide-root
    pipeline runs next to the lean one on every worker, as in the benchmark."""
    from badread_b200.engine import FragmentBatch
    em, qm = load_models('nanopore2023', 'nanopore2023')
    O, orc = _oracle(em, qm)
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    rnd = random.Random(4242)
    lens = [rnd.choice([300, 2500, 9000]) + rnd.randrange(100) for _ in range(280)]
    lens += [22000, 31000, 48000, 75000, 120000, 149690]
    batch = FragmentBatch()
    frags, idents, ridx = [], [], []
    for i, n in enumerate(lens):
        frags.append(_np_dna(5000 + i, n))
        idents.append(rnd.choice([0.99, 0.96, 0.93, 0.87]))
        ridx.append(2 * i + 1)
        batch.add_literal_read(ridx[-1], frags[-1], idents[-1])
    res, total = engine.sequence_batch(batch)
    outs, _ = orc.sequence_batch(frags, idents, engine.seed, ridx, n_threads=16)
    bad = [i for i in range(len(frags)) if res.read(i) != (outs[i][0], outs[i][1])
           or (res.records[i].matches, res.records[i].columns) != (outs[i][2], outs[i][3])]
    assert not bad, [(i, lens[i], idents[i]) for i in bad[:10]]


@pytest.mark.parametrize('knob,value', [('BADREAD_B200_LOWMEM', '1'), ('BADREAD_B200_RING_T', '2'), ('BADREAD_B200_RING_T', '8'),
                                        ('BADREAD_B200_LPT', '0')])
def test_alternative_builds_match_oracle(monkeypatch, knob, value):
    """The builds behind the tuning knobs write the same reads as the defaults: BADREAD_B200_LOWMEM=1 (window / leaf
    aligners that keep checkpoints and re-run tiles into shared memory instead of a per-column history in global memory:
    7x less DRAM traffic, measured slower), BADREAD_B200_RING_T=2 / 8 (columns per tick of the traceback's staging ring),
    BADREAD_B200_LPT=0 (node queues walked in push order)."""
    from badread_b200.engine import Engine, FragmentBatch
    monkeypatch.setenv(knob, value)
    eng = Engine(device=0, seed=99)
    try:
        em, qm = load_models('nanopore2023', 'nanopore2023')
        O, orc = _oracle(em, qm)
        eng.set_error_model(em)
        eng.set_qscore_model(qm)
        rnd = random.Random(31)
        lens = [rnd.choice([400, 1200, 3000, 7000]) + rnd.randrange(90) for _ in range(300)] + [26000, 52000]
        batch = FragmentBatch()
        frags, idents, ridx = [], [], []
        for i, n in enumerate(lens):
            frags.append(_np_dna(8000 + i, n))
            idents.append(rnd.choice([0.97, 0.92, 0.85, 0.78]))
            ridx.append(3 * i)
            batch.add_literal_read(ridx[-1], frags[-1], idents[-1])
        res, total = eng.sequence_batch(batch)
        outs, _ = orc.sequence_batch(frags, idents, 99, ridx, n_threads=16)
        bad = [i for i in range(len(frags)) if res.read(i) != (outs[i][0], outs[i][1])
               or (res.records[i].matches, res.records[i].columns) != (outs[i][2], outs[i][3])]
        assert not bad, [(i, lens[i], idents[i]) for i in bad[:10]]
    finally:
        eng.close()
