"""
Re-runs of a batch.  A run is enqueued without host round trips, so the error-loop rounds, the joined-read buffers
(slack), the Hirschberg levels, the node queues and the split-score scratch are sized from the fragment lengths before
it starts.  When the device reports one of them too small, the fetch raises it and runs the batch again (at most three
times).  Here every limit is made too small - by its starting value (BADREAD_B200_ROUNDS / _SLACK / _EXTRA_LEVELS /
_LR_CAP) or by inputs that outgrow it - and each case checks the reasons bb_last_run_retries reports and every read
against the oracle: sequence, quality, matches, columns, loop and change counts, identity re-measurements, and outputs
packed without gaps.  Split batches where only some workers run again, limits that stay raised on the context, and a
batch that cannot be fitted are covered too.
"""
import concurrent.futures
import os

import numpy as np
import pytest

from conftest import load_models
from test_rerun_inputs import INSERT_MODEL, SLIP_FIRST_INDEX, SLIP_MODEL, SLIP_SEED, model, slip_fragments

pytestmark = pytest.mark.gpu

SEED = SLIP_SEED
ROUNDS, SLACK, LEVELS, QUEUES, SCRATCH = 1, 2, 4, 8, 16
_ORACLE_CACHE = {}


def _dna(seed, n):
    return np.frombuffer(b'ACGT', dtype=np.uint8)[np.random.RandomState(seed).randint(0, 4, n)].tobytes().decode('ascii')


def _engine(monkeypatch, **env):
    from badread_b200.engine import Engine
    for k, v in env.items():
        monkeypatch.setenv('BADREAD_B200_' + k, str(v))
    eng = Engine(device=0, seed=SEED)
    for k in env:
        monkeypatch.delenv('BADREAD_B200_' + k)
    return eng


def _oracle(key, em, qm, reads):
    """Oracle (seq, qual, stats) of every read, host threads over the reads (cached per input set)."""
    if key not in _ORACLE_CACHE:
        from oracle import oracle as O
        orc = O.Oracle(em, qm)
        with concurrent.futures.ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as ex:
            futs = [ex.submit(orc.sequence_fragment, f, ident, SEED, ri, with_stats=True) for f, ident, ri in reads]
            _ORACLE_CACHE[key] = [fu.result() for fu in futs]
    return _ORACLE_CACHE[key]


def _batch(reads):
    from badread_b200.engine import FragmentBatch
    batch = FragmentBatch()
    for frag, ident, ri in reads:
        batch.add_literal_read(ri, frag, ident)
    return batch


def _run(eng, em, qm, reads, split_calls=False):
    eng.set_error_model(em)
    eng.set_qscore_model(qm)
    batch = _batch(reads)
    if split_calls:
        eng.upload_batch(batch)
        eng.run_batch()
        return eng.fetch_batch()
    return eng.sequence_batch(batch)


def _check(res, total, reads, want):
    n = len(reads)
    assert total == sum(res.records[i].out_len for i in range(n))
    spans = sorted((res.records[i].out_off, res.records[i].out_len) for i in range(n) if res.records[i].out_len)
    if spans:
        assert spans[0][0] == 0 and all(a + la == b for (a, la), (b, _) in zip(spans, spans[1:]))   # packed, no overlap
        assert spans[-1][0] + spans[-1][1] == total
    bad = []
    for i, (frag, ident, _) in enumerate(reads):
        s, q, _, st = want[i]
        rec = res.records[i]
        got = (res.read(i), rec.matches, rec.columns, rec.loop_count, rec.change_count, rec.n_alignments, rec.flags,
               rec.frag_len)
        if got != ((s, q), st['matches'], st['columns'], st['loop_count'], st['change_count'], st['n_alignments'], 0,
                   len(frag)):
            bad.append((i, len(frag), ident))
    assert not bad, bad[:10]


def _mixed_reads(lowest=0.75):
    """About 300 reads of 1 b - 30 kb and three of 60-100 kb, identities `lowest`-0.99."""
    rs = np.random.RandomState(8080)
    lens = [int(x) for x in np.concatenate([[1, 2, 7], rs.randint(20, 3000, 200), rs.randint(3000, 30000, 97)])]
    lens += [61000, 83000, 100000]
    return [(_dna(30000 + i, n), float(rs.uniform(lowest, 0.99)), 10000 + 3 * i) for i, n in enumerate(lens)]


def _insert_reads(lens, idents, first):
    return [(_dna(first + i, n), ident, first + 2 * i) for i, (n, ident) in enumerate(zip(lens, idents))]


@pytest.fixture(scope='module')
def insert_models(tmp_path_factory):
    return model(tmp_path_factory.mktemp('rerun'), INSERT_MODEL, 'insert.txt'), load_models('random', 'ideal')[1]


@pytest.mark.parametrize('knob,value,reason', [('ROUNDS', 1, ROUNDS), ('SLACK', 0.3, SLACK), ('EXTRA_LEVELS', -4, LEVELS),
                                               ('LR_CAP', 256, SCRATCH)])
def test_each_limit_forced_by_its_starting_value(monkeypatch, knob, value, reason):
    """One limit started too small on a mixed nanopore2023 batch: the fetch runs the batch again for that reason and the
    reads equal the oracle's.  SLACK=0.3 leaves most joined reads without room; EXTRA_LEVELS=-4 stops the 100 kb reads'
    Hirschberg trees four levels early; LR_CAP=256 gives the wide roots too few split-score rows; ROUNDS=1 leaves the
    reads whose first horizon of changes is too short in the loop (no nanopore2023 read at 0.75-0.99 needs a second
    round, so that case runs nanopore2020 at 0.55-0.99).  The node queues (BB_RERUN_QUEUES) cannot be forced: they hold
    seq_cap / 256 + 4 n + 1024 nodes per level, and a read only enters the alignment when it fits seq_cap, where its
    leaves of >= 900 bases number far fewer - a small slack makes reads go without room instead."""
    name, lowest = ('nanopore2020', 0.55) if knob == 'ROUNDS' else ('nanopore2023', 0.75)
    em, qm = load_models(name, name)
    reads = _mixed_reads(lowest)
    want = _oracle(('mixed', name), em, qm, reads)
    eng = _engine(monkeypatch, **{knob: value})
    try:
        res, total = _run(eng, em, qm, reads)
        n_reruns, reasons = eng.last_run_retries()
        assert n_reruns >= 1 and reasons & reason, (n_reruns, reasons)
        _check(res, total, reads, want)
    finally:
        eng.close()


def test_loop_rounds_outgrown_without_overrides(monkeypatch, tmp_path):
    """Reads that need 4-6 error-loop rounds (the homopolymer-slippage model; test_rerun_inputs pins the count on the
    emulated device code): three rounds are enqueued, the replay kernel reports reads still pending and the batch runs
    again with six."""
    em = model(tmp_path, SLIP_MODEL, 'slip.txt')
    qm = load_models('random', 'ideal')[1]
    reads = [(f, ident, SLIP_FIRST_INDEX + i) for i, (f, ident) in enumerate(slip_fragments())]
    want = _oracle('slip', em, qm, reads)
    eng = _engine(monkeypatch)
    try:
        res, total = _run(eng, em, qm, reads)
        n_reruns, reasons = eng.last_run_retries()
        assert n_reruns == 1 and reasons == ROUNDS, (n_reruns, reasons)
        _check(res, total, reads, want)
    finally:
        eng.close()


# reads of the insertion model: 20-150 kb at identity 0.55-0.7 (joined reads 1.5x and more), 1.6 Mb of fragments
INFLATE = ([20000, 35000, 52000, 75000, 110000, 150000, 27000, 64000, 41000, 88000, 130000, 30000, 97000, 46000, 120000],
           [0.55, 0.6, 0.65, 0.7, 0.58, 0.62, 0.68, 0.55, 0.6, 0.66, 0.7, 0.57, 0.63, 0.69, 0.59])


def test_inflating_reads_outgrow_the_read_buffers(monkeypatch, insert_models):
    """Every read grows to 1.5x its fragment or more: the joined reads do not fit the 1.25x buffers (BB_RERUN_SLACK).
    First GPU run of a k=3 model.  The split-score scratch has no natural trigger here: with insertions only, a node's
    band is about the length gained plus twice the slack in its bound, below the rows sized from the expected edits.
    The per-warp strip buffer (error 4) is sized from the longest fragment, and every node's target is a slice of a
    fragment, so no read below 256 kb reaches it either."""
    em, qm = insert_models
    reads = _insert_reads(*INFLATE, 40000)
    want = _oracle('inflate', em, qm, reads)
    eng = _engine(monkeypatch)
    try:
        res, total = _run(eng, em, qm, reads)
        n_reruns, reasons = eng.last_run_retries()
        print(f'inflating reads: {n_reruns} re-runs, reasons {reasons:#x}')
        assert n_reruns >= 1 and reasons & SLACK, (n_reruns, reasons)
        assert not reasons & (LEVELS | QUEUES), reasons
        _check(res, total, reads, want)
    finally:
        eng.close()


def _split_inflating(worker):
    """A batch for the default two-worker context where only `worker` outgrows its read buffers: 150 reads of 100-400 b
    and five reads of 82-100 kb at identity 1 (no changes), and five reads of 82-100 kb at 0.55 that grow to 1.5x with the
    insertion model.  The split deals the reads longest first, alternately to workers 0 and 1; the long reads alternate
    between the two kinds so that the inflating ones all land on `worker`."""
    infl, plain = [100000, 96000, 92000, 88000, 84000], [98000, 94000, 90000, 86000, 82000]
    if worker == 1:
        infl, plain = plain, infl
    reads = [(_dna(71000 + i, 100 + 2 * i), 1.0, 71000 + 2 * i) for i in range(150)]
    reads += [(_dna(72000 + i, n), 0.55, 72001 + 2 * i) for i, n in enumerate(infl)]
    reads += [(_dna(73000 + i, n), 1.0, 73001 + 2 * i) for i, n in enumerate(plain)]
    return reads


@pytest.mark.parametrize('worker', [0, 1])
@pytest.mark.parametrize('split_calls', [False, True])
def test_split_batch_where_one_worker_runs_again(monkeypatch, insert_models, worker, split_calls):
    """Only worker 0 or only worker 1 of the default two-worker context runs again (its reads need 1.5x their fragments,
    the other worker's need 1x).  Through bb_sequence_batch (the block copies enqueued early are replaced when a worker
    ran again and the later blocks moved) and through upload / run / fetch."""
    em, qm = insert_models
    reads = _split_inflating(worker)
    want = _oracle(('split', worker), em, qm, reads)
    eng = _engine(monkeypatch)
    try:
        res, total = _run(eng, em, qm, reads, split_calls)
        n_reruns, reasons = eng.last_run_retries()
        assert n_reruns == 1 and reasons == SLACK, (n_reruns, reasons)
        _check(res, total, reads, want)
    finally:
        eng.close()


@pytest.mark.parametrize('split_calls', [False, True])
def test_head_batch_context_runs_again(monkeypatch, insert_models, split_calls):
    """Three workers with a head batch of the longest reads on worker 0: 48 reads of 20-22 kb at 0.55 that grow to 1.5x
    (the head takes about 18 of them, the others share the rest) and 272 reads of 100-400 b at identity 1.  The
    checkpoint builds of the lane aligners (LOWMEM=1, same reads) keep the scratch of three workers small enough to sit
    next to the suite's shared two-worker engine on an 80 GB card."""
    em, qm = insert_models
    reads = [(_dna(90000 + i, 20000 + 41 * i), 0.55, 90000 + i) for i in range(48)]
    reads += [(_dna(91000 + i, 100 + i), 1.0, 91000 + i) for i in range(272)]
    want = _oracle('head', em, qm, reads)
    eng = _engine(monkeypatch, SUBBATCHES=3, HEAD_WORKER=1, LOWMEM=1)
    try:
        res, total = _run(eng, em, qm, reads, split_calls)
        n_reruns, reasons = eng.last_run_retries()
        assert n_reruns >= 1 and reasons & SLACK, (n_reruns, reasons)
        _check(res, total, reads, want)
    finally:
        eng.close()


def test_rerun_with_output_buffers_too_small(monkeypatch, insert_models):
    """A split batch that runs again and whose reads do not fit the caller's buffers: BB_ERR_CAPACITY with the needed
    size after the re-run, then the fetch with larger buffers gives the reads."""
    em, qm = insert_models
    reads = _split_inflating(1)
    want = _oracle(('split', 1), em, qm, reads)
    need = sum(len(w[0]) for w in want)
    eng = _engine(monkeypatch)
    try:
        eng._ensure_out(int((need - 4096) / 1.25) - 2000)    # pinned buffers 2 kb short of the reads
        small = eng._out_cap
        assert small < need
        res, total = _run(eng, em, qm, reads)
        assert total == need and eng._out_cap > small
        assert eng.last_run_retries()[0] == 1
        _check(res, total, reads, want)
    finally:
        eng.close()


def test_raised_limits_stay_on_the_context(monkeypatch, insert_models):
    """The Engine that just ran a batch again runs it once more without re-running and writes the same reads; a different
    batch on it (worker 0 of a split batch outgrowing its buffers) equals the oracle's reads, as on a fresh Engine."""
    em, qm = insert_models
    reads = _insert_reads(*INFLATE, 40000)
    eng = _engine(monkeypatch)
    try:
        res, total = _run(eng, em, qm, reads)
        assert eng.last_run_retries()[0] >= 1
        first = [res.read(i) for i in range(len(reads))]
        res, total2 = _run(eng, em, qm, reads)
        assert eng.last_run_retries() == (0, 0)
        assert total2 == total and [res.read(i) for i in range(len(reads))] == first
        other = _split_inflating(0)
        res, total = _run(eng, em, qm, other)
        _check(res, total, other, _oracle(('split', 0), em, qm, other))
    finally:
        eng.close()


def test_config5_tail_reads(monkeypatch):
    """Reads of 160-250 kb at identity 0.8-0.9 (the gamma tail of --length 40000,20000): whichever limits they outgrow,
    the reads equal the oracle's."""
    em, qm = load_models('nanopore2023', 'nanopore2023')
    reads = [(_dna(120000 + i, n), ident, 120000 + i) for i, (n, ident) in enumerate(((160000, 0.9), (210000, 0.85), (250000, 0.8)))]
    want = _oracle('tail', em, qm, reads)
    eng = _engine(monkeypatch)
    try:
        res, total = _run(eng, em, qm, reads)
        n_reruns, reasons = eng.last_run_retries()
        print(f'config-5 tail: {n_reruns} re-runs, reasons {reasons:#x}')
        assert not reasons & QUEUES
        _check(res, total, reads, want)
    finally:
        eng.close()


def test_batch_that_cannot_fit_fails_cleanly(monkeypatch):
    """EXTRA_LEVELS=-40 leaves a 100 kb read's tree unfinished after three growths of 8 levels: bb_sequence_batch fails
    with "did not fit after growing" (a host-side error, no reads), and the same Engine then runs the next batch
    correctly."""
    from badread_b200.engine import EngineError
    em, qm = load_models('nanopore2023', 'nanopore2023')
    eng = _engine(monkeypatch, EXTRA_LEVELS=-40)
    try:
        big = [(_dna(150000, 100000), 0.9, 150000)]
        with pytest.raises(EngineError, match='did not fit after growing'):
            _run(eng, em, qm, big)
        n_reruns, reasons = eng.last_run_retries()
        assert n_reruns == 3 and reasons & LEVELS, (n_reruns, reasons)
        reads = _mixed_reads()[:100]     # (one worker: the second worker of the context still starts 40 levels short)
        want = _oracle(('mixed', 'nanopore2023'), em, qm, _mixed_reads())[:100]
        res, total = _run(eng, em, qm, reads)
        _check(res, total, reads, want)
    finally:
        eng.close()


def test_config1_batch_does_not_rerun(engine):
    """A batch shaped like the benchmark's (nanopore2023, 300 reads of up to 60 kb at 0.85-0.99) runs once."""
    em, qm = load_models('nanopore2023', 'nanopore2023')
    rs = np.random.RandomState(11)
    reads = [(_dna(200000 + i, int(n)), float(rs.uniform(0.85, 0.99)), 200000 + i)
             for i, n in enumerate(np.minimum(rs.gamma(2.0, 8000.0, 300).astype(int) + 1, 60000))]
    res, total = _run(engine, em, qm, reads)
    assert engine.last_run_retries() == (0, 0)
