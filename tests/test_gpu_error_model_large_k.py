"""
Error models of k up to 16 on the GPU: `error_model --k_size 13 / 16` equal the reference's files
(tests/golden/models/error_model_k13 / _k16, oracle/make_golden_large_k.py), the hash-table k-mer index
(bb_upload_error_model_kmers) gives the dense upload's reads for a k = 7 model, and the k = 13 and k = 16 models
simulate the oracle's reads (Philox) - through sequence_batch and upload/run/fetch, on the default two-worker context and
on a three-worker context with a head batch (k = 16 through bb_k_mutate_chain), and through `simulate`.
"""
import concurrent.futures
import contextlib
import gzip
import io
import os
import subprocess
import sys
import types

import numpy as np
import pytest

from conftest import load_models

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.realpath(__file__))
MODELS = os.path.join(HERE, 'golden', 'models')
SEED = 4321
_CACHE = {}


def model_file(name):
    return os.path.join(MODELS, name + '.txt.gz')


def _golden(name):
    with gzip.open(model_file(name), 'rt') as f:
        return f.read()


def _models(em_name):
    from badread_b200.error_model import ErrorModel
    from badread_b200.qscore_model import QScoreModel
    if em_name not in _CACHE:
        sink = io.StringIO()
        _CACHE[em_name] = (ErrorModel(model_file(em_name), sink), QScoreModel(model_file('qscore_model_k9'), sink))
    return _CACHE[em_name]


def _reference():
    from badread_b200.misc import load_fasta
    refs = load_fasta(os.path.join(MODELS, 'ref.fasta'))[0]
    return refs['ctgA'] + refs['ctgB'], [(0, len(refs['ctgA'])), (len(refs['ctgA']), len(refs['ctgB']))]


def _plans(n_reads=300, seed=77):
    """About 300 fragments of 0.3-100 kb as segment lists over the two contigs (both strands; reads longer than a contig
    are several slices joined), some with literal N runs or random literal stretches between slices."""
    rs = np.random.RandomState(seed)
    _, contigs = _reference()
    lens = np.concatenate([rs.randint(300, 5000, n_reads - 50), rs.randint(5000, 30000, 40), rs.randint(30000, 100001, 10)])
    plans = []
    for i, n in enumerate(lens.tolist()):
        segs, left = [], n
        while left > 0:
            r = rs.rand()
            if r < 0.04:
                m = min(left, int(rs.randint(5, 60)))
                segs.append(('lit', 'N' * m))
            elif r < 0.08:
                m = min(left, int(rs.randint(50, 800)))
                segs.append(('lit', ''.join('ACGT'[x] for x in rs.randint(0, 4, m))))
            else:
                start, clen = contigs[int(rs.randint(0, 2))]
                m = min(left, int(rs.randint(200, clen)))
                off = int(rs.randint(0, clen - m + 1))
                segs.append(('ref', start + off, m, bool(rs.rand() < 0.5)))
            left -= m
        plans.append((segs, float(rs.uniform(0.75, 0.99)), 50000 + 7 * i))
    return plans


def _materialise(ref, segs):
    from badread_b200.misc import reverse_complement
    parts = []
    for s in segs:
        if s[0] == 'lit':
            parts.append(s[1])
        else:
            piece = ref[s[1]:s[1] + s[2]]
            parts.append(reverse_complement(piece) if s[3] else piece)
    return ''.join(parts)


def _batch(plans):
    from badread_b200.engine import FragmentBatch
    batch = FragmentBatch()
    for segs, ident, ri in plans:
        for s in segs:
            if s[0] == 'lit':
                batch.add_literal_segment(s[1])
            else:
                batch.add_ref_segment(s[1], s[2], s[3])
        batch.end_read(ri, ident)
    return batch


def _oracle(key, em, qm, reads, seed=SEED):
    key = (key, seed)
    if key not in _CACHE:
        from oracle.oracle_kmers import make_oracle
        orc = make_oracle(em, qm)
        with concurrent.futures.ThreadPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as ex:
            futs = [ex.submit(orc.sequence_fragment, f, ident, seed, ri, with_stats=True) for f, ident, ri in reads]
            _CACHE[key] = [fu.result() for fu in futs]
    return _CACHE[key]


def _run(eng, em, qm, plans, split_calls, index='auto'):
    ref, _ = _reference()
    eng.upload_reference(ref.encode())
    eng.set_error_model(em, index=index)
    eng.set_qscore_model(qm)
    batch = _batch(plans)
    if split_calls:
        eng.upload_batch(batch)
        eng.run_batch()
        return eng.fetch_batch()[0]
    return eng.sequence_batch(batch)[0]


def _check(res, reads, want):
    bad = []
    for i, (frag, _, _) in enumerate(reads):
        s, q, _, st = want[i]
        rec = res.records[i]
        got = (res.read(i), rec.matches, rec.columns, rec.loop_count, rec.change_count, rec.n_alignments, rec.flags, rec.frag_len)
        if got != ((s, q), st['matches'], st['columns'], st['loop_count'], st['change_count'], st['n_alignments'], 0, len(frag)):
            bad.append((i, len(frag)))
    assert not bad, bad[:10]


def _hit_fraction(em, reads):
    """Share of the fragments' k-mer positions that have a row in the model (from the host tables)."""
    k = em.kmer_size
    rows = set(em.alternatives)
    hits = total = 0
    for frag, _, _ in reads[:60]:
        total += max(0, len(frag) - k + 1)
        hits += sum(frag[x:x + k] in rows for x in range(len(frag) - k + 1))
    return hits / total


def _engine(monkeypatch, **env):
    from badread_b200.engine import Engine
    for k, v in env.items():
        monkeypatch.setenv('BADREAD_B200_' + k, str(v))
    eng = Engine(device=0, seed=SEED)
    for k in env:
        monkeypatch.delenv('BADREAD_B200_' + k)
    return eng


# ------------------------------------------------------------------------------------------------ builder
@pytest.mark.parametrize('k', [13, 16])
def test_error_model_large_k_equals_the_reference_output(k):
    """bb_count_kmer_alternatives_wide (128-bit keys, 16-byte atomicCAS) + the sparse host aggregation: the reference's
    file byte for byte."""
    from badread_b200.model_builders import make_error_model
    args = types.SimpleNamespace(reference=os.path.join(MODELS, 'ref.fasta'), reads=os.path.join(MODELS, 'reads.fastq'),
                                 alignment=os.path.join(MODELS, 'reads.paf'), max_alignments=None, k_size=k, max_alt=25)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        make_error_model(args, output=io.StringIO())
    assert out.getvalue() == _golden(f'error_model_k{k}')


def test_error_model_command_line_k16():
    root = os.path.join(HERE, '..')
    p = subprocess.run([sys.executable, '-m', 'badread_b200', 'error_model', '--reference', os.path.join(MODELS, 'ref.fasta'),
                        '--reads', os.path.join(MODELS, 'reads.fastq'), '--alignment', os.path.join(MODELS, 'reads.paf'),
                        '--k_size', '16'], cwd=root, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert p.returncode == 0, p.stderr.decode()[-500:]
    assert p.stdout.decode() == _golden('error_model_k16')


# ------------------------------------------------------------------------------------------------ simulation
def test_hash_index_gives_the_dense_reads_for_k7(monkeypatch):
    """nanopore2023 (k = 7) through bb_upload_error_model_kmers: every record field, sequence and quality equal the dense
    upload's, on a mixed batch of about 300 reads up to 100 kb.  (Each test here runs on a context of its own and
    closes it: the scratch that 100 kb reads grow would stay on the suite's shared context.)"""
    em, qm = load_models('nanopore2023', 'nanopore2023')
    plans = _plans(seed=7)
    out = {}
    eng = _engine(monkeypatch)
    try:
        for index in ('auto', 'hash'):
            res = _run(eng, em, qm, plans, split_calls=False, index=index)
            out[index] = (res.table().copy(), [res.read(i) for i in range(len(plans))])
    finally:
        eng.close()
    ta, tb = out['auto'][0], out['hash'][0]
    for name in ta.dtype.names:
        if name not in ('loop_kcycles', 'align_kcycles'):
            assert np.array_equal(ta[name], tb[name]), name
    assert out['auto'][1] == out['hash'][1]


@pytest.mark.parametrize('em_name,split_calls', [('error_model_k13', False), ('error_model_k16', False),
                                                 ('error_model_k16', True)])
def test_large_k_models_match_oracle(monkeypatch, em_name, split_calls):
    em, qm = _models(em_name)
    plans = _plans()
    ref, _ = _reference()
    reads = [(_materialise(ref, segs), ident, ri) for segs, ident, ri in plans]
    assert _hit_fraction(em, reads) > 0.35      # (the reads behind the model cover about half of each strand)
    want = _oracle(('plans', em_name), em, qm, reads)
    eng = _engine(monkeypatch)
    try:
        _check(_run(eng, em, qm, plans, split_calls), reads, want)
    finally:
        eng.close()


@pytest.mark.parametrize('split_calls', [False, True])
def test_k16_on_a_head_batch_context(monkeypatch, split_calls):
    """Three workers with a head batch of the longest reads: k = 16 rows through bb_k_mutate_chain (16 slots per
    candidate: exactly its shared-memory width) and the table shared by the sub-contexts."""
    em, qm = _models('error_model_k16')
    plans = _plans(n_reads=300, seed=99)
    ref, _ = _reference()
    reads = [(_materialise(ref, segs), ident, ri) for segs, ident, ri in plans]
    want = _oracle(('plans99', 'k16'), em, qm, reads)
    eng = _engine(monkeypatch, SUBBATCHES=3, HEAD_WORKER=1, LOWMEM=1)
    try:
        res = _run(eng, em, qm, plans, split_calls)
        _check(res, reads, want)
    finally:
        eng.close()


def test_simulate_command_line_with_k16_model():
    """`simulate --error_model error_model_k16.txt.gz` on the fixture reference: every emitted read equals the
    oracle's."""
    from badread_b200 import simulate as S
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.fragment_lengths import FragmentLengths
    from badread_b200.identities import Identities
    from oracle.oracle_kmers import make_oracle
    args = parse_args(['simulate', '--reference', os.path.join(MODELS, 'ref.fasta'), '--quantity', '3x', '--length',
                       '3000,2000', '--seed', '9', '--error_model', model_file('error_model_k16'), '--qscore_model',
                       model_file('qscore_model_k9')])
    check_simulate_args(args)
    out, err = io.StringIO(), io.StringIO()
    S.simulate(args, output=err, stdout=out)
    lines = out.getvalue().strip().split('\n')
    records = {lines[i][1:].split(' ')[0]: (lines[i][1:], lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    assert len(records) >= 20
    sink = io.StringIO()
    ref = S.Reference(args.reference, sink)
    fl = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, sink)
    S.adjust_depths(ref, fl, args, np.random.RandomState(9))
    planner = S.ReadPlanner(args, ref, fl, Identities(args.mean_identity, args.identity_stdev, args.max_identity, sink), 9)
    em, qm = _models('error_model_k16')
    orc = make_oracle(em, qm)
    checked = 0
    for idx in range(len(records) + 50):
        pieces, info, ident, name = planner.plan(idx)
        rec = records.get(str(name))
        if rec is None:
            continue
        seq, qual, actual = orc.sequence_fragment(planner.materialise(pieces), ident, 9, read_index=idx)
        assert (rec[1], rec[2]) == (seq, qual)
        checked += 1
    assert checked == len(records)
