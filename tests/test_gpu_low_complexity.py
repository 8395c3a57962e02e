"""
The GPU's aligners, error loop and whole reads on low-complexity sequence, against the numpy DP and the oracle.

Homopolymers, short tandem repeats, satellites and junk fragments tie many co-optimal alignments: Hirschberg split
rows tie in long runs across lanes and chunks, the traceback's I > D > diagonal preference walks the band's edges,
and a homopolymer query against a homopolymer column makes the Myers match mask all ones, so the add's carry runs
through every word of a chunk.  A kernel that broke a tie the wrong way would still find an alignment of the right
distance, but not the same CIGAR, and the read's qualities (or its window identities, hence the read itself) would
differ.  Uniform random DNA, which the other GPU tests use, seldom gets there.  The generators and the numpy DP are
those of test_low_complexity_oracle.py.
"""
import functools
import io
import random
import zlib

import numpy as np
import pytest

from conftest import load_models
from test_gpu_cli import _run as run_simulate
from test_gpu_kernel_work import CLASS_NAMES, LANE8_COLS_DEFAULT, WIDE, LANE8, check_against_prediction, route
from test_low_complexity_oracle import (NAIVE_CELLS, dna, edit_distance, genome_like, junk_fragment, partner,
                                        repeat_pairs, rephase, satellite, stretch, tandem)

pytestmark = pytest.mark.gpu

SEED = 2718
MODELS = [('nanopore2023', 'nanopore2023'), ('pacbio2021', 'pacbio2021'), ('random', 'ideal')]


# -------------------------------------------------------------------------------------------------- single pairs
def _long_pairs():
    """Pairs beyond the full-matrix checker's size, up to 60 kb a side, and the tall and wide leaves of
    test_gpu_parity.py built from repeats."""
    rnd = random.Random(62)
    out = []
    for n, rate in ((9000, 0.02), (20000, 0.05), (60000, 0.01)):
        s, r = genome_like(rnd, n, n_runs=1)
        out += [(partner(rnd, s, r, rate), s), (s, stretch(rnd, s, r))]
    for n in (12000, 30000):
        junk, unit = junk_fragment(rnd, n)
        out.append((partner(rnd, junk, [(0, n, unit)], 0.03), junk))
    sat, unit = satellite(rnd, 171, 40000, 0.02)
    out.append((partner(rnd, sat, [], 0.02), sat))
    base = rnd.choice('ACGT')
    hp = dna(rnd, 500) + base * 9000 + dna(rnd, 500)
    out.append((hp, dna(rnd, 500) + base * 8700 + dna(rnd, 500)))
    strs = tandem('CAG', 3000)
    out.append((strs, tandem('CAG', 700)))                           # tall leaf: 3 strips, few columns
    out.append((base * 40, base * 30000))                            # wide leaf
    out.append((tandem('AC', 40), rephase(rnd, tandem('AC', 30000), [(0, 30000, 'AC')])))
    return out


def test_align_path_on_repeats_matches_references(engine):
    """engine.align_path (the warp aligner) on every repetitive pair: the numpy DP's distance and the full-matrix
    checker's ops up to its size, the oracle's banded ops beyond it."""
    from oracle import oracle as O
    for q, t, family in repeat_pairs():
        got_ops, got_d = engine.align_path(q, t)
        assert got_d == edit_distance(q, t), (family, len(q), len(t))
        assert got_ops == O.align_path(q, t, naive=True)[0], (family, len(q), len(t))
    for q, t in _long_pairs():
        assert len(q) * len(t) > NAIVE_CELLS or min(len(q), len(t)) <= 700
        want = O.align_path(q, t)
        assert engine.align_path(q, t) == want, (len(q), len(t))


# --------------------------------------------------------------------------------------------------- whole reads
WINDOW_LENGTHS = [1, 2, 5, 30, 200, 985, 986, 987, 1000, 1001, 1400, 3000, 9000, 20000]
LONG_REPEAT_CASES = [(25000, 0.95, 'junk'), (40000, 0.9, 'satellite'), (60000, 0.8, 'genome'), (100000, 0.9, 'genome'),
                     (150000, 0.75, 'junk'), (150000, 0.9, 'genome')]


def _fragment(rnd, n, family):
    """A fragment of n bases of one family and its repeat intervals."""
    if family == 'junk':
        f, unit = junk_fragment(rnd, n)
        return f, [(0, n, unit)]
    if family == 'homopolymer':
        base = rnd.choice('ACGT')
        flank = n // 8
        return dna(rnd, flank) + base * (n - 2 * flank) + dna(rnd, flank), [(flank, n - flank, base)]
    if family == 'str':
        unit = dna(rnd, rnd.randint(2, 6))
        return tandem(unit, n), [(0, n, unit)]
    if family == 'satellite':
        f, unit = satellite(rnd, rnd.randint(20, 200), n, rnd.choice([0.01, 0.02, 0.03]))
        return f, [(0, n, unit)]
    return genome_like(rnd, n, n_runs=rnd.choice([0, 0, 2]))


FAMILIES = ('junk', 'homopolymer', 'str', 'satellite', 'genome')


def _read_batch(model, long_cases, n_short):
    rnd = random.Random(zlib.crc32(model.encode()))
    frags, idents, repeats = [], [], []

    def add(n, ident, family):
        f, r = _fragment(rnd, n, family)
        frags.append(f)
        idents.append(ident)
        repeats.append(r)

    for i, n in enumerate(WINDOW_LENGTHS * 2):
        add(n, rnd.choice([1.0, 0.97, 0.9, 0.83, 0.75]) if i >= len(WINDOW_LENGTHS) else 0.93, FAMILIES[i % len(FAMILIES)])
    for n, ident, family in long_cases:
        add(n, ident, family)
    for i in range(n_short):
        add(rnd.choice([40, 300, 900, 1500, 2600, 4000, 9000]) + rnd.randrange(50), rnd.choice([1.0, 0.98, 0.93, 0.88, 0.8, 0.75]),
            FAMILIES[i % len(FAMILIES)])
    return frags, idents, [11 * i + 5 for i in range(len(frags))], repeats


def _engine(em, qm):
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=SEED)
    eng.set_error_model(em)
    eng.set_qscore_model(qm)
    return eng


def _literal_batch(frags, idents, ridx):
    from badread_b200.engine import FragmentBatch
    batch = FragmentBatch()
    for f, t, r in zip(frags, idents, ridx):
        batch.add_literal_read(r, f, t)
    return batch


def _collect(res, n):
    """What a batch gave every read, copied out before its context (and the output buffers) go."""
    out = []
    for i in range(n):
        r = res.records[i]
        out.append((res.read(i), (r.matches, r.columns), r.flags, r.frag_len, (r.loop_count, r.change_count, r.n_alignments)))
    return out


def _mismatches(got, outs, frags):
    bad = []
    for i, (o, g) in enumerate(zip(outs, got)):
        st = o[4]
        want = ((o[0], o[1]), (o[2], o[3]), 0, len(frags[i]), (st['loop_count'], st['change_count'], st['n_alignments']))
        if g != want:
            bad.append((i, len(frags[i])))
    return bad


@functools.lru_cache(maxsize=None)
def _run_batch(model):
    """One batch of repetitive fragments for a model pair, through the oracle (with trees) and a fresh context."""
    from oracle import oracle as O
    em, qm = load_models(*model)
    heavy = model[0] == 'nanopore2023'
    frags, idents, ridx, repeats = _read_batch(model[0], LONG_REPEAT_CASES if heavy else LONG_REPEAT_CASES[-1:],
                                               120 if heavy else 40)
    orc = O.Oracle(em, qm)
    outs, _ = orc.sequence_batch(frags, idents, SEED, ridx, n_threads=16, with_stats=True)
    eng = _engine(em, qm)
    try:
        res, _ = eng.sequence_batch(_literal_batch(frags, idents, ridx))
        got = _collect(res, len(frags))
        work = eng.last_run_work()
    finally:
        eng.close()
    return {'model': model, 'frags': frags, 'idents': idents, 'ridx': ridx, 'repeats': repeats, 'outs': outs,
            'got': got, 'work': work, 'pad': orc.k}


@pytest.fixture(params=MODELS, ids=['-'.join(m) for m in MODELS])
def reads(request):
    return _run_batch(request.param)


@pytest.fixture
def nanopore_reads():
    """The kernel-class batch: the nanopore2023 one, with reads up to 150 kb."""
    return _run_batch(MODELS[0])


def test_repetitive_reads_match_oracle(reads):
    """Every read byte for byte, its loop statistics, matches / columns and fragment length, and no flags."""
    bad = _mismatches(reads['got'], reads['outs'], reads['frags'])
    assert not bad, bad[:10]
    lengths = {len(f) for f in reads['frags']}
    assert {985, 986, 1000, 150000} <= lengths


def _inside_repeat_classes(trees, repeats, pad):
    """Per node class, the nodes below the roots whose target slice lies wholly inside one repeat interval of the
    fragment (the target is the fragment with `pad` bases either side); the query slice of such a node is the read's
    copy of that stretch of the repeat, as the alignment path crosses the node's columns inside it."""
    counts = [0] * 5
    for tree, reps in zip(trees, repeats):
        for d, _, nn, t0, mm, best, is_leaf, _ in tree:
            if d == 0 or is_leaf:
                continue
            lo, hi = t0 - pad, t0 - pad + mm
            if any(s <= lo and hi <= e for s, e, _ in reps):
                counts[route(nn, mm, best, LANE8_COLS_DEFAULT)[1]] += 1
    return counts


def test_kernel_classes_match_tree_prediction(nanopore_reads):
    """The device's per-level, per-class node counts and leaf counts equal the routing rule applied to the oracle's
    trees; every window, node and leaf kernel took work; and every node class took nodes that lie inside a repeat."""
    reads = nanopore_reads
    trees = [o[4]['tree'] for o in reads['outs']]
    work = reads['work']
    check_against_prediction(work, trees, LANE8_COLS_DEFAULT)
    totals = np.asarray(work['levels']).sum(axis=0)
    summary = dict({k: v for k, v in work.items() if k != 'levels'}, **dict(zip(('node_' + c for c in CLASS_NAMES), totals.tolist())))
    print('\nper-kernel work of the repetitive batch:', summary)
    assert all(v > 0 for v in summary.values()), summary
    inside = _inside_repeat_classes(trees, reads['repeats'], reads['pad'])
    print('nodes inside a repeat per class:', dict(zip(CLASS_NAMES, inside)))
    assert all(x > 0 for x in inside), inside


SETTINGS = [
    ({'BADREAD_B200_LOWMEM': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_RING_T': '2'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_RING_T': '8'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_LANE8_COLS': '0'}, 0),
    ({'BADREAD_B200_LANE8_COLS': '100000'}, 100000),
    ({'BADREAD_B200_QUAD': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_PAIR_CTAS': '2'}, LANE8_COLS_DEFAULT),
]


@pytest.mark.parametrize('env,lane8_cols', SETTINGS, ids=['-'.join(f'{k[13:]}={v}' for k, v in e.items()) for e, _ in SETTINGS])
def test_repetitive_reads_under_alternative_builds(nanopore_reads, monkeypatch, env, lane8_cols):
    """A fresh context per build or routing setting: the nanopore2023 batch's reads equal the oracle's and its node
    and leaf counts the prediction for that setting.  BADREAD_B200_QUAD=1 and PAIR_CTAS=2 put the multi-warp mailbox
    hand-over on repetitive chunks."""
    reads = nanopore_reads
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = _engine(*load_models(*reads['model']))
    try:
        res, _ = eng.sequence_batch(_literal_batch(reads['frags'], reads['idents'], reads['ridx']))
        got = _collect(res, len(reads['frags']))
        work = eng.last_run_work()
    finally:
        eng.close()
    bad = _mismatches(got, reads['outs'], reads['frags'])
    assert not bad, bad[:10]
    check_against_prediction(work, [o[4]['tree'] for o in reads['outs']], lane8_cols)
    totals = np.asarray(work['levels']).sum(axis=0)
    if lane8_cols == 0:
        assert totals[LANE8] == 0
    if lane8_cols > LANE8_COLS_DEFAULT:
        assert totals[LANE8] > np.asarray(reads['work']['levels']).sum(axis=0)[LANE8]
    if 'BADREAD_B200_QUAD' in env or 'BADREAD_B200_PAIR_CTAS' in env:
        assert totals[WIDE] > 0


# ---------------------------------------------------------------------------------------------------- end to end
def _repetitive_reference(path):
    """Three contigs dominated by homopolymers, STRs and satellites."""
    rnd = random.Random(404)
    contigs = []
    s, _ = genome_like(rnd, 30000)
    contigs.append(('>repeats circular=true', s))
    parts = []
    while sum(map(len, parts)) < 20000:
        parts.append(satellite(rnd, rnd.randint(20, 200), rnd.randint(1000, 4000), 0.02)[0])
        parts.append(rnd.choice('ACGT') * rnd.randint(5, 60))
    contigs.append(('>satellites', ''.join(parts)))
    parts = []
    while sum(map(len, parts)) < 12000:
        parts.append(tandem(dna(rnd, rnd.randint(2, 6)), rnd.randint(30, 600)))
        parts.append(rnd.choice('ACGT') * rnd.randint(8, 200))
    contigs.append(('>strs depth=2', ''.join(parts)))
    path.write_text(''.join(f'{h}\n{s}\n' for h, s in contigs))


def test_simulate_repetitive_reference_with_junk_matches_oracle(tmp_path):
    """`simulate` on a repetitive reference with nanopore2023 models and many junk reads (under a k-mer error model):
    every emitted read equals the oracle's for the fragment the planner gives it."""
    from badread_b200 import simulate as S
    from badread_b200.error_model import ErrorModel
    from badread_b200.fragment_lengths import FragmentLengths
    from badread_b200.identities import Identities
    from badread_b200.qscore_model import QScoreModel
    from oracle import oracle as O
    _repetitive_reference(tmp_path / 'ref.fasta')
    args, fastq, _ = run_simulate(tmp_path, extra=['--quantity', '3x', '--error_model', 'nanopore2023',
                                                   '--qscore_model', 'nanopore2023', '--junk_reads', '25'])
    lines = fastq.strip().split('\n')
    records = {lines[i][1:].split(' ')[0]: (lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    assert len(records) >= 30
    sink = io.StringIO()
    ref = S.Reference(args.reference, sink)
    fl = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, sink)
    S.adjust_depths(ref, fl, args, np.random.RandomState(5))
    planner = S.ReadPlanner(args, ref, fl, Identities(args.mean_identity, args.identity_stdev, args.max_identity, sink), 5)
    orc = O.Oracle(ErrorModel(args.error_model, sink), QScoreModel(args.qscore_model, sink))
    checked = junk = 0
    for idx in range(len(records) + 50):
        pieces, info, ident, name = planner.plan(idx)
        rec = records.get(str(name))
        if rec is None:
            continue
        seq, qual, _ = orc.sequence_fragment(planner.materialise(pieces), ident, 5, read_index=idx)
        assert rec == (seq, qual), (idx, info)
        checked += 1
        junk += any('junk_seq' in x for x in info)
    assert checked == len(records)
    print(f'\n{checked} reads, {junk} of them junk')
    assert junk >= 5, junk
