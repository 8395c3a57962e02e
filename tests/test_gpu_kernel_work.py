"""
Which alignment kernels did the work: the device's per-kernel task counts (Engine.last_run_work) against the oracle's
Hirschberg trees of the same reads.

The final alignment of a batch is spread over eleven persistent kernels, and a routing rule picks the kernel of every
task (bb_tasks.cuh bb_push_task, bb_api.cu enqueue_error_loop).  A kernel that received no work would still leave every
read correct, so the read-level parity tests cannot tell whether a class of kernels ran at all.  Here the routing rule
is restated in Python and applied to the oracle's tree of every read: the tree is a fixed function of the inputs (each
split row comes from exact scores under edlib's rules; whether a node is a leaf depends only on its size), so below the
roots the device's per-level, per-class node counts are predicted exactly.  Root bands come from the device's
injected-edit bound instead of the exact score, so the roots are checked by their number only.
"""
import random

import numpy as np
import pytest

from conftest import load_models, random_dna
from test_gpu_parity import LONG_CASES, _np_dna

pytestmark = pytest.mark.gpu

SEED = 4321
LANE8, LEAN1, LEAN2, LEAN4, WIDE = range(5)
CLASS_NAMES = ('lane8', 'lean1', 'lean2', 'lean4', 'wide')
LANE8_COLS_DEFAULT = 4096


# ---------------------------------------------------------------------------------------- the routing rule, restated
def _half(x):
    return -((-x) // 2) if x < 0 else x // 2   # C's truncating division by 2


def bb_band(n, m, k):
    """bb_align.cuh bb_band: the band (a, b) of a path of cost <= k from (0, 0) to (n, m)."""
    a = max(0, _half(k - (n - m)))
    b = max(0, _half(k + (n - m)))
    if a + b < 1:
        b = 1
    return a, b


def bb_task_band(nn, mm, k):
    """bb_tasks.cuh bb_task_band: k clamped to [|nn - mm|, max(nn, mm)], both sides rounded up to even."""
    k = min(max(k, abs(nn - mm)), max(nn, mm))
    a, b = bb_band(nn, mm, k)
    return a + (a & 1), b + (b & 1)


def bb_lane_words(a, b):
    return ((a + b) >> 5) + 2


def bb_pick_L(a, b, K, max_l):
    """bb_align.cuh bb_pick_L<MAXL>: the fewest words per lane that fit the band into K lanes (0: none up to MAXL)."""
    L = 1
    while L <= max_l:
        if (a + b) // (32 * L) + 2 <= K:
            return L
        L *= 2
    return 0


def bb_uses_traceback(n, m):
    return 20 * ((n + 63) // 64) * m + 8 * m < 1048576


def route(nn, mm, best, lane8_cols):
    """bb_push_task's choice for a task with both sides non-empty: ('leaf', 0 lane / 1 warp) or ('node', class)."""
    a, b = bb_task_band(nn, mm, best)
    lw = bb_lane_words(a, b)
    if bb_uses_traceback(nn, mm):
        return 'leaf', 0 if (lw <= 8 and mm <= 2048) else 1
    if lw <= 8 and mm <= lane8_cols:
        return 'node', LANE8
    return 'node', {1: LEAN1, 2: LEAN2, 4: LEAN4}.get(bb_pick_L(a, b, 16, 4), WIDE)


def predict(trees, lane8_cols):
    """Per-depth node totals, per-depth per-class nodes below the roots, root leaves and leaves below the roots per
    kernel, from the oracle trees (depth, q0, nn, t0, mm, best, is_leaf, target_has_non_acgt)."""
    depth_nodes, classes, root_leaves, leaves = {}, {}, 0, [0, 0]
    for tree in trees:
        for d, _, nn, _, mm, best, is_leaf, _ in tree:
            kind, which = route(nn, mm, best, lane8_cols)
            assert (kind == 'leaf') == bool(is_leaf), (nn, mm)
            if is_leaf:
                if d == 0:
                    root_leaves += 1
                else:
                    leaves[which] += 1
                continue
            depth_nodes[d] = depth_nodes.get(d, 0) + 1
            if d >= 1:
                classes.setdefault(d, [0] * 5)[which] += 1
    return {'depth_nodes': depth_nodes, 'classes': classes, 'root_leaves': root_leaves, 'leaves': leaves}


def check_against_prediction(work, trees, lane8_cols):
    """Assertions 2-4 of the coverage batch: every level's total, every class below the roots, the leaves."""
    p = predict(trees, lane8_cols)
    levels = work['levels']
    deepest = max(p['depth_nodes'])
    assert deepest < len(levels), (deepest, len(levels))
    for d, row in enumerate(levels):
        assert sum(row) == p['depth_nodes'].get(d, 0), f'level {d}: device {sum(row)} nodes, oracle tree {p["depth_nodes"].get(d, 0)}'
        if d >= 1:
            want = p['classes'].get(d, [0] * 5)
            for c in range(5):
                assert row[c] == want[c], f'level {d}, class {CLASS_NAMES[c]}: device {row[c]} nodes, oracle tree {want[c]}'
    assert work['root_leaf_lane'] + work['root_leaf_warp'] == p['root_leaves']
    assert work['leaf_lane'] - work['root_leaf_lane'] == p['leaves'][0]
    assert work['leaf_warp'] - work['root_leaf_warp'] == p['leaves'][1]
    return p


# ---------------------------------------------------------------------------------------------------- the batch
def _n_runs_fragment(rnd, n):
    """ACGT with single Ns and runs of 50-3000 Ns: nodes whose target holds non-ACGT bases take the bit-plane passes'
    exact per-column path."""
    s = list(_np_dna(rnd.randrange(1 << 30), n))
    for _ in range(rnd.randint(3, 8)):
        s[rnd.randrange(n)] = 'N'
    for _ in range(rnd.randint(1, 3)):
        run = rnd.randint(50, 3000)
        p = rnd.randrange(n - run)
        s[p:p + run] = 'N' * run
    return ''.join(s)


def _coverage_batch():
    rnd = random.Random(2027)
    frags, idents = [], []
    for i, (n, ident) in enumerate(LONG_CASES):
        frags.append(_np_dna(977 + i, n))
        idents.append(ident)
    # a read far enough from its fragment that nodes below the root are wider than the warp pair's 32 x 32 words
    # (a + b >= 31 * 1024) and take the strip path
    frags.append(_np_dna(5151, 150000))
    idents.append(0.55)
    for _ in range(10):
        frags.append(_n_runs_fragment(rnd, rnd.randint(20000, 60000)))
        idents.append(rnd.choice([0.75, 0.8, 0.85, 0.9, 0.93, 0.97]))
    for i in range(240):
        n = rnd.choice([1, 40, 300, 900, 1500, 2600, 4000, 9000]) + rnd.randrange(50)
        frags.append(random_dna(rnd, n, 'ACGT' if i % 11 else 'ACGTN'))
        idents.append(rnd.choice([1.0, 0.98, 0.93, 0.88, 0.8, 0.7]))
    ridx = [7 * i + 3 for i in range(len(frags))]
    return frags, idents, ridx


def _engine():
    from badread_b200.engine import Engine
    em, qm = load_models('nanopore2023', 'nanopore2023')
    eng = Engine(device=0, seed=SEED)
    eng.set_error_model(em)
    eng.set_qscore_model(qm)
    return eng


def _batch(frags, idents, ridx):
    from badread_b200.engine import FragmentBatch
    batch = FragmentBatch()
    for f, t, r in zip(frags, idents, ridx):
        batch.add_literal_read(r, f, t)
    return batch


def _check_reads(res, outs, frags):
    bad = []
    for i in range(len(frags)):
        rec, o = res.records[i], outs[i]
        st = o[4]
        if (res.read(i) != (o[0], o[1]) or (rec.matches, rec.columns) != (o[2], o[3]) or rec.flags != 0
                or (rec.loop_count, rec.change_count, rec.n_alignments) != (st['loop_count'], st['change_count'], st['n_alignments'])):
            bad.append((i, len(frags[i])))
    assert not bad, bad[:10]


@pytest.fixture(scope='module')
def coverage():
    from oracle import oracle as O
    em, qm = load_models('nanopore2023', 'nanopore2023')
    frags, idents, ridx = _coverage_batch()
    outs, _ = O.Oracle(em, qm).sequence_batch(frags, idents, SEED, ridx, n_threads=16, with_stats=True)
    eng = _engine()
    try:
        batch = _batch(frags, idents, ridx)
        res, _ = eng.sequence_batch(batch)
        _check_reads(res, outs, frags)
        work = eng.last_run_work()
        # the same upload run twice: the counts start from zero on every run
        eng.upload_batch(batch)
        again = []
        for _ in range(2):
            eng.run_batch()
            r, _ = eng.fetch_batch()
            again.append(([r.read(i) for i in range(len(frags))], eng.last_run_work()))
    finally:
        eng.close()
    return {'frags': frags, 'idents': idents, 'ridx': ridx, 'outs': outs, 'trees': [o[4]['tree'] for o in outs],
            'work': work, 'again': again}


def _summary(work):
    totals = np.asarray(work['levels']).sum(axis=0)
    return dict({k: v for k, v in work.items() if k != 'levels'}, **dict(zip(('node_' + c for c in CLASS_NAMES), totals.tolist())))


# ---------------------------------------------------------------------------------------------------- the tests
def test_coverage_batch_counts_match_oracle_tree(coverage):
    """The default context: every read equals the oracle's, every level's nodes and every class below the roots are
    the restated rule applied to the oracle trees, and every window, node and leaf kernel took work."""
    work, trees, outs = coverage['work'], coverage['trees'], coverage['outs']
    check_against_prediction(work, trees, LANE8_COLS_DEFAULT)
    s = _summary(work)
    print('\nper-kernel work of the coverage batch:', s)
    for k, v in s.items():
        assert v > 0, (k, s)
    assert s['window_lane4'] + s['window_lane8'] + s['window_warp'] >= sum(o[4]['n_alignments'] for o in outs)
    # premises of the batch, from the oracle trees: the strip path below the roots, and non-ACGT targets in every
    # node class
    strip, non_acgt = 0, [0] * 5
    for tree in trees:
        for d, _, nn, _, mm, best, is_leaf, na in tree:
            if d == 0 or is_leaf:
                continue
            cls = route(nn, mm, best, LANE8_COLS_DEFAULT)[1]
            a, b = bb_task_band(nn, mm, best)
            if cls == WIDE and bb_pick_L(a, b, 32, 32) == 0:
                strip += 1
            non_acgt[cls] += na
    print('strip nodes below the roots:', strip, ' nodes with non-ACGT targets per class:', dict(zip(CLASS_NAMES, non_acgt)))
    assert strip > 0
    assert all(x > 0 for x in non_acgt), non_acgt


def test_repeated_run_gives_identical_counts(coverage):
    (reads0, work0), (reads1, work1) = coverage['again']
    assert work0 == work1 == coverage['work']
    assert reads0 == reads1
    assert reads0 == [(o[0], o[1]) for o in coverage['outs']]


# Routing knobs and grid shapes, each on a context of its own.  The window counts are the same in all of them: the
# three window kernels apply the same fall-through conditions in both builds (history and BADREAD_B200_LOWMEM=1
# checkpoints), and which windows a read needs depends on the read alone.  This batch forms no head batch with three
# workers (it has fewer than 16 reads of at least 0.6x the longest), so BADREAD_B200_HEAD_WORKER=1 splits it three ways
# like any other; test_gpu_parity.py covers the head batch's reads.
MATRIX = [
    ({'BADREAD_B200_LANE8_COLS': '0'}, 0),
    ({'BADREAD_B200_LANE8_COLS': '100000'}, 100000),
    ({'BADREAD_B200_QUAD': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_PAIR_CTAS': '2'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_GRID_DIV': '64'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_SUBBATCHES': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_SUBBATCHES': '4'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_SUBBATCHES': '3', 'BADREAD_B200_HEAD_WORKER': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_LOWMEM': '1'}, LANE8_COLS_DEFAULT),
    ({'BADREAD_B200_LPT': '0'}, LANE8_COLS_DEFAULT),
]


@pytest.mark.parametrize('env,lane8_cols', MATRIX, ids=['-'.join(f'{k[13:]}={v}' for k, v in e.items()) for e, _ in MATRIX])
def test_routing_and_grid_settings(coverage, monkeypatch, env, lane8_cols):
    """BADREAD_B200_GRID_DIV=64 puts every grid pgrid sizes at its floor of sm_count / 2 CTAs, so that each CTA loops
    over many tasks; BADREAD_B200_QUAD=1 routes wide nodes to the 8-warp kernel with its shared-memory mailbox."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = _engine()
    try:
        res, _ = eng.sequence_batch(_batch(coverage['frags'], coverage['idents'], coverage['ridx']))
        _check_reads(res, coverage['outs'], coverage['frags'])
        work = eng.last_run_work()
    finally:
        eng.close()
    check_against_prediction(work, coverage['trees'], lane8_cols)
    base = coverage['work']
    for k in ('window_lane4', 'window_lane8', 'window_warp'):
        assert work[k] == base[k], (k, work[k], base[k])
    totals = np.asarray(work['levels']).sum(axis=0)
    if lane8_cols == 0:
        assert all(row[LANE8] == 0 for row in work['levels'])
    if lane8_cols > LANE8_COLS_DEFAULT:
        assert totals[LANE8] > np.asarray(base['levels']).sum(axis=0)[LANE8]
    if env.get('BADREAD_B200_QUAD') == '1':
        assert totals[WIDE] > 0
