"""CPU checks of the oracle's record of a final alignment's Hirschberg tree (the ground truth the GPU kernel-work
tests predict per-level, per-class task counts from): the banded tree equals the full-matrix checker's, the tree's
leaves rebuild the alignment, and the tree of a read is the final alignment's alone, the same from a batch's threads."""
import random

from conftest import load_models, mutate, random_dna


def _cases(rnd, count):
    for _ in range(count):
        n = rnd.randint(1, 300)
        a = random_dna(rnd, n)
        b = mutate(rnd, a, rnd.choice([0.02, 0.1, 0.3, 0.9])) if rnd.random() < 0.8 else random_dna(rnd, rnd.randint(1, 250), 'ACGTN')
        yield a, b


def test_banded_tree_equals_full_matrix_tree():
    """With the traceback limit forced low, small inputs split into Hirschberg trees several levels deep: every node
    (position, size, best score, leaf or not) of the banded aligner equals the full-matrix checker's."""
    from oracle import oracle as O
    rnd = random.Random(5)
    deepest = 0
    try:
        for limit in (1024 * 1024, 2000, 300):
            O.set_traceback_limit(limit)
            for a, b in _cases(rnd, 150):
                got = O.align_path(a, b, with_tree=True)
                want = O.align_path(a, b, naive=True, with_tree=True)
                assert got == want, (limit, len(a), len(b))
                assert got[:2] == O.align_path(a, b)
                deepest = max([deepest] + [e[0] for e in got[2]])
    finally:
        O.set_traceback_limit(1024 * 1024)
    assert deepest >= 4


def _rebuild(q, t, tree, naive):
    """The alignment's ops from its tree in call order: every recorded node must be the next one the recursion
    reaches; a leaf contributes the traceback of its own pair, and a side left empty by a split its 'I' or 'D' run."""
    from oracle import oracle as O
    it = iter(tree)
    nxt = [next(it, None)]

    def take():
        e = nxt[0]
        nxt[0] = next(it, None)
        return e

    def build(depth, q0, nn, t0, mm):
        if nn == 0:
            return 'D' * mm
        if mm == 0:
            return 'I' * nn
        e = take()
        assert e is not None and e[:5] == (depth, q0, nn, t0, mm), (e, (depth, q0, nn, t0, mm))
        best, is_leaf, non_acgt = e[5:]
        assert non_acgt == int(any(c not in 'ACGT' for c in t[t0:t0 + mm]))
        if is_leaf:
            ops, d = O.align_path(q[q0:q0 + nn], t[t0:t0 + mm], naive=naive)
            assert d == best
            return ops
        left_w = mm // 2
        f = nxt[0]
        left_nn = f[2] if f is not None and f[:2] == (depth + 1, q0) and f[3] == t0 else 0
        ops = build(depth + 1, q0, left_nn, t0, left_w) + build(depth + 1, q0 + left_nn, nn - left_nn, t0 + left_w, mm - left_w)
        assert sum(c != '=' for c in ops) == best
        return ops

    ops = build(0, 0, len(q), 0, len(t))
    assert nxt[0] is None
    return ops


def test_tree_leaves_rebuild_the_alignment():
    from oracle import oracle as O
    rnd = random.Random(8)
    try:
        for limit in (2000, 300):
            O.set_traceback_limit(limit)
            for naive in (False, True):
                for a, b in _cases(rnd, 60):
                    ops, _, tree = O.align_path(a, b, naive=naive, with_tree=True)
                    assert _rebuild(a, b, tree, naive) == ops
    finally:
        O.set_traceback_limit(1024 * 1024)
    # at the default limit: a 6 kb pair splits twice
    a = random_dna(rnd, 6000)
    b = mutate(rnd, a, 0.1)
    ops, _, tree = O.align_path(a, b, with_tree=True)
    assert max(e[0] for e in tree) >= 2 and _rebuild(a, b, tree, False) == ops


def test_read_tree_is_the_final_alignment_and_thread_safe():
    """sequence_fragment's tree is that of the final alignment (the untrimmed read against the padded fragment), not
    of the error loop's window alignments; sequence_batch's threads each record their own reads' trees."""
    from oracle import oracle as O
    rnd = random.Random(9)
    em, qm = load_models('nanopore2023', 'nanopore2023')
    orc = O.Oracle(em, qm)
    frags = [random_dna(rnd, n, 'ACGT' if i % 3 else 'ACGTN') for i, n in enumerate((3, 900, 2600, 5200, 7000, 12000))]
    idents = [0.9, 0.85, 0.95, 0.8, 0.9, 0.75]
    outs, _ = orc.sequence_batch(frags, idents, 21, list(range(len(frags))), n_threads=4, with_stats=True)
    plain, _ = orc.sequence_batch(frags, idents, 21, list(range(len(frags))), n_threads=4)
    for i, f in enumerate(frags):
        s, q, _, st = orc.sequence_fragment(f, idents[i], 21, read_index=i, with_stats=True)
        assert outs[i][:4] == plain[i]
        assert (outs[i][0], outs[i][1], outs[i][2], outs[i][3]) == (s, q, st.pop('matches'), st.pop('columns'))
        assert outs[i][4] == st
        tree = st['tree']
        assert tree[0][:5] == (0, 0, st['untrimmed_len'], 0, len(f) + 2 * orc.k)
        assert [e[0] for e in tree].count(0) == 1
        assert sum(e[2] for e in tree if e[6]) <= st['untrimmed_len']
    assert any(len(o[4]['tree']) > 1 for o in outs) and st['n_alignments'] > 0
    # an armed recorder is consumed by the next final alignment only
    assert O.align_path('ACGT', 'ACGA') == ('===X', 1)
    assert O.align_path('ACGT', 'ACGA', with_tree=True)[2] == [(0, 0, 4, 0, 4, 1, 1, 0)]
