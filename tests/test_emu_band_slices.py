"""
The lane aligners' traceback history holds only the band's slice of every column: bb_band_words(a, b) words from row
max(0, c - a) on (bb_lane_step), staged by bb_ring_tick and walked at bit ti - max(0, tj - a).  These cases put the slice
edges where they can go wrong, under the emulator against the oracle: bands of a + b + 1 rows just below, at and above
one and two words, the smallest band and the largest each window build admits (bb_lane_words == LW, a slice of LW - 1
words); columns left of the band's top (c < a, the slice clamped at row 0) in every case; query lengths that are not a
multiple of 32; non-ACGT target characters.  bb_band makes a + b >= 1, so the smallest band has two rows; the leaves'
bands are even on both sides, so theirs have an odd number of rows.
"""
import random

import pytest

from conftest import mutate, random_dna


@pytest.fixture(scope='module')
def emu():
    from emu import emu as E
    E.build()
    return E


def lane_words(a, b):
    return ((a + b) >> 5) + 2


def window_band(qn, tm, uw):
    """bb_band of a window as bb_k_window_lane_hist computes it from the injected-edit bound uw."""
    uw = min(max(uw, abs(qn - tm)), max(qn, tm))
    a, b = max(0, (uw - (qn - tm)) // 2), max(0, (uw + (qn - tm)) // 2)
    return (a, 1) if a + b < 1 else (a, b)


def window_changes(rnd, frag, rows, alphabet):
    """Changes whose last identity re-measurement has a band of exactly `rows` rows (a + b + 1) over the whole fragment
    (one window: the fragment is at most 1000 bases).  Distinct positions, y of them 2-character insertions, the rest
    substitutions: uw = N + y and a + b = uw - (N & 1); below 25 rows, 25 changes on fewer positions (the last change
    of a position is its state)."""
    t = rows - 1
    if t < 24:   # one insertion makes a > 0; a + b = p + y - (p & 1)
        p, y = (t, 1) if t % 2 else (t - 1, 2)
        n_total = 25
    else:
        p = n_total = 25 if t < 50 else 50 if t < 100 else 100 if t < 200 else 200
        y = t - p + (p & 1)
    pos = rnd.sample(range(len(frag)), p)
    changes = []
    for i, q in enumerate(pos):
        if i < y:
            changes.append((q, frag[q] + rnd.choice(alphabet)))
        else:
            changes.append((q, rnd.choice([c for c in alphabet if c != frag[q]])))
    changes += [changes[0]] * (n_total - len(changes))
    return changes


def oracle_window(frag, changes, a):
    applied = dict(changes[:25 * a])
    return ''.join(applied.get(i, frag[i]) for i in range(len(frag)))


@pytest.mark.parametrize('lw', [4, 8])
def test_window_hist_band_slice_edges(emu, lw):
    from oracle import oracle as O
    rnd = random.Random(90 + lw)
    largest = 32 * (lw - 1)                     # a + b + 1 with bb_lane_words(a, b) == lw
    cases = [(2, 999, 'ACGT'), (31, 1000, 'ACGT'), (32, 700, 'ACGT'), (33, 333, 'ACGTN'), (largest, 1000, 'ACGT')]
    if lw == 8:
        cases += [(63, 999, 'ACGT'), (64, 960, 'ACGTN'), (65, 1000, 'ACGT')]
    for rows, frag_len, alphabet in cases:
        frag = random_dna(rnd, frag_len)
        changes = window_changes(rnd, frag, rows, alphabet)
        got = emu.window_lane(frag, changes, 11, 3 + rows, lw=lw, hist=1)
        assert len(got) == len(changes) // 25
        for a_idx, (matches, cols) in enumerate(got, start=1):
            target = oracle_window(frag, changes, a_idx)
            seen = {q for q, _ in changes[:25 * a_idx]}
            applied = dict(changes[:25 * a_idx])
            uw = sum(max(1, len(applied[q])) for q in seen)
            a, b = window_band(frag_len, len(target), uw)
            if a_idx == len(got):
                assert a + b + 1 == rows, (rows, a, b)
            if lane_words(a, b) > lw:
                assert (matches, cols) == (-1, -1)
                continue
            ops, _ = O.align_path(frag, target)
            assert (matches, cols) == (ops.count('='), len(ops)), (lw, rows, frag_len, a_idx, a, b)
            if a_idx == len(got):
                assert a > 0                    # columns c < a: the slice clamped at row 0
                if rows == largest:
                    assert lane_words(a, b) == lw


def leaf_band(nn, mm, k):
    """bb_task_band of a root: bb_band of the clamped bound, even on both sides."""
    k = min(max(k, abs(nn - mm)), max(nn, mm))
    a, b = max(0, (k - (nn - mm)) // 2), max(0, (k + (nn - mm)) // 2)
    if a + b < 1:
        b = 1
    return a + (a & 1), b + (b & 1)


def test_leaf_hist_band_slice_edges(emu):
    """bb_k_leaf_lane_hist on roots that are leaves (their band from the read's bound): the band's rows against the
    oracle's ops for the same query and target."""
    from oracle import oracle as O
    rnd = random.Random(77)
    cases = [(3, 999, 0.0, 'ACGT'), (31, 1000, 0.01, 'ACGT'), (33, 700, 0.01, 'ACGTN'), (63, 1500, 0.02, 'ACGT'),
             (65, 1201, 0.02, 'ACGTN'), (223, 1600, 0.06, 'ACGT')]
    for rows, m, rate, alphabet in cases:
        frag = random_dna(rnd, m, alphabet)
        base = mutate(rnd, frag, rate)
        for extra in range(8):      # query lengths until the band's rows come out exactly (they step by 2 or 4)
            seq = base + random_dna(rnd, extra)
            n = len(seq)
            ops, d = O.align_path(seq, frag)
            k = next((k for k in range(max(d, abs(n - m)), max(n, m) + 1) if sum(leaf_band(n, m, k)) + 1 == rows), None)
            if k is not None:
                break
        assert k is not None, (rows, m)
        a, b = leaf_band(n, m, k)
        assert lane_words(a, b) <= 8 and (a > 0 or rows == 3), (rows, n, m, d, a, b)
        assert emu.tasks_align(seq, frag, k) == ops, (rows, n, m, k)
