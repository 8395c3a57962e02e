"""
The oracle's aligner on low-complexity sequence, against references that share none of its code.

Real genomes are full of homopolymers, short tandem repeats (STRs) and satellites, and `simulate` makes junk reads of
a 1-5 base unit repeated over the whole fragment.  On such input many alignments are co-optimal, so the rule of
DESIGN.md §1 decides between them all the time: the traceback prefers I over D over the diagonal, and a Hirschberg
node splits at the smallest interior query row whose forward and reverse column scores sum to the node's distance,
then at row -1, then at row |q| - 1.  Inside a repeat long runs of rows tie for that split, and they cross 32-row
boundaries.  Uniform random DNA seldom ties.

The references are an int64 numpy edit-distance DP written here (one query row at a time; the left-neighbour term as
a running minimum) and the oracle's full-matrix checker (align_path(..., naive=True)).  Neither uses the bit vectors,
the bands or the banded Hirschberg passes.  The device's task pipeline, run here under the warp emulator, is held to the
same ops.  The generators below are shared with tests/test_gpu_low_complexity.py.
"""
import functools
import random

import numpy as np
import pytest

NAIVE_CELLS = 5 * 10 ** 7      # the full-matrix checker holds (n + 1) x (m + 1) int32 matrices
DEFAULT_LIMIT = 1024 * 1024


# ------------------------------------------------------------------------------------------------------ generators
def dna(rnd, n, alphabet='ACGT'):
    if n <= 0:
        return ''
    a = np.frombuffer(alphabet.encode('ascii'), dtype=np.uint8)
    return a[np.random.RandomState(rnd.randrange(1 << 30)).randint(0, len(a), n)].tobytes().decode('ascii')


def tandem(unit, n):
    return (unit * (n // len(unit) + 1))[:n]


def junk_fragment(rnd, n):
    """The read planner's junk fragment (simulate.ReadPlanner.get_fragment): a unit of 1-5 random bases, repeated."""
    p = rnd.randint(1, 5)
    unit = dna(rnd, p)
    return (unit * (int(round(n / p)) + 1))[:n], unit


def diverge(rnd, unit, rate):
    """A copy of unit with every base substituted (2/3) or deleted or followed by an insertion (1/3) at rate."""
    out = []
    for c in unit:
        x = rnd.random()
        if x >= rate:
            out.append(c)
        elif x < rate / 3:
            continue
        elif x < 2 * rate / 3:
            out.append(c + rnd.choice('ACGT'))
        else:
            out.append(rnd.choice([b for b in 'ACGT' if b != c]))
    return ''.join(out)


def satellite(rnd, unit_len, n, rate):
    """Copies of one random unit, each diverged at rate, cut to n bases."""
    unit = dna(rnd, unit_len)
    out, size = [], 0
    while size < n:
        out.append(diverge(rnd, unit, rate))
        size += len(out[-1])
    return ''.join(out)[:n], unit


class Layout(object):
    """A sequence put together piece by piece, with the interval [start, end) and the unit of every repeat in it."""

    def __init__(self):
        self.parts, self.repeats, self.n = [], [], 0

    def add(self, s, unit=None):
        if unit is not None and s:
            self.repeats.append((self.n, self.n + len(s), unit))
        self.parts.append(s)
        self.n += len(s)
        return self

    def done(self):
        return ''.join(self.parts), self.repeats


# A chunk of the lane and warp aligners is one 32 * L-row Myers word for L = 1, 2, 4, 8, 16.
CHUNK_ROWS = (32, 64, 128, 256, 512)
HP_RUNS = (1, 2, 5, 31, 32, 33, 63, 64, 65, 127, 255, 300, 511, 512, 513, 1000, 1023, 2047, 3000, 5000)


def homopolymer_layouts(rnd):
    """Homopolymers of 1-5000 bases in random DNA; one end of each run on a multiple of 32, 64, 128, 256 or 512, or
    one base either side of it (the start in half the cases, the end in the other half).  In every other layout the
    run holds the sequence's midpoint, where a Hirschberg root splits the target."""
    out, i = [], 0
    for rows in CHUNK_ROWS:
        for off in (-1, 0, 1):
            for at_end in (True, False):
                run = HP_RUNS[i % len(HP_RUNS)]
                centred = i % 2 == 0
                i += 1
                k = max(1, -(-(run + 2) // rows)) if at_end else rnd.randint(1, 3)
                edge = rows * k + off
                start = edge - run if at_end else edge
                base = rnd.choice('ACGT')
                prefix = dna(rnd, start)
                while prefix and prefix[-1] == base:            # the run is exactly `run` bases long
                    prefix = prefix[:-1] + rnd.choice([b for b in 'ACGT' if b != base])
                suffix = dna(rnd, rnd.randrange(max(0, start - run), start + run) if centred else rnd.randint(40, 300))
                while suffix and suffix[0] == base:
                    suffix = rnd.choice([b for b in 'ACGT' if b != base]) + suffix[1:]
                out.append(Layout().add(prefix).add(base * run, base).add(suffix).done())
    return out


def str_layouts(rnd):
    """STRs of 2-6 base units filling most of the sequence, and junk fragments of every unit length."""
    out = []
    for unit_len in range(2, 7):
        for n in (150, 700, 2100):
            unit = dna(rnd, unit_len)
            while len(set(unit)) == 1:
                unit = dna(rnd, unit_len)
            lay = Layout().add(dna(rnd, rnd.randint(0, 40))).add(tandem(unit, n), unit).add(dna(rnd, rnd.randint(0, 40)))
            out.append(lay.done())
    for n in (40, 333, 1000, 2500, 4000):
        for _ in range(2):
            junk, unit = junk_fragment(rnd, n)
            out.append(Layout().add(junk, unit).done())
    return out


def satellite_layouts(rnd):
    """Satellites: units of 20-200 bases repeated with 1-3 % divergence."""
    out = []
    for unit_len, n, rate in ((20, 900, 0.01), (37, 2000, 0.03), (64, 2600, 0.02), (120, 3000, 0.01), (200, 4000, 0.03),
                              (171, 1500, 0.02)):
        sat, unit = satellite(rnd, unit_len, n, rate)
        out.append(Layout().add(dna(rnd, rnd.randint(20, 200))).add(sat, unit).add(dna(rnd, rnd.randint(20, 200))).done())
    return out


def genome_like(rnd, n, n_runs=0):
    """Random DNA with homopolymers (mostly 4-12 bases, some up to 80) about every 60 bases, STRs of 2-6 base units
    about every 400 bases and a diverged satellite about every 4 kb; n_runs runs of 20-400 Ns over random stretches."""
    lay = Layout()
    while lay.n < n:
        lay.add(dna(rnd, int(rnd.expovariate(1 / 40))))
        x = rnd.random()
        if x < 0.75:
            base = rnd.choice('ACGT')
            lay.add(base * (rnd.randint(4, 12) if rnd.random() < 0.9 else rnd.randint(13, 80)), base)
        elif x < 0.985:
            unit = dna(rnd, rnd.randint(2, 6))
            lay.add(tandem(unit, len(unit) * rnd.randint(5, 40)), unit)
        else:
            sat, unit = satellite(rnd, rnd.randint(20, 200), rnd.randint(400, 3000), rnd.choice([0.01, 0.02, 0.03]))
            lay.add(sat, unit)
        if n_runs and rnd.random() < n_runs * 60 / n:
            run = rnd.randint(20, 400)
            lay.add('N' * run, 'N')
    seq, repeats = lay.done()
    return seq[:n], [(s, min(e, n), u) for s, e, u in repeats if s < n]


def partner(rnd, seq, repeats, rate, run_bias=0.8):
    """A mutated copy of seq with about rate * len(seq) edits.  A share run_bias of them fall inside the repeats, as the
    insertion or deletion of one whole unit in phase (a length change inside a homopolymer or an STR, the edit that
    ties the most paths); the rest are substitutions, insertions and deletions of one base anywhere."""
    n = len(seq)
    spans = [(s, e, u) for s, e, u in repeats if e > s]
    weights = [e - s for s, e, _ in spans]
    edits = {}
    for _ in range(max(1, int(round(rate * n)))):
        if spans and rnd.random() < run_bias:
            s, e, u = rnd.choices(spans, weights)[0]
            p = rnd.randrange(s, e)
            edits[p] = ('del', len(u)) if rnd.random() < 0.5 else ('ins', seq[p:p + len(u)] if p + len(u) <= e else u)
        elif n:
            p = rnd.randrange(n)
            kind = rnd.choice(('sub', 'ins', 'del'))
            edits[p] = ('del', 1) if kind == 'del' else (kind, rnd.choice([b for b in 'ACGT' if b != seq[p]]))
    out, i = [], 0
    while i < n:
        e = edits.get(i)
        if e is None:
            out.append(seq[i])
            i += 1
        elif e[0] == 'del':
            i += e[1]
        else:
            out.append(e[1] + seq[i] if e[0] == 'ins' else e[1])
            i += 1
    return ''.join(out) or 'A'


def rephase(rnd, seq, repeats):
    """seq with every repeat replaced by the same repeat in another phase (units of 2 or more bases) or by another
    unit of the same length (homopolymers and runs of N become a run of another base)."""
    out, pos = [], 0
    for s, e, u in repeats:
        if s < pos:
            continue
        out.append(seq[pos:s])
        if len(u) > 1 and len(set(u)) > 1:
            shift = rnd.randrange(1, len(u))
            out.append(tandem(u[shift:] + u[:shift], e - s))
        else:
            out.append(rnd.choice([b for b in 'ACGT' if b != u[0]]) * (e - s))
        pos = e
    out.append(seq[pos:])
    return ''.join(out)


def stretch(rnd, seq, repeats):
    """seq with every exact repeat of 40 bases or more made longer or shorter by whole units, by a tenth to a third of
    its length: a homopolymer or STR that differs by d bases between the two sides ties about d rows of a split."""
    out, pos = [], 0
    for s, e, u in repeats:
        if s < pos or e - s < 40 or seq[s:e] != tandem(u, e - s):
            continue
        d = len(u) * max(1, rnd.randint((e - s) // 10, (e - s) // 3) // len(u))
        out.append(seq[pos:s])
        out.append(tandem(u, e - s + (d if rnd.random() < 0.5 else -d)))
        pos = e
    out.append(seq[pos:])
    return ''.join(out)


def repeat_layouts(seed):
    """Every layout family: (sequence, repeats, family)."""
    rnd = random.Random(seed)
    out = [(s, r, 'homopolymer') for s, r in homopolymer_layouts(rnd)]
    out += [(s, r, 'str') for s, r in str_layouts(rnd)]
    out += [(s, r, 'satellite') for s, r in satellite_layouts(rnd)]
    for n, n_runs in ((1200, 0), (2500, 0), (4000, 2), (6000, 0), (3000, 3)):
        s, r = genome_like(rnd, n, n_runs)
        out.append((s, r, 'genome'))
    return out


@functools.lru_cache(maxsize=None)
def repeat_pairs(seed=61):
    """(query, target, family) pairs: every layout against mutated partners at several rates (each way round), against
    a copy whose repeats are longer or shorter, and against a copy in another phase or unit; at most NAIVE_CELLS cells
    each."""
    rnd = random.Random(seed + 1)
    pairs = []
    for i, (seq, repeats, family) in enumerate(repeat_layouts(seed)):
        rate = (0.004, 0.02, 0.06, 0.15)[i % 4]
        other = partner(rnd, seq, repeats, rate)
        pairs.append((seq, other, family))
        pairs.append((other, seq, family))
        longer = stretch(rnd, seq, repeats)
        if longer != seq:
            pairs.append((longer, seq, family) if i % 2 else (seq, longer, family))
        if i % 3 == 0:
            pairs.append((rephase(rnd, seq, repeats), seq, family))
    return [p for p in pairs if len(p[0]) * len(p[1]) <= NAIVE_CELLS]


# ---------------------------------------------------------------------------------------------- the numpy reference
def _codes(s):
    return np.frombuffer(s.encode('latin-1'), dtype=np.uint8)


def dp_last_column(q, t):
    """D(q[:i + 1], t) for every i in [0, len(q)), int64, one query row at a time.  Within a row
    D[i][j] = min(tmp[j], D[i][j - 1] + 1) with tmp[j] = min(D[i-1][j-1] + (q[i] != t[j]), D[i-1][j] + 1), which
    unrolls to D[i][j] = min over k <= j of tmp[k] + j - k = j + cummin(tmp[k] - k)."""
    qa, ta = _codes(q), _codes(t)
    m = len(ta)
    j = np.arange(m + 1, dtype=np.int64)
    mismatch = {c: (ta != c).astype(np.int64) for c in np.unique(qa)}
    row = j.copy()
    tmp = np.empty(m + 1, dtype=np.int64)
    out = np.empty(len(qa), dtype=np.int64)
    for i, c in enumerate(qa):
        tmp[0] = i + 1
        np.minimum(row[:-1] + mismatch[c], row[1:] + 1, out=tmp[1:])
        row = j + np.minimum.accumulate(tmp - j)
        out[i] = row[-1]
    return out


def edit_distance(q, t):
    if not q or not t:
        return max(len(q), len(t))
    return int(dp_last_column(q, t)[-1])


def split_sums(q, t):
    """The root split of a Hirschberg node q x t (target split at len(t) // 2): for query rows r = -1 .. len(q) - 1,
    the distance of q[:r + 1] to the left half plus that of q[r + 1:] to the right half (index r + 1)."""
    n, m = len(q), len(t)
    left_w, right_w = m // 2, m - m // 2
    L = dp_last_column(q, t[:left_w])
    R = dp_last_column(q[::-1], t[::-1][:right_w])
    sums = np.empty(n + 1, dtype=np.int64)
    sums[0] = left_w + R[n - 1]
    sums[1:n] = L[:n - 1] + R[n - 2::-1]
    sums[n] = L[n - 1] + right_w
    return sums


def rule_split(sums):
    """DESIGN.md §1: the smallest interior row with the smallest sum, then row -1, then row n - 1."""
    n = len(sums) - 1
    best = sums.min()
    interior = np.flatnonzero(sums[1:n] == best)
    if interior.size:
        return int(interior[0])
    return -1 if sums[0] == best else n - 1


def tied_rows(sums):
    """The rows (-1 .. n - 1) whose sum is the smallest."""
    return np.flatnonzero(sums == sums.min()) - 1


def straddles_32(rows):
    """Two consecutive tied rows r, r + 1 with r + 1 a multiple of 32."""
    s = set(rows.tolist())
    return any(r + 1 in s and (r + 1) % 32 == 0 for r in s)


def check_ops(ops, q, t, dist):
    """ops spells an alignment of q to t of cost dist."""
    i = j = 0
    for c in ops:
        if c in '=X':
            assert (q[i] == t[j]) == (c == '='), (i, j, c)
            i += 1
            j += 1
        elif c == 'I':
            i += 1
        else:
            assert c == 'D', c
            j += 1
    assert (i, j) == (len(q), len(t))
    assert sum(c != '=' for c in ops) == dist


def tree_root_split(tree):
    """The split row the root of a Hirschberg tree chose (None when the root is a leaf)."""
    root = tree[0]
    if root[6]:
        return None
    nxt = tree[1] if len(tree) > 1 else None
    left_nn = nxt[2] if nxt is not None and nxt[0] == 1 and nxt[1] == 0 and nxt[3] == 0 else 0
    return left_nn - 1


# ---------------------------------------------------------------------------------------------------- the tests
def test_numpy_dp_matches_full_matrix_distance():
    """The numpy DP against the full-matrix checker's distance on small pairs, repetitive and random, either side as
    short as one base; its split sums have the distance as their minimum."""
    from oracle import oracle as O
    rnd = random.Random(3)
    cases = [('A', 'A'), ('A', 'C'), ('A', 'AAAA'), ('AAAA', 'A'), ('ACAC', 'CACA'), ('NNNA', 'ANNN'), ('AAAAAAAA', 'AAAA')]
    for _ in range(120):
        kind = rnd.randrange(4)
        n = rnd.randint(1, 300)
        if kind == 0:
            a = dna(rnd, n, 'ACGTN')
            b = dna(rnd, rnd.randint(1, 300))
        elif kind == 1:
            a = rnd.choice('ACGT') * n
            b = partner(rnd, a, [(0, n, a[0])], 0.05)
        elif kind == 2:
            a, unit = junk_fragment(rnd, n)
            b = partner(rnd, a, [(0, n, unit)], rnd.choice([0.01, 0.1]))
        else:
            a, r = genome_like(rnd, n)
            b = rephase(rnd, a, r) if rnd.random() < 0.5 else partner(rnd, a, r, 0.05)
        cases.append((a, b))
    for a, b in cases:
        d = edit_distance(a, b)
        assert d == O.align_path(a, b, naive=True)[1], (a, b)
        if len(b) >= 2:
            assert split_sums(a, b).min() == d


def test_banded_equals_full_matrix_on_repeats():
    """At the default traceback limit: the banded aligner's ops, distance and Hirschberg tree equal the full-matrix
    checker's on every repetitive pair, the distance equals the numpy DP's, and the ops spell an alignment of that
    cost."""
    from oracle import oracle as O
    pairs = repeat_pairs()
    split_roots = 0
    for q, t, family in pairs:
        got = O.align_path(q, t, with_tree=True)
        want = O.align_path(q, t, naive=True, with_tree=True)
        assert got == want, (family, len(q), len(t))
        assert got[1] == edit_distance(q, t), (family, len(q), len(t))
        check_ops(got[0], q, t, got[1])
        split_roots += not got[2][0][6]
    assert split_roots >= 20, split_roots        # Hirschberg roots at the default limit, not only leaves


@pytest.mark.parametrize('limit', [300, 2000])
def test_banded_tree_equals_full_matrix_at_low_limits(limit):
    """With the traceback limit forced low, pairs of up to 2500 bases split into trees many levels deep whose nodes
    lie inside the repeats: the banded tree and ops equal the full-matrix checker's."""
    from oracle import oracle as O
    pairs = [p for p in repeat_pairs() if max(len(p[0]), len(p[1])) <= 2500]
    deepest = 0
    try:
        O.set_traceback_limit(limit)
        for q, t, family in pairs:
            got = O.align_path(q, t, with_tree=True)
            want = O.align_path(q, t, naive=True, with_tree=True)
            assert got == want, (limit, family, len(q), len(t))
            deepest = max([deepest] + [e[0] for e in got[2]])
    finally:
        O.set_traceback_limit(DEFAULT_LIMIT)
    assert len(pairs) >= 60 and deepest >= 6, (len(pairs), deepest)


def test_root_splits_tie_and_follow_the_rule():
    """The premise of this file, counted with the numpy DP: most root splits have two or more tied rows, some have 32
    or more, and some ties run across a multiple of 32.  And the oracle's banded root (traceback limit 300, so that
    every root large enough splits) chose the row the rule picks among them."""
    from oracle import oracle as O
    pairs = [p for p in repeat_pairs() if len(p[1]) >= 2]
    n_tied, n_tied32, n_straddle, checked = 0, 0, 0, 0
    try:
        O.set_traceback_limit(300)
        for q, t, family in pairs:
            sums = split_sums(q, t)
            rows = tied_rows(sums)
            n_tied += rows.size >= 2
            n_tied32 += rows.size >= 32
            n_straddle += straddles_32(rows)
            _, dist, tree = O.align_path(q, t, with_tree=True)
            assert sums.min() == dist
            split = tree_root_split(tree)
            if split is not None:
                assert split == rule_split(sums), (family, len(q), len(t), split, rows[:8].tolist())
                checked += 1
    finally:
        O.set_traceback_limit(DEFAULT_LIMIT)
    print(f'\n{len(pairs)} root splits: {n_tied} with >= 2 tied rows, {n_tied32} with >= 32, {n_straddle} across a '
          f'multiple of 32; {checked} checked against the oracle tree')
    assert n_tied >= 0.5 * len(pairs), (n_tied, len(pairs))
    assert n_tied32 >= 20 and n_straddle >= 20, (n_tied32, n_straddle)
    assert checked >= 0.9 * len(pairs)


def test_device_task_pipeline_on_repeats_under_emulator():
    """The device's final-alignment task pipeline, warps emulated on the CPU, on the pairs whose root is a Hirschberg
    node: the oracle's ops.  Its node kernels pick the split row among the tied ones, and a rule that took another
    tied row would still align at the same distance but give other ops."""
    from emu import emu as E
    from oracle import oracle as O
    E.build()
    checked = 0
    for q, t, family in repeat_pairs():
        if 20 * ((len(q) + 63) // 64) * len(t) + 8 * len(t) < DEFAULT_LIMIT:
            continue
        ops, d = O.align_path(q, t)
        assert E.tasks_align(q, t, d) == ops, (family, len(q), len(t))
        checked += 1
    assert checked >= 20, checked


def test_generators():
    """The generators make what the tests above rely on: run ends on and next to every chunk multiple, and repeat
    intervals that hold their unit."""
    rnd = random.Random(1)
    hits = set()
    for seq, repeats in homopolymer_layouts(rnd):
        (s, e, u), = repeats
        assert seq[s:e] == u * (e - s) and (s == 0 or seq[s - 1] != u) and (e == len(seq) or seq[e] != u)
        for rows in CHUNK_ROWS:
            for off in (-1, 0, 1):
                if (e - off) % rows == 0 or (s - off) % rows == 0:
                    hits.add((rows, off))
    assert hits == {(rows, off) for rows in CHUNK_ROWS for off in (-1, 0, 1)}
    for seq, repeats, family in repeat_layouts(61):
        for s, e, u in repeats:
            if family != 'satellite' and not (family == 'genome' and len(u) >= 20):
                assert seq[s:e] == tandem(u, e - s), (family, s, e, u)
