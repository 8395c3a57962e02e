"""
The counting kernels of the model builders (csrc/bb_models.cuh) against a count made from the definition
(tests/model_counts_ref.py: gapped column strings, string windows, insertion-ordered dicts; no packed keys, no length
limits).  CPU tier:

* the definitional count writes the nine committed model files of tests/golden/models, i.e. it equals the unmodified
  reference wherever the golden data goes, and the digests of tests/golden/golden_model_stress.json
  (oracle/make_golden_model_stress.py: the unmodified reference on a seeded hot + diverse + edges mix);
* the device code under the emulator, behind the unchanged host code, writes the definitional model files on seeded
  inputs the golden data does not reach, and what the count call returns - keys, first-occurrence stamps, counts or
  histograms, `overall`, overflow list - is decoded here into strings and equals the definitional dicts entry by entry;
* both builders' behaviour on a quality character outside Phred+33.

tests/test_gpu_model_counts.py runs the same comparisons on the device at full size.
"""
import contextlib
import gzip
import io
import json
import os
import types

import numpy as np
import pytest

import model_counts_ref as R

HERE = os.path.dirname(os.path.realpath(__file__))
DATA = os.path.join(HERE, 'golden', 'models')
STRESS = os.path.join(HERE, 'golden', 'golden_model_stress.json')
ERROR_KS = [3, 7, 12, 13, 16]
QSCORE_KS = [(1, 6), (5, 0), (9, 6), (13, 2)]
CIGAR_MAX = 29          # symbols a CIGAR key holds


def kmer_max_len(k):
    """Read k-mer bases a key holds: the bits 2k + 6 leave in 64, or the low word of a 128-bit key."""
    return 32 if k > 12 else 29 - k


# ------------------------------------------------------------------------------------------------ inputs and the definition
class Case(object):
    """A data set written to disk and loaded by the builders' own loaders, with its definitional counts (cached)."""

    def __init__(self, dataset, directory):
        from badread_b200 import model_builders as mb
        os.makedirs(directory, exist_ok=True)
        self.args = dataset.write(str(directory))
        self.alns, self.reads, self.refs = R.load(self.args)
        assert len(self.alns) == len(dataset.paf)        # the loader's filters kept every alignment
        self.flat = mb.FlatAlignments(self.alns, self.reads, self.refs, io.StringIO(), 1000)
        self._cache = {}

    def error(self, k):
        if k not in self._cache:
            self._cache[k] = R.count_error_model(self.alns, self.reads, self.refs, k)
        return self._cache[k]

    def qscore(self, k, max_del):
        if (k, max_del) not in self._cache:
            self._cache[k, max_del] = R.count_qscore_model(self.alns, self.reads, self.refs, k, max_del)
        return self._cache[k, max_del]

    def long_kmer_windows(self, k):
        """(alignment, r, k) of the windows that go to the overflow list: first and last base agree, the reference k-mer is
        ACGT and the read k-mer is longer than a key holds (its alphabet is the host's to check)."""
        out, limit = [], kmer_max_len(k)
        for a, aln in enumerate(self.alns):
            read_cols, ref_cols, _ = R.columns(aln, self.reads, self.refs)
            if k + ref_cols.count(b'-') <= limit:       # (no window of it has that many inserted bases)
                continue
            out.extend((a, r, k) for r, (f, d) in enumerate(R.error_windows(read_cols, ref_cols, k))
                       if len(d) > limit and d[0] == f[0] and d[-1] == f[-1] and not f.translate(None, b'ACGT'))
        return out

    def odd_cigar_windows(self, k, max_del):
        """(alignment, i, kk) of the windows with a CIGAR longer than a key holds, (alignment, i, -kk) of those whose
        quality is not a Phred+33 character."""
        out = []
        for a, aln in enumerate(self.alns):
            read_cols, ref_cols, qual = R.columns(aln, self.reads, self.refs)
            if b'D' not in R.cigar_columns(read_cols, ref_cols) and min(qual, default=33) >= 33 and max(qual, default=33) < 127:
                continue
            for kk in range(1, k + 1, 2):
                for i, (c, q) in enumerate(R.qscore_windows(read_cols, ref_cols, qual, kk, max_del)):
                    if not 33 <= q < 127:
                        out.append((a, i, -kk))
                    elif len(c) > CIGAR_MAX:
                        out.append((a, i, kk))
        return out


def run_builder(mb, which, args, **kw):
    fn = mb.make_error_model if which == 'error' else mb.make_qscore_model
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        fn(types.SimpleNamespace(**{**vars(args), **kw}), output=io.StringIO())
    return out.getvalue()


# ------------------------------------------------------------------------------------------------ decoding the raw return
def _letters(codes, width):
    """(n,) packed words, base j at bits 2j -> (n, width) ASCII matrix."""
    shifts = np.uint64(2) * np.arange(width, dtype=np.uint64)
    return np.frombuffer(b'ACGT', dtype=np.uint8)[((codes[:, None] >> shifts) & np.uint64(3)).astype(np.int64)]


def decode_kmer_entries(raw, k):
    """{(reference k-mer, read k-mer): (count, (alignment, r))} of what the k-mer count call returned."""
    keys, first, counts = raw[0], raw[1], raw[2]
    if k > 12:
        read_bits, refcode, lens = keys[:, 0], keys[:, 1] >> np.uint64(6), (keys[:, 1] & np.uint64(63)).astype(np.int64)
    else:
        refcode, lens = keys >> np.uint64(64 - 2 * k), ((keys >> np.uint64(58 - 2 * k)) & np.uint64(63)).astype(np.int64)
        read_bits = keys & np.uint64((1 << (58 - 2 * k)) - 1)
    n = len(first)
    ref_m = _letters(refcode, k)[:, ::-1].tobytes().decode() if n else ''        # (first base in the highest bits)
    width = int(lens.max()) if n else 1
    read_m = _letters(read_bits, width).tobytes().decode() if n else ''
    out = {}
    for j, (ln, c, st) in enumerate(zip(lens.tolist(), counts[:, 0].tolist(), first.tolist())):
        key = (ref_m[j * k:(j + 1) * k], read_m[j * width:j * width + ln])
        assert key not in out, f'the key of {key} came back twice'
        out[key] = (c, (st >> 32, st & 0xffffffff))
    return out


def decode_cigar_entries(raw):
    """{CIGAR: ({quality: count}, (alignment, window size, i))} of what the CIGAR count call returned."""
    keys, first, counts = raw[0], raw[1], raw[2]
    n = len(first)
    lens = (keys >> np.uint64(58)).astype(np.int64)
    width = int(lens.max()) if n else 1
    shifts = np.uint64(2) * np.arange(width, dtype=np.uint64)
    text = np.frombuffer(b'=XID', dtype=np.uint8)[((keys[:, None] >> shifts) & np.uint64(3)).astype(np.int64)].tobytes().decode()
    rows, cols = np.nonzero(counts)
    hists = [{} for _ in range(n)]
    for j, q, c in zip(rows.tolist(), cols.tolist(), counts[rows, cols].tolist()):
        hists[j][q] = c
    out = {}
    for j, (ln, st) in enumerate(zip(lens.tolist(), first.tolist())):
        cigar = text[j * width:j * width + ln]
        assert cigar not in out, f'the key of {cigar} came back twice'
        out[cigar] = (hists[j], (st >> 36, 2 * ((st >> 32) & 15) + 1, st & 0xffffffff))
    return out


def _same_entries(got, want, what):
    missing, extra = [x for x in want if x not in got], [x for x in got if x not in want]
    assert not missing and not extra, f'{what}: missing {missing[:5]} ({len(missing)}), not in the definition {extra[:5]} ({len(extra)})'
    wrong = [(x, got[x], want[x]) for x in want if got[x] != want[x]]
    assert not wrong, f'{what}: (key, returned, definition) {wrong[:5]} ({len(wrong)} differ)'


def check_kmer_entries(raw, case, k):
    """Count and first occurrence of every (reference k-mer, read k-mer) a key holds; the overflow list is exactly the
    windows a key does not hold.  -> (entries, overflow windows)."""
    counts, first, _ = case.error(k)
    limit = kmer_max_len(k)
    want = {(f, d): (c, first[f, d]) for f, alts in counts.items() for d, c in alts.items() if len(d) <= limit}
    _same_entries(decode_kmer_entries(raw, k), want, f'k-mer entries, k = {k}')
    ovf = sorted(zip(*(o.tolist() for o in raw[4])))
    assert ovf == sorted(case.long_kmer_windows(k)), f'overflow list, k = {k}'
    return len(want), len(ovf)


def check_cigar_entries(raw, case, k, max_del):
    """Histogram and first occurrence of every CIGAR a key holds, `overall`, and the overflow list."""
    hist, first, overall, _ = case.qscore(k, max_del)
    want = {c: (h, first[c]) for c, h in hist.items() if len(c) <= CIGAR_MAX}
    _same_entries(decode_cigar_entries(raw), want, f'CIGAR entries, k = {k}, max_del = {max_del}')
    assert {q: int(c) for q, c in enumerate(raw[3].tolist()) if c} == overall
    ovf = sorted(zip(*(o.tolist() for o in raw[4])))
    assert ovf == sorted(case.odd_cigar_windows(k, max_del)), f'overflow list, k = {k}, max_del = {max_del}'
    return len(want), len(ovf)


def check_error_model(mb, case, k, max_alt=25):
    """make_error_model over `mb._count` (whatever it is patched to): the definitional file, and every raw entry."""
    raws, inner = [], mb._count

    def recording(*a, **kw):
        raws.append(inner(*a, **kw))
        return raws[-1]
    mb._count = recording
    try:
        text = run_builder(mb, 'error', case.args, k_size=k, max_alt=max_alt)
    finally:
        mb._count = inner
    want = R.error_model_text(case.error(k)[0], max_alt)
    stats = check_kmer_entries(raws[0], case, k)
    assert text.splitlines()[:3] == want.splitlines()[:3]
    assert text == want
    return stats


def check_qscore_model(mb, case, k, max_del, min_occur=1, max_output=1000000):
    raws, inner = [], mb._count

    def recording(*a, **kw):
        raws.append(inner(*a, **kw))
        return raws[-1]
    mb._count = recording
    try:
        text = run_builder(mb, 'qscore', case.args, k_size=k, max_del=max_del, min_occur=min_occur, max_output=max_output)
    finally:
        mb._count = inner
    hist, _, overall, _ = case.qscore(k, max_del)
    want = R.qscore_model_text(hist, overall, min_occur, max_output)
    stats = check_cigar_entries(raws[0], case, k, max_del)
    assert text.splitlines()[:3] == want.splitlines()[:3]
    assert text == want
    return stats


# ------------------------------------------------------------------------------------------------ the definition is pinned
def _golden(name):
    with gzip.open(os.path.join(DATA, name + '.txt.gz'), 'rt') as f:
        return f.read()


@pytest.fixture(scope='module')
def golden_inputs():
    args = types.SimpleNamespace(reference=os.path.join(DATA, 'ref.fasta'), reads=os.path.join(DATA, 'reads.fastq'),
                                 alignment=os.path.join(DATA, 'reads.paf'))
    return (args,) + R.load(args)


@pytest.mark.parametrize('name,k,max_alt,max_alignments', [('error_model_k7', 7, 25, None), ('error_model_k5_alt3', 5, 3, None),
                                                           ('error_model_k4_max50', 4, 25, 50), ('error_model_k13', 13, 25, None),
                                                           ('error_model_k16', 16, 25, None)])
def test_definitional_error_model_is_the_references(golden_inputs, name, k, max_alt, max_alignments):
    from badread_b200 import model_builders as mb
    args, alns, reads, refs = golden_inputs
    if max_alignments:
        alns = mb.load_alignments(args.alignment, max_alignments, output=io.StringIO())
    assert R.error_model_text(R.count_error_model(alns, reads, refs, k)[0], max_alt) == _golden(name)


@pytest.mark.parametrize('name,k,max_del,min_occur,max_output', [('qscore_model_k9', 9, 6, 3, 10000), ('qscore_model_k5_del3', 5, 3, 1, 10000),
                                                                 ('qscore_model_k9_max40', 9, 6, 100, 40),
                                                                 ('qscore_model_k9_all', 9, 6, 1, 1000000)])
def test_definitional_qscore_model_is_the_references(golden_inputs, name, k, max_del, min_occur, max_output):
    _, alns, reads, refs = golden_inputs
    hist, _, overall, _ = R.count_qscore_model(alns, reads, refs, k, max_del)
    assert R.qscore_model_text(hist, overall, min_occur, max_output) == _golden(name)


@pytest.fixture(scope='module')
def stress_case(tmp_path_factory):
    return Case(R.stress_mix(), tmp_path_factory.mktemp('stress'))


def stress_text_from_definition(case, which, kw):
    if which == 'error':
        return R.error_model_text(case.error(kw['k_size'])[0], kw['max_alt'])
    hist, _, overall, _ = case.qscore(kw['k_size'], kw['max_del'])
    return R.qscore_model_text(hist, overall, kw['min_occur'], kw['max_output'])


@pytest.mark.parametrize('name,which,kw', R.STRESS_MODELS, ids=[m[0] for m in R.STRESS_MODELS])
def test_definitional_count_is_the_references_on_the_stress_mix(stress_case, name, which, kw):
    """The unmodified reference's files for a mix the golden set does not have (low complexity, 25-30 % errors, the
    hand-built edges), by their digests."""
    with open(STRESS) as f:
        want = json.load(f)[name]
    assert R.stress_digest(stress_text_from_definition(stress_case, which, kw)) == want


# ------------------------------------------------------------------------------------------------ device code under the emulator
def emulated_count(which, flat, k, max_del=0, device=0):
    """model_builders._count by the device code under the emulator, every table starting at 256 slots."""
    from emu import emu as E
    from emu import emu_large_k as EL
    if which == 'kmers_wide':
        return EL.count_kmers_wide(flat, k, cap=256)
    return E.count_windows(which, flat, k, max_del, cap=256)


@pytest.fixture(scope='module')
def emulated():
    from emu import emu as E
    from emu import emu_large_k as EL
    from badread_b200 import model_builders as mb
    E.build()
    EL.build()
    inner, mb._count = mb._count, emulated_count
    yield mb
    mb._count = inner


@pytest.fixture(scope='module')
def cases(tmp_path_factory):
    """edges: the 21 hand-built alignments; hot: 80 of the low-complexity set (16 000 windows per k, 8 + 8 tie
    alignments); diverse: 12 noisy alignments of 500 reference bases."""
    return {'edges': Case(R.edges(), tmp_path_factory.mktemp('edges')), 'hot': Case(R.hot(80), tmp_path_factory.mktemp('hot')),
            'diverse': Case(R.diverse(12, 500), tmp_path_factory.mktemp('diverse'))}


@pytest.mark.parametrize('k', ERROR_KS)
@pytest.mark.parametrize('data', ['edges', 'hot', 'diverse'])
def test_error_model_kernel_under_the_emulator_counts_the_definition(emulated, cases, data, k):
    check_error_model(emulated, cases[data], k)


@pytest.mark.parametrize('k,max_del', QSCORE_KS)
@pytest.mark.parametrize('data', ['edges', 'hot', 'diverse'])
def test_qscore_model_kernel_under_the_emulator_counts_the_definition(emulated, cases, data, k, max_del):
    check_qscore_model(emulated, cases[data], k, max_del)


def test_max_alt_min_occur_and_max_output_under_the_emulator(emulated, cases):
    check_error_model(emulated, cases['diverse'], 3, max_alt=2)
    check_qscore_model(emulated, cases['diverse'], 5, 3, min_occur=4, max_output=50)


def test_the_edges_are_in_the_edge_set(cases):
    """Both sides of every limit occur: read k-mers of max_len and max_len + 1 bases at every k, CIGARs of 29 and 30
    symbols at both window sizes, quality bins 0 and 93, and windows that count on both sides of an N."""
    case = cases['edges']
    for k in ERROR_KS:
        lens = {len(d) for alts in case.error(k)[0].values() for d in alts}
        assert {kmer_max_len(k), kmer_max_len(k) + 1} <= lens, k
        assert case.long_kmer_windows(k)
    for k, max_del in [(9, 6), (13, 2)]:
        hist, _, overall, _ = case.qscore(k, max_del)
        assert {CIGAR_MAX, CIGAR_MAX + 1} <= {len(c) for c in hist}
        assert overall[0] > 0 and overall[93] > 0
    assert any(c.startswith('D') for c in case.qscore(9, 6)[0])         # the 'D' columns in front of the first read base


def test_hot_set_has_ties_only_the_first_occurrence_breaks(cases):
    """Alternatives of one reference k-mer with equal counts, and CIGARs with equal totals, first seen in different
    alignments: their order in the file is the order of the stamps alone."""
    case = cases['hot']
    counts, first, _ = case.error(7)
    alts = counts['AAAAAAA']
    tied = [d for d in alts if alts[d] == alts['AAACAAAA'] and d != 'AAAAAAA']
    assert len({first['AAAAAAA', d][0] for d in tied}) >= 2 and any('G' in d for d in tied) and alts['AAACAAAA'] >= 8
    hist, first, _, _ = case.qscore(9, 6)
    totals = {c: sum(h.values()) for c, h in hist.items()}
    assert totals['=I='] == totals['==I'] >= 16


# ------------------------------------------------------------------------------------------------ not a quality character
def test_quality_character_outside_phred33(emulated, tmp_path):
    """A blank among the qualities: qscore_model exits with the host's message (the kernel hands every window whose
    middle base has it to the overflow list with a negative size, and counts it nowhere); error_model does not look at
    qualities."""
    case = Case(R.edges(bad_quality=True), tmp_path)
    with pytest.raises(SystemExit) as e:
        run_builder(emulated, 'qscore', case.args, k_size=9, max_del=6, min_occur=1, max_output=100)
    assert str(e.value) == "Error: quality character ' ' outside the Phred+33 range"
    raw = emulated_count('cigars', case.flat, 9, 6)
    odd = [w for w in case.odd_cigar_windows(9, 6) if w[2] < 0]
    assert len(odd) == 5 and sorted(w for w in zip(*(o.tolist() for o in raw[4])) if w[2] < 0) == sorted(odd)
    assert int(raw[3].sum()) == sum(case.qscore(9, 6)[2].values()) - 1
    check_error_model(emulated, case, 7)
