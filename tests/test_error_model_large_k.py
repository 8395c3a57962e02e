"""
Error models of k up to 16 on the CPU: the oracle with a sorted-code k-mer index (oracle/oracle_kmers.py) pinned to the
reference
(tests/golden/golden_sequence_fragment_large_k.json, oracle/make_golden_large_k.py), the 128-bit-key counting kernel of
`error_model` under the warp emulator behind the unchanged host code (byte for byte the reference's k = 13 and k = 16
files), K1 with the hash-table index (badread_b200/csrc/bb_em_tables.h), the error loop behind it against the oracle, and
the host tables of ErrorModel.
"""
import contextlib
import gzip
import io
import json
import os
import random
import types

import numpy as np
import pytest

from conftest import random_dna

HERE = os.path.dirname(os.path.realpath(__file__))
MODELS = os.path.join(HERE, 'golden', 'models')
_CACHE = {}


def model_file(name):
    return os.path.join(MODELS, name + '.txt.gz')


def error_model(name):
    from badread_b200.error_model import ErrorModel
    if name not in _CACHE:
        _CACHE[name] = ErrorModel(model_file(name), io.StringIO())
    return _CACHE[name]


def oracle_for(em_name, qm_name='qscore_model_k9'):
    from badread_b200.qscore_model import QScoreModel
    from oracle.oracle_kmers import make_oracle
    key = ('oracle', em_name, qm_name)
    if key not in _CACHE:
        _CACHE[key] = make_oracle(error_model(em_name), QScoreModel(model_file(qm_name), io.StringIO()))
    return _CACHE[key]


def reference_contigs():
    from badread_b200.misc import load_fasta
    return load_fasta(os.path.join(MODELS, 'ref.fasta'))[0]


def rows_by_kmer(em):
    """{k-mer: row} from the model's tables (the definition the index must reproduce)."""
    t = em.to_device_tables()
    return {em._kmer_of_row(r): r for r in range(len(t['row_off']) - 1)}


@pytest.fixture(scope='module')
def emu():
    from emu import emu_large_k as EL
    EL.build()
    return EL


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_oracle_sequence_fragment_matches_reference_with_large_k():
    """sequence_fragment (Mersenne Twister) with the k = 13 and k = 16 models: the oracle's sorted-code index gives the
    reference's reads, on reference slices of both strands, N runs and random fragments."""
    from oracle import oracle as O
    with open(os.path.join(HERE, 'golden', 'golden_sequence_fragment_large_k.json')) as f:
        cases = json.load(f)['sequence_fragment']
    assert {c['error_model'] for c in cases} == {'error_model_k13', 'error_model_k16'}
    assert {'ref_fwd', 'ref_rev', 'ref_n_run', 'inserted_n', 'random'} <= {c['kind'] for c in cases}
    for c in cases:
        seq, qual, ident = oracle_for(c['error_model'], c['qscore_model']).sequence_fragment(
            c['fragment'], c['identity'], c['seed'], mode=O.RNG_MT)
        assert (seq, qual, ident) == (c['seq'], c['qual'], c['actual_identity']), (c['error_model'], c['kind'])


# ------------------------------------------------------------------------------------------------ builder
@pytest.mark.parametrize('k', [13, 16])
def test_wide_counting_kernel_under_the_emulator_gives_the_reference_file(monkeypatch, emu, k):
    """`error_model --k_size 13 / 16`: bbm_k_kmer_alternatives with 128-bit keys (claimed by the emulator's 16-byte
    atomicCAS) from a table far too small to start with, behind the host code of make_error_model, writes the reference's
    file byte for byte (k-mer order, %.6f fractions, ties by first occurrence, the 30-base insertion through the
    overflow list)."""
    from badread_b200 import model_builders as mb
    calls = []

    def counted(which, flat, kk, max_del=0, device=0):
        assert which == 'kmers_wide' and kk == k
        calls.append(which)
        return emu.count_kmers_wide(flat, kk, cap=256)
    monkeypatch.setattr(mb, '_count', counted)
    args = types.SimpleNamespace(reference=os.path.join(MODELS, 'ref.fasta'), reads=os.path.join(MODELS, 'reads.fastq'),
                                 alignment=os.path.join(MODELS, 'reads.paf'), max_alignments=None, k_size=k, max_alt=25)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        mb.make_error_model(args, output=io.StringIO())
    with gzip.open(model_file(f'error_model_k{k}'), 'rt') as f:
        want = f.read()
    assert calls == ['kmers_wide']
    assert out.getvalue().splitlines()[:3] == want.splitlines()[:3]
    assert out.getvalue() == want


def test_builder_refuses_k_above_16(monkeypatch):
    from badread_b200 import model_builders as mb
    monkeypatch.setattr(mb, '_count', lambda *a, **kw: pytest.fail('no count for k = 17'))
    args = types.SimpleNamespace(reference=os.path.join(MODELS, 'ref.fasta'), reads=os.path.join(MODELS, 'reads.fastq'),
                                 alignment=os.path.join(MODELS, 'reads.paf'), max_alignments=None, k_size=17, max_alt=25)
    with pytest.raises(SystemExit, match='k > 16'):
        mb.make_error_model(args, output=io.StringIO())


# ------------------------------------------------------------------------------------------------ K1 and the loop
@pytest.mark.parametrize('name', ['error_model_k13', 'error_model_k16'])
def test_fragment_builder_with_hash_index(emu, name):
    """bb_k_build_fragments<.., true>: every position's row is the model's row of the k-mer that starts there, -1 for
    k-mers without a row and for k-mers holding an N; on reference slices of both strands, an N run and literals."""
    from badread_b200.misc import reverse_complement
    em = error_model(name)
    k = em.kmer_size
    rows = rows_by_kmer(em)
    refs = reference_contigs()
    ref = refs['ctgA'] + refs['ctgB']
    rnd = random.Random(k)
    lit = random_dna(rnd, 300) + 'NNNN' + random_dna(rnd, 50)
    segments = [(0, 1000, 2000), (1, 30000, 1500), (0, 24000 + 6900, 300), (2, 0, len(lit)), (0, 5, 2 * k - 3)]
    frag, kidx = emu.build_kidx_hash(ref, lit, segments, k, em.to_device_tables()['kmer_codes'], 11, 7)
    body = (ref[1000:3000] + reverse_complement(ref[30000:31500]) + ref[30900:31200] + lit + ref[5:5 + 2 * k - 3])
    assert frag[k:len(frag) - k] == body
    want = [rows.get(frag[x:x + k], -1) for x in range(len(frag) - k + 1)]
    assert kidx == want
    hits = sum(r >= 0 for r in want)
    assert hits > 0.4 * len(want)                      # reference k-mers have rows (about half of them) ...
    assert any('N' in frag[x:x + k] for x in range(len(want)))
    assert all(r < 0 for x, r in enumerate(want) if 'N' in frag[x:x + k])   # ... N k-mers and the literals do not
    lit0 = k + 2000 + 1500 + 300
    assert sum(r >= 0 for r in want[lit0:lit0 + 300 - k]) <= 2


def test_error_loop_with_k16_table_matches_oracle(emu):
    """The error loop behind K1's hash index (bb_k_mutate, the window kernels, bb_k_replay, bb_k_join) for the k = 16
    model equals the oracle (Philox): loop and change counts, alignments, the mutated read."""
    em = error_model('error_model_k16')
    orc = oracle_for('error_model_k16')
    refs = reference_contigs()
    rnd = random.Random(16)
    cases = [(refs['ctgA'][2000:2800], 0.85), (refs['ctgB'][3000:3400], 0.9), (random_dna(rnd, 300), 0.8),
             (refs['ctgB'][6950:7300], 0.88)]
    rows = rows_by_kmer(em)
    for n, (frag, ident) in enumerate(cases):
        seed, read = 100 + n, 3 * n + 1
        joined, st = emu.error_loop_kmers(frag, ident, seed, read, em)
        seq, _, _, want = orc.sequence_fragment(frag, ident, seed, read, with_stats=True)
        assert {x: st[x] for x in ('loop_count', 'change_count', 'n_alignments', 'untrimmed_len')} == \
            {x: want[x] for x in ('loop_count', 'change_count', 'n_alignments', 'untrimmed_len')}, (n, ident)
        assert joined[st['start_trim']:len(joined) - st['end_trim']] == seq, (n, ident)
    assert sum(cases[0][0][x:x + 16] in rows for x in range(800 - 15)) > 400     # the model's rows are drawn from


# ------------------------------------------------------------------------------------------------ host tables
@pytest.mark.parametrize('name', ['error_model_k13', 'error_model_k16'])
def test_error_model_tables_round_trip(name):
    """ErrorModel holds no 4^k array for k > 12 and says so; alternatives / probabilities / add_errors_to_kmer work from
    the rows, and every line of the file comes back."""
    em = error_model(name)
    k = int(name.rsplit('k', 1)[1])
    t = em.to_device_tables()
    assert em.kmer_size == k and t['index'] == 'hash' and 'kmer_to_row' not in t
    with gzip.open(model_file(name), 'rt') as f:
        lines = f.read().splitlines()
    assert len(em.alternatives) == len(lines) == len(t['row_off']) - 1
    for line in lines[:200] + lines[-200:]:
        parts = [x.split(',') for x in line.strip().split(';') if x]
        kmer = parts[0][0]
        assert [''.join(a) for a in em.alternatives[kmer]] == [p[0] for p in parts]
        assert em.probabilities[kmer] == [float(p[1]) for p in parts]
    random.seed(5)
    kmer = lines[0].split(',')[0]
    for _ in range(20):
        assert len(em.add_errors_to_kmer(kmer)) == k


def test_builtin_k7_model_keeps_the_dense_index():
    from conftest import load_models
    em, _ = load_models('nanopore2023', 'nanopore2023')
    t = em.to_device_tables()
    assert t['index'] == 'dense' and t['kmer_to_row'].size == 4 ** 7


def test_hash_table_builder(emu):
    """Every row is found through the table, absent codes miss, a repeated code and k outside 3..16 are refused."""
    em = error_model('error_model_k16')
    codes = em.to_device_tables()['kmer_codes']
    rnd = np.random.RandomState(1)
    # a 'fragment' of the literal k-mers of some rows and of random codes, looked up through K1
    pick = rnd.choice(codes.size, 200, replace=False)
    present = set(codes.tolist())
    absent = [c for c in rnd.randint(0, 4 ** 16, 400, dtype=np.int64).tolist() if c not in present][:200]
    kmers = [''.join('ACGT'[(int(c) >> (2 * (15 - j))) & 3] for j in range(16)) for c in list(codes[pick]) + absent]
    lit = ''.join(kmers)
    _, kidx = emu.build_kidx_hash('', lit, [(2, 0, len(lit))], 16, codes, 1, 1)
    got = [kidx[16 + 16 * i] for i in range(len(kmers))]
    assert got[:200] == pick.tolist()
    assert got[200:] == [-1] * len(absent)
    dup = codes.copy()
    dup[17] = dup[3]
    with pytest.raises(ValueError, match='same k-mer'):
        emu.build_kidx_hash('', 'ACGT' * 10, [(2, 0, 40)], 16, dup, 1, 1)
    with pytest.raises(ValueError, match='3..16'):
        emu.build_kidx_hash('', 'ACGT' * 10, [(2, 0, 40)], 17, codes[:4], 1, 1)


def test_k17_model_is_refused_with_the_new_limit(tmp_path):
    from badread_b200.error_model import ErrorModel
    p = tmp_path / 'k17.txt'
    p.write_text('A' * 17 + ',0.9;' + 'A' * 16 + 'CA,0.1;\n')
    with pytest.raises(SystemExit, match='k > 16'):
        ErrorModel(str(p), io.StringIO())


def test_sorted_code_oracle_equals_the_dense_oracle():
    """Where both exist (k = 7 here) the sorted-code oracle finds the dense index's rows: the same reads, counts and
    alignments as oracle.Oracle, in both RNG modes."""
    from badread_b200.qscore_model import QScoreModel
    from oracle import oracle as O
    from oracle.oracle_kmers import OracleKmers
    em = error_model('error_model_k7')
    qm = QScoreModel(model_file('qscore_model_k9'), io.StringIO())
    dense, sparse = O.Oracle(em, qm), OracleKmers(em, qm)
    refs = reference_contigs()
    rnd = random.Random(7)
    frags = [refs['ctgA'][100:1600], refs['ctgB'][6900:7500], random_dna(rnd, 700), refs['ctgA'][9000:9013]]
    for n, frag in enumerate(frags):
        for mode in (O.RNG_PHILOX, O.RNG_MT):
            want = dense.sequence_fragment(frag, 0.85, 50 + n, n, mode=mode, with_stats=True)
            assert sparse.sequence_fragment(frag, 0.85, 50 + n, n, mode=mode, with_stats=True) == want, (n, mode)
