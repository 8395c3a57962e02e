"""
Qscore models with CIGAR keys of more than 31 symbols - the k=9, max_del=6 models `qscore_model` builds by default hold
keys of up to 9 + 8*6 = 57 symbols - on the CPU: the oracle pinned to the reference on such models
(tests/golden/golden_get_qscores_long.json, oracle/make_golden_long_qscores.py), the host tables, the round trip from
`qscore_model` to loadable device tables, and the K5 device code (bb_k_qscores_pair with the tables of the shared
builder, csrc/bb_qscore_tables.h; tests/emu/emu_qscores.cpp) under the warp emulator against the oracle.
"""
import contextlib
import io
import json
import os
import random
import statistics

import pytest

from conftest import mutate, random_dna

HERE = os.path.dirname(os.path.realpath(__file__))
MODELS = os.path.join(HERE, 'golden', 'models')
_CACHE = {}


def model_file(name):
    return os.path.join(MODELS, name + '.txt.gz')


def qscore_model(name):
    from badread_b200.qscore_model import QScoreModel
    if name not in _CACHE:
        _CACHE[name] = QScoreModel(model_file(name), io.StringIO())
    return _CACHE[name]


def oracle_for(qm_name, em_name='random'):
    from badread_b200.error_model import ErrorModel
    from oracle import oracle as O
    em = ErrorModel(model_file(em_name) if em_name.startswith('error_model') else em_name, io.StringIO())
    return O.Oracle(em, qscore_model(qm_name))


def golden():
    with open(os.path.join(HERE, 'golden', 'golden_get_qscores_long.json')) as f:
        return json.load(f)


def long_key_bases(qm, seq, frag):
    """How many bases of get_qscores(seq, frag) draw from a key of more than 31 symbols: the window choice of
    qscore_model.get_qscores + QScoreModel.get_qscore (qscore_model.py:32-75, 273-287) restated over the oracle's
    CIGAR."""
    from oracle import oracle as O
    full_cigar = O.align_path(seq, frag)[0]
    pos = [j for j, c in enumerate(full_cigar) if c != 'D']
    margins = (qm.kmer_size - 1) // 2
    count = 0
    for i in range(len(seq)):
        start, end = i - margins, i + margins
        while start < 0 or end >= len(seq):
            start += 1
            end -= 1
        cigar = full_cigar[pos[start]:pos[end] + 1]
        while cigar not in qm.scores:
            cigar = cigar[1:-1].strip('D')
        count += len(cigar) > 31
    return count


def motif_pair(rnd, n):
    """A fragment of about n bases from ACCCCCC blocks and random stretches, and a read of it that drops whole C runs
    (deletion runs of 6 between single matches: long-key windows), keeps some runs, and has scattered errors."""
    frag, seq = [], []
    while sum(map(len, frag)) < n:
        if rnd.random() < 0.5:
            r = rnd.randint(4, 20)
            frag.append(('A' + 'C' * 6) * r)
            seq.append(''.join('A' if rnd.random() < 0.85 else rnd.choice(['G', 'AT', 'ACCCCCC']) for _ in range(r)))
        else:
            block = random_dna(rnd, rnd.randint(30, 300))
            frag.append(block)
            seq.append(mutate(rnd, block, rnd.choice([0.0, 0.03, 0.1])))
    return ''.join(seq), ''.join(frag)


@pytest.fixture(scope='module')
def emu():
    from emu import emu_qscores as EQ
    EQ.build()
    return EQ


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_oracle_get_qscores_matches_reference_on_long_keys():
    from badread_b200.qscore_model import qscore_char_to_error_prob
    from oracle import oracle as O
    cases = golden()['get_qscores']
    assert len(cases) >= 10
    for c in cases:
        qual, matches, cols = oracle_for(c['qscore_model']).get_qscores(c['seq'], c['frag'], c['seed'], mode=O.RNG_MT)
        assert qual == c['qual'], (c['pair'], c['qscore_model'])
        assert matches / cols == c['actual_identity']
        assert 1.0 - statistics.mean(qscore_char_to_error_prob(q) for q in qual) == c['identity_by_qscores']


def test_oracle_sequence_fragment_matches_reference_on_long_keys():
    from oracle import oracle as O
    cases = golden()['sequence_fragment']
    assert len(cases) >= 5
    for c in cases:
        orc = oracle_for(c['qscore_model'], c['error_model'])
        seq, qual, ident = orc.sequence_fragment(c['fragment'], c['identity'], c['seed'], mode=O.RNG_MT)
        assert (seq, qual, ident) == (c['seq'], c['qual'], c['actual_identity']), len(c['fragment'])


def test_golden_pairs_select_long_keys():
    """The fixture's pairs really reach keys of more than 31 symbols (the first pair: 35 of its 340 bases under
    qscore_model_k9_all), and the runs of seven C's miss them."""
    by = {(c['pair'], c['qscore_model']): c for c in golden()['get_qscores']}
    qm_all, qm_k9 = qscore_model('qscore_model_k9_all'), qscore_model('qscore_model_k9')
    c = by[('collapsed_runs', 'qscore_model_k9_all')]
    assert long_key_bases(qm_all, c['seq'], c['frag']) == 35
    c = by[('runs_of_seven', 'qscore_model_k9_all')]
    assert long_key_bases(qm_all, c['seq'], c['frag']) == 0
    total_all = sum(long_key_bases(qm_all, c['seq'], c['frag']) for c in by.values() if c['qscore_model'] == 'qscore_model_k9_all')
    total_k9 = sum(long_key_bases(qm_k9, c['seq'], c['frag']) for c in by.values() if c['qscore_model'] == 'qscore_model_k9')
    assert total_all >= 100 and total_k9 >= 10, (total_all, total_k9)


# ------------------------------------------------------------------------------------------------ host tables
@pytest.mark.parametrize('name,n_long', [('qscore_model_k9', 2), ('qscore_model_k9_all', 12)])
def test_device_tables_of_models_with_long_keys(name, n_long):
    """to_device_tables() takes keys of any length: key_chars / key_off carry every key, `keys` the packed form of
    those of at most 31 symbols and 0 for the longer ones."""
    from badread_b200.qscore_model import pack_cigar
    qm = qscore_model(name)
    t = qm.to_device_tables()
    cigars = list(qm.scores)
    assert t['n_keys'] == len(cigars) and len(t['key_off']) == len(cigars) + 1
    chars = bytes(t['key_chars']).decode()
    assert [chars[t['key_off'][i]:t['key_off'][i + 1]] for i in range(len(cigars))] == cigars
    assert sum(len(c) > 31 for c in cigars) == n_long and max(len(c) for c in cigars) <= 57
    assert [int(k) for k in t['keys']] == [pack_cigar(c) if len(c) <= 31 else 0 for c in cigars]


def test_round_trip_from_qscore_model_to_device_tables(monkeypatch, tmp_path):
    """`qscore_model` with the command line's defaults (k=9, max_del=6; min_occur lowered to 2 for this small data set),
    its counting kernels under the emulator, writes a model that loads and turns into device tables, long keys
    included."""
    from emu import emu as E
    from badread_b200 import model_builders as mb
    from badread_b200.__main__ import parse_args
    from badread_b200.qscore_model import QScoreModel
    E.build()
    monkeypatch.setattr(mb, '_count', E.count_windows)
    a = parse_args(['qscore_model', '--reference', os.path.join(MODELS, 'ref.fasta'), '--reads',
                    os.path.join(MODELS, 'reads.fastq'), '--alignment', os.path.join(MODELS, 'reads.paf'), '--min_occur', '2'])
    assert (a.k_size, a.max_del) == (9, 6)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        mb.make_qscore_model(a, output=io.StringIO())
    path = tmp_path / 'model.txt'
    path.write_text(out.getvalue())
    qm = QScoreModel(str(path), io.StringIO())
    t = qm.to_device_tables()
    assert qm.kmer_size == 9 and t['n_keys'] == len(qm.scores)
    long_keys = [c for c in qm.scores if len(c) > 31]
    assert long_keys and sum(int(k) == 0 for k in t['keys']) == len(long_keys)


# ------------------------------------------------------------------------------------------------ K5 under the emulator
def test_emulated_qscores_match_oracle_on_hand_made_pairs(emu):
    """bb_k_qscores_pair with the tables of the shared builder: the packed table for short windows, the side table for
    windows of more than 31 symbols, the fall-back to the next smaller window on a miss.  Philox mode."""
    from oracle import oracle as O
    n_long = 0
    for i, c in enumerate(golden()['get_qscores']):
        qm = qscore_model(c['qscore_model'])
        seq, frag = c['seq'], c['frag']
        d = O.align_path(seq, frag)[1]
        want = oracle_for(c['qscore_model']).get_qscores(seq, frag, 55, read_index=i)
        assert emu.get_qscores_cigars(seq, frag, d + 3, qm, 55, i) == want, (c['pair'], c['qscore_model'])
        n_long += long_key_bases(qm, seq, frag)
    assert n_long >= 100


def test_emulated_qscores_match_oracle_on_mutated_random_pairs(emu):
    from oracle import oracle as O
    rnd = random.Random(41)
    n_long = 0
    for it, n in enumerate((1000, 1800, 2600, 3500, 5000)):
        seq, frag = motif_pair(rnd, n)
        name = 'qscore_model_k9_all' if it % 2 == 0 else 'qscore_model_k9'
        qm = qscore_model(name)
        d = O.align_path(seq, frag)[1]
        want = oracle_for(name).get_qscores(seq, frag, 7, read_index=100 + it)
        assert emu.get_qscores_cigars(seq, frag, d + rnd.choice([0, 10]), qm, 7, 100 + it) == want, (n, name)
        n_long += long_key_bases(qm, seq, frag)
    assert n_long >= 100, n_long


def test_builder_rejects_bad_keys(emu):
    """bb_build_qscore_tables (behind bb_upload_qscore_model_cigars) refuses a symbol outside =XID and an empty key,
    with a message."""
    import numpy as np
    t = qscore_model('qscore_model_k9').to_device_tables()

    def with_keys(cigars):
        chars = ''.join(cigars).encode()
        off = np.cumsum([0] + [len(c) for c in cigars]).astype(np.int32)
        return dict(t, n_keys=len(cigars), key_chars=np.frombuffer(chars, dtype=np.uint8).copy(), key_off=off,
                    row_off=t['row_off'][:len(cigars) + 1])
    seq, frag = 'ACGTACGTA', 'ACGTACGTA'
    with pytest.raises(ValueError, match=r"'=M=' holds a symbol other than =XID"):
        emu.get_qscores_cigars(seq, frag, 0, with_keys(['=', 'X', 'I', '=M=']), 1, 0)
    with pytest.raises(ValueError, match='empty CIGAR key'):
        emu.get_qscores_cigars(seq, frag, 0, with_keys(['=', 'X', '', 'I']), 1, 0)
    with_keys(['=', 'X', 'I'])   # the helper itself builds valid tables
    assert emu.get_qscores_cigars(seq, frag, 0, with_keys(['=', 'X', 'I']), 1, 0)[1:] == (9, 9)


def test_repeated_keys_and_windows_beyond_the_longest_key(emu):
    """Like the dict assignment in QScoreModel.load_from_file, a key given twice maps to its later row, in the packed
    table and in the side table alike; a window longer than every key of the model falls back to the next smaller
    window without a look-up."""
    import numpy as np
    run = 'D' * 6
    short3, long7, long9 = run.join('=' * 3), run.join('=' * 7), run.join('=' * 9)   # 15, 43, 57 symbols
    frag, seq = ('A' + 'C' * 6) * 8 + 'A', 'A' * 9     # =D6=D6...= : 9 matches, 8 deletion runs

    def tables(cigars, scores):
        chars = ''.join(cigars).encode()
        return {'kmer_size': 9, 'n_keys': len(cigars), 'key_chars': np.frombuffer(chars, dtype=np.uint8).copy(),
                'key_off': np.cumsum([0] + [len(c) for c in cigars]).astype(np.int32),
                'row_off': np.arange(len(cigars) + 1, dtype=np.int32), 'scores': np.asarray(scores, dtype=np.uint8),
                'cum': np.ones(len(cigars), dtype=np.float64)}
    t = tables(['=', 'X', 'I', short3, long7, long9, short3, long7], [1, 2, 3, 4, 5, 6, 40, 41])
    qual = emu.get_qscores_cigars(seq, frag, 60, t, 1, 0)[0]
    # bases 0, 8: '='; 1, 7: short3; 2, 6: the 5-base window (29 symbols) misses -> short3; 3, 5: long7; 4: long9
    assert [ord(q) - 33 for q in qual] == [1, 40, 40, 41, 6, 41, 40, 40, 1]
    t = tables(['=', 'X', 'I', short3, long7], [1, 2, 3, 4, 5])
    qual = emu.get_qscores_cigars(seq, frag, 60, t, 1, 0)[0]
    assert [ord(q) - 33 for q in qual] == [1, 4, 4, 5, 5, 5, 4, 4, 1]
