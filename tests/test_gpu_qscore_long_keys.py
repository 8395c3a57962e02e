"""
Qscore models with CIGAR keys of more than 31 symbols on the GPU (the k=9, max_del=6 models of tests/golden/models):
bb_get_qscores, bb_sequence_batch and `simulate` equal the oracle in Philox mode, and the side-table branch of
bb_k_qscores is taken inside a batch.
"""
import ctypes
import io
import os
import random

import numpy as np
import pytest

from conftest import random_dna
from test_qscore_long_keys import MODELS, golden, long_key_bases, model_file, oracle_for, qscore_model

pytestmark = pytest.mark.gpu


def error_model(name):
    from badread_b200.error_model import ErrorModel
    return ErrorModel(model_file(name), io.StringIO())


def test_get_qscores_entry_matches_oracle_on_hand_made_pairs(engine):
    n_long = 0
    for i, c in enumerate(golden()['get_qscores']):
        qm = qscore_model(c['qscore_model'])
        engine.set_qscore_model(qm)
        want = oracle_for(c['qscore_model']).get_qscores(c['seq'], c['frag'], engine.seed, read_index=900 + i)
        assert engine.get_qscores(c['seq'], c['frag'], read_index=900 + i) == want, (c['pair'], c['qscore_model'])
        n_long += long_key_bases(qm, c['seq'], c['frag'])
    assert n_long >= 100


def _check_batch(engine, em, qm, frags, idents, first_index):
    from badread_b200.engine import FragmentBatch
    from oracle import oracle as O
    engine.set_error_model(em)
    engine.set_qscore_model(qm)
    batch = FragmentBatch()
    for i, (frag, ident) in enumerate(zip(frags, idents)):
        batch.add_literal_read(first_index + i, frag, ident)
    res, total = engine.sequence_batch(batch)
    assert total == sum(res.records[i].out_len for i in range(len(frags)))
    outs, _ = O.Oracle(em, qm).sequence_batch(frags, idents, engine.seed, [first_index + i for i in range(len(frags))],
                                             n_threads=8)
    for i in range(len(frags)):
        assert res.read(i) == (outs[i][0], outs[i][1]), (i, len(frags[i]), idents[i])
        rec = res.records[i]
        assert (rec.matches, rec.columns) == (outs[i][2], outs[i][3])


def test_batch_with_a_long_key_model_matches_oracle(engine):
    """error_model_k7 + qscore_model_k9_all on 300 reads of 0.3-20 kb, enough to be dealt out over the workers."""
    rnd = random.Random(4242)
    frags = [random_dna(rnd, rnd.choice([300, 800, 1500, 3000, 6000, 20000]) + rnd.randrange(0, 200)) for _ in range(300)]
    idents = [rnd.choice([0.98, 0.93, 0.87, 0.8]) for _ in frags]
    _check_batch(engine, error_model('error_model_k7'), qscore_model('qscore_model_k9_all'), frags, idents, 20000)


def _oracle_long_key_bases(orc, qm, frags, idents, seed, first_index):
    """Bases of the reads that draw from keys of more than 31 symbols: the oracle's padded fragment and untrimmed read
    (its debug capture) through the restated window choice."""
    from oracle import oracle as O
    L = O.lib()
    L.bo_debug_arm.argtypes = [ctypes.c_int]
    L.bo_debug_get.restype = ctypes.c_int64
    L.bo_debug_get.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
    L.bo_debug_arm(1)
    total = 0
    try:
        for i, (frag, ident) in enumerate(zip(frags, idents)):
            orc.sequence_fragment(frag, ident, seed, read_index=first_index + i)
            got = []
            for which in (0, 1):
                n = L.bo_debug_get(which, None, 0)
                buf = np.zeros(max(n, 1), dtype=np.uint8)
                L.bo_debug_get(which, buf.ctypes.data_as(ctypes.c_void_p), n)
                got.append(bytes(buf[:n]).decode('latin-1'))
            total += long_key_bases(qm, got[1], got[0])
    finally:
        L.bo_debug_arm(0)
    return total


def test_batch_takes_the_long_key_branch(engine, tmp_path):
    """A hand-written k=8 error model that drops the six C's of ACCCCCCA nine times in ten and leaves the other 8-mers of
    ACCCCCC repeats alone, on fragments of such repeats: the reads align with runs of six deletions between single
    matches, and hundreds of their bases draw from the model's keys of 33 to 57 symbols.  Every read equals the
    oracle's."""
    from badread_b200.error_model import ErrorModel
    from oracle import oracle as O
    repeats = 'ACCCCCC' * 3
    path = tmp_path / 'collapse_runs.txt'
    path.write_text(''.join('ACCCCCCA,0.1;AA,0.9;\n' if j == 0 else f'{repeats[j:j + 8]},1.0;\n' for j in range(7)))
    em = ErrorModel(str(path), io.StringIO())
    qm = qscore_model('qscore_model_k9_all')
    rnd = random.Random(77)
    frags, idents = [], []
    for i in range(200):
        parts = []
        for _ in range(rnd.randint(1, 6)):
            parts.append(('A' + 'C' * 6) * rnd.randint(10, 80))
            parts.append(random_dna(rnd, rnd.randint(0, 150)))
        frags.append(''.join(parts))
        idents.append(rnd.choice([0.4, 0.5, 0.6]))
    n_long = _oracle_long_key_bases(O.Oracle(em, qm), qm, frags[:40], idents[:40], engine.seed, 70000)
    assert n_long >= 500, n_long     # 1176 in the first 40 reads
    _check_batch(engine, em, qm, frags, idents, 70000)


def test_simulate_command_line_with_long_key_models(tmp_path):
    """`simulate --error_model error_model_k7.txt.gz --qscore_model qscore_model_k9_all.txt.gz`: every emitted read
    equals the oracle's sequence_fragment for the same fragment, identity, seed and read index."""
    from badread_b200 import simulate as S
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.error_model import ErrorModel
    from badread_b200.fragment_lengths import FragmentLengths
    from badread_b200.identities import Identities
    from badread_b200.qscore_model import QScoreModel
    from oracle import oracle as O
    args = parse_args(['simulate', '--reference', os.path.join(MODELS, 'ref.fasta'), '--quantity', '3x', '--length',
                       '3000,2000', '--seed', '8', '--error_model', model_file('error_model_k7'), '--qscore_model',
                       model_file('qscore_model_k9_all')])
    check_simulate_args(args)
    out, err = io.StringIO(), io.StringIO()
    S.simulate(args, output=err, stdout=out)
    lines = out.getvalue().strip().split('\n')
    records = {lines[i][1:].split(' ')[0]: (lines[i][1:], lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    assert len(records) >= 20
    sink = io.StringIO()
    ref = S.Reference(args.reference, sink)
    fl = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, sink)
    S.adjust_depths(ref, fl, args, np.random.RandomState(8))
    planner = S.ReadPlanner(args, ref, fl, Identities(args.mean_identity, args.identity_stdev, args.max_identity, sink), 8)
    orc = O.Oracle(ErrorModel(args.error_model, sink), QScoreModel(args.qscore_model, sink))
    checked = 0
    for idx in range(len(records) + 50):
        pieces, info, ident, name = planner.plan(idx)
        rec = records.get(str(name))
        if rec is None:
            continue
        seq, qual, actual = orc.sequence_fragment(planner.materialise(pieces), ident, 8, read_index=idx)
        assert (rec[1], rec[2]) == (seq, qual)
        assert f'read_identity={actual * 100.0:.3f}%' in rec[0]
        checked += 1
    assert checked == len(records)
