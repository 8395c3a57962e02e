#!/usr/bin/env python3
"""
make_golden_long_qscores.py - generates tests/golden/golden_get_qscores_long.json by running the UNMODIFIED reference
(/root/reference) with `edlib` supplied by oracle/edlib_shim, like make_golden.py (which it leaves alone: re-running
that script rewrites the other fixtures).  TEST INFRASTRUCTURE.

The qscore models are the k=9, max_del=6 models of tests/golden/models (written by `qscore_model` from the synthetic
data set of make_golden_models.py).  They hold CIGAR keys of more than 31 symbols, up to 9 + 8*6 = 57; the pairs
here are made so that the windows of many bases are such keys:

  get_qscores        hand-made pairs under qscore_model_k9_all and qscore_model_k9: a read that keeps only the A of
                     every ACCCCCC of its fragment (D runs of 6 between matches), and variants - runs of 7 C's (the
                     model holds them as D*6, so those windows miss and fall back), X and I next to the deletion runs,
                     long-key windows at both read ends (where the window is pulled in)
  sequence_fragment  error_model_k7 + qscore_model_k9_all on random and ACCCCCC-motif fragments
"""
import io
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.join(HERE, 'edlib_shim'))
sys.path.insert(0, os.path.join(HERE, '..'))
sys.path.insert(0, '/root/reference')

import badread.error_model as rem  # noqa: E402
import badread.qscore_model as rqm  # noqa: E402
import badread.simulate as rsim  # noqa: E402

MODELS = os.path.join(HERE, '..', 'tests', 'golden', 'models')
OUT = os.path.join(HERE, '..', 'tests', 'golden', 'golden_get_qscores_long.json')


def hand_made_pairs(rnd):
    """(name, seq, frag) pairs whose alignments hold runs of deletions between single matches."""
    def dna(n):
        return ''.join(rnd.choice('ACGT') for _ in range(n))
    motif6, motif7 = 'A' + 'C' * 6, 'A' + 'C' * 7
    pairs = []
    frag = motif6 * 40 + dna(300)
    pairs.append(('collapsed_runs', 'A' * 40 + frag[280:], frag))
    frag = motif7 * 40 + dna(300)
    pairs.append(('runs_of_seven', 'A' * 40 + frag[320:], frag))
    frag = motif6 * 20 + motif7 * 10 + motif6 * 20 + dna(200)
    pairs.append(('runs_of_six_and_seven', 'A' * 50 + frag[7 * 20 + 8 * 10 + 7 * 20:], frag))
    frag = motif6 * 40 + dna(300)
    read = []
    for j in range(40):   # a few A's become mismatches, a few are followed by an inserted T
        read.append('G' if j % 13 == 6 else 'A')
        if j % 17 == 11:
            read.append('T')
    pairs.append(('mismatches_and_insertions', ''.join(read) + frag[280:], frag))
    mid = dna(200)
    frag = motif6 * 30 + mid + motif6 * 30 + 'A'
    pairs.append(('both_ends', 'A' * 30 + mid + 'A' * 31, frag))
    frag = motif6 * 12
    pairs.append(('all_collapsed', 'A' * 12, frag))
    return pairs


def main():
    sink = io.StringIO()
    rnd = random.Random(20261015)
    qms = {name: rqm.QScoreModel(os.path.join(MODELS, name + '.txt.gz'), sink)
           for name in ('qscore_model_k9_all', 'qscore_model_k9')}
    em = rem.ErrorModel(os.path.join(MODELS, 'error_model_k7.txt.gz'), sink)

    qs = []
    for name, seq, frag in hand_made_pairs(rnd):
        for qm_name, qm in qms.items():
            seed = rnd.randint(0, 2 ** 32 - 1)
            random.seed(seed)
            qual, actual, by_q = rqm.get_qscores(seq, frag, qm)
            qs.append({'pair': name, 'qscore_model': qm_name, 'seq': seq, 'frag': frag, 'seed': seed, 'qual': qual,
                       'actual_identity': actual, 'identity_by_qscores': by_q})

    frags = []
    for length, ident in ((300, 0.9), (1200, 0.85), (2500, 0.95)):
        frags.append((''.join(rnd.choice('ACGT') for _ in range(length)), ident))
    frags.append((('A' + 'C' * 6) * 60, 0.8))
    frags.append((('A' + 'C' * 6) * 100 + ''.join(rnd.choice('ACGT') for _ in range(400)), 0.7))
    cases = []
    for frag, ident in frags:
        seed = rnd.randint(0, 2 ** 32 - 1)
        random.seed(seed)
        seq, qual, actual, _ = rsim.sequence_fragment(frag, ident, em, qms['qscore_model_k9_all'])
        cases.append({'error_model': 'error_model_k7', 'qscore_model': 'qscore_model_k9_all', 'fragment': frag,
                      'identity': ident, 'seed': seed, 'seq': seq, 'qual': qual, 'actual_identity': actual})

    with open(OUT, 'w') as f:
        json.dump({'get_qscores': qs, 'sequence_fragment': cases}, f)
    print('wrote', len(qs), 'get_qscores cases,', len(cases), 'sequence_fragment cases')


if __name__ == '__main__':
    main()
