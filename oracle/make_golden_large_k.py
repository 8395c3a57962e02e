#!/usr/bin/env python3
"""
make_golden_large_k.py - fixtures for error models of k = 13 and k = 16, made by running the UNMODIFIED reference
(a checkout of rrwick/Badread named by BADREAD_REFERENCE; `edlib` supplied by oracle/edlib_shim) on the builder data
set of make_golden_models.py (tests/golden/models: ref.fasta, reads.fastq, reads.paf).  TEST INFRASTRUCTURE.

  models/error_model_k13.txt.gz   badread.error_model.make_error_model, k_size=13, run directly
  models/error_model_k16.txt.gz   the same with k_size=16, run with `itertools` in badread.error_model's namespace
                                  replaced by a shim (below): the reference cannot enumerate 4^16 k-mers
  golden_sequence_fragment_large_k.json
                                  badread.simulate.sequence_fragment (Mersenne Twister, random.seed per case) with both
                                  models and qscore_model_k9: fragments cut from ref.fasta on both strands (about half
                                  of their k-mers have a row), fragments with N runs, random fragments (almost every k-mer misses),
                                  lengths from a few bases below 2k up to a few kb

The shim's product('ACGT', repeat=k) yields, in sorted order, every ACGT k-mer of the reference's two strands instead
of all 4^k.  The reference only ever indexes its dict with reference k-mers that are ACGT-only (its only_acgt test
comes before the lookup), and every such k-mer is a k-mer of one of the two strands, so the dict it builds holds every
key the full run would use.  Its final loop prints k-mers in product order, and sorted order over 'ACGT' is that order,
so the file is the one the full run would print.  The script checks this at k = 13: the shimmed run must give the same
bytes as the direct one.

Run once; the fixtures are committed, the reference is not needed at test time.
"""
import contextlib
import gzip
import io
import itertools
import json
import os
import random
import sys
import types

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.join(HERE, 'edlib_shim'))
sys.path.insert(0, os.path.join(HERE, '..'))
if not os.environ.get('BADREAD_REFERENCE'):
    sys.exit('set BADREAD_REFERENCE to a checkout of rrwick/Badread')
sys.path.insert(0, os.environ['BADREAD_REFERENCE'])

import badread.error_model as rem  # noqa: E402
import badread.misc as rmisc  # noqa: E402
import badread.qscore_model as rqm  # noqa: E402
import badread.simulate as rsim  # noqa: E402

MODELS = os.path.join(HERE, '..', 'tests', 'golden', 'models')
OUT_JSON = os.path.join(HERE, '..', 'tests', 'golden', 'golden_sequence_fragment_large_k.json')
MAX_ALT = 25


class ReferenceKmers(object):
    """Stands in for the `itertools` module inside badread.error_model: product('ACGT', repeat=k) yields the sorted
    ACGT k-mers of both strands of `refs`; every other name is the real module's."""

    def __init__(self, refs):
        self._refs = refs

    def product(self, alphabet, repeat):
        assert alphabet == 'ACGT'
        kmers = set()
        for seq in self._refs.values():
            for s in (seq, rmisc.reverse_complement(seq)):
                for i in range(len(s) - repeat + 1):
                    kmer = s[i:i + repeat]
                    if rmisc.only_acgt(kmer):
                        kmers.add(kmer)
        return iter(sorted(kmers))

    def __getattr__(self, name):
        return getattr(itertools, name)


def run_make_error_model(k, shim):
    args = types.SimpleNamespace(reference=os.path.join(MODELS, 'ref.fasta'), reads=os.path.join(MODELS, 'reads.fastq'),
                                 alignment=os.path.join(MODELS, 'reads.paf'), max_alignments=None, k_size=k,
                                 max_alt=MAX_ALT)
    buf, sink = io.StringIO(), io.StringIO()
    real = rem.itertools
    if shim:
        rem.itertools = ReferenceKmers(rmisc.load_fasta(args.reference)[0])
    try:
        with contextlib.redirect_stdout(buf):
            rem.make_error_model(args, output=sink)
    finally:
        rem.itertools = real
    return buf.getvalue()


def write_model(text, name):
    with gzip.GzipFile(os.path.join(MODELS, name), 'wb', mtime=0) as f:   # (mtime 0: reproducible bytes)
        f.write(text.encode())
    print(name, len(text.splitlines()), 'lines', os.path.getsize(os.path.join(MODELS, name)), 'bytes')


def fragments(rnd, refs, k):
    """(kind, fragment, identity) cases for a k-mer size k."""
    a, b = refs['ctgA'], refs['ctgB']
    rc = rmisc.reverse_complement
    out = []
    for n, ident in ((2 * k - 3, 0.85), (2 * k + 2, 0.9), (400, 0.8), (1500, 0.9), (3500, 0.95)):
        s = rnd.randint(0, len(a) - n)
        out.append(('ref_fwd', a[s:s + n], ident))
        s = rnd.randint(0, 6000 - n) if n < 6000 else 0
        out.append(('ref_rev', rc(b[s:s + n]), ident))
    out.append(('ref_n_run', b[6700:7400], 0.85))                       # the contig's own 40 N's
    mid = a[10000:11200]
    out.append(('inserted_n', mid[:500] + 'N' * 25 + mid[500:], 0.9))
    out.append(('scattered_n', ''.join('N' if rnd.random() < 0.01 else c for c in a[14000:15000]), 0.88))
    for n, ident in ((2 * k - 2, 0.9), (800, 0.85), (2500, 0.92)):
        out.append(('random', ''.join(rnd.choice('ACGT') for _ in range(n)), ident))
    return out


def main():
    text13 = run_make_error_model(13, shim=False)
    shimmed13 = run_make_error_model(13, shim=True)
    assert shimmed13 == text13, 'the k-mer shim changed the k = 13 model'
    print('k = 13: the shimmed run equals the direct run')
    write_model(text13, 'error_model_k13.txt.gz')
    write_model(run_make_error_model(16, shim=True), 'error_model_k16.txt.gz')

    sink = io.StringIO()
    refs = rmisc.load_fasta(os.path.join(MODELS, 'ref.fasta'))[0]
    qm = rqm.QScoreModel(os.path.join(MODELS, 'qscore_model_k9.txt.gz'), sink)
    rnd = random.Random(20261016)
    cases = []
    for k in (13, 16):
        em_name = f'error_model_k{k}'
        em = rem.ErrorModel(os.path.join(MODELS, em_name + '.txt.gz'), sink)
        for kind, frag, ident in fragments(rnd, refs, k):
            seed = rnd.randint(0, 2 ** 32 - 1)
            random.seed(seed)
            seq, qual, actual, _ = rsim.sequence_fragment(frag, ident, em, qm)
            cases.append({'error_model': em_name, 'qscore_model': 'qscore_model_k9', 'kind': kind, 'fragment': frag,
                          'identity': ident, 'seed': seed, 'seq': seq, 'qual': qual, 'actual_identity': actual})
    with open(OUT_JSON, 'w') as f:
        json.dump({'sequence_fragment': cases}, f)
    print('wrote', len(cases), 'sequence_fragment cases')


if __name__ == '__main__':
    main()
