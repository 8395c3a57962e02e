#!/usr/bin/env python3
"""
make_golden_model_stress.py - one more pin of the model builders' tests to the unmodified reference, at a size and on
sequence the data set of make_golden_models.py does not have.  TEST INFRASTRUCTURE.

Writes the seeded mix of tests/model_counts_ref.py (stress_mix: 400 low-complexity alignments with tied alternatives, 60
alignments with 25-30 % errors, the hand-built edges) to a temporary directory, runs the UNMODIFIED reference
(/root/reference; its `edlib` import is satisfied by oracle/edlib_shim, which these two commands never call) on it -

  error_model_k7, error_model_k12      badread.error_model.make_error_model
  qscore_model_k9                      badread.qscore_model.make_qscore_model (max_del 6, min_occur 1)

- and stores, per file, the SHA-256, the line count and the first and last three lines in
tests/golden/golden_model_stress.json.  tests/test_model_counts.py holds the definitional count to these digests,
tests/test_gpu_model_counts.py the device.

Alignments the reference cannot run are left out of the mix (model_counts_ref.STRESS_LEFT_OUT; the definitional count
and the device still meet them in the other tests):
  edge_starts_with_i   after its first window the reference's error-model loop skips the leading insertion columns and
                       lands on reference base 0 again, so its next window has k + 1 reference bases and its own
                       `assert len(ref_kmer) == args.k_size` fails
  edge_starts_with_d   the same in the qscore loop with leading deletion columns
                       (`assert len(read_kmer.replace(' ', '')) == len(read_kmer_qual) == k_size`)
  edge_ends_with_d     the reference's align_sequences indexes its per-read-base error list at the read's length
                       (IndexError)
For the same reasons the diverse alignments of the mix are cut to start and end on an aligned column.

Run once in the build container (a few minutes: the reference's loops are pure Python, and it makes a dict of all 4^12
k-mers); the fixture is committed, the reference is not needed at test time.
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.realpath(__file__))
OUT = os.path.join(HERE, '..', 'tests', 'golden', 'golden_model_stress.json')
sys.path.insert(0, os.path.join(HERE, '..', 'tests'))
sys.path.insert(0, os.path.join(HERE, '..'))

import model_counts_ref as R  # noqa: E402


def main():
    sys.path.insert(0, os.path.join(HERE, 'edlib_shim'))
    sys.path.insert(0, '/root/reference')
    import badread.error_model as rem
    import badread.qscore_model as rqm
    result = {}
    with tempfile.TemporaryDirectory() as tmp:
        args = R.stress_mix().write(tmp)
        for name, which, kw in R.STRESS_MODELS:
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                (rem.make_error_model if which == 'error' else rqm.make_qscore_model)(
                    types.SimpleNamespace(**{**vars(args), **kw}), output=io.StringIO())
            result[name] = R.stress_digest(buf.getvalue())
            print(name, result[name]['lines'], 'lines', result[name]['sha256'][:16])
    with open(OUT, 'w') as f:
        json.dump(result, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
