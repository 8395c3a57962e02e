#!/usr/bin/env python3
"""
make_golden_plot.py - fixtures for `badread_b200 plot`.  TEST INFRASTRUCTURE.

Runs the UNMODIFIED reference's plot (/root/reference: badread.plot_window_identity.plot_window_identity with --no_plot)
on the model builders' data set (tests/golden/models: ref.fasta, reads.fastq, reads.paf) and writes
tests/golden/golden_plot.json:

  stdout     what the reference prints (loaders' progress, then one repr line per chosen alignment)
  cases      for windows 1, 7, 100, 1000 and 2500, with and without --qual: per chosen alignment the number of points
             get_window_means returned, SHA-256 of the packed positions (int64), identities (float64) and qualities
             (float64) over all alignments, and a few sample values (as float.hex)

The reference imports matplotlib at module level and draws with it; a stub module in sys.modules stands in for it
(--no_plot never draws), the way oracle/edlib_shim stands in for edlib.  Run once; the fixture is committed.
"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
DATA = os.path.join(HERE, '..', 'tests', 'golden', 'models')
OUT = os.path.join(HERE, '..', 'tests', 'golden', 'golden_plot.json')
WINDOWS = (1, 7, 100, 1000, 2500)


def stub_matplotlib():
    mpl = types.ModuleType('matplotlib')
    mpl.axes = types.ModuleType('matplotlib.axes')
    mpl.axes.Axes = type('Axes', (), {})
    mpl.projections = types.ModuleType('matplotlib.projections')
    mpl.projections.register_projection = lambda cls: None
    mpl.pyplot = types.ModuleType('matplotlib.pyplot')
    for name, mod in (('matplotlib', mpl), ('matplotlib.axes', mpl.axes), ('matplotlib.projections', mpl.projections),
                      ('matplotlib.pyplot', mpl.pyplot)):
        sys.modules[name] = mod


def digest(values, dtype):
    return hashlib.sha256(np.asarray(values, dtype=dtype).tobytes()).hexdigest()


def main():
    stub_matplotlib()
    sys.path.insert(0, os.path.join(HERE, 'edlib_shim'))
    sys.path.insert(0, '/root/reference')
    import badread.plot_window_identity as rp

    calls = []
    original = rp.get_window_means

    def recording(*a, **kw):
        result = original(*a, **kw)
        calls.append(result)
        return result

    rp.get_window_means = recording
    out = {'inputs': 'tests/golden/models: ref.fasta, reads.fastq, reads.paf', 'cases': []}
    stdout = None
    for window in WINDOWS:
        for qual in (False, True):
            args = argparse.Namespace(reference=os.path.join(DATA, 'ref.fasta'), reads=os.path.join(DATA, 'reads.fastq'),
                                      alignment=os.path.join(DATA, 'reads.paf'), window=window, qual=qual, no_plot=True)
            calls.clear()
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                rp.plot_window_identity(args, output=buf)
            if stdout is None:
                stdout = buf.getvalue()
            assert buf.getvalue() == stdout
            per = 2 if qual else 1
            ident = [calls[i] for i in range(0, len(calls), per)]
            quals = [calls[i + 1] for i in range(0, len(calls), per)] if qual else []
            positions = [p for pos, _ in ident for p in pos]
            identities = [v for _, m in ident for v in m]
            case = {'window': window, 'qual': qual, 'counts': [len(m) for _, m in ident],
                    'positions_sha256': digest(positions, np.int64), 'identity_sha256': digest(identities, np.float64),
                    'min_identity': float.hex(min(identities)) if identities else None,
                    'samples': [[a, j, pos[j], float.hex(m[j])] for a, (pos, m) in enumerate(ident) if m
                                for j in (0, len(m) // 2, len(m) - 1)][:12]}
            if qual:
                assert all(len(q) == len(m) for (_, q), (_, m) in zip(quals, ident))
                case['qual_sha256'] = digest([v for _, q in quals for v in q], np.float64)
                case['qual_samples'] = [[a, j, float.hex(q[j])] for a, (_, q) in enumerate(quals) if q
                                        for j in (0, len(q) - 1)][:8]
            out['cases'].append(case)
    out['stdout'] = stdout
    with open(OUT, 'w') as f:
        json.dump(out, f, indent=1)
        f.write('\n')
    print(f'wrote {OUT}: {len(out["cases"])} cases, {stdout.count(chr(10))} stdout lines')


if __name__ == '__main__':
    main()
