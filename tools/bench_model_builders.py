#!/usr/bin/env python3
"""
bench_model_builders.py - `badread error_model` / `badread qscore_model` (SURVEY.md 8f row f4) on a synthetic data set,
this repo's GPU builders next to the unmodified reference (oracle/_ref + oracle/edlib_shim, one process - the
reference's builders are single-threaded Python), with the two model files compared byte for byte.

    python tools/bench_model_builders.py [--reads 600] [--length 8000] [--skip_reference]

Prints one JSON object: alignment columns per second of each command for both implementations (whole command: parsing,
counting, sorting, printing), the share of the GPU counting call in this repo's time, and whether the files are equal.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), '..')
sys.path.insert(0, ROOT)
ACGT = np.frombuffer(b'ACGT', dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for x, y in zip(b'ACGTN', b'TGCAN'):
    COMP[x] = y


def make_data(directory, n_reads, length, seed=7):
    rs = np.random.RandomState(seed)
    ref = ACGT[rs.randint(0, 4, 2_000_000)]
    with open(os.path.join(directory, 'ref.fasta'), 'wb') as f:
        f.write(b'>chr\n' + ref.tobytes() + b'\n')
    columns = 0
    with open(os.path.join(directory, 'reads.fastq'), 'wb') as fq, open(os.path.join(directory, 'reads.paf'), 'w') as paf:
        for i in range(n_reads):
            n = int(rs.randint(length // 2, length * 3 // 2))
            start = int(rs.randint(0, ref.size - n))
            strand = '+' if rs.rand() < 0.5 else '-'
            seg = ref[start:start + n]
            if strand == '-':
                seg = COMP[seg[::-1]]
            u = rs.rand(n)
            deleted = u < 0.03
            deleted[0] = deleted[-1] = False
            sub = (u >= 0.03) & (u < 0.06)
            ins_after = np.where(rs.rand(n) < 0.025, rs.randint(1, 4, n), 0)
            ins_after[-1] = 0
            ins_after[deleted] = 0
            bases = seg.copy()
            bases[sub] = ACGT[rs.randint(0, 4, int(sub.sum()))]
            # columns: per reference base one M or D column, then its insertion columns
            per_base = 1 + ins_after
            out_len = int((~deleted).sum() + ins_after.sum())
            read = np.empty(out_len, dtype=np.uint8)
            kinds = np.empty(int(per_base.sum()), dtype=np.uint8)       # 0 M, 1 I, 2 D per column
            col = np.cumsum(per_base) - per_base
            kinds[:] = 1
            kinds[col] = np.where(deleted, 2, 0)
            is_read = kinds != 2
            read_cols = np.flatnonzero(is_read)
            vals = np.empty(kinds.size, dtype=np.uint8)
            vals[:] = ACGT[rs.randint(0, 4, kinds.size)]
            vals[col] = bases
            read[:] = vals[read_cols]
            change = np.flatnonzero(np.diff(kinds)) + 1
            bounds = np.concatenate([[0], change, [kinds.size]])
            runs = [(int(bounds[j + 1] - bounds[j]), 'MID'[kinds[bounds[j]]]) for j in range(len(bounds) - 1)]
            if strand == '-':
                runs = runs[::-1]
            cigar = ''.join(f'{c}{k}' for c, k in runs)
            matches = int(((kinds[col] == 0) & ~sub).sum())
            qual = (33 + rs.randint(2, 41, out_len)).astype(np.uint8)
            fq.write(b'@r%d\n' % i + read.tobytes() + b'\n+\n' + qual.tobytes() + b'\n')
            paf.write('\t'.join([f'r{i}', str(out_len), '0', str(out_len), strand, 'chr', str(ref.size), str(start),
                                 str(start + n), str(matches), str(kinds.size), '60', f'AS:i:{2 * matches - kinds.size}',
                                 f'cg:Z:{cigar}']) + '\n')
            columns += kinds.size
    return columns


def run(fn, args):
    out = io.StringIO()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(out):
        fn(args, output=io.StringIO())
    return out.getvalue(), time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=600)
    ap.add_argument('--length', type=int, default=8000)
    ap.add_argument('--skip_reference', action='store_true')
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        columns = make_data(d, a.reads, a.length)
        base = dict(reference=os.path.join(d, 'ref.fasta'), reads=os.path.join(d, 'reads.fastq'),
                    alignment=os.path.join(d, 'reads.paf'), max_alignments=None)
        em_args = types.SimpleNamespace(k_size=7, max_alt=25, **base)
        qm_args = types.SimpleNamespace(k_size=9, max_del=6, min_occur=100, max_output=10000, **base)
        from badread_b200 import model_builders as mb
        count_s = [0.0]
        inner = mb._count

        def timed_count(*x, **kw):
            t0 = time.perf_counter()
            r = inner(*x, **kw)
            count_s[0] += time.perf_counter() - t0
            return r
        mb._count = timed_count
        run(mb.make_error_model, em_args)     # warm-up: CUDA context, module load
        count_s[0] = 0.0
        ours_em, t_em = run(mb.make_error_model, em_args)
        c_em, count_s[0] = count_s[0], 0.0
        ours_qm, t_qm = run(mb.make_qscore_model, qm_args)
        c_qm = count_s[0]
        res = {'metric': 'alignment columns/s', 'data': f'synthetic: {a.reads} reads of ~{a.length} bases on a 2 Mb reference, '
               f'3 % deletions, 3 % substitutions, 2.5 % insertion sites; {columns} alignment columns',
               'b200': {'error_model': columns / t_em, 'qscore_model': columns / t_qm, 'error_model_s': t_em,
                        'qscore_model_s': t_qm, 'gpu_count_call_s': {'error_model': c_em, 'qscore_model': c_qm},
                        'note': 'whole command: parse FASTA / FASTQ / PAF, choose and flatten the alignments (Python), '
                                'count on the GPU (bb_count_*: copies + kernels), sort and print'}}
        if not a.skip_reference:
            sys.path.insert(0, os.path.join(ROOT, 'oracle', 'edlib_shim'))
            sys.path.insert(0, os.path.join(ROOT, 'oracle', '_ref'))
            import badread.error_model as rem
            import badread.qscore_model as rqm
            ref_em, r_em = run(rem.make_error_model, em_args)
            ref_qm, r_qm = run(rqm.make_qscore_model, qm_args)
            res['reference'] = {'error_model': columns / r_em, 'qscore_model': columns / r_qm, 'error_model_s': r_em,
                                'qscore_model_s': r_qm, 'note': 'unmodified badread (oracle/_ref), one process'}
            res['parity'] = {'error_model_identical': ours_em == ref_em, 'qscore_model_identical': ours_qm == ref_qm,
                             'error_model_lines': len(ours_em.splitlines()), 'qscore_model_lines': len(ours_qm.splitlines())}
            res['speedup'] = {'error_model': r_em / t_em, 'qscore_model': r_qm / t_qm}
        print(json.dumps(res))
        if 'parity' in res and not (res['parity']['error_model_identical'] and res['parity']['qscore_model_identical']):
            sys.exit(3)


if __name__ == '__main__':
    main()
