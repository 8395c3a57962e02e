#!/usr/bin/env python3
"""
BAM input of the model builders on one GPU.  The data set is the golden one of tests/golden/models (reads.fastq,
reads.paf) repeated --copies times under new read names, written as FASTQ + PAF and as BAM (BGZF by zlib level 6, the
converter of tests/test_model_builders_alignments.py).  Measures:
  * the card's name, power limit and top SM clock;
  * the inflate of that BAM: the whole bgzf.decompress call (host walk, copies both ways, kernel), the kernel alone
    (torch.profiler, CUDA activities, in a run of its own), and zlib member by member on one thread of this host;
  * the wall time of `python -m badread_b200 error_model` from the BAM alone against the same build from FASTQ + PAF,
    alternating, and that both write the same model.
Prints one JSON line.  Usage: tools/bench_bam_input.py [--copies C] [--repeats R]
"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import test_model_builders_alignments as T  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi failed: {q.stderr.strip()[:200]}'


def data_set(tmp, copies):
    reads = T.read_fastq(os.path.join(T.DATA, 'reads.fastq'))
    refs = T.read_refs(os.path.join(T.DATA, 'ref.fasta'))
    paf = open(os.path.join(T.DATA, 'reads.paf')).read().splitlines()
    all_reads, all_paf = {}, []
    for c in range(copies):
        for n, r in reads.items():
            all_reads[f'{n}_{c}'] = r
        for line in paf:
            f = line.split('\t')
            all_paf.append('\t'.join([f'{f[0]}_{c}'] + f[1:]))
    paths = {k: os.path.join(tmp, 'reads.' + k) for k in ('fastq', 'paf', 'bam')}
    with open(paths['fastq'], 'w') as f:
        f.write(''.join(f'@{n}\n{s}\n+\n{q}\n' for n, (s, q) in all_reads.items()))
    with open(paths['paf'], 'w') as f:
        f.write('\n'.join(all_paf) + '\n')
    raw = T.bam_bytes(T.paf_to_records(all_paf, all_reads), refs)
    with open(paths['bam'], 'wb') as f:
        f.write(b''.join(T.bgzf_member(raw[i:i + T.CHUNK], 6) for i in range(0, len(raw), T.CHUNK)) + T.EOF)
    return paths, len(raw), len(all_paf)


def build(argv):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.environ.get('PYTHONPATH', '')]))
    t0 = time.perf_counter()
    p = subprocess.run([sys.executable, '-m', 'badread_b200', 'error_model'] + argv, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, timeout=3600)
    wall = time.perf_counter() - t0
    if p.returncode:
        raise RuntimeError(p.stderr.decode(errors='replace')[-500:])
    return wall, p.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--copies', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    res = {'card': card()}
    tmp = tempfile.mkdtemp()
    paths, raw_bytes, n_records = data_set(tmp, a.copies)
    comp = open(paths['bam'], 'rb').read()
    res.update(records=n_records, bam_bytes=len(comp), inflated_bytes=raw_bytes)

    from badread_b200.bgzf import decompress
    out = decompress(comp)                       # warm-up: context, module load
    assert bytes(out) == gzip.decompress(comp)
    calls = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        decompress(comp)
        calls.append(time.perf_counter() - t0)
    res['call_s'] = calls
    res['call_MB_per_s'] = raw_bytes / min(calls) / 1e6
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decompress(comp)
        torch.cuda.synchronize()
    k_ms = sum((ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total) / 1e3
               for ev in prof.events() if 'infl_k_members' in ev.name)
    res['kernel_ms'] = k_ms
    res['kernel_MB_per_s'] = raw_bytes / (k_ms / 1e3) / 1e6 if k_ms else None
    # zlib member by member (gzip.decompress copies the rest of the stream per member, which is quadratic)
    zl = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        view, pos, parts = memoryview(comp), 0, []
        while pos < len(comp):
            end = pos + int.from_bytes(comp[pos + 16:pos + 18], 'little') + 1
            parts.append(zlib.decompress(view[pos + 18:end - 8], -15))
            pos = end
        zl.append(time.perf_counter() - t0)
        assert b''.join(parts) == bytes(out)
    res['zlib_one_thread_s'] = zl
    res['zlib_one_thread_MB_per_s'] = raw_bytes / min(zl) / 1e6

    ref = os.path.join(T.DATA, 'ref.fasta')
    runs = {'bam': [], 'fastq_paf': []}
    outs = {}
    for _ in range(a.repeats):
        runs['bam'].append(None)
        runs['bam'][-1], outs['bam'] = build(['--reference', ref, '--alignment', paths['bam']])
        runs['fastq_paf'].append(None)
        runs['fastq_paf'][-1], outs['paf'] = build(['--reference', ref, '--reads', paths['fastq'], '--alignment', paths['paf']])
    res['error_model_wall_s'] = runs
    res['same_model'] = outs['bam'] == outs['paf']
    for p in paths.values():
        os.unlink(p)
    os.rmdir(tmp)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
