#!/usr/bin/env python3
"""
bench_plot.py - `badread_b200 plot --windows` on a seeded synthetic set: wall time with its stage split, peak device
memory, and for scale the pure-Python time of the reference's per-base loops (align_sequences + get_window_means) on a
prefix of the alignments.

    python tools/bench_plot.py [--mb 300] [--read_kb 20] [--window 100] [--qual] [--gz] [--out DIR]

The set: one random contig, reads cut from it on both strands with ~8 % substitutions and a 1-3 base insertion or
deletion every ~60 bases, PAF with cg:Z: tags.  Stages: load (FASTQ parsed on the GPU, PAF parsed, best alignment per
read), gather (aligned slices on the GPU), kernel (bb_window_series: all passes, copies to the host included), format
and write (the rest of writing the table: bb_window_format and the file or BGZF writer).  Peak device memory is
sampled from cudaMemGetInfo every 5 ms (the library allocates outside PyTorch's allocator).  Prints one JSON line with
the card's name and power limit.  Writes the data set and the table to a temporary directory unless --out names one.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)

_COMP = bytes.maketrans(b'ACGT', b'TGCA')


def make_set(d, total_mb, read_kb, seed=1):
    rs = np.random.RandomState(seed)
    acgt = np.frombuffer(b'ACGT', np.uint8)
    n_reads = max(1, int(total_mb * 1000 // read_kb))
    ctg = acgt[rs.randint(0, 4, max(2_000_000, read_kb * 3000))].tobytes()
    with open(os.path.join(d, 'ref.fasta'), 'wb') as f:
        f.write(b'>c\n' + ctg + b'\n')
    fq, paf = open(os.path.join(d, 'reads.fastq'), 'wb'), open(os.path.join(d, 'aln.paf'), 'w')
    for i in range(n_reads):
        n = int(read_kb * 1000 * (0.5 + rs.rand()))
        fs = int(rs.randint(0, len(ctg) - 2 * n))
        m_len = rs.randint(20, 100, n // 20 + 2)
        kinds = rs.randint(0, 2, m_len.size)            # 0: insertion, 1: deletion after each M run
        ind = rs.randint(1, 4, m_len.size)
        parts, runs, fp, rp = [], [], 0, 0
        for m, k, x in zip(m_len.tolist(), kinds.tolist(), ind.tolist()):
            if rp >= n:
                break
            seg = bytearray(ctg[fs + fp:fs + fp + m])
            parts.append(bytes(seg))
            runs.append(f'{m}M')
            fp += m
            rp += m
            if k == 0:
                parts.append(acgt[rs.randint(0, 4, x)].tobytes())
                runs.append(f'{x}I')
                rp += x
            else:
                runs.append(f'{x}D')
                fp += x
        runs.append('10M')
        parts.append(ctg[fs + fp:fs + fp + 10])
        fp += 10
        rp += 10
        seq = np.frombuffer(b''.join(parts), np.uint8).copy()
        sub = rs.rand(seq.size) < 0.08
        seq[sub] = acgt[rs.randint(0, 4, int(sub.sum()))]
        strand = '+' if i % 2 == 0 else '-'
        s = seq.tobytes()
        if strand == '-':
            s = s.translate(_COMP)[::-1]   # (the runs stay: PAF's CIGAR is in the reference's orientation)
        q = (33 + rs.randint(5, 40, len(s))).astype(np.uint8).tobytes()
        fq.write(b'@r%d\n%s\n+\n%s\n' % (i, s, q))
        cols = rp + sum(int(r[:-1]) for r in runs if r.endswith('D'))
        paf.write(f'r{i}\t{len(s)}\t0\t{len(s)}\t{strand}\tc\t{len(ctg)}\t{fs}\t{fs + fp}\t{int(cols * 0.9)}\t{cols}\t60'
                  f'\tAS:i:{cols}\tcg:Z:{"".join(runs)}\n')
    fq.close()
    paf.close()
    return n_reads


def python_loops(reads, refs, alns, window, budget):
    """The reference's per-base loops (align_sequences' error list and get_window_means' running sum) over the first
    alignments, `budget` read positions in all: (seconds, positions)."""
    from badread_b200.misc import reverse_complement
    t0, done = time.perf_counter(), 0
    for a in alns:
        if done >= budget:
            break
        seq, _ = reads[a.read_name]
        read = seq[a.read_start:a.read_end]
        ref = refs[a.ref_name][a.ref_start:a.ref_end]
        if a.strand == '-':
            ref = reverse_complement(ref)
        e, rp, fp = [0] * len(read), 0, 0
        for count, kind in a.runs:
            if kind == 'M':
                for i in range(count):
                    if read[rp + i] != ref[fp + i]:
                        e[rp + i] += 1
                rp += count
                fp += count
            elif kind == 'I':
                for i in range(count):
                    e[rp + i] += 1
                rp += count
            elif kind == 'D':
                e[rp] += count
                fp += count
        s, means = sum(e[:window]), []
        for i in range(len(e) - window):
            means.append(100.0 * (1.0 - s / window))
            s += e[i + window] - e[i]
        done += len(read)
    return time.perf_counter() - t0, done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mb', type=float, default=300, help='aligned read bases, in Mb')
    ap.add_argument('--read_kb', type=int, default=20)
    ap.add_argument('--window', type=int, default=100)
    ap.add_argument('--qual', action='store_true')
    ap.add_argument('--gz', action='store_true')
    ap.add_argument('--python_mb', type=float, default=2, help='positions for the pure-Python loops, in Mb')
    ap.add_argument('--out', help='directory for the data set and the table (default: a temporary one)')
    args = ap.parse_args()
    import torch
    from badread_b200 import misc, plot
    from badread_b200 import model_builders as mb

    d = args.out or tempfile.mkdtemp(prefix='bench_plot_')
    os.makedirs(d, exist_ok=True)
    t = time.perf_counter()
    n_reads = make_set(d, args.mb, args.read_kb)
    t_make = time.perf_counter() - t
    ref, reads, paf = (os.path.join(d, x) for x in ('ref.fasta', 'reads.fastq', 'aln.paf'))
    table = os.path.join(d, 'windows.tsv' + ('.gz' if args.gz else ''))

    torch.cuda.init()
    free0, total = torch.cuda.mem_get_info(0)
    low = [free0]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            time.sleep(0.005)

    th = threading.Thread(target=sample, daemon=True)
    th.start()
    stages = {}
    try:
        t0 = time.perf_counter()
        refs = misc.load_fasta(ref)[0]
        a = argparse.Namespace(reference=ref, reads=reads, alignment=paf, max_alignments=None)
        inp = mb._DeviceInputs(a, refs, io.StringIO())
        stages['load'] = time.perf_counter() - t0
        try:
            t = time.perf_counter()
            flat = inp.flatten(io.StringIO(), 1000, np.zeros((inp.n, 3), np.int64))
            stages['gather'] = time.perf_counter() - t
            read_start = inp.a['read_start'][inp.chosen]
            names = [inp.read_names[i] for i in inp.a['read_id'][inp.chosen].tolist()]
            t = time.perf_counter()
            for _ in plot._passes(flat, args.window, args.qual):
                pass
            stages['kernel'] = time.perf_counter() - t
            t = time.perf_counter()
            plot.write_windows(table, flat, names, read_start, args.window, args.qual)
            stages['format_write'] = time.perf_counter() - t - stages['kernel']    # (write_windows runs the passes again)
            positions = int(flat.read_off[-1])
        finally:
            inp.close()
        wall = time.perf_counter() - t0
    finally:
        stop.set()
        th.join()
    r, f, alns = mb.load_fastq(reads, output=io.StringIO()), refs, mb.load_alignments(paf, output=io.StringIO())
    py_s, py_n = python_loops(r, f, alns, args.window, int(args.python_mb * 1e6))
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    print(json.dumps({'reads': n_reads, 'aligned_positions': positions, 'window': args.window, 'qual': args.qual,
                      'gz': args.gz, 'make_set_s': round(t_make, 2), 'wall_s': round(wall, 3),
                      'stages_s': {k: round(v, 3) for k, v in stages.items()},
                      'table_bytes': os.path.getsize(table), 'peak_device_mb_sampled': round((free0 - low[0]) / 2**20, 1),
                      'python_loops': {'positions': py_n, 'seconds': round(py_s, 3),
                                       'positions_per_s': round(py_n / py_s) if py_s else None},
                      'gpu': smi[0] if smi else None}))


if __name__ == '__main__':
    main()
