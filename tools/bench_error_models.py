#!/usr/bin/env python3
"""
bench_error_models.py - the cost of an error model's k-mer index.  One config-1-sized batch (bench.py's workload: 5 Mb
synthetic reference, 50x, nanopore2023 qscore model, seed 1) is run with three error models:

  nanopore2023 dense   the built-in k = 7 model with its dense kmer_to_row[4^7] (bb_upload_error_model)
  nanopore2023 hash    the same model through the hash-table index (bb_upload_error_model_kmers): the lookup cost in K1
  synthetic k16        a seeded k = 16 model with one row for every distinct 16-mer of the reference's two strands
                       (millions of rows): keep the 16-mer (p ~ U(0.85, 0.95)), drop one seeded base (p = 0.03), or make
                       one random change (the remainder).  Its tables are built with numpy here, not read from a model
                       file (ErrorModel's text loader walks the rows in Python)

For each: rows and entries, the host time to load / build the tables, the upload time, the device memory of the
tables, and the median over the timed runs of the build_fragments stage (K1) and of the whole step (bb_last_run_ms),
after one warm-up run.  Needs a GPU.

    python tools/bench_error_models.py [--runs 5] [--reads N]

Prints one JSON object.
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), '..')
sys.path.insert(0, ROOT)


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


class TableModel(object):
    """Flat error-model tables built directly (the to_device_tables() surface Engine.set_error_model reads)."""

    def __init__(self, tables):
        self._t = tables

    def to_device_tables(self):
        return dict(self._t)


def kmer_codes_of(seq, k):
    """Distinct 2-bit codes of the ACGT k-mers of both strands of `seq` (uint8 bases)."""
    lut = np.full(256, 4, dtype=np.uint8)
    for i, c in enumerate(b'ACGT'):
        lut[c] = i
    out = []
    for strand in (0, 1):
        b = lut[seq]
        if strand:
            b = np.where(b < 4, 3 - b, 4)[::-1]
        n = b.size - k + 1
        code = np.zeros(n, dtype=np.int64)
        bad = np.zeros(n, dtype=bool)
        for j in range(k):
            w = b[j:j + n]
            bad |= w > 3
            code = code * 4 + (w & 3)
        out.append(code[~bad])
    return np.unique(np.concatenate(out))


def synthetic_k16(seq, seed=16):
    k = 16
    rs = np.random.RandomState(seed)
    codes = kmer_codes_of(seq, k)
    n = codes.size
    keep = rs.uniform(0.85, 0.95, n)
    drop = np.full(n, 0.03)
    rest = 1.0 - keep - drop
    cum = np.empty(3 * n)
    cum[0::3] = keep
    cum[1::3] = keep + drop
    cum[2::3] = keep + drop + rest
    flags = np.tile(np.asarray([1, 0, 2], dtype=np.uint8), n)
    bases = np.frombuffer(b'ACGT', dtype=np.uint8)[(codes[:, None] >> (2 * (k - 1 - np.arange(k)))) & 3]   # (n, k)
    ident = (1 | (bases.astype(np.uint32) << 8))                                                          # inline slots
    dropped = ident.copy()
    pos = rs.randint(1, k - 1, n)                     # (the first and last base stay, as in a built model)
    dropped[np.arange(n), pos] = 0                    # an empty slot string
    slots = np.empty((3 * n, k), dtype=np.uint32)
    slots[0::3] = ident
    slots[1::3] = dropped
    slots[2::3] = 0xFFFFFFFF
    return TableModel({'k': k, 'type': 1, 'index': 'hash', 'kmer_codes': codes,
                       'row_off': np.arange(0, 3 * n + 1, 3, dtype=np.int32), 'cum': cum, 'flags': flags,
                       'slots': np.ascontiguousarray(slots.reshape(-1)), 'pool': np.zeros(1, dtype=np.uint8)})


def table_bytes(t, index):
    n_rows = len(t['row_off']) - 1
    ne = int(t['row_off'][-1])
    common = t['row_off'].nbytes + ne * 8 + ne + ne * t['k'] * 4 + t['pool'].nbytes + 32 * n_rows
    if index == 'dense':
        return common + t['kmer_to_row'].nbytes
    bits = 6
    while (1 << bits) < 2 * n_rows:
        bits += 1
    return common + 8 * (1 << bits)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--runs', type=int, default=5, help='timed runs per setup')
    ap.add_argument('--reads', type=int, default=None, help='cap on the reads of the batch (default: config 1 in full)')
    a = ap.parse_args()
    import bench
    from badread_b200.engine import Engine
    from badread_b200.error_model import ErrorModel
    wl = bench.Workload(1, 0, 1, 'weak', max_reads=a.reads)
    if len(wl.batches) != 1:
        sys.exit(f'expected one batch, the workload has {len(wl.batches)}')
    t0 = time.perf_counter()
    builtin = ErrorModel('nanopore2023', io.StringIO())
    load_builtin = time.perf_counter() - t0
    t0 = time.perf_counter()
    synth = synthetic_k16(wl.ref.concat)
    load_synth = time.perf_counter() - t0
    setups = [('nanopore2023_dense', builtin, 'auto', 'dense', load_builtin),
              ('nanopore2023_hash', builtin, 'hash', 'hash', load_builtin),
              ('synthetic_k16', synth, 'auto', 'hash', load_synth)]
    eng = Engine(device=0, seed=bench.SEED)
    eng.upload_reference(wl.ref.concat)
    eng.set_qscore_model(wl.models[1])
    result = {'gpu': gpu_name_and_power_limit(), 'reads': wl.n_reads, 'fragment_bases': wl.frag_bases, 'runs': a.runs,
              'times': 'ms; stages: CUDA events of bb_last_run_ms, medians over the runs', 'setups': {}}
    for name, em, index, kind, load_s in setups:
        t = em.to_device_tables()
        t0 = time.perf_counter()
        eng.set_error_model(em, index=index)
        upload_s = time.perf_counter() - t0
        eng.upload_batch(wl.batches[0])
        eng.run_batch()
        eng.last_run_ms()
        k1, total = [], []
        for _ in range(a.runs):
            eng.run_batch()
            step, stages = eng.last_run_ms()
            k1.append(stages['build_fragments'])
            total.append(step)
        _, emitted = eng.fetch_batch()
        result['setups'][name] = {
            'k': int(t['k']), 'index': kind, 'rows': len(t['row_off']) - 1, 'entries': int(t['row_off'][-1]),
            'host_load_s': round(load_s, 3), 'upload_s': round(upload_s, 3),
            'device_table_mb': round(table_bytes(t, kind) / 2 ** 20, 1), 'emitted_bases': int(emitted),
            'build_fragments_ms_median': statistics.median(k1), 'build_fragments_ms_min': min(k1),
            'step_ms_median': statistics.median(total)}
    eng.close()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
