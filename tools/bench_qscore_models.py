#!/usr/bin/env python3
"""
bench_qscore_models.py - the cost of qscore-model keys of more than 31 symbols in K5 (bb_k_qscores).  One config-1-sized
batch (bench.py's workload: 5 Mb synthetic reference, 50x, nanopore2023 error model, seed 1) is run with the same error
model and two qscore models: the built-in nanopore2023 (keys of at most 21 symbols, the packed table alone) and
tests/golden/models/qscore_model_k9_all.txt.gz (k=9, max_del=6, keys of up to 57 symbols, so windows that the packed
key cannot hold are looked up in the side table).  Reports the `qscores` stage time of bb_last_run_ms for each, over
repeated runs of the uploaded batch (after one warm-up run per model).  Needs a GPU.

    python tools/bench_qscore_models.py [--runs 5] [--reads N]

Prints one JSON object.
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), '..')
sys.path.insert(0, ROOT)


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--runs', type=int, default=5, help='timed runs per model')
    ap.add_argument('--reads', type=int, default=None, help='cap on the reads of the batch (default: config 1 in full)')
    a = ap.parse_args()
    import bench
    from badread_b200.engine import Engine
    from badread_b200.qscore_model import QScoreModel
    wl = bench.Workload(1, 0, 1, 'weak', max_reads=a.reads)
    if len(wl.batches) != 1:
        sys.exit(f'expected one batch, the workload has {len(wl.batches)}')
    models = {'nanopore2023': wl.models[1],
              'qscore_model_k9_all': QScoreModel(os.path.join(ROOT, 'tests', 'golden', 'models', 'qscore_model_k9_all.txt.gz'),
                                                 io.StringIO())}
    eng = Engine(device=0, seed=bench.SEED)
    eng.upload_reference(wl.ref.concat)
    eng.set_error_model(wl.models[0])
    result = {'gpu': gpu_name_and_power_limit(), 'reads': wl.n_reads, 'fragment_bases': wl.frag_bases, 'runs': a.runs,
              'stage': 'qscores (bb_k_qscores, CUDA events of bb_last_run_ms)', 'models': {}}
    for name, qm in models.items():
        eng.set_qscore_model(qm)
        eng.upload_batch(wl.batches[0])
        eng.run_batch()
        eng.last_run_ms()
        q_ms, total_ms = [], []
        for _ in range(a.runs):
            eng.run_batch()
            total, stages = eng.last_run_ms()
            q_ms.append(stages['qscores'])
            total_ms.append(total)
        _, emitted = eng.fetch_batch()
        t = qm.to_device_tables()
        result['models'][name] = {
            'keys': int(t['n_keys']), 'keys_over_31_symbols': int((t['keys'] == 0).sum()),
            'longest_key': max(len(c) for c in qm.scores), 'emitted_bases': int(emitted),
            'qscores_ms_median': statistics.median(q_ms), 'qscores_ms_min': min(q_ms), 'qscores_ms_max': max(q_ms),
            'run_ms_median': statistics.median(total_ms)}
    eng.close()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
