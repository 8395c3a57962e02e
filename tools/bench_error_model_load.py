"""Error model file loading: the host loader (ErrorModel(file)) against the device loader (DeviceErrorModel, one engine)
on seeded synthetic models written in the builders' form: a k = 7 model the size of a nanopore text model (16 384 rows,
27 entries each) and k = 16 models of 1 M and 10 M rows (three alternatives each).  Each load runs in a process of its
own and reports its wall time, its stage split (device), its peak host RSS and its peak device memory (sampled with
cudaMemGetInfo every 2 ms), with the card's name and power limit.  Both routes' tables are compared on every model whose
host load is measured.  Writes profile_out/bench_error_model_load.json (git-ignored) unless --out names another file.

    python tools/bench_error_model_load.py [--skip-host-over ROWS]
"""
import argparse
import gzip
import json
import os
import pathlib
import resource
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def synthetic_text(k, n_rows, n_alts, seed):
    """n_rows distinct k-mers, each with itself, n_alts - 2 single substitutions and one deletion, probabilities '%.6f'."""
    rng = np.random.default_rng(seed)
    codes = np.arange(4 ** k, dtype=np.int64) if n_rows == 4 ** k else rng.choice(4 ** k, size=n_rows, replace=False)
    rng.shuffle(codes)
    letters = np.frombuffer(b'ACGT', np.uint8)
    kmers = letters[(codes[:, None] >> (2 * np.arange(k - 1, -1, -1)))[:, :] & 3]
    fields = []

    def prob():   # '0.dddddd'
        d = rng.integers(0, 10, size=(n_rows, 6), dtype=np.uint8) + ord('0')
        head = np.tile(np.frombuffer(b'0.', np.uint8), (n_rows, 1))
        return np.concatenate([head, d], axis=1)

    sep = lambda c: np.full((n_rows, 1), ord(c), np.uint8)  # noqa: E731
    fields += [kmers, sep(','), prob(), sep(';')]
    for a in range(n_alts - 2):
        alt = kmers.copy()
        pos = 1 + a % (k - 2)
        alt[:, pos] = letters[(codes + 1 + a // (k - 2)) % 4]
        fields += [alt, sep(','), prob(), sep(';')]
    fields += [np.delete(kmers, k // 2, axis=1), sep(','), prob(), sep(';'), sep('\n')]
    return np.concatenate(fields, axis=1).tobytes()


def one(route, path):
    """One load in this process -> JSON line."""
    import io
    import torch
    from badread_b200.engine import Engine
    from badread_b200.error_model import DeviceErrorModel, ErrorModel
    out = {'route': route}
    if route == 'host':
        rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
        t = time.perf_counter()
        m = ErrorModel(path, io.StringIO())
        out['wall_s'] = time.perf_counter() - t
        out['rows'] = len(m._tables['row_off']) - 1
        np.savez(path + '.host.npz', **m._tables)
    else:
        eng = Engine(device=0, seed=1)
        free0 = torch.cuda.mem_get_info(0)[0]
        peak = [0]
        stop = threading.Event()

        def sample():
            while not stop.is_set():
                peak[0] = max(peak[0], free0 - torch.cuda.mem_get_info(0)[0])
                time.sleep(0.002)

        th = threading.Thread(target=sample)
        rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
        th.start()
        t = time.perf_counter()
        m = DeviceErrorModel.load(path, [eng], io.StringIO())
        out['wall_s'] = time.perf_counter() - t
        stop.set()
        th.join()
        out['info'] = m.info
        out['peak_device_bytes'] = int(peak[0])
        out['rows'] = m.info['n_rows']
        if os.path.exists(path + '.host.npz'):
            with np.load(path + '.host.npz') as h:
                out['tables_equal'] = all(np.array_equal(h[key], m._tables[key]) and h[key].dtype == m._tables[key].dtype
                                          for key in h.files) and sorted(h.files) == sorted(m._tables)
        eng.close()
    out['rss_before_kb'] = rss0
    out['peak_rss_kb'] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--one', nargs=2, metavar=('ROUTE', 'FILE'))
    ap.add_argument('--skip-host-over', type=int, default=2_000_000, help='rows above which the host loader is not run')
    ap.add_argument('--out', default=str(ROOT / 'profile_out' / 'bench_error_model_load.json'),
                    help='the JSON file of the results')
    a = ap.parse_args()
    if a.one:
        return one(*a.one)
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()
    results = {'card': card[0] if card else 'unknown', 'models': []}
    with tempfile.TemporaryDirectory() as tmp:
        for label, k, rows, alts in (('k7_nanopore_size', 7, 16384, 27), ('k16_1M', 16, 1_000_000, 3),
                                     ('k16_10M', 16, 10_000_000, 3)):
            path = os.path.join(tmp, f'{label}.txt.gz')
            text = synthetic_text(k, rows, alts, seed=k + rows)
            with gzip.open(path, 'wb', compresslevel=1) as f:
                f.write(text)
            entry = {'model': label, 'k': k, 'rows': rows, 'text_bytes': len(text), 'file_bytes': os.path.getsize(path)}
            del text
            for route in ('host', 'device'):
                if route == 'host' and rows > a.skip_host_over:
                    entry['host'] = 'not measured'
                    continue
                r = subprocess.run([sys.executable, __file__, '--one', route, path], capture_output=True, text=True)
                if r.returncode:
                    entry[route] = {'error': r.stderr[-2000:]}
                else:
                    entry[route] = json.loads(r.stdout.strip().splitlines()[-1])
            results['models'].append(entry)
            print(json.dumps(entry), flush=True)
    pathlib.Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    pathlib.Path(a.out).write_text(json.dumps(results, indent=1))


if __name__ == '__main__':
    main()
