#!/usr/bin/env python3
"""
bench_builder_routes.py - `badread error_model` from FASTQ + PAF on the two routes of model_builders.device_route: the
host route (load_fastq, load_alignments, FlatAlignments in Python) and the device route (the FASTQ inflated and parsed
on the GPU, the PAF parsed by bb_aln_parse, the aligned slices gathered on the GPU), alternating, on the synthetic data
of tools/bench_model_builders.py, plain and gzipped.

    python tools/bench_builder_routes.py [--reads 2000] [--length 8000] [--runs 3]

Each run is a process of its own (its peak RSS is its own).  Prints one JSON object: the card and its power limit, and
per run the whole-command wall time, the stage split, the peak host RSS, the peak device memory in use (cudaMemGetInfo
sampled every 5 ms, above what the process held before the command) and whether the model file equals the host route's.
The device route's stages: 'read' (the file into page-locked memory), 'inflate_parse' (bb_fastq_parse: upload,
inflate, parse kernels, names to the host; not split further), 'alignments' (PAF parse and choice), 'join_gather'
(bb_flat_build: join, planning, upload, gather kernel), 'count'.  The host route's: 'reads', 'alignments', 'flatten',
'count'.  Needs a GPU: without one the device route fails.
"""
import argparse
import contextlib
import ctypes
import hashlib
import io
import json
import os
import resource
import subprocess
import sys
import tempfile
import threading
import time
import types

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))


def _timed(obj, name, stage, split):
    inner = getattr(obj, name)

    def wrapper(*a, **kw):
        t0 = time.perf_counter()
        try:
            return inner(*a, **kw)
        finally:
            split[stage] = split.get(stage, 0.0) + time.perf_counter() - t0
    setattr(obj, name, wrapper)


class _DeviceMemory(object):
    """The peak of (total - free) device memory, sampled every 5 ms, above the level at start."""

    def __init__(self):
        self.rt = ctypes.CDLL('libcudart.so.12')
        self.base = self.peak = self._used()
        self.stop = False
        self.thread = threading.Thread(target=self._poll, daemon=True)
        self.thread.start()

    def _used(self):
        free, total = ctypes.c_size_t(), ctypes.c_size_t()
        self.rt.cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total))
        return total.value - free.value

    def _poll(self):
        while not self.stop:
            self.peak = max(self.peak, self._used())
            time.sleep(0.005)

    def close(self):
        self.stop = True
        self.thread.join()
        return self.peak - self.base


def child(route, reads, paf, reference):
    """One run of error_model on `route`: prints its JSON record."""
    from badread_b200 import engine
    from badread_b200 import model_builders as mb
    split = {}
    mb.device_route = lambda args, fmt: route == 'device'
    if route == 'device':
        _timed(engine, 'FastaFile', 'read', split)
        _timed(mb._lib.lib(), 'bb_fastq_parse', 'inflate_parse', split)
        _timed(mb, '_parse_records', 'alignments', split)
        _timed(mb._lib.lib(), 'bb_flat_build', 'join_gather', split)
    else:
        _timed(mb, 'load_fastq', 'reads', split)
        _timed(mb, 'load_alignments', 'alignments', split)
        _timed(mb, 'FlatAlignments', 'flatten', split)
    _timed(mb, '_count', 'count', split)
    if mb._lib.lib().bb_device_count() < 1:
        sys.exit('bench_builder_routes: no CUDA device')
    mem = _DeviceMemory()
    args = types.SimpleNamespace(reference=reference, reads=reads, alignment=paf, max_alignments=None, k_size=7, max_alt=25)
    out = io.StringIO()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(out):
        mb.make_error_model(args, output=io.StringIO())
    wall = time.perf_counter() - t0
    peak_dev = mem.close()
    print(json.dumps({'route': route, 'wall_s': wall, 'stages_s': split,
                      'peak_rss_mb': resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024,
                      'peak_device_mb': peak_dev / 2 ** 20, 'model_sha1': hashlib.sha1(out.getvalue().encode()).hexdigest()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=2000)
    ap.add_argument('--length', type=int, default=8000)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--child', nargs=4, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(*a.child)
    from bench_model_builders import make_data
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True).stdout.strip()
    with tempfile.TemporaryDirectory() as d:
        columns = make_data(d, a.reads, a.length)
        plain = os.path.join(d, 'reads.fastq')
        subprocess.run(['gzip', '-6', '-k', plain], check=True)
        res = {'gpu': gpu, 'data': f'synthetic: {a.reads} reads of ~{a.length} bases, {columns} alignment columns',
               'runs': []}
        for kind, reads in (('plain', plain), ('gzip', plain + '.gz')):
            want = None
            for i in range(a.runs):
                for route in ('host', 'device'):
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', route, reads,
                                        os.path.join(d, 'reads.paf'), os.path.join(d, 'ref.fasta')],
                                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, universal_newlines=True)
                    if p.returncode:
                        sys.exit(f'{route} run failed: {p.stderr[-2000:]}')
                    r = json.loads(p.stdout.strip().splitlines()[-1])
                    want = want or (r['model_sha1'] if route == 'host' else None)
                    r.update(fastq=kind, run=i, identical_to_host=r.pop('model_sha1') == want)
                    res['runs'].append(r)
        print(json.dumps(res))


if __name__ == '__main__':
    main()
