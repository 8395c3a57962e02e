"""Loading the simulate reference from plain gzip: BASELINE config 4's reference (24 contigs of 125 Mb, written by
tools/bench_reference_load.py's writer) compressed by zlib at level 6 as one gzip member per contig (as `pigz -6` or a
concatenation of `gzip -6` files gives, no BGZF fields), and as BGZF.

Three legs, alternating, each in a process of its own: the host route (Python's gzip inflates, then bb_fasta_parse
parses the text on the device), the device route (Engine.load_fasta: the file inflated in parallel chunks on the GPU),
and BGZF for reference.  Per leg: wall time, the inflater's stats, and in a separate profiled run the per-kernel CUDA
times from torch.profiler.  The card's name and power limit are read in the same call.  Prints one JSON line.

    python tools/bench_gzip_input.py [--contigs 24] [--contig_mb 125] [--reps 2] [--out DIR]

With --sweep the three legs are replaced by the inflater alone (bgzf.gunzip) on the gzip file at several chunk sizes,
each in a profiled process of its own, for each library given with --lib (builds with other constants, such as
GZ_CANDIDATES, linked by the caller): the per-kernel times and the stats of each.

    python tools/bench_gzip_input.py --sweep 16,32,64,128,256 [--lib path.so ...]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib
from multiprocessing import Pool

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def _member(args):
    path, lo, hi = args
    with open(path, 'rb') as f:
        f.seek(lo)
        data = f.read(hi - lo)
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    return co.compress(data) + co.flush()


def write_gzip(plain, out, n_contigs):
    """One level-6 gzip member per contig of the plain file, compressed side by side."""
    with open(plain, 'rb') as f:
        text = f.read()
    starts, at = [], 0
    while True:
        at = text.find(b'>', at)
        if at < 0:
            break
        starts.append(at)
        at += 1
    del text
    bounds = starts + [os.path.getsize(plain)]
    with Pool(min(n_contigs, os.cpu_count() or 1)) as pool, open(out, 'wb') as fo:
        for m in pool.imap(_member, [(plain, a, b) for a, b in zip(bounds[:-1], bounds[1:])]):
            fo.write(m)


def _kernel_times(prof):
    out = {}
    for ev in prof.key_averages():
        dev_us = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0) or 0
        name = ev.key.replace('(anonymous namespace)::', '').replace('void ', '').split('(')[0]
        if dev_us and (name.startswith(('gz_k_', 'infl_k_', 'fasta_k_')) or 'Memcpy' in name):
            out[name] = round(dev_us / 1e3, 3)
    return out


def sweep_leg(lib_path, path, chunk_kib):
    """The inflater alone on the file, in a profiled run, with the library at lib_path (default: the tree's)."""
    import pathlib
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    from badread_b200 import _lib
    if lib_path != '-':
        _lib.LIB_PATH = pathlib.Path(lib_path)
    from badread_b200.bgzf import gunzip
    with open(path, 'rb') as f:
        data = f.read()
    gunzip(zlib.compress(b'>a\nACGT\n', wbits=31))   # (library load and CUDA context, not timed)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        out, stats = gunzip(data, chunk_bytes=chunk_kib << 10)
        wall = time.perf_counter() - t0
    k = _kernel_times(prof)
    return {'lib': os.path.basename(lib_path), 'chunk_kib': chunk_kib, 'bytes_out': len(out), 'wall_s': wall, 'stats': stats,
            'kernels_ms': k, 'gz_kernels_ms': round(sum(v for n, v in k.items() if n.startswith('gz_k_')), 3)}


def leg(route, path, profile):
    import torch  # noqa: F401  (the profiler)
    import numpy as np
    from badread_b200.engine import Engine, FastaFile
    eng = Engine(device=0, seed=0)
    ctx = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as tprofile
        ctx = tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
        ctx.__enter__()
    res = {'route': route}
    t0 = time.perf_counter()
    if route == 'host':   # the route before the device inflater: Python's gzip, then the device parse of the text
        import gzip
        with open(path, 'rb') as f:
            text = gzip.decompress(f.read())
        res['host_inflate_s'] = time.perf_counter() - t0
        fasta = FastaFile.__new__(FastaFile)
        fasta._lib, fasta._pinned, fasta.gzip, fasta.data = None, None, False, np.frombuffer(text, np.uint8)
    else:
        fasta = FastaFile(path)
    res['file_s'] = time.perf_counter() - t0
    table = eng.load_fasta(fasta)
    res['wall_s'] = time.perf_counter() - t0
    fasta.close()
    if ctx is not None:
        ctx.__exit__(None, None, None)
        res['kernels_ms'] = _kernel_times(ctx)
    res['bases'] = int(sum(table[1]))
    res['stats'] = eng.last_gzip_stats()
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--contigs', type=int, default=24)
    ap.add_argument('--contig_mb', type=float, default=125)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None, help='directory for the reference files (default: a temporary one)')
    ap.add_argument('--sweep', default=None, help='chunk sizes in KiB, comma-separated: the inflater alone at each')
    ap.add_argument('--lib', action='append', default=None, help='with --sweep: a library build to sweep (repeatable)')
    ap.add_argument('--leg', nargs=3, default=None, help=argparse.SUPPRESS)
    ap.add_argument('--sweep_leg', nargs=3, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.leg:
        print(json.dumps(leg(a.leg[0], a.leg[1], a.leg[2] == '1')))
        return
    if a.sweep_leg:
        print(json.dumps(sweep_leg(a.sweep_leg[0], a.sweep_leg[1], int(a.sweep_leg[2]))))
        return
    from bench_reference_load import write_reference
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory(dir=a.out) as tmp:
        plain, bz, gz = (os.path.join(tmp, n) for n in ('ref.fa', 'ref.bgzf.fa.gz', 'ref.fa.gz'))
        write_reference(plain, bz, a.contigs, int(a.contig_mb * 1e6))
        t0 = time.perf_counter()
        write_gzip(plain, gz, a.contigs)
        result = {'gpu': gpu[0] if gpu else None, 'contigs': a.contigs, 'contig_bases': int(a.contig_mb * 1e6),
                  'plain_bytes': os.path.getsize(plain), 'gzip_bytes': os.path.getsize(gz), 'bgzf_bytes': os.path.getsize(bz),
                  'gzip_write_s': time.perf_counter() - t0, 'legs': []}
        os.unlink(plain)
        if a.sweep:
            for lib in a.lib or ['-']:
                for kib in (int(x) for x in a.sweep.split(',')):
                    p = subprocess.run([sys.executable, __file__, '--sweep_leg', lib, gz, str(kib)], cwd=ROOT,
                                       capture_output=True, text=True)
                    result['legs'].append(json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else
                                          {'lib': lib, 'chunk_kib': kib, 'error': p.stderr[-2000:]})
            print(json.dumps(result))
            return
        routes = (('host', gz), ('device', gz), ('bgzf', bz))
        for rep in range(a.reps + 1):   # the last round profiled
            for route, path in routes:
                p = subprocess.run([sys.executable, __file__, '--leg', route, path, '1' if rep == a.reps else '0'], cwd=ROOT,
                                   capture_output=True, text=True)
                r = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else {'route': route, 'error': p.stderr[-2000:]}
                r['profiled'] = rep == a.reps
                result['legs'].append(r)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
