#!/usr/bin/env python3
"""
BGZF output (`simulate --gzip`) on one GPU, config 1 of bench.py (5 Mb circular reference, 50x, nanopore2023):
  * the card's name and power limit;
  * the compressor on config 1's FASTQ: kernel time (torch.profiler, CUDA activities, in a run of its own), and the whole
    Engine.bgzf_compress call with the host-to-device copy of the FASTQ and the device-to-host copy of the members;
  * the compression ratio against zlib levels 1 and 6 on the same 65 280-byte chunks of a prefix of that FASTQ, zlib timed
    on one thread of this host;
  * the wall time of `python -m badread_b200 simulate` for config 1 to /dev/null, with and without --gzip, alternating.
Prints one JSON line.  Usage: tools/bench_bgzf.py [--repeats R] [--zlib-mb M]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')

import bench  # noqa: E402

CHUNK = 65280


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi failed: {q.stderr.strip()[:200]}'


def simulate(fasta, out_path, gz, cfg):
    argv = [sys.executable, '-m', 'badread_b200', 'simulate', '--reference', fasta, '--quantity', cfg['quantity'],
            '--seed', str(bench.SEED)] + cfg['extra'] + (['--gzip'] if gz else [])
    env = dict(os.environ, BADREAD_B200_TIMING='1', PYTHONPATH=os.pathsep.join([ROOT, os.environ.get('PYTHONPATH', '')]))
    t0 = time.perf_counter()
    with open(out_path, 'wb') as out:
        p = subprocess.run(argv, env=env, stdout=out, stderr=subprocess.PIPE, timeout=600)
    wall = time.perf_counter() - t0
    if p.returncode:
        raise RuntimeError(p.stderr.decode(errors='replace')[-500:])
    line = [ln for ln in p.stderr.decode(errors='replace').splitlines() if ln.startswith('BADREAD_B200_TIMING ')][-1]
    st = json.loads(line.split(' ', 1)[1])
    return {'process_wall_s': wall, 'simulate_loop_s': st['batches_s'], 'bases': st['bases']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--zlib-mb', type=int, default=64, help='prefix of the FASTQ that zlib compresses (MB)')
    a = ap.parse_args()
    cfg = bench.CONFIGS[1]
    res = {'card': card(), 'config': cfg['label']}
    tmp = tempfile.mkdtemp()
    fasta, fastq = os.path.join(tmp, 'ref.fasta'), os.path.join(tmp, 'reads.fastq')
    with open(fasta, 'wb') as f:
        for name, n, seed, depth, circ in cfg['contigs']:
            hdr = f'>{name}' + (f' depth={depth:g}' if depth != 1.0 else '') + (' circular=true' if circ else '')
            f.write(hdr.encode() + b'\n' + bench._synth_contig(seed, n).tobytes() + b'\n')

    # the FASTQ itself (also the first, untimed run: caches warm)
    simulate(fasta, fastq, False, cfg)
    with open(fastq, 'rb') as f:
        data = f.read()
    res['fastq_bytes'] = len(data)

    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=1)
    comp, _ = eng.bgzf_compress(data, 0, final=True)   # warm-up: scratch, pinned buffer, modules
    comp = bytes(comp)
    calls = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        eng.bgzf_compress(data, 0, final=True)
        calls.append(time.perf_counter() - t0)
    res['compressed_bytes'] = len(comp)
    res['ratio'] = len(data) / len(comp)
    res['call_s'] = calls
    res['call_GB_per_s'] = len(data) / min(calls) / 1e9

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.bgzf_compress(data, 0, final=True)
        torch.cuda.synchronize()
    kernels, copies = {}, {}
    for ev in prof.events():
        name = ev.name
        dt = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        if 'bgzf_k_' in name:   # (mangled or not: bgzf_k_compress, bgzf_k_lines, bgzf_k_scan, bgzf_k_pack)
            key = name[name.index('bgzf_k_'):].split('(')[0].split('P')[0]
            kernels[key] = kernels.get(key, 0.0) + dt / 1e3
        elif 'Memcpy' in name or 'memcpy' in name:
            copies[name] = copies.get(name, 0.0) + dt / 1e3
    res['kernel_ms'] = kernels
    res['copy_ms'] = copies
    k_total = sum(kernels.values())
    res['kernel_GB_per_s'] = len(data) / (k_total / 1e3) / 1e9 if k_total else None
    eng.close()

    # zlib on this host, the same chunks of a prefix
    pre = data[:a.zlib_mb << 20]
    zl = {}
    for level in (1, 6):
        t0 = time.perf_counter()
        size = sum(len(zlib.compress(pre[i:i + CHUNK], level)) - 6 + 26 for i in range(0, len(pre), CHUNK))
        zl[f'level{level}'] = {'ratio': len(pre) / size, 'MB_per_s_one_thread': len(pre) / (time.perf_counter() - t0) / 1e6}
    eng2 = Engine(device=0, seed=1)
    res['ratio_on_zlib_prefix'] = len(pre) / len(bytes(eng2.bgzf_compress(pre, 0, final=True)[0]))
    eng2.close()
    res['zlib'] = zl
    res['zlib_prefix_bytes'] = len(pre)

    # the command line to /dev/null, alternating
    runs = {'plain': [], 'gzip': []}
    for _ in range(a.repeats):
        for gz in (False, True):
            runs['gzip' if gz else 'plain'].append(simulate(fasta, os.devnull, gz, cfg))
    res['simulate'] = runs
    for p in (fasta, fastq):
        os.unlink(p)
    os.rmdir(tmp)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
