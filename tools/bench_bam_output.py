#!/usr/bin/env python3
"""
BAM output (`simulate --bam`) on one GPU, config 1 of bench.py (5 Mb circular reference, 50x, nanopore2023):
  * the card's name and power limit;
  * the wall time of the simulate loop (`python -m badread_b200 simulate`, BADREAD_B200_TIMING) plain, with --gzip and
    with --bam, alternating, each writing its file to a temporary directory;
  * the sizes of the three files and the bytes that cross PCIe on each path;
  * the record kernel and the compressor's kernels (torch.profiler, CUDA activities) over a whole --bam run in this
    process;
  * ptxas's resource lines of the new kernels, from the build's logs.
Prints one JSON line.  Usage: tools/bench_bam_output.py [--repeats R]
"""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')

import bench  # noqa: E402

MODES = {'plain': [], 'gzip': ['--gzip'], 'bam': ['--bam']}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    return q.stdout.strip() if q.returncode == 0 else f'nvidia-smi failed: {q.stderr.strip()[:200]}'


def argv_of(fasta, cfg, mode):
    return ['simulate', '--reference', fasta, '--quantity', cfg['quantity'], '--seed', str(bench.SEED)] + cfg['extra'] + \
        MODES[mode]


def simulate(fasta, out_path, mode, cfg):
    env = dict(os.environ, BADREAD_B200_TIMING='1', PYTHONPATH=os.pathsep.join([ROOT, os.environ.get('PYTHONPATH', '')]))
    t0 = time.perf_counter()
    with open(out_path, 'wb') as out:
        p = subprocess.run([sys.executable, '-m', 'badread_b200'] + argv_of(fasta, cfg, mode), env=env, stdout=out,
                           stderr=subprocess.PIPE, timeout=900)
    wall = time.perf_counter() - t0
    if p.returncode:
        raise RuntimeError(p.stderr.decode(errors='replace')[-500:])
    line = [ln for ln in p.stderr.decode(errors='replace').splitlines() if ln.startswith('BADREAD_B200_TIMING ')][-1]
    st = json.loads(line.split(' ', 1)[1])
    return {'process_wall_s': round(wall, 3), 'simulate_loop_s': round(st['batches_s'], 3), 'reads': st['reads'],
            'bases': st['bases']}


def profile_bam(fasta, cfg):
    """Kernel and copy times of a whole --bam run in this process."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from badread_b200.__main__ import check_simulate_args, parse_args
    from badread_b200.simulate import simulate as run
    torch.cuda.init()
    args = parse_args(argv_of(fasta, cfg, 'bam'))
    check_simulate_args(args)
    sink = io.BytesIO()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(args, output=io.StringIO(), stdout=sink)
        torch.cuda.synchronize()
    kernels, copies = {}, {}
    for ev in prof.events():
        name = ev.name
        dt = (ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total) / 1e3
        for k in ('bam_k_records', 'bgzf_k_compress_bam', 'bgzf_k_scan', 'bgzf_k_pack'):
            if k in name:
                kernels[k] = kernels.get(k, 0.0) + dt
        if 'Memcpy' in name or 'memcpy' in name:
            copies[name] = copies.get(name, 0.0) + dt
    return {'kernel_ms': {k: round(v, 3) for k, v in kernels.items()},
            'copy_ms': {k: round(v, 3) for k, v in sorted(copies.items(), key=lambda x: -x[1])[:6]},
            'bam_bytes': len(sink.getvalue())}


def ptxas_lines():
    out = {}
    for log in ('bb_tu_bam_out', 'bb_tu_bgzf'):
        path = os.path.join(ROOT, 'badread_b200', 'csrc', 'build', log + '.ptxas.log')
        if not os.path.isfile(path):
            continue
        name = None
        for ln in open(path):
            m = re.search(r"Compiling entry function '(\w+)'", ln)
            if m:
                name = m.group(1)
            elif name and ('bam' in name) and ('Used' in ln or 'spill' in ln):
                out.setdefault(name, []).append(ln.split(':', 1)[-1].strip())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    cfg = bench.CONFIGS[1]
    res = {'card': card(), 'config': cfg['label']}
    tmp = tempfile.mkdtemp()
    fasta = os.path.join(tmp, 'ref.fasta')
    with open(fasta, 'wb') as f:
        for name, n, seed, depth, circ in cfg['contigs']:
            hdr = f'>{name}' + (f' depth={depth:g}' if depth != 1.0 else '') + (' circular=true' if circ else '')
            f.write(hdr.encode() + b'\n' + bench._synth_contig(seed, n).tobytes() + b'\n')

    # one untimed run of each (caches warm), keeping the files for their sizes
    sizes = {}
    for mode in MODES:
        path = os.path.join(tmp, 'out.' + mode)
        first = simulate(fasta, path, mode, cfg)
        sizes[mode] = os.path.getsize(path)
        os.unlink(path)
    res['reads'], res['bases'] = first['reads'], first['bases']
    res['bytes'] = sizes
    res['bam_over_gzip'] = round(sizes['bam'] / sizes['gzip'], 4)
    n = first['reads']
    fastq_headers = sizes['plain'] - 2 * first['bases'] - 4 * n   # '@', '\n', '+\n', '\n' and the header text
    # bytes over PCIe: plain and --gzip copy the bases and qualities down (2 per base); --gzip copies the FASTQ back up
    # and its members down; --bam (one GPU) uploads a 32-byte record descriptor, an 8-byte position and the name and CO
    # text per read (about the FASTQ header text) and copies the members down.  Descriptors of the batches are the same.
    res['pcie_bytes'] = {'plain': 2 * first['bases'], 'gzip': 2 * first['bases'] + sizes['plain'] + sizes['gzip'],
                         'bam': 40 * n + fastq_headers + sizes['bam']}

    runs = {m: [] for m in MODES}
    for _ in range(a.repeats):
        for mode in MODES:
            runs[mode].append(simulate(fasta, os.path.join(tmp, 'out.' + mode), mode, cfg))
            os.unlink(os.path.join(tmp, 'out.' + mode))
    res['simulate'] = runs
    res['simulate_loop_s'] = {m: [r['simulate_loop_s'] for r in v] for m, v in runs.items()}
    res['profile_bam'] = profile_bam(fasta, cfg)
    res['ptxas'] = ptxas_lines()
    os.unlink(fasta)
    os.rmdir(tmp)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
