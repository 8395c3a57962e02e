"""Loading the simulate reference: the host loader (misc.load_fasta_arrays + Engine.upload_reference) against the GPU
loader (Engine.load_fasta) on BASELINE config 4's reference, 24 contigs of 125 Mb, written as a plain FASTA of 60-column
lines and as BGZF.

Per loader and file: wall time split into file read, parse on the host, host-to-device copy, inflate kernel, parse kernels
and gather (kernel and copy times from torch.profiler's CUDA activities), and peak host RSS; each leg runs in a process
of its own.  Then the setup_s that `simulate --quantity 10000` reports for both files.  The card's name and power limit
are read in the same call.  Prints one JSON line.

    python tools/bench_reference_load.py [--contigs 24] [--contig_mb 125] [--out DIR]
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)


def write_reference(path_plain, path_bgzf, n_contigs, contig_len):
    import numpy as np
    from badread_b200.bgzf import EOF_MEMBER
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=0)
    with open(path_plain, 'wb') as fp, open(path_bgzf, 'wb') as fz:
        pending = b''
        for c in range(n_contigs):
            rs = np.random.RandomState(4000 + c)
            bases = np.frombuffer(b'ACGT', np.uint8)[rs.randint(0, 4, contig_len)]
            full = contig_len // 60 * 60
            grid = np.empty((full // 60, 61), np.uint8)
            grid[:, :60] = bases[:full].reshape(-1, 60)
            grid[:, 60] = 10
            text = grid.tobytes() + (bases[full:].tobytes() + b'\n' if contig_len > full else b'')
            text = f'>contig_{c + 1} depth=1\n'.encode() + text
            fp.write(text)
            data = pending + text
            members, used = eng.bgzf_compress(data, final=False)
            fz.write(members.tobytes())
            pending = data[used:]
        members, _ = eng.bgzf_compress(pending, final=True)
        fz.write(members.tobytes())
        fz.write(EOF_MEMBER)
    eng.close()


def _kernel_times(prof):
    """Sums of CUDA kernel and memcpy times (ms) by what they are."""
    out = {'h2d_ms': 0.0, 'inflate_kernel_ms': 0.0, 'parse_kernels_ms': 0.0, 'gather_ms': 0.0}
    for ev in prof.events():
        name = ev.name
        dev_us = getattr(ev, 'device_time', None) or getattr(ev, 'cuda_time', 0) or 0
        if ev.device_type is None or str(ev.device_type) != 'DeviceType.CUDA':
            continue
        if 'Memcpy HtoD' in name:
            out['h2d_ms'] += dev_us / 1e3
        elif 'infl_k_members' in name:
            out['inflate_kernel_ms'] += dev_us / 1e3
        elif 'fasta_k_gather' in name:
            out['gather_ms'] += dev_us / 1e3
        elif 'fasta_k_' in name:
            out['parse_kernels_ms'] += dev_us / 1e3
    return out


def leg(loader, path, profile):
    """One load in this process -> dict of times and peak RSS."""
    import torch  # noqa: F401  (the profiler)
    from badread_b200.engine import Engine, FastaFile
    eng = Engine(device=0, seed=0)
    res = {'loader': loader, 'file': os.path.basename(path)}
    ctx = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as tprofile
        ctx = tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
        ctx.__enter__()
    t0 = time.perf_counter()
    if loader == 'host':
        from badread_b200.misc import load_fasta_arrays
        import numpy as np
        t_read = time.perf_counter()
        names, arrays, *_ = load_fasta_arrays(path)   # reads (and inflates) the file and parses it
        concat = np.concatenate(arrays)
        res['read_and_parse_s'] = time.perf_counter() - t_read
        t_up = time.perf_counter()
        eng.upload_reference(concat)
        res['upload_s'] = time.perf_counter() - t_up
        n = concat.size
    else:
        t_read = time.perf_counter()
        fasta = FastaFile(path)
        res['file_read_s'] = time.perf_counter() - t_read
        t_up = time.perf_counter()
        table = eng.load_fasta(fasta)
        fasta.close()
        res['device_load_s'] = time.perf_counter() - t_up
        n = sum(table[1])
    res['wall_s'] = time.perf_counter() - t0
    if ctx is not None:
        ctx.__exit__(None, None, None)
        res.update(_kernel_times(ctx))
    res['bases'] = int(n)
    res['peak_rss_gb'] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    eng.close()
    return res


def setup_s(path):
    env = dict(os.environ, BADREAD_B200_TIMING='1')
    argv = [sys.executable, '-m', 'badread_b200', 'simulate', '--reference', path, '--quantity', '10000', '--seed', '1']
    p = subprocess.run(argv, cwd=ROOT, env=env, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True, check=True)
    line = [x for x in p.stderr.splitlines() if x.startswith('BADREAD_B200_TIMING ')][-1]
    return json.loads(line.split(' ', 1)[1])['setup_s']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--contigs', type=int, default=24)
    ap.add_argument('--contig_mb', type=float, default=125)
    ap.add_argument('--out', default=None, help='directory for the two reference files (default: a temporary one)')
    ap.add_argument('--leg', nargs=3, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.leg:
        print(json.dumps(leg(a.leg[0], a.leg[1], a.leg[2] == '1')))
        return
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory(dir=a.out) as tmp:
        plain, bz = os.path.join(tmp, 'ref.fa'), os.path.join(tmp, 'ref.fa.gz')
        t0 = time.perf_counter()
        write_reference(plain, bz, a.contigs, int(a.contig_mb * 1e6))
        result = {'gpu': gpu[0] if gpu else None, 'contigs': a.contigs, 'contig_bases': int(a.contig_mb * 1e6),
                  'plain_bytes': os.path.getsize(plain), 'bgzf_bytes': os.path.getsize(bz),
                  'write_s': time.perf_counter() - t0, 'legs': []}
        for loader in ('host', 'device'):
            for path in (plain, bz):
                for profile in (False, True):   # wall times without the profiler; kernel times from a profiled run
                    p = subprocess.run([sys.executable, __file__, '--leg', loader, path, '1' if profile else '0'], cwd=ROOT,
                                       capture_output=True, text=True)
                    r = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else \
                        {'loader': loader, 'file': os.path.basename(path), 'error': p.stderr[-2000:]}
                    r['profiled'] = profile
                    result['legs'].append(r)
        result['setup_s'] = {'plain': setup_s(plain), 'bgzf': setup_s(bz)}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
