#!/usr/bin/env python3
"""
bench.py - simulated Gbases/s of the Badread error-injection hot path on H100 (BASELINE.json metric).

A "step" is one pass of the hot path (sequence_fragment for every read of the workload).  `--config N` selects
BASELINE.json configs[N]; the default, N = 1, is the configuration the metric is quoted on:
  1  5 Mb synthetic circular reference (RandomState(1001)), 50x, nanopore2023 error + qscore models, all defaults
     (~16.4 k reads, ~248 Mbases per step)
  2  same reference, 200x, nanopore2020 models, --identity 90,98,5 --glitches 1000,100,100  (~66 k reads, ~1 Gbase)
  3  100 Mb: 10 linear contigs + 3 circular plasmids, 50x, pacbio2021 models, --chimeras 10  (~5 Gbases, split over N)
  4  3 Gb: 24 linear contigs, 30x, nanopore2023, --length 40000,20000                     (~90 Gbases, split over N)

  value     whole-job Gbases/s with the reference, the model tables and the fragment descriptors resident in HBM
            (bb_batch_run only; with several batches per step the descriptor upload and the fetch of each batch sit
            outside the timed spans)
  e2e       the same through bb_sequence_batch with HOST buffers: descriptor H2D + seq/qual D2H inside the timing
  roofline  dominant stage: algorithmic bytes per emitted base / its CUDA-event duration, against the measured HBM copy
            peak (MEASURED_PEAKS.json); DRAM traffic and instruction counts come from the newest ncu pass committed
            under profiles/ (tools/profile_step.sh)
  parity    the GPU reads of the timed workload against the CPU oracle for the same read indices: the whole workload
            for configs 1-2, the first 10 000 read indices for configs 3-4 (SURVEY.md 8d); a mismatch fails the run
  cpu_baseline  the CPU oracle port (oracle/badread_oracle.c, Philox mode, pthreads over reads) on those same reads
  --impl reference   times only that CPU port on all host threads (the reference is pure Python + an un-vendored edlib;
            its C restatement is pinned byte-for-byte to it in tests/)
  --dump-outputs DIR   after the timed steps, writes what the last timed step returned for a fixed, seeded sample of its
            reads (rank 0): DIR/read_index.npy, one DIR/<field>.npy per record field and the reads' sequence and quality
            bytes concatenated in DIR/seq.npy / DIR/qual.npy (float64 / float32, under 64 MB in all), so that two builds
            can be compared output for output

Multi-GPU (torchrun, one rank per GPU): reads shard by index (rank g owns indices g, g+N, ...), no data-path
collective; the collectives are the barrier, the SUM of emitted bases / mismatches and the MAX of elapsed time (NCCL).
`--scaling weak` (default for configs 1-2): every rank processes a full config-sized share; `--scaling strong`
(default for configs 3-4, which BASELINE.json defines as sharded jobs): the one job is split over the N GPUs.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, ROOT)
os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')   # before torch / the library initialize CUDA (see _lib.py)

SEED = 1
PARITY_PREFIX = 10000   # SURVEY.md 8d: first 10 000 read indices for the sharded configs

_ACGT = np.frombuffer(b'ACGT', dtype=np.uint8)


def log(*a):
    print(*a, file=sys.stderr, flush=True)


# ------------------------------------------------------------------------------------------------ workloads
def _synth_contig(seed, n):
    """RandomState(seed).randint(0, 4, n) -> ACGT, in chunks (identical stream, bounded memory)."""
    rs = np.random.RandomState(seed)
    out = np.empty(n, dtype=np.uint8)
    step = 1 << 24
    for lo in range(0, n, step):
        hi = min(n, lo + step)
        out[lo:hi] = _ACGT[rs.randint(0, 4, hi - lo)]
    return out


CONFIGS = {
    1: {'label': 'BASELINE.json configs[1]: 5 Mb synthetic circular ref (RandomState(1001)), 50x, nanopore2023 '
                 'error+qscore, default identity/length/adapters/glitches, seed 1',
        'contigs': [('chr1', 5_000_000, 1001, 1.0, True)], 'quantity': '50x',
        'extra': ['--error_model', 'nanopore2023', '--qscore_model', 'nanopore2023'], 'scaling': 'weak', 'parity': 'full'},
    2: {'label': 'BASELINE.json configs[2]: 5 Mb synthetic circular ref (RandomState(1001)), 200x, nanopore2020 '
                 'error+qscore, identity 90,98,5, glitches 1000,100,100, seed 1',
        'contigs': [('chr1', 5_000_000, 1001, 1.0, True)], 'quantity': '200x',
        'extra': ['--error_model', 'nanopore2020', '--qscore_model', 'nanopore2020', '--identity', '90,98,5',
                  '--glitches', '1000,100,100'], 'scaling': 'weak', 'parity': 'full'},
    3: {'label': 'BASELINE.json configs[3]: 100 Mb synthetic ref (10 linear contigs x 9.95 Mb RandomState(2001+i), '
                 'circular plasmids 300 kb depth=2, 150 kb depth=5, 50 kb depth=10), 50x, pacbio2021, chimeras 10, seed 1',
        'contigs': [(f'contig{i + 1}', 9_950_000, 2001 + i, 1.0, False) for i in range(10)] +
                   [('plasmid1', 300_000, 2011, 2.0, True), ('plasmid2', 150_000, 2012, 5.0, True),
                    ('plasmid3', 50_000, 2013, 10.0, True)], 'quantity': '50x',
        'extra': ['--error_model', 'pacbio2021', '--qscore_model', 'pacbio2021', '--chimeras', '10'],
        'scaling': 'strong', 'parity': 'prefix'},
    4: {'label': 'BASELINE.json configs[4]: 3 Gb synthetic ref (24 linear contigs x 125 Mb RandomState(3001+i)), 30x, '
                 'nanopore2023, length 40000,20000, seed 1',
        'contigs': [(f'chr{i + 1}', 125_000_000, 3001 + i, 1.0, False) for i in range(24)], 'quantity': '30x',
        'extra': ['--error_model', 'nanopore2023', '--qscore_model', 'nanopore2023', '--length', '40000,20000'],
        'scaling': 'strong', 'parity': 'prefix'},
}


class SynthReference(object):
    """The attributes of simulate.Reference, built in memory (no FASTA round trip for a 3 Gb reference)."""

    def __init__(self, contigs):
        self.names = [c[0] for c in contigs]
        self.lengths = [int(c[1]) for c in contigs]
        self.depths = [float(c[3]) for c in contigs]
        self.circular = [bool(c[4]) for c in contigs]
        self.left_hairpin = [False] * len(contigs)
        self.right_hairpin = [False] * len(contigs)
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int64)
        self.concat = np.empty(int(self.offsets[-1]), dtype=np.uint8)
        for i, c in enumerate(contigs):
            self.concat[self.offsets[i]:self.offsets[i + 1]] = _synth_contig(c[2], int(c[1]))

    @property
    def size(self):
        return int(sum(self.lengths))


class Workload(object):
    """This rank's reads of one step, planned by the native planner and cut into batches."""

    def __init__(self, cfg_id, rank, world, scaling, max_reads=None, batch_reads=32768, threads=None):
        from badread_b200 import simulate as S
        from badread_b200.__main__ import check_simulate_args, parse_args
        from badread_b200.error_model import ErrorModel
        from badread_b200.fragment_lengths import FragmentLengths
        from badread_b200.identities import Identities
        from badread_b200.planner import NativePlanner
        from badread_b200.qscore_model import QScoreModel
        cfg = CONFIGS[cfg_id]
        self.cfg, self.rank, self.world = cfg, rank, world
        t0 = time.perf_counter()
        self.ref = SynthReference(cfg['contigs'])
        t_ref = time.perf_counter() - t0
        fd, placeholder = tempfile.mkstemp(suffix='.fasta')   # only so that the CLI's argument checks see a file
        os.write(fd, b'>placeholder\nACGT\n')
        os.close(fd)
        args = parse_args(['simulate', '--reference', placeholder, '--quantity', cfg['quantity'], '--seed', str(SEED)] +
                          cfg['extra'])
        check_simulate_args(args)
        os.unlink(placeholder)
        sink = io.StringIO()
        fl = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, sink)
        S.adjust_depths(self.ref, fl, args, np.random.RandomState(SEED))
        ids = Identities(args.mean_identity, args.identity_stdev, args.max_identity, sink)
        self.models = (ErrorModel(args.error_model, sink), QScoreModel(args.qscore_model, sink))
        self.planner = NativePlanner(args, self.ref, fl, ids, SEED, n_threads=threads)
        target = S.get_target_size(self.ref.size, args.quantity)
        # weak: this rank plans until ITS error-free total reaches the whole job's target (every rank = one full
        # config-sized share); strong: until it reaches target / world (the one job split over the ranks).  Reads
        # come out ~1 % shorter or longer than their fragments, so these are the job's read counts to within that.
        my_target = target if scaling == 'weak' else (target + world - 1) // world
        t0 = time.perf_counter()
        self.batches, self.n_reads, self.frag_bases = [], 0, 0
        i = 0
        chunk = max(256, min(batch_reads, int(my_target / max(1.0, float(args.mean_frag_length)) * 1.02) + 64))
        while self.frag_bases < my_target and (max_reads is None or self.n_reads < max_reads):
            n = min(chunk, batch_reads)
            if max_reads is not None:
                n = min(n, max_reads - self.n_reads)
            pb = self.planner.plan(rank + world * i, n, stride=world)
            cum = np.cumsum(pb.frag_len.astype(np.int64))
            need = my_target - self.frag_bases
            keep = n if cum[-1] < need else int(np.searchsorted(cum, need) + 1)
            if keep < n:
                pb = self.planner.plan(rank + world * i, keep, stride=world)
            self.batches.append(pb.detach())
            self.n_reads += keep
            self.frag_bases += int(cum[keep - 1])
            i += keep
        self.t_plan = time.perf_counter() - t0
        self.target = target
        log(f'[rank {rank}] reference built in {t_ref:.1f} s; planned {self.n_reads} reads ({self.frag_bases} fragment '
            f'bases, {len(self.batches)} batch(es)) in {self.t_plan:.2f} s with the native planner')

    def h2d_bytes(self):
        return sum(b.h2d_bytes() for b in self.batches)

    def prefix_reads(self, limit):
        """(batch, position) of this rank's reads with global index < limit (None: all)."""
        out = []
        for bi, b in enumerate(self.batches):
            idx = b.read_index
            sel = np.arange(len(b)) if limit is None else np.nonzero(idx < limit)[0]
            out += [(bi, int(j)) for j in sel]
        return out


# ------------------------------------------------------------------------------------------------ measurement helpers
class ClockSampler(object):
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, device):
        self.device = device
        self.proc = None
        self.path = None

    def start(self):
        try:
            fd, self.path = tempfile.mkstemp(suffix='.csv')
            os.close(fd)
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.device), f'--query-gpu={self.Q}',
                                          '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=open(self.path, 'w'), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        out = {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': []}
        if self.proc is None:
            return out
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, reasons, mx = [], set(), None
        try:
            for line in open(self.path):
                parts = [x.strip() for x in line.split(',')]
                if len(parts) < 9:
                    continue
                try:
                    sm.append(float(parts[1]))
                    mx = float(parts[2])
                except ValueError:
                    continue
                for name, val in zip(('hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap'), parts[5:9]):
                    if val.lower() == 'active':
                        reasons.add(name)
            os.unlink(self.path)
        except Exception:
            pass
        if sm:
            out['sm_mhz'] = float(np.median(sm))
            out['sm_max_mhz'] = mx
            out['samples'] = len(sm)
        out['reasons'] = sorted(reasons)
        return out


def cpu_port_run(wl, picks, n_threads):
    """Runs the CPU oracle port (Philox mode, pthreads over reads) over the reads `picks` = [(batch, position)].
    Returns (outputs, bases, seconds); outputs[i] = (seq, qual, matches, columns)."""
    from oracle import oracle as O
    orc = O.Oracle(*wl.models)
    frs = [wl.batches[b].fragment(j, wl.ref.concat) for b, j in picks]
    ids = [float(wl.batches[b].target_identity[j]) for b, j in picks]
    idx = [int(wl.batches[b].read_index[j]) for b, j in picks]
    t0 = time.perf_counter()
    outs, bases = orc.sequence_batch(frs, ids, SEED, idx, n_threads=n_threads)
    return outs, bases, time.perf_counter() - t0


def algorithmic_warp_inst(block_steps):
    """Integer work the path needs, as warp instructions: the oracle counts the 64-row block updates of the passes a path
    needs (both passes of every Hirschberg node, the history pass of every leaf and of every identity re-measurement,
    bands from exact scores; not the distance search in front).  One 64-row update = two 32-row word updates of ~13
    integer operations each (Myers / Hyyro: 8 logic, 1 add, 2 shifts, 2 for the carries), 32 lanes per warp instruction."""
    return block_steps * 2 * 13 / 32.0


def parity_check(res, picks, outs):
    """GPU reads of one batch (BatchResult) against the oracle's for the same read indices: sequences, quality strings,
    alignment counts.  Returns the mismatching picks."""
    bad = []
    for (b, j), o in zip(picks, outs):
        rec = res.records[j]
        if res.read(j) != (o[0], o[1]) or (rec.matches, rec.columns) != (o[2], o[3]):
            bad.append((b, j))
    return bad


class OutputSample(object):
    """--dump-outputs: a fixed sample of this rank's reads (RandomState(SEED) over the planned reads, at most 4096 reads
    and about 6 Mbases of fragments) as the timed path returns them in a BatchResult: the record fields that do not
    depend on timing or on the layout of the output buffers, and the sequence and quality bytes."""
    FIELDS = ('out_len', 'frag_len', 'matches', 'columns', 'loop_count', 'change_count', 'n_alignments', 'flags')
    MAX_BYTES = 64 << 20

    def __init__(self, wl, max_reads=4096, max_frag_bases=6_000_000):
        every = [(b, j) for b, batch in enumerate(wl.batches) for j in range(len(batch))]
        self.want, bases = {}, 0
        for k in np.random.RandomState(SEED).permutation(len(every))[:max_reads]:
            b, j = every[k]
            bases += int(wl.batches[b].frag_len[j])
            if bases > max_frag_bases:
                break
            self.want.setdefault(b, []).append(j)
        self.got = {}

    def take(self, bi, res, read_index):
        """Copies the wanted reads of batch `bi` out of `res` (its buffers are reused by the next fetch)."""
        for j in self.want.get(bi, ()):
            rec = res.records[j]
            seq, qual = res.read(j)
            self.got[int(read_index[j])] = ([float(getattr(rec, f)) for f in self.FIELDS], seq, qual)

    def write(self, d):
        os.makedirs(d, exist_ok=True)
        idx = sorted(self.got)
        fields = np.array([self.got[i][0] for i in idx], dtype=np.float64).reshape(len(idx), len(self.FIELDS))
        seq = np.frombuffer(''.join(self.got[i][1] for i in idx).encode('latin-1'), dtype=np.uint8).astype(np.float32)
        qual = np.frombuffer(''.join(self.got[i][2] for i in idx).encode('latin-1'), dtype=np.uint8).astype(np.float32)
        assert seq.nbytes + qual.nbytes + fields.nbytes + 8 * len(idx) < self.MAX_BYTES, 'output sample too large'
        np.save(os.path.join(d, 'read_index.npy'), np.array(idx, dtype=np.float64))
        for k, f in enumerate(self.FIELDS):
            np.save(os.path.join(d, f'{f}.npy'), fields[:, k])
        np.save(os.path.join(d, 'seq.npy'), seq)
        np.save(os.path.join(d, 'qual.npy'), qual)
        return len(idx), int(seq.size)


def reference_shim_rate(cfg, n_procs, quantity_bases):
    """BASELINE.md's primary CPU baseline: the UNMODIFIED reference (`badread.simulate.simulate`, copied into oracle/_ref
    by `make -C oracle ref`) with `edlib` provided by oracle/edlib_shim (the oracle's aligner; the real wheel
    is absent), run the way its README recommends for parallelism: n independent processes with --quantity target/n and
    different seeds.  Returns the cpu_baseline-style object, or None with a reason."""
    ref_dir = os.path.join(ROOT, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref_dir, 'badread')):
        return {'value': None, 'kind': 'reference', 'sample': 'oracle/_ref is not installed'}
    try:
        fd, fasta = tempfile.mkstemp(suffix='.fasta')
        with os.fdopen(fd, 'wb') as f:
            for name, n, seed, depth, circ in cfg['contigs']:
                hdr = f'>{name}' + (f' depth={depth:g}' if depth != 1.0 else '') + (' circular=true' if circ else '')
                f.write(hdr.encode() + b'\n' + _synth_contig(seed, n).tobytes() + b'\n')
        env = dict(os.environ)
        env['PYTHONPATH'] = os.pathsep.join([os.path.join(ROOT, 'oracle', 'edlib_shim'), ref_dir, env.get('PYTHONPATH', '')])
        for v in ('OMP_NUM_THREADS', 'OPENBLAS_NUM_THREADS', 'MKL_NUM_THREADS'):
            env[v] = '1'   # one thread per reference process (numpy would start a pool per process)
        runner = ('import sys\nfrom badread.__main__ import main\nmain()\n')
        t0 = time.perf_counter()
        procs = []
        for i in range(n_procs):
            argv = [sys.executable, '-c', runner, 'simulate', '--reference', fasta, '--quantity', str(quantity_bases),
                    '--seed', str(SEED + i)] + cfg['extra']
            procs.append(subprocess.Popen(argv, env=env, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL))
        bases = 0
        deadline = t0 + 180.0   # a reported baseline must not hold the bench up
        try:
            for p in procs:
                out, _ = p.communicate(timeout=max(1.0, deadline - time.perf_counter()))
                if p.returncode != 0:
                    raise RuntimeError(f'reference process exited with {p.returncode}')
                lines = out.split(b'\n')
                bases += sum(len(lines[j]) for j in range(1, len(lines), 4))
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
            os.unlink(fasta)
        dt = time.perf_counter() - t0
        return {'value': bases / dt / 1e9, 'unit': 'Gbases/s', 'cores': n_procs, 'kind': 'reference',
                'sample': f'unmodified badread.simulate (oracle/_ref) + oracle/edlib_shim: {n_procs} processes x --quantity '
                          f'{quantity_bases} with seeds {SEED}..{SEED + n_procs - 1}, {bases} bases in {dt:.1f} s wall of the '
                          f'slowest (model loading, ~3 s per process, included)'}
    except Exception as e:   # a reported baseline, never a reason to fail the bench
        return {'value': None, 'kind': 'reference', 'sample': f'failed: {e}'}


def cli_e2e(cfg, n_gpus=1):
    """The real command line end to end: `python -m badread_b200 simulate ...` on the config's reference written as FASTA,
    FASTQ to /dev/null.  Returns wall seconds of the whole process and of its simulate loop (planning + GPU + FASTQ
    assembly + write; engines, reference and tables already resident), as the tool itself reports them."""
    try:
        fd, fasta = tempfile.mkstemp(suffix='.fasta')
        with os.fdopen(fd, 'wb') as f:
            for name, n, seed, depth, circ in cfg['contigs']:
                hdr = f'>{name}' + (f' depth={depth:g}' if depth != 1.0 else '') + (' circular=true' if circ else '')
                f.write(hdr.encode() + b'\n' + _synth_contig(seed, n).tobytes() + b'\n')
        env = dict(os.environ)
        env['BADREAD_B200_TIMING'] = '1'
        env['PYTHONPATH'] = os.pathsep.join([ROOT, env.get('PYTHONPATH', '')])
        argv = [sys.executable, '-m', 'badread_b200', 'simulate', '--reference', fasta, '--quantity', cfg['quantity'],
                '--seed', str(SEED), '--gpus', str(n_gpus)] + cfg['extra']
        t0 = time.perf_counter()
        with open(os.devnull, 'wb') as null:
            p = subprocess.run(argv, env=env, stdout=null, stderr=subprocess.PIPE, timeout=240)
        wall = time.perf_counter() - t0
        os.unlink(fasta)
        if p.returncode != 0:
            return {'value': None, 'note': f'exit code {p.returncode}: {p.stderr.decode(errors="replace")[-300:]}'}
        line = [ln for ln in p.stderr.decode(errors='replace').splitlines() if ln.startswith('BADREAD_B200_TIMING ')][-1]
        st = json.loads(line.split(' ', 1)[1])
        return {'value': st['bases'] / st['batches_s'] / 1e9, 'unit': 'Gbases/s', 'gpus': n_gpus, 'reads': st['reads'],
                'bases': st['bases'], 'simulate_loop_s': st['batches_s'], 'process_wall_s': wall, 'setup_s': st['setup_s'],
                'nccl_stop_condition': st.get('nccl_stop_condition'),
                'note': '`python -m badread_b200 simulate` > /dev/null; value = bases / simulate loop (native planner + '
                        'bb_sequence_batch + FASTQ assembly + write), models, reference and engines resident'}
    except Exception as e:
        return {'value': None, 'note': f'failed: {e}'}


def peaks():
    path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    try:
        with open(path) as f:
            return float(json.load(f)['hbm_gbs']), 'measured (MEASURED_PEAKS.json hbm_gbs)'
    except Exception:
        return 3350.0, 'not measured: H100 SXM data sheet, 3.35 TB/s'


def newest_profile(suffix):
    """profiles/<tag>_<suffix>.json with the highest tag (r1c < r2a < r2b ...), written by tools/profile_step.sh."""
    d = os.path.join(ROOT, 'profiles')
    try:
        names = sorted(n for n in os.listdir(d) if n.endswith(f'_{suffix}.json'))
    except OSError:
        return None, None
    if not names:
        return None, None
    try:
        with open(os.path.join(d, names[-1])) as f:
            return json.load(f), f'profiles/{names[-1]}'
    except Exception:
        return None, None


# ------------------------------------------------------------------------------------------------ main
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', type=str, default='b200', choices=['b200', 'reference'])
    ap.add_argument('--config', type=int, default=1, choices=sorted(CONFIGS), help='index into BASELINE.json configs')
    ap.add_argument('--scaling', type=str, default=None, choices=['weak', 'strong'])
    ap.add_argument('--reads', type=int, default=None, help='cap on the reads per rank and step (a bounded sample; stated in config)')
    ap.add_argument('--batch_reads', type=int, default=32768, help='reads per device batch')
    ap.add_argument('--profile', action='store_true', help='skip the e2e, parity and CPU legs (for runs under ncu)')
    ap.add_argument('--no_parity', action='store_true', help='skip the parity + CPU baseline leg')
    ap.add_argument('--ref_shim_bases', type=int, default=300000,
                    help='bases per process of the reference-with-shim baseline leg (0: skip it)')
    ap.add_argument('--dump-outputs', type=str, default=None, metavar='DIR',
                    help='write a fixed sample of what the last timed step returned to DIR/<name>.npy')
    a = ap.parse_args()
    if a.dump_outputs and a.impl != 'b200':
        ap.error('--dump-outputs writes the outputs of the GPU path (--impl b200)')
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    n_cores = os.cpu_count() or 1
    cfg = CONFIGS[a.config]
    scaling = a.scaling or cfg['scaling']
    config = {'workload': cfg['label'], 'sharding': f'read index mod {world}',
              'cache': 'inputs (>= 250 MB of fragments per step) exceed the 50 MB L2'}
    if a.reads is not None:
        config['sample'] = f'bounded to the first {a.reads} reads per rank and step (--reads)'
    dtype = 'u8/int32 (+f64 identity estimate)'

    if a.impl == 'reference':
        if rank != 0:
            return 0
        # the CPU port over the reads rank 0 of an N = 1 run processes per step, on all host threads
        wl = Workload(a.config, 0, 1, scaling, max_reads=a.reads, batch_reads=a.batch_reads)
        limit = None if cfg['parity'] == 'full' else PARITY_PREFIX
        picks = wl.prefix_reads(limit)
        n_warm = max(64, len(picks) // 8)
        outs, bases, dt = cpu_port_run(wl, picks[:n_warm], n_cores)   # probe (= the size of a warm-up step)
        budget = 280.0
        est_full = dt / max(1, bases) * sum(int(wl.batches[b].frag_len[j]) for b, j in picks)
        n_timed = len(picks)
        if est_full * a.steps > budget:   # keep the whole reference run within a few minutes
            n_timed = max(64, int(len(picks) * budget / (est_full * a.steps)))
        for _ in range(max(0, a.warmup - 1)):
            cpu_port_run(wl, picks[:n_warm], n_cores)
        tot_b, tot_t = 0, 0.0
        for _ in range(a.steps):
            _, bases, dt = cpu_port_run(wl, picks[:n_timed], n_cores)
            tot_b += bases
            tot_t += dt
        val = tot_b / tot_t / 1e9
        what = 'every read of the workload' if n_timed == wl.n_reads else f'the first {n_timed} of {wl.n_reads} reads of the workload'
        sample = f'{what} per step ({tot_b // max(1, a.steps)} bases, {tot_t / max(1, a.steps):.2f} s) on {n_cores} threads; ' \
                 f'warm-up steps run the first {n_warm} reads'
        line = {'impl': 'reference', 'metric': 'simulated Gbases/sec', 'value': val, 'unit': 'Gbases/s', 'n_gpus': a.gpus,
                'steps': a.steps, 'warmup': a.warmup, 'ms_per_step': tot_t / max(1, a.steps) * 1e3,
                'higher_is_better': True, 'scaling': scaling, 'vs_baseline': None, 'dtype': dtype,
                'data': 'synthetic', 'config': config,
                'cpu_baseline': {'value': val, 'unit': 'Gbases/s', 'cores': n_cores, 'kind': 'port', 'sample': sample},
                'e2e': {'value': val, 'unit': 'Gbases/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
                'gpu_launches': 0}
        print(json.dumps(line), flush=True)
        return 0

    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local_rank)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))

    from badread_b200.engine import Engine, comm_unique_id, nccl_available
    wl = Workload(a.config, rank, world, scaling, max_reads=a.reads, batch_reads=a.batch_reads,
                  threads=max(1, n_cores // world))
    eng = Engine(device=local_rank, seed=SEED)
    t0 = time.perf_counter()
    eng.upload_reference(wl.ref.concat)
    eng.set_error_model(wl.models[0])
    eng.set_qscore_model(wl.models[1])
    log(f'[rank {rank}] reference + tables uploaded in {time.perf_counter() - t0:.2f} s')
    nb = len(wl.batches)
    config['batches_per_step'] = nb
    lib_nccl = False
    if dist is not None and nccl_available():   # the library's own communicator for the SUM of emitted bases
        import torch
        box = [comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        eng.comm_init_rank(box[0], rank, world)
        lib_nccl = True

    def barrier():
        eng.synchronize()
        if dist is not None:
            dist.barrier()

    # ---- device-resident timing: bb_batch_run only
    sampler = ClockSampler(local_rank)
    stage_acc = {}
    state = {'dev_ms': 0.0, 'uploaded': False}

    sample = OutputSample(wl) if a.dump_outputs and rank == 0 else None

    def resident_step(timed, last=False):
        """One step; returns the seconds spent in bb_batch_run (+ completion) and the emitted bases (None if not fetched).
        The last timed step hands what it fetched to the output sample."""
        spent, emitted = 0.0, None
        for bi, b in enumerate(wl.batches):
            if nb > 1 or not state['uploaded']:
                eng.upload_batch(b)
                state['uploaded'] = True
            t = time.perf_counter()
            eng.run_batch()
            total_ms, stages = eng.last_run_ms()   # waits for the batch's last event
            spent += time.perf_counter() - t
            if timed:
                state['dev_ms'] += total_ms
                for k, v in stages.items():
                    stage_acc[k] = stage_acc.get(k, 0.0) + v
            if nb > 1 or not timed:
                res_b, n_b = eng.fetch_batch()
                emitted = (emitted or 0) + n_b
                if last and sample is not None:
                    sample.take(bi, res_b, b.read_index)
        return spent, emitted

    sampler.start()   # nvidia-smi needs ~0.5 s for its first sample: it runs from the warm-up steps (same load) on
    bases = 0
    for _ in range(max(1, a.warmup)):
        _, bases = resident_step(False)
    launches0 = eng.launch_count()
    barrier()
    t0 = time.perf_counter()
    run_s = 0.0
    for step in range(a.steps):
        s_, e_ = resident_step(True, last=step == a.steps - 1)
        run_s += s_
        if e_ is not None:
            bases = e_
    barrier()
    wall = time.perf_counter() - t0
    elapsed = wall if nb == 1 else run_s   # several batches: only the bb_batch_run spans count (see the docstring)
    clocks = sampler.stop()
    launches = eng.launch_count() - launches0
    if os.environ.get('BADREAD_B200_TRACE') == '1':   # diagnostics: timeline of the last timed run
        trace = os.path.join(tempfile.gettempdir(), f'trace_config{a.config}_rank{rank}.csv')
        eng.trace_dump(trace)
        log(f'[rank {rank}] launch timeline of the last timed run: {trace}')
    if sample is not None:
        if nb == 1:   # one batch: the timed runs leave their reads on the device; the last run's are fetched here
            sample.take(0, eng.fetch_batch()[0], wl.batches[0].read_index)
        n_s, b_s = sample.write(a.dump_outputs)
        log(f'[rank 0] outputs of the last timed step: {n_s} reads, {b_s} bases written to {a.dump_outputs}')
    dev_ms = state['dev_ms']

    # ---- end to end through bb_sequence_batch: host descriptors in, host seq/qual out, every step
    bases_e2e, e2e_elapsed, res = bases, float('nan'), None
    if not a.profile:
        eng.sequence_batch(wl.batches[0])
        barrier()
        t1 = time.perf_counter()
        for _ in range(a.steps):
            bases_e2e = 0
            for b in wl.batches:
                res, n_b = eng.sequence_batch(b)
                bases_e2e += n_b
        barrier()
        e2e_elapsed = time.perf_counter() - t1
    d2h = 2 * bases_e2e + wl.n_reads * 48
    log(f'[rank {rank}] timed: {elapsed / a.steps * 1e3:.1f} ms/step resident, {e2e_elapsed / a.steps * 1e3:.1f} ms/step end to end')

    # ---- parity + CPU baseline on the same reads
    cpu_g, cpu_desc, parity, alg_inst_G = None, 'skipped', None, None
    if not a.profile and not a.no_parity:
        limit = None if cfg['parity'] == 'full' else PARITY_PREFIX
        picks = wl.prefix_reads(limit)
        if world > 1 and limit is None:   # N ranks share the host cores: every rank checks the first 4096 of its reads
            picks = picks[:4096]
        threads = max(1, n_cores // world)
        n_bad, cpu_bases, cpu_dt = 0, 0, 0.0
        from oracle import oracle as _O
        _O.block_steps_reset()
        for bi in sorted(set(b for b, _ in picks)):
            # nb == 1: `res` still holds the reads fetched by the last end-to-end step; otherwise the batch is run again
            # (the pinned output buffers are reused by every call, so each batch is compared before the next one runs)
            r_b = res if nb == 1 else eng.sequence_batch(wl.batches[bi])[0]
            mine = [(b, j) for b, j in picks if b == bi]
            o, cb, cd = cpu_port_run(wl, mine, threads)
            bad = parity_check(r_b, mine, o)
            n_bad += len(bad)
            if bad:
                log(f'[rank {rank}] PARITY MISMATCH in batch {bi}: read indices '
                    f'{[int(wl.batches[b].read_index[j]) for b, j in bad[:8]]}')
            cpu_bases += cb
            cpu_dt += cd
        cpu_g = cpu_bases / cpu_dt / 1e9 if cpu_dt > 0 else None
        if cpu_bases > 0:   # scaled from the reads the oracle ran to this rank's whole step
            alg_inst_G = algorithmic_warp_inst(_O.block_steps()) * (bases_e2e / cpu_bases) / 1e9
        log(f'[rank {rank}] parity leg: {len(picks)} reads, {n_bad} mismatches, oracle {cpu_dt:.1f} s')
        what = ('the whole workload' if len(picks) == wl.n_reads else f'the first {len(picks)} reads of this rank') if limit is None \
            else f'read indices < {limit} of this rank'
        cpu_desc = f'{what}: {len(picks)} reads, {cpu_bases} bases in {cpu_dt:.2f} s on {threads} threads'
        parity = {'reads_checked': len(picks), 'bases_checked': int(cpu_bases), 'mismatches': int(n_bad),
                  'scope': ('whole workload' if world == 1 else 'the first 4096 reads of every rank') if limit is None
                  else f'first {limit} read indices (SURVEY.md 8d)',
                  'against': 'oracle/badread_oracle.c (Philox mode), same read indices: seq, qual, matches/columns'}

    ref_shim, cli = None, None
    # (only the 5 Mb configs: the reference's loader turns a 3 Gb FASTA into tens of GB of Python objects PER PROCESS -
    # running it on all cores at once took the whole box down, twice)
    if rank == 0 and world == 1 and not a.profile and not a.no_parity and a.ref_shim_bases > 0 and a.config in (1, 2):
        t_leg = time.perf_counter()
        ref_shim = reference_shim_rate(cfg, min(n_cores, 32), a.ref_shim_bases)
        log(f'[rank 0] reference-with-shim leg: {time.perf_counter() - t_leg:.1f} s: {ref_shim.get("value")}')
    if rank == 0 and world == 1 and not a.profile and not a.no_parity and a.config in (1, 2):
        eng.close()   # the command line creates its own engine on the same GPU
        t_leg = time.perf_counter()
        cli = cli_e2e(cfg)
        log(f'[rank 0] command-line leg: {time.perf_counter() - t_leg:.1f} s: {cli.get("value")} {cli.get("note", "")[:120]}')

    tot_bases, max_elapsed, max_e2e = float(bases), elapsed, e2e_elapsed
    if dist is not None:
        import torch
        tb = torch.tensor([float(bases), float(parity['reads_checked'] if parity else 0),
                           float(parity['mismatches'] if parity else 0), float(parity['bases_checked'] if parity else 0)],
                          device='cuda', dtype=torch.float64)
        dist.all_reduce(tb, op=dist.ReduceOp.SUM)
        tm = torch.tensor([elapsed, e2e_elapsed], device='cuda', dtype=torch.float64)
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
        tot_bases, max_elapsed, max_e2e = float(tb[0].item()), float(tm[0].item()), float(tm[1].item())
        if lib_nccl:   # the product's collective: bb_allreduce_bases (must agree with torch's)
            tot_lib = eng.allreduce_bases(int(bases))
            assert tot_lib == int(tot_bases), (tot_lib, tot_bases)
            config['bases_sum'] = 'bb_allreduce_bases (NCCL, in the library)'
        if parity:
            parity['reads_checked'], parity['mismatches'] = int(tb[1].item()), int(tb[2].item())
            parity['bases_checked'] = int(tb[3].item())
            parity['scope'] += f'; summed over {world} ranks'
    if rank != 0:
        eng.close()
        if dist is not None:
            dist.barrier()
            dist.destroy_process_group()
        return 0

    value = tot_bases * a.steps / max_elapsed / 1e9
    e2e_value = tot_bases * a.steps / max_e2e / 1e9
    kernels = {k: v / a.steps for k, v in stage_acc.items() if k not in ('total', 'host_scan')}
    dom = max(kernels, key=kernels.get)
    peak, peak_src = peaks()
    # algorithmic bytes per emitted base (SURVEY.md 8d, DESIGN.md): 1 reference read + 1 sequence write + 1 quality write
    alg_bytes_per_base = 3.0
    achieved = alg_bytes_per_base * bases / (kernels[dom] * 1e-3) / 1e9
    traffic, traffic_src = None, None
    tj, tj_name = newest_profile('traffic')
    if tj is not None and a.config == 1:
        try:  # DRAM bytes of the stage's kernels over one step, from the newest committed ncu pass
            traffic = float(tj['per_stage'][dom]['dram_GB']) * 1e9
            traffic_src = f'{tj_name} (ncu dram__bytes_read.sum + dram__bytes_write.sum, one step)'
        except Exception:
            pass
    alu = None
    ij, ij_name = newest_profile('inst')
    if ij is not None and a.config == 1:
        try:  # integer ALU-pipe accounting: warp instructions of one step over the measured step time
            ginst = float(ij['warp_inst_G_per_step'])
            import torch
            sm_count, smsp = torch.cuda.get_device_properties(local_rank).multi_processor_count, 4
            clk_ghz = (clocks.get('sm_mhz') or 1980.0) / 1e3
            peak_alu = sm_count * smsp * clk_ghz * 0.5   # LOP3/IADD3/SHF: one warp instruction per 2 clocks per SMSP
            ach = ginst / (dev_ms / a.steps * 1e-3)
            alu = {'achieved': ach, 'peak': peak_alu, 'unit': 'G warp-inst/s', 'frac': ach / peak_alu,
                   'warp_inst_G_per_step': ginst, 'source': f'{ij_name} (ncu smsp__inst_executed.sum)'}
            if alg_inst_G is not None:   # what the path needs (oracle's block-update count of this run's reads), not what was issued
                alu['algorithmic_warp_inst_G_per_step'] = alg_inst_G
                alu['algorithmic_frac'] = alg_inst_G / (dev_ms / a.steps * 1e-3) / peak_alu
                alu['issued_over_algorithmic'] = ginst / alg_inst_G
                alu['algorithmic_source'] = ('oracle block-update count of the parity leg\'s reads (64-row updates of the Hirschberg '
                                             'node, leaf and window passes with exact bands) x 2 words x 13 ops / 32 lanes')
        except Exception:
            pass
    roofline = {'bound': 'hbm', 'kernel': dom, 'achieved': achieved, 'peak': peak, 'unit': 'GB/s', 'frac': achieved / peak,
                'traffic': traffic, 'traffic_source': traffic_src, 'peak_source': peak_src, 'kernel_ms': kernels[dom],
                'algorithmic_bytes_per_step': alg_bytes_per_base * bases, 'alu_pipe': alu,
                'note': 'stage = all kernels of that stage of the path; the path is bit-vector DP bound by the integer '
                        'ALU pipe (0.5 warp-inst/clk/SMSP), not by HBM: the HBM fraction is small by construction, see '
                        'DESIGN.md for the ALU-pipe accounting'}
    line = {'metric': 'simulated Gbases/sec', 'value': value, 'unit': 'Gbases/s', 'n_gpus': world, 'steps': a.steps,
            'warmup': a.warmup, 'ms_per_step': max_elapsed / a.steps * 1e3, 'higher_is_better': True, 'scaling': scaling,
            'vs_baseline': None, 'dtype': dtype, 'data': 'synthetic', 'config': config,
            'reads_per_step_rank0': wl.n_reads, 'bases_per_step_rank0': bases,
            'device_ms_per_step_rank0': dev_ms / a.steps, 'stage_ms_rank0': {k: v / a.steps for k, v in stage_acc.items()},
            'plan_s_rank0': wl.t_plan, 'clocks': clocks,
            'e2e': {'value': e2e_value, 'unit': 'Gbases/s', 'h2d_bytes_per_step': int(wl.h2d_bytes()), 'd2h_bytes_per_step': int(d2h)},
            'gpu_launches': int(launches),
            'roofline': roofline,
            'cpu_baseline': {'value': cpu_g, 'unit': 'Gbases/s', 'cores': max(1, n_cores // world), 'kind': 'port', 'sample': cpu_desc},
            'cpu_baseline_reference': ref_shim, 'cli_e2e': cli,
            'parity': parity}
    print(json.dumps(line), flush=True)
    eng.close()
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()
    if parity is not None and parity['mismatches']:
        log(f'PARITY FAILURE: {parity}')
        return 3
    return 0


if __name__ == '__main__':
    sys.exit(main())
