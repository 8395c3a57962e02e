"""
simulate - driver of `badread simulate` on the GPU, mirroring the reference's badread/simulate.py.

What runs where:
  * sequence_fragment (simulate.py:256-358) - the hot path - runs on the GPU for batches of reads
    (Engine.sequence_batch -> bb_sequence_batch).  `sequence_fragment(fragment, target_identity, error_model,
    qscore_model)` below keeps the reference's single-read signature (a batch of one).
  * the fragment builder (simulate.py:91-253, 361-387, 459-482) stays on the host but emits fragment DESCRIPTORS
    (slices of the HBM-resident reference on either strand + literal bytes) instead of Python strings, so a
    15 kb read costs a few dozen bytes of host->device traffic.
  * the driver loop (simulate.py:63-86): reads are numbered 0,1,2,...; every read draws from its own random
    streams keyed by (seed, read index) - host draws from per-read `random.Random` / numpy RandomState, device
    draws from Philox (csrc/bb_rng.cuh).  The reference's single sequential Mersenne-Twister stream is
    data-dependent per read and cannot be reproduced in parallel; with per-read streams the FASTQ depends only
    on --seed, never on batch size or GPU count.  Reads are emitted in index order until the total reaches the
    target (simulate.py:63), skipping empty reads (simulate.py:70).

Derived from Badread (Copyright 2018 Ryan Wick, rrwick@gmail.com, https://github.com/rrwick/Badread), which is free
software under the GNU General Public License version 3 or later; this file mirrors the named parts of the
reference's interface and is distributed under the same licence (see LICENSE and NOTICE at the repository root).
"""
import random
import statistics
import sys
import uuid

import numpy as np

from . import settings
from .engine import Engine, FastaFile, FragmentBatch, default_engine, next_read_index, run_each
from .error_model import ErrorModel, load_error_model
from .fragment_lengths import FragmentLengths
from .identities import Identities
from .misc import float_to_str, load_fasta, load_fasta_arrays, str_is_int
from .qscore_model import QScoreModel, qscore_char_to_error_prob
from .version import __version__

_BASES = np.frombuffer(b'ACGT', dtype=np.uint8)
import time as _time  # noqa: E402
_T_IMPORT = _time.perf_counter()


# ------------------------------------------------------------------------------------------ single read
def sequence_fragment(fragment, target_identity, error_model, qscore_model):
    """simulate.py:256-358 with the reference's signature: returns (seq, qual, actual_identity,
    identity_by_qscores). Runs on the GPU as a batch of one read."""
    eng = default_engine(error_model=error_model, qscore_model=qscore_model)
    batch = FragmentBatch()
    batch.add_literal_read(next_read_index(), fragment, target_identity)
    res, _ = eng.sequence_batch(batch)
    seq, qual = res.read(0)
    actual_identity = res.identity(0)
    if len(qual) > 0:
        identity_by_qscores = 1.0 - statistics.mean(qscore_char_to_error_prob(q) for q in qual)
    else:
        identity_by_qscores = 0.0
    return seq, qual, actual_identity, identity_by_qscores


# ------------------------------------------------------------------------------------------ reference
class Reference(object):
    """Contigs of the reference FASTA, concatenated for upload (load_reference, simulate.py:494-507)."""

    def __init__(self, filename, output=sys.stderr):
        print('', file=output)
        print(f'Loading reference from {filename}', file=output)
        self.names, arrays, depths, circular, left_hairpin, right_hairpin = load_fasta_arrays(filename)
        self.lengths = [int(a.size) for a in arrays]
        self.depths = [depths[n] for n in self.names]
        self.circular = [circular[n] for n in self.names]
        self.left_hairpin = [left_hairpin[n] for n in self.names]
        self.right_hairpin = [right_hairpin[n] for n in self.names]
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int64)
        self.concat = np.concatenate(arrays) if arrays else np.zeros(0, dtype=np.uint8)
        self._report(output)

    def _report(self, output):
        plural = '' if len(self.names) == 1 else 's'
        print(f'  {len(self.names):,} contig{plural}:', file=output)
        for i, name in enumerate(self.names):
            circular_linear = 'circular' if self.circular[i] else 'linear'
            print(f'    {name}: {self.lengths[i]:,} bp, {circular_linear}, {self.depths[i]:.2f}x depth', file=output)
        if len(self.names) > 1:
            print(f'  total size: {sum(self.lengths):,} bp', file=output)

    @property
    def size(self):
        return int(sum(self.lengths))


class DeviceReference(Reference):
    """The reference FASTA loaded by the engines themselves: each one reads the file's bytes from one page-locked copy,
    parses them on its GPU and keeps the contigs there (Engine.load_fasta), so the bases never exist on the host.  The
    host keeps what the planner reads: names, lengths, depths and flags.  concat is None."""

    def __init__(self, filename, engines, output=sys.stderr):
        print('', file=output)
        print(f'Loading reference from {filename}', file=output)
        fasta = FastaFile(filename)
        tables = [None] * len(engines)

        def load(g):
            tables[g] = engines[g].load_fasta(fasta)

        try:
            run_each(len(engines), load)
        finally:
            fasta.close()
        self.names, self.lengths, depths, circular, left_hairpin, right_hairpin = tables[0]
        self.depths = [depths[n] for n in self.names]
        self.circular = [circular[n] for n in self.names]
        self.left_hairpin = [left_hairpin[n] for n in self.names]
        self.right_hairpin = [right_hairpin[n] for n in self.names]
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int64)
        self.concat = None
        self._report(output)


def adjust_depths(ref, frag_lengths, args, rng):
    """simulate.py:516-536."""
    sampled = np.asarray([frag_lengths.get_fragment_length(rng) for _ in range(100000)], dtype=np.int64)
    total = int(sampled.sum())
    for i in range(len(ref.names)):
        ref_len = ref.lengths[i]
        if not args.small_plasmid_bias and ref.circular[i]:
            passing_total = int(sampled[sampled <= ref_len].sum())
            if passing_total == 0:
                sys.exit('Error: fragment length distribution incompatible with reference lengths '
                         '- try running with --small_plasmid_bias to avoid this error')
            ref.depths[i] *= total / passing_total
        if not ref.circular[i]:
            passing_total = int(np.minimum(sampled, ref_len).sum())
            ref.depths[i] *= total / passing_total


# ------------------------------------------------------------------------------------------ fragment builder
class Piece(object):
    """One run of a fragment: a reference slice ('+' / '-' strand coordinates of that strand) or literal bytes."""
    __slots__ = ('contig', 'strand', 'start', 'length', 'data')

    def __init__(self, contig=None, strand=None, start=0, length=0, data=None):
        self.contig, self.strand, self.start, self.length, self.data = contig, strand, start, length, data

    def slice(self, lo, hi):
        if self.data is not None:
            return Piece(data=self.data[lo:hi], length=hi - lo)
        return Piece(self.contig, self.strand, self.start + lo, hi - lo)


def literal(data):
    if isinstance(data, str):
        data = data.encode('latin-1')
    return Piece(data=data, length=len(data))


def slice_pieces(pieces, lo, hi):
    out, pos = [], 0
    for p in pieces:
        a, b = max(lo, pos), min(hi, pos + p.length)
        if a < b:
            out.append(p.slice(a - pos, b - pos))
        pos += p.length
        if pos >= hi:
            break
    return out


def random_bases(nrng, n):
    return _BASES[nrng.randint(0, 4, size=n)].tobytes() if n > 0 else b''


class ReadPlanner(object):
    """The host-side fragment builder: build_fragment and friends (simulate.py:91-253, 361-387, 459-482) with
    per-read random streams, producing pieces + the FASTQ header info + the target identity."""

    def __init__(self, args, ref, frag_lengths, identities, seed):
        self.args, self.ref, self.frag_lengths, self.identities, self.seed = args, ref, frag_lengths, identities, seed
        self.start_adapt_rate, self.start_adapt_amount = adapter_parameters(args.start_adapter)
        self.end_adapt_rate, self.end_adapt_amount = adapter_parameters(args.end_adapter)
        self.weights = [d * l for d, l in zip(ref.depths, ref.lengths)]  # get_ref_contig_weights :118-121

    def streams(self, read_index):
        key = (int(self.seed) & 0xffffffffffffffff, int(read_index))
        rng = random.Random((key[0] << 64) | (key[1] << 1) | 1)
        nrng = np.random.RandomState([key[0] & 0xffffffff, key[0] >> 32, key[1] & 0xffffffff, key[1] >> 32, 0xB200])
        return rng, nrng

    def plan(self, read_index):
        rng, nrng = self.streams(read_index)
        args = self.args
        pieces = self.get_start_adapter(rng, nrng)
        info = []
        frag, frag_info = self.get_fragment(rng, nrng)
        pieces += frag
        info.append(','.join(frag_info))
        while rng.random() < args.chimeras / 100:  # simulate.py:101-110
            info.append('chimera')
            if rng.random() < settings.CHIMERA_END_ADAPTER_CHANCE:
                pieces.append(literal(args.end_adapter_seq))
            if rng.random() < settings.CHIMERA_START_ADAPTER_CHANCE:
                pieces.append(literal(args.start_adapter_seq))
            frag, frag_info = self.get_fragment(rng, nrng)
            pieces += frag
            info.append(','.join(frag_info))
        pieces += self.get_end_adapter(rng, nrng)
        pieces = [p for p in pieces if p.length > 0]
        pieces = self.add_glitches(pieces, nrng)
        target_identity = self.identities.get_identity(nrng)
        read_name = uuid.UUID(int=rng.getrandbits(128))
        return pieces, info, target_identity, read_name

    # simulate.py:148-165
    def get_fragment(self, rng, nrng):
        fragment_length = self.frag_lengths.get_fragment_length(nrng)
        draw = rng.random()  # get_fragment_type :168-180
        junk_rate, random_rate = self.args.junk_reads / 100, self.args.random_reads / 100
        if draw < junk_rate:
            repeat_length = rng.randint(1, 5)  # get_junk_fragment :249-253
            repeat_count = int(round(fragment_length / repeat_length)) + 1
            junk = (random_bases(nrng, repeat_length) * repeat_count)[:fragment_length]
            return [literal(junk)], ['junk_seq']
        if draw < junk_rate + random_rate:
            return [literal(random_bases(nrng, fragment_length))], ['random_seq']
        for _ in range(1000):
            pieces, info = self.get_real_fragment(fragment_length, rng)
            if pieces:
                return pieces, info
        sys.exit('Error: failed to generate any sequence fragments - are your read lengths '
                 'incompatible with your reference contig lengths?')

    # simulate.py:183-246
    def get_real_fragment(self, fragment_length, rng):
        ref = self.ref
        if len(ref.names) == 1:
            c = 0
        else:
            c = rng.choices(range(len(ref.names)), weights=self.weights)[0]
        info = [ref.names[c]]
        length = ref.lengths[c]
        if rng.random() < 0.5:
            strand, other = '+', '-'
        else:
            strand, other = '-', '+'
        info.append(strand + 'strand')
        hairpin_at_end = ref.right_hairpin[c] if strand == '+' else ref.left_hairpin[c]
        if fragment_length >= length and not ref.circular[c] and not hairpin_at_end:
            info.append('0-' + str(length))
            return [Piece(c, strand, 0, length)], info
        if fragment_length > length and ref.circular[c]:
            return [], ''
        start_pos = rng.randint(0, length - 1)
        end_pos = start_pos + fragment_length
        if ref.circular[c]:
            info.append(f'{start_pos}-{end_pos}')
            if end_pos <= length:
                return [Piece(c, strand, start_pos, end_pos - start_pos)], info
            looped_end_pos = end_pos - length
            assert looped_end_pos > 0
            return [Piece(c, strand, start_pos, length - start_pos), Piece(c, strand, 0, looped_end_pos)], info
        if end_pos > length:
            if hairpin_at_end:
                fwd_len = length - start_pos
                left_over_bases = min(fragment_length - fwd_len, fwd_len)
                info.append(f'{start_pos}-{length} (hairpin) 0-{left_over_bases}')
                return [Piece(c, strand, start_pos, fwd_len), Piece(c, other, 0, left_over_bases)], info
            end_pos = length
        info.append(f'{start_pos}-{end_pos}')
        return [Piece(c, strand, start_pos, end_pos - start_pos)], info

    # simulate.py:361-387
    def get_start_adapter(self, rng, nrng):
        adapter, rate, amount = self.args.start_adapter_seq, self.start_adapt_rate, self.start_adapt_amount
        if not adapter or rate == 0.0 or amount == 0.0:
            return []
        if rng.random() < rate:
            if amount == 1.0:
                return [literal(adapter)]
            frag_len = get_adapter_frag_length(amount, adapter, nrng)
            return [literal(adapter[len(adapter) - frag_len:])]
        return []

    def get_end_adapter(self, rng, nrng):
        adapter, rate, amount = self.args.end_adapter_seq, self.end_adapt_rate, self.end_adapt_amount
        if not adapter or rate == 0.0 or amount == 0.0:
            return []
        if rng.random() < rate:
            if amount == 1.0:
                return [literal(adapter)]
            return [literal(adapter[:get_adapter_frag_length(amount, adapter, nrng)])]
        return []

    # simulate.py:459-482
    def add_glitches(self, pieces, nrng):
        rate, size, skip = self.args.glitch_rate, self.args.glitch_size, self.args.glitch_skip
        if rate == 0:
            return pieces
        total = sum(p.length for p in pieces)
        i = 0
        out = []
        while True:
            dist_to_glitch = int(nrng.geometric(p=1 / rate if rate > 1 else 1))
            out += slice_pieces(pieces, i, min(i + dist_to_glitch, total))
            i += dist_to_glitch
            if i >= total:
                break
            if size > 0:
                out.append(literal(random_bases(nrng, int(nrng.geometric(p=1 / size if size > 1 else 1)))))
            if skip > 0:
                i += int(nrng.geometric(p=1 / skip if skip > 1 else 1))
            if i >= total:
                break
        return [p for p in out if p.length > 0]

    def add_to_batch(self, batch, read_index, pieces, target_identity):
        ref = self.ref
        for p in pieces:
            if p.data is not None:
                batch.add_literal_segment(p.data)
            elif p.strand == '+':
                batch.add_ref_segment(ref.offsets[p.contig] + p.start, p.length, reverse=False)
            else:  # slice [start, start+len) of the reverse complement == revcomp of forward [L-start-len, L-start)
                fwd_start = ref.lengths[p.contig] - p.start - p.length
                batch.add_ref_segment(ref.offsets[p.contig] + fwd_start, p.length, reverse=True)
        batch.end_read(read_index, target_identity)

    def materialise(self, pieces):
        """The fragment as a Python string (tests and the oracle-side checks; the GPU gathers it itself)."""
        from .misc import reverse_complement
        ref = self.ref
        out = []
        for p in pieces:
            if p.data is not None:
                out.append(bytes(p.data))
            else:
                o = int(ref.offsets[p.contig])
                if p.strand == '+':
                    out.append(ref.concat[o + p.start:o + p.start + p.length].tobytes())
                else:
                    fwd_start = ref.lengths[p.contig] - p.start - p.length
                    out.append(reverse_complement(ref.concat[o + fwd_start:o + fwd_start + p.length].tobytes()))
        return b''.join(out).decode('latin-1')


def get_adapter_frag_length(amount, adapter, nrng):
    beta_a = 2.0 * amount
    beta_b = 2.0 - beta_a
    return round(int(len(adapter) * nrng.beta(beta_a, beta_b)))


def adapter_parameters(param_str):
    parts = param_str.split(',')
    if len(parts) == 2:
        try:
            return [float(x) / 100 for x in parts]
        except ValueError:
            pass
    sys.exit('Error: adapter parameters must be two comma-separated values between 0 and 1')


def build_random_adapters(args, rng):
    """simulate.py:422-432."""
    random_start, random_end = False, False
    if str_is_int(args.start_adapter_seq):
        args.start_adapter_seq = ''.join('ACGT'[rng.randint(0, 3)] for _ in range(int(args.start_adapter_seq)))
        random_start = True
    if str_is_int(args.end_adapter_seq):
        args.end_adapter_seq = ''.join('ACGT'[rng.randint(0, 3)] for _ in range(int(args.end_adapter_seq)))
        random_end = True
    return random_start, random_end


def get_target_size(ref_size, quantity):
    """simulate.py:124-145."""
    try:
        return int(quantity)
    except ValueError:
        pass
    quantity = quantity.lower()
    try:
        last_char = quantity[-1]
        value = float(quantity[:-1])
        if last_char == 'x':
            return int(round(value * ref_size))
        elif last_char == 'g':
            return int(round(value * 1000000000))
        elif last_char == 'm':
            return int(round(value * 1000000))
        elif last_char == 'k':
            return int(round(value * 1000))
    except (ValueError, IndexError):
        pass
    sys.exit('Error: could not parse quantity\n'
             '--quantity must be either an absolute value (e.g. 250M) or a relative depth (e.g. 25x)')


# ------------------------------------------------------------------------------------------ banner
def print_intro(output):
    print('', file=output)
    print(f'Badread v{__version__}', file=output)
    print('long read simulation', file=output)


def print_glitch_summary(glitch_rate, glitch_size, glitch_skip, output):
    print('', file=output)
    if glitch_rate == 0:
        print('Reads will have no glitches', file=output)
    else:
        print('Read glitches:', file=output)
        print(f'  rate (mean distance between glitches) = {float_to_str(glitch_rate):>5}', file=output)
        print(f'  size (mean length of random sequence) = {float_to_str(glitch_size):>5}', file=output)
        print(f'  skip (mean sequence lost per glitch)  = {float_to_str(glitch_skip):>5}', file=output)


def print_adapter_summary(start_rate, start_amount, start_seq, end_rate, end_amount, end_seq, random_start,
                          random_end, output):
    print('', file=output)
    if start_seq and start_rate > 0.0 and start_amount > 0.0:
        print('Start adapter:', file=output)
        print(f'  seq: {start_seq}{" (randomly generated)" if random_start else ""}', file=output)
        print(f'  rate:   {start_rate * 100.0:.1f}%', file=output)
        print(f'  amount: {start_amount * 100.0:.1f}%', file=output)
    else:
        print('Start adapter: none', file=output)
    print('', file=output)
    if end_seq and end_rate > 0.0 and end_amount > 0.0:
        print('End adapter:', file=output)
        print(f'  seq: {end_seq}{" (randomly generated)" if random_end else ""}', file=output)
        print(f'  rate:   {end_rate * 100.0:.1f}%', file=output)
        print(f'  amount: {end_amount * 100.0:.1f}%', file=output)
    else:
        print('End adapter: none', file=output)


def print_other_problem_summary(args, output):
    print('', file=output)
    print('Other problems:', file=output)
    print(f'  chimera join rate: {args.chimeras}%', file=output)
    print(f'  junk read rate:    {args.junk_reads}%', file=output)
    print(f'  random read rate:  {args.random_reads}%', file=output)


def print_progress(count, bp, target, output):
    plural = ' ' if count == 1 else 's'
    percent = int(1000.0 * bp / target) / 10
    if percent > 100.0:
        percent = 100.0
    print(f'\rSimulating: {count:,} read{plural}  {bp:,} bp  {percent:.1f}%', file=output, flush=True, end='')


# ------------------------------------------------------------------------------------------ driver
def simulate(args, output=sys.stderr, stdout=None):
    """simulate.py:32-88. FASTQ goes to stdout, everything else to `output`."""
    stdout = sys.stdout if stdout is None else stdout
    print_intro(output)
    seed = args.seed if args.seed is not None else random.SystemRandom().getrandbits(63)
    setup_rng = random.Random(seed)
    setup_nrng = np.random.RandomState(seed & 0xffffffff)
    n_gpus = max(1, int(getattr(args, 'gpus', 1) or 1))
    engines = [Engine(device=g, seed=seed) for g in range(n_gpus)]   # each GPU parses the reference itself
    try:
        _simulate(args, output, stdout, seed, setup_rng, setup_nrng, engines)
    finally:
        for eng in engines:
            eng.close()


def _simulate(args, output, stdout, seed, setup_rng, setup_nrng, engines):
    """simulate() once its engines exist: the reference is loaded onto them, then the reads are simulated."""
    ref = DeviceReference(args.reference, engines, output)
    frag_lengths = FragmentLengths(args.mean_frag_length, args.frag_length_stdev, output)
    adjust_depths(ref, frag_lengths, args, setup_nrng)
    identities = Identities(args.mean_identity, args.identity_stdev, args.max_identity, output)
    error_model = load_error_model(args.error_model, engines, output)
    qscore_model = QScoreModel(args.qscore_model, output)
    print_glitch_summary(args.glitch_rate, args.glitch_size, args.glitch_skip, output)
    random_start, random_end = build_random_adapters(args, setup_rng)
    planner = ReadPlanner(args, ref, frag_lengths, identities, seed)
    print_adapter_summary(planner.start_adapt_rate, planner.start_adapt_amount, args.start_adapter_seq,
                          planner.end_adapt_rate, planner.end_adapt_amount, args.end_adapter_seq,
                          random_start, random_end, output)
    print_other_problem_summary(args, output)
    target_size = get_target_size(ref.size, args.quantity)
    print('', file=output)
    print(f'Target read set size: {target_size:,} bp', file=output)
    print('', file=output)

    import os
    import time
    t_loop = time.perf_counter()
    stats = run_batches(args, ref, frag_lengths, identities, error_model, qscore_model, seed, target_size, engines, output,
                        stdout)
    print('\n', file=output)
    if os.environ.get('BADREAD_B200_TIMING') == '1':   # one machine-readable line for bench.py's cli_e2e leg
        import json
        stats['loop_s'] = time.perf_counter() - t_loop
        stats['setup_s'] = t_loop - _T_IMPORT
        print('BADREAD_B200_TIMING ' + json.dumps(stats), file=output, flush=True)


def _write_fastq(stdout, buf):
    """FASTQ bytes to the caller's stream: the binary layer of a real file / pipe, or a text stream (tests)."""
    raw = getattr(stdout, 'buffer', None)
    if raw is not None:
        stdout.flush()
        raw.write(memoryview(buf))
    else:
        stdout.write(bytes(buf).decode('latin-1'))


def _binary(stdout):
    """The binary layer of a real file / pipe, or the stream itself when it takes bytes (tests)."""
    raw = getattr(stdout, 'buffer', None)
    if raw is None:
        return stdout
    stdout.flush()
    return raw


def run_batches(args, ref, frag_lengths, identities, error_model, qscore_model, seed, target_size, engines, output, stdout):
    """The driver loop of simulate.py:63-86 over batches of reads on the engines (one per GPU, each holding the
    reference; the caller closes them).  Reads are numbered 0, 1, 2, ...; a batch of B
    indices is dealt out over the GPUs (GPU g takes indices = g mod G), planned by the native planner, sequenced on
    the GPUs side by side (one host thread each) and written in index order until the total reaches the target, so
    the FASTQ is independent of the batch size and of the number of GPUs.  With --gzip the GPUs compress the FASTQ to
    BGZF (badread_b200/bgzf.py) before it is written; with --bam they build and compress unaligned BAM records of the
    same reads instead (badread_b200/bam.py)."""
    from .planner import NativePlanner, fastq_format_sharded
    from ._lib import ReadResult
    import os
    n_gpus = len(engines)
    planners = []
    threads_each = max(1, (os.cpu_count() or 1) // n_gpus)
    for eng in engines:
        eng.set_error_model(error_model)
        eng.set_qscore_model(qscore_model)
        planners.append(NativePlanner(args, ref, frag_lengths, identities, seed, n_threads=threads_each))

    use_nccl = False
    if n_gpus > 1:   # the stop condition's SUM over the GPUs goes through NCCL when the library can load it
        from .engine import allreduce_bases_all, comm_init_all, nccl_available
        if nccl_available():
            comm_init_all(engines)
            use_nccl = True

    count, total_size, next_index = 0, 0, 0
    mean_len = max(1.0, float(args.mean_frag_length))
    max_batch = int(getattr(args, 'batch_reads', 0) or 16384) * n_gpus
    import time
    t_first = time.perf_counter()   # engines, reference and tables are resident: the simulate loop proper starts here
    out_buf = None
    empty = np.zeros(1, dtype=np.uint8)
    writer = None
    bam = getattr(args, 'bam', False)
    if bam:   # records built and compressed on the GPUs: the bases and qualities stay on the device
        from .bam import BAMWriter
        writer = BAMWriter(engines, _binary(stdout))
    elif getattr(args, 'gzip', False):
        from .bgzf import BGZFWriter
        writer = BGZFWriter(engines, _binary(stdout))
    print_progress(count, total_size, target_size, output)
    try:
        while total_size < target_size:
            want = int((target_size - total_size) / mean_len * 1.05) + 8
            n_batch = max(1, min(max_batch, want))
            planned, results = [None] * n_gpus, [None] * n_gpus

            def work(g):
                n_g = len(range(g, n_batch, n_gpus))
                planned[g] = planners[g].plan(next_index + g, n_g, stride=n_gpus)
                if not n_g:
                    results[g] = None
                elif bam:
                    results[g] = engines[g].run_batch_results(planned[g])[0]
                else:
                    results[g] = engines[g].sequence_batch(planned[g])[0]

            run_each(n_gpus, work)
            recs = [r.records if r is not None else (ReadResult * 1)() for r in results]
            if bam:
                n_emit, bases = writer.write_batch(planned, recs, total_size, target_size)
            else:
                seqs = [r.seq if r is not None else empty for r in results]
                quals = [r.qual if r is not None else empty for r in results]
                buf, n_emit, bases, _, out_buf = fastq_format_sharded(planned, recs, seqs, quals, 0, total_size, target_size,
                                                                      out=out_buf)
                if writer is None:
                    _write_fastq(stdout, buf)
                else:
                    writer.write(buf)
            if use_nccl:
                # every GPU learns the batch's total from one all-reduce: more than was written means the target was
                # reached inside this batch (the FASTQ stops after the read that reaches it, simulate.py:63)
                produced = allreduce_bases_all(engines, [r.total_bases() if r is not None else 0 for r in results])
                assert produced >= bases and (produced == bases or total_size + bases >= target_size)
            total_size += bases
            count += n_emit
            print_progress(count, total_size, target_size, output)
            next_index += n_batch
        if writer is not None:
            writer.close()
        return {'reads': count, 'bases': total_size, 'gpus': n_gpus, 'batches_s': time.perf_counter() - t_first,
                'nccl_stop_condition': bool(use_nccl)}
    finally:
        for pl in planners:
            pl.close()
