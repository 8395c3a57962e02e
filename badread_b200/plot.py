"""
plot.py - `badread plot` (plot_window_identity.py of the reference) without the drawing: the identity along each read
over a sliding window, and optionally the mean qscore, computed on the GPU and written as a table (--windows).

The reads and alignments come in through the model builders' routes (model_builders._inputs): the same choice of one
alignment per read, the same progress text on `output` (without their "Processing alignments" line, which the
reference's plot does not print) and one line per chosen alignment, Alignment's repr.  Every chosen alignment is checked
before anything is written: where the reference would crash on it or plot positions its CIGAR does not describe, this
exits with an error naming it.  The series come from bb_window_series (csrc/bb_plot.cuh) in passes of a bounded number of
read positions, and native host threads format the table (bb_window_format); a name ending in .gz gets BGZF,
compressed on the GPU.
"""
import argparse
import ctypes
import io
import sys

import numpy as np

from . import _lib
from .misc import load_fasta
from .model_builders import DeviceFlat, _DeviceInputs, _inputs, _ptr

PASS_POSITIONS = 1 << 26    # read positions per pass of bb_window_series (at least the longest alignment's)
FORMAT_LINES = 1 << 22      # table lines per bb_window_format call


def plot_window_identity(args, output=sys.stdout):
    """plot_window_identity.plot_window_identity: prints the loaders' progress and every chosen alignment to `output`;
    with args.windows writes the window table there."""
    refs = load_fasta(args.reference)[0]
    margs = argparse.Namespace(**vars(args))
    margs.max_alignments = None         # (plot reads every alignment)
    inputs = _inputs(margs, refs, output, need_qual=args.qual)
    try:
        names, reprs, read_start = _describe(inputs)
        slice_len = np.zeros((inputs.n, 3), dtype=np.int64)
        if isinstance(inputs, _DeviceInputs):
            flat = inputs.flatten(io.StringIO(), 1000, slice_len) if inputs.n else None
        else:
            flat = inputs.flatten(io.StringIO(), 1000) if inputs.n else None
            slice_len[:] = _host_slice_lengths(inputs)
        if flat is not None:
            _check(flat, slice_len, args.qual, names, reprs)
        for r in reprs:
            print(r, file=output)
        output.flush()
        if args.windows is not None:
            write_windows(args.windows, flat, names, read_start, args.window, args.qual)
    finally:
        inputs.close()


def _describe(inputs):
    """Per chosen alignment: read name, repr (Alignment.__repr__) and read start."""
    if isinstance(inputs, _DeviceInputs):
        a, ch = inputs.a, inputs.chosen
        names = [inputs.read_names[i] for i in a['read_id'][ch].tolist()]
        cols, matches = a['columns'][ch].tolist(), (a['columns'][ch].astype(np.int64) - a['nm'][ch]).tolist()
        reprs = ['%s:%d-%d(%s),%s:%d-%d(%.3f%%)' % (n, rs, re_, '-' if f & 16 else '+', inputs.ref_names[ri], fs, fe,
                                                   100.0 * m / c)
                 for n, rs, re_, f, ri, fs, fe, m, c in zip(names, a['read_start'][ch].tolist(), a['read_end'][ch].tolist(),
                                                             a['flag'][ch].tolist(), a['ref_id'][ch].tolist(),
                                                             a['ref_start'][ch].tolist(), a['ref_end'][ch].tolist(), matches,
                                                             cols)]
        return names, reprs, a['read_start'][ch].astype(np.int64)
    alns = inputs.alignments
    return ([x.read_name for x in alns], [repr(x) for x in alns],
            np.asarray([x.read_start for x in alns], dtype=np.int64))


def _host_slice_lengths(inputs):
    """The lengths of every chosen alignment's sequence, quality and reference slices (Python's slicing)."""
    out = np.zeros((inputs.n, 3), dtype=np.int64)
    for i, x in enumerate(inputs.alignments):
        seq, qual = inputs.reads[x.read_name]
        out[i] = (len(seq[x.read_start:x.read_end]), len(qual[x.read_start:x.read_end]),
                  len(inputs.refs[x.ref_name][x.ref_start:x.ref_end]))
    return out


def _check(flat, slice_len, want_qual, names, reprs):
    """Exits naming the first alignment whose CIGAR does not fit its slices: its read span is not the read slice's length,
    a D run starts after the last read base, an M run reaches past the reference slice, or (with qualities) its quality
    slice is shorter than its read slice."""
    n = flat.n
    span = np.diff(flat.read_off)
    ops = flat.ops[:int(flat.ops_off[-1])]
    kind, count = ops & 3, (ops >> 2).astype(np.int64)
    owner = np.repeat(np.arange(n), np.diff(flat.ops_off))
    p0, r0 = flat.op_read0[:ops.size].astype(np.int64), flat.op_ref0[:ops.size].astype(np.int64)
    bad = np.zeros((n, 4), dtype=bool)
    bad[:, 0] = span != slice_len[:, 0]
    np.logical_or.at(bad[:, 1], owner[(kind == 2) & (p0 == span[owner])], True)
    m_end = np.zeros(n, dtype=np.int64)
    np.maximum.at(m_end, owner[kind == 0], (r0 + count)[kind == 0])
    bad[:, 2] = m_end > slice_len[:, 2]
    if want_qual:
        bad[:, 3] = slice_len[:, 1] < slice_len[:, 0]
    rows = np.flatnonzero(bad.any(axis=1))
    if rows.size == 0:
        return
    i = int(rows[0])
    what = int(np.flatnonzero(bad[i])[0])
    why = [f'its CIGAR covers {int(span[i])} read bases but the aligned part of the read has {int(slice_len[i, 0])}',
           'its CIGAR has a deletion after the last aligned read base',
           f'its CIGAR reaches past the aligned part of the reference ({int(slice_len[i, 2])} bases)',
           f'the read has fewer qualities ({int(slice_len[i, 1])}) than bases ({int(slice_len[i, 0])}) in the aligned part'][what]
    sys.exit(f'Error: alignment {reprs[i]} of read {names[i]}: {why}')


def _passes(flat, window, want_qual, device=0, budget=PASS_POSITIONS):
    """bb_window_series over the alignments in passes of at most max(budget, longest alignment + 1) read positions:
    yields (first alignment, alignments, identity, mean qscore or None)."""
    L = _lib.lib()
    sizes = np.diff(flat.read_off) + 1
    budget = max(int(budget), int(sizes.max()) if sizes.size else 1)
    if isinstance(flat, DeviceFlat):
        read, qual, ref, ops, p0, r0 = flat.device_pointers
    else:
        read, qual, ref, ops, p0, r0 = (_ptr(x) for x in (flat.read, flat.qual, flat.ref, flat.ops, flat.op_read0, flat.op_ref0))
    first = 0
    while first < flat.n:
        ends = np.cumsum(sizes[first:])
        n = int(np.searchsorted(ends, budget, side='right'))
        points = np.maximum(np.diff(flat.read_off[first:first + n + 1]) - window, 0)
        total = int(points.sum())
        ident = np.empty(max(total, 1), dtype=np.float64)
        mq = np.empty(max(total, 1), dtype=np.float64) if want_qual else None
        got = ctypes.c_int64(0)
        rc = L.bb_window_series(device, flat.n, read, qual if want_qual else None, ref, _ptr(flat.read_off), _ptr(flat.ref_off),
                                ops, p0, r0, _ptr(flat.ops_off), window, int(want_qual), first, n, _ptr(ident),
                                _ptr(mq) if want_qual else None, ctypes.byref(got))
        if rc != _lib.BB_OK:
            sys.exit(L.bb_model_error().decode(errors='replace') or f'Error: bb_window_series failed ({rc})')
        assert got.value == total
        yield first, n, ident[:total], (mq[:total] if want_qual else None)
        first += n


def window_series(flat, read_start, window, want_qual, device=0, budget=PASS_POSITIONS):
    """The window series of a flat set (FlatAlignments or DeviceFlat) as numpy arrays: (point_off [n + 1] with alignment
    a's windows at [point_off[a], point_off[a + 1]), positions (int64), identities (float64), mean qscores (float64, or
    None without want_qual)).  budget: read positions per pass of the kernel."""
    parts = list(_passes(flat, window, want_qual, device, budget))
    points = np.maximum(np.diff(flat.read_off) - window, 0)
    point_off = np.concatenate([[0], np.cumsum(points)]).astype(np.int64)
    ident = np.concatenate([p[2] for p in parts]) if parts else np.zeros(0)
    mq = (np.concatenate([p[3] for p in parts]) if parts else np.zeros(0)) if want_qual else None
    return point_off, _positions(point_off, np.asarray(read_start, dtype=np.int64) + window // 2), ident, mq


def _positions(point_off, pos0):
    counts = np.diff(point_off)
    return np.repeat(pos0 - point_off[:-1], counts) + np.arange(int(point_off[-1]), dtype=np.int64)


def write_windows(filename, flat, names, read_start, window, want_qual, device=0, budget=PASS_POSITIONS):
    """The table of --windows: "name\\tposition\\tidentity[\\tmean qscore]" per window, values as '%.4f'; BGZF when the
    name ends in .gz."""
    L = _lib.lib()
    blob = ''.join(names).encode()
    name_off = np.concatenate([[0], np.cumsum([len(x.encode()) for x in names])]).astype(np.int64)
    pos0 = np.asarray(read_start, dtype=np.int64) + window // 2
    names_buf = np.frombuffer(blob or b'\0', dtype=np.uint8)
    with open(filename, 'wb') as out:
        sink = out
        if filename.endswith('.gz'):
            from . import bgzf
            from .engine import Engine
            engine = Engine(device=device, seed=0)
            sink = bgzf.BGZFWriter([engine], out)
        try:
            for first, n, ident, mq in (_passes(flat, window, want_qual, device, budget) if flat is not None else ()):
                point_off = np.concatenate([[0], np.cumsum(np.maximum(np.diff(flat.read_off[first:first + n + 1]) - window, 0))])
                point_off = point_off.astype(np.int64)
                longest = int(np.diff(name_off[first:first + n + 1]).max())
                line = int(L.bb_window_line_bound(longest))
                buf = np.empty(min(int(point_off[-1]), FORMAT_LINES) * line + 1, dtype=np.uint8)
                for lo in range(0, int(point_off[-1]), FORMAT_LINES):
                    hi = min(lo + FORMAT_LINES, int(point_off[-1]))
                    got = ctypes.c_int64(0)
                    rc = L.bb_window_format(n, _ptr(names_buf), _ptr(name_off[first:]), _ptr(pos0[first:]), _ptr(point_off),
                                            _ptr(ident), _ptr(mq) if want_qual else None, lo, hi, _ptr(buf), buf.size,
                                            ctypes.byref(got))
                    if rc != _lib.BB_OK:
                        raise RuntimeError(f'bb_window_format failed ({rc})')
                    sink.write(memoryview(buf)[:got.value])
            if sink is not out:
                sink.close()
        finally:
            if sink is not out:
                engine.close()
