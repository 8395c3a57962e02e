"""ctypes front end of tests/emu/emu_fastq.cpp: the FASTQ parser and the slice gather's device code under the warp
emulator, with the host planning of bb_flat_build (fq_plan) as the library runs it.  TEST INFRASTRUCTURE."""
import ctypes
import os
import pathlib
import subprocess
import types

import numpy as np

HERE = pathlib.Path(os.path.dirname(os.path.realpath(__file__)))
LIB = HERE / 'libemu_fastq.so'
TILE, LPT = 16384, 16       # the device's FQ_TILE and FQ_LINES_PER_THREAD


def build():
    root = HERE.parent.parent
    srcs = [HERE / 'emu_fastq.cpp', HERE / 'cuda_emu.h', root / 'badread_b200' / 'csrc' / 'bb_fastq.cuh',
            root / 'include' / 'badread_b200.h']
    if not LIB.is_file() or any(LIB.stat().st_mtime < s.stat().st_mtime for s in srcs):
        # 64 threads per tile (two warps: the cross-warp step of the block scan runs) and 16 in the scan CTAs (so that
        # their threads take several tiles each on small inputs)
        subprocess.run(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-fno-gnu-unique',
                        '-DFQ_THREADS=64', '-DFQ_SCAN_THREADS=16', '-o', str(LIB), str(srcs[0])], check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(str(LIB))
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        L.emu_fastq_parse.restype = ctypes.c_int
        L.emu_fastq_parse.argtypes = [ctypes.c_char_p, i64, i32, i32, vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i64)]
        L.emu_fastq_flat.restype = ctypes.c_int
        L.emu_fastq_flat.argtypes = [ctypes.c_char_p, i64, vp, i64, ctypes.c_char_p, vp, vp, i32, vp, vp, vp, vp, i64, vp, vp] + [vp] * 9 + [vp]
        _lib = L
    return _lib


class ParseError(ValueError):
    pass


def parse(text, tile=TILE, lpt=LPT):
    """The records' spans (n, 6): name, sequence and quality [lo, hi), as bb_fastq_parse finds them.  Raises ParseError
    with bb_fastq_parse's reason for a header without a name ('name', record) or a truncated last record ('truncated',
    record)."""
    text = bytes(text)
    cap = text.count(b'\n') + 1
    recs = np.zeros((cap, 6), np.int64)
    n_rec, err = ctypes.c_int64(0), ctypes.c_int64(0)
    rc = lib().emu_fastq_parse(text, len(text), tile, lpt, recs.ctypes.data, cap, ctypes.byref(n_rec), ctypes.byref(err))
    if rc:
        raise RuntimeError(f'emu_fastq_parse failed ({rc})')
    if err.value >= 0:
        raise ParseError(('truncated' if err.value & 1 else 'name', err.value >> 1))
    return recs[:n_rec.value]


def load(text, tile=TILE, lpt=LPT):
    """{name: (upper-case sequence, qualities)} of the parsed records, as load_fastq returns it (the last record of a
    repeated name)."""
    text = bytes(text)
    out = {}
    for nl, nh, sl, sh, ql, qh in parse(text, tile, lpt).tolist():
        out[text[nl:nh].decode()] = (text[sl:sh].upper().decode(), text[ql:qh].decode())
    return out


def flat(text, paf, refs, tile=TILE, lpt=LPT):
    """What bb_flat_build makes of a FASTQ text, a PAF file and load_fasta's refs, with the alignments chosen as the
    device route chooses them: a FlatAlignments look-alike, or ('read' / 'reference' / 'ascii', alignment) for a
    failure."""
    from badread_b200 import _lib, misc
    from badread_b200 import model_builders as mb
    text = bytes(text)
    recs = parse(text, tile, lpt)
    name_off = np.concatenate([[0], np.cumsum(recs[:, 1] - recs[:, 0])]).astype(np.int64)
    names = b''.join(text[a:b] for a, b in recs[:, :2].tolist()) or b'\0'
    handle = mb._parse_records(str(paf), 'paf', None)
    try:
        v, n, ref_names, _, a = mb._record_arrays(handle)
        best = mb._best_per_read(a, n)
        chosen = mb._usable(best, a['columns'][best], a['columns'][best].astype(np.int64) - a['nm'][best]).astype(np.int64)
        contig_at, contig_len, contigs, total = mb._touched_contigs(a['ref_id'][chosen], ref_names, refs)
        sizes, failed = np.zeros(3, np.int64), np.zeros(2, np.int64)
        comp = np.frombuffer(misc._COMP_TABLE, np.uint8).copy()
        recs_c = np.ascontiguousarray(recs) if recs.size else np.zeros((1, 6), np.int64)
        common = [text, len(text), recs_c.ctypes.data, len(recs), names, name_off.ctypes.data, ctypes.addressof(v), len(chosen),
                  chosen.ctypes.data if chosen.size else None, contig_at.ctypes.data, contig_len.ctypes.data, contigs.ctypes.data,
                  total, comp.ctypes.data, sizes.ctypes.data]
        L = lib()
        rc = L.emu_fastq_flat(*common, *([None] * 9), failed.ctypes.data)
        if rc == 0:
            nr, nf, no = (int(x) for x in sizes)
            out = types.SimpleNamespace(n=len(chosen), read=np.zeros(max(nr, 1), np.uint8), qual=np.zeros(max(nr, 1), np.uint8),
                                        ref=np.zeros(max(nf, 1), np.uint8), ops=np.zeros(max(no, 1), np.uint32),
                                        op_read0=np.zeros(max(no, 1), np.int32), op_ref0=np.zeros(max(no, 1), np.int32),
                                        read_off=np.zeros(len(chosen) + 1, np.int64), ref_off=np.zeros(len(chosen) + 1, np.int64),
                                        ops_off=np.zeros(len(chosen) + 1, np.int64))
            rc = L.emu_fastq_flat(*common, *(getattr(out, f).ctypes.data for f in
                                             ('read', 'qual', 'ref', 'ops', 'op_read0', 'op_ref0', 'read_off', 'ref_off', 'ops_off')),
                                  failed.ctypes.data)
            if rc == 0:
                return out
        return ({1: 'read', 2: 'reference', 3: 'ascii', 4: 'cigar'}[int(failed[1])], int(failed[0]))
    finally:
        _lib.lib().bb_aln_free(handle)
